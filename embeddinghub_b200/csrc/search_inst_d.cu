// K2 instantiations over fp32 rows of dpad 1024 .. 2048 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<1024, float>;
template struct SearchShape<1536, float>;
template struct SearchShape<2048, float>;
}  // namespace ehb
