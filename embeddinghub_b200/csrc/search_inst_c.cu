// K2 instantiations over fp32 rows of dpad 512 .. 768 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<512, float>;
template struct SearchShape<768, float>;
}  // namespace ehb
