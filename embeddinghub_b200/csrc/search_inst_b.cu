// K2 instantiations over fp32 rows of dpad 256 .. 384 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<256, float>;
template struct SearchShape<384, float>;
}  // namespace ehb
