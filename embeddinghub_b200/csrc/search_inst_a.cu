// K2 instantiations over fp32 rows of dpad 32 .. 128 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<32, float>;
template struct SearchShape<64, float>;
template struct SearchShape<128, float>;
}  // namespace ehb
