// K2 instantiations over the bf16 shadow of dpad 32 .. 128 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<32, __nv_bfloat16>;
template struct SearchShape<64, __nv_bfloat16>;
template struct SearchShape<128, __nv_bfloat16>;
}  // namespace ehb
