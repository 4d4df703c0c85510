// K2 instantiations over the bf16 shadow of dpad 256 .. 512 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<256, __nv_bfloat16>;
template struct SearchShape<384, __nv_bfloat16>;
template struct SearchShape<512, __nv_bfloat16>;
}  // namespace ehb
