// K2 instantiations over the wide rows, dpad 3072 .. 4096, fp32 and the bf16 shadow (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<3072, float>;
template struct SearchShape<4096, float>;
template struct SearchShape<3072, __nv_bfloat16>;
template struct SearchShape<4096, __nv_bfloat16>;
}  // namespace ehb
