// K2 instantiations over the bf16 shadow of dpad 1536 .. 2048 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<1536, __nv_bfloat16>;
template struct SearchShape<2048, __nv_bfloat16>;
}  // namespace ehb
