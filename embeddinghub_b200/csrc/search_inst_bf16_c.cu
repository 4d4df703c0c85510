// K2 instantiations over the bf16 shadow of dpad 768 .. 1024 (see search_impl.cuh)
#include "search_impl.cuh"
namespace ehb {
template struct SearchShape<768, __nv_bfloat16>;
template struct SearchShape<1024, __nv_bfloat16>;
}  // namespace ehb
