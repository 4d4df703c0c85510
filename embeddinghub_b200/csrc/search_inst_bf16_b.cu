// K2 instantiations over bf16 rows (row shapes of the bf16 walk; see search_impl.cuh and walk.cuh)
#include "search_impl.cuh"
namespace ehb {
cudaError_t launch_search_bf16_d256(EHB_SEARCH_ARGS) { return launch_search_kpl<8, 8, __nv_bfloat16>(EHB_SEARCH_PASS); }
cudaError_t launch_search_bf16_d384(EHB_SEARCH_ARGS) { return launch_search_kpl<8, 12, __nv_bfloat16>(EHB_SEARCH_PASS); }
cudaError_t launch_search_bf16_d512(EHB_SEARCH_ARGS) { return launch_search_kpl<8, 16, __nv_bfloat16>(EHB_SEARCH_PASS); }
}  // namespace ehb
