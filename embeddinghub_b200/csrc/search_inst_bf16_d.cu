// K2 instantiations over bf16 rows (row shapes of the bf16 walk; see search_impl.cuh and walk.cuh)
#include "search_impl.cuh"
namespace ehb {
cudaError_t launch_search_bf16_d1536(EHB_SEARCH_ARGS) { return launch_search_kpl<32, 12, __nv_bfloat16>(EHB_SEARCH_PASS); }
cudaError_t launch_search_bf16_d2048(EHB_SEARCH_ARGS) { return launch_search_kpl<32, 16, __nv_bfloat16>(EHB_SEARCH_PASS); }
}  // namespace ehb
