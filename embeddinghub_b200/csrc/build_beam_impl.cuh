// K5 wide form (ef_construction 257 .. 4096): the kernels BuildShape::launch runs for efc > kMaxRegEfc and the
// occupancy of its persistent construction search (included by build_inst_beam_*.cu only, so that the register
// form's translation units do not instantiate them).
#pragma once
#include "build_impl.cuh"

namespace ehb {

template <uint32_t DPAD>
BuildSearchBeamKernel BuildBeamShape<DPAD>::search(bool hasdel) {
  constexpr int LPV = row_lpv(DPAD * 4u), NQ = row_nq(DPAD, DPAD * 4u);
  return hasdel ? build_search_beam_kernel<LPV, NQ, true> : build_search_beam_kernel<LPV, NQ, false>;
}
template <uint32_t DPAD>
BuildRowsKernel BuildBeamShape<DPAD>::rows(int mode) {
  constexpr int LPV = row_lpv(DPAD * 4u), NQ = row_nq(DPAD, DPAD * 4u);
  return mode == kBuildUpdate ? update_neighbors_wide_kernel<LPV, NQ> : repair_rows_wide_kernel<LPV, NQ>;
}
template <uint32_t DPAD>
cudaError_t BuildBeamShape<DPAD>::warps(const BuildGraph& bg, const WalkCfg& cfg, int sms, uint32_t* out) {
  return resident_warps((const void*)search(bg.g.deleted != nullptr), build_warp_smem(cfg, DPAD), sms, out);
}

}  // namespace ehb
