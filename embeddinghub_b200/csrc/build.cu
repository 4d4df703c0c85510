// K5 — batched HNSW construction on the GPU.
//
// Replaces the reference's build path: ANNIndex::set -> hnswlib addPoint
// (embeddinghub/embeddingstore/index.cc:20-37), driven one row at a time by
// Version::create_ann_index (version.cc:64-74).  Same algorithm per point —
// greedy descent through the upper layers, an ef_construction beam search per
// layer, hnswlib's getNeighborsByHeuristic2 neighbour selection, mutual
// connection with re-pruning of full rows — but a whole wave of points is
// linked per launch:
//   phase A (build_search_kernel, one warp per new point): search the already
//     linked graph, select <= M neighbours per layer, write the point's own
//     rows, emit one (target row, source, distance) record per selected edge;
//   phase B (count / alloc / scatter kernels): bucket the edge records by target
//     row with atomics (no global sort);
//   phase C (merge_rows_kernel, one warp per touched row): append the incoming
//     links, or, when the row would overflow, re-select the row with the same
//     heuristic over (existing + incoming) — what mutuallyConnectNewElement
//     does one edge at a time.
// Results are deterministic: candidates are ordered by (distance, id) before
// any selection, so atomic arrival order never matters.
// The kernels are in build_impl.cuh, instantiated per row shape in build_inst_*.cu (ef_construction <= 256) and
// build_inst_beam_*.cu (the wide form, up to 4096).
#include "kernels.h"

namespace ehb {

cudaError_t launch_build_batch(const BuildGraph& bg, const WalkCfg& cfg, const uint32_t* ids, uint32_t first,
                               uint32_t b, int mode, BuildBuffers& bb, uint32_t wpb, const BuildBeam& bm,
                               cudaStream_t s) {
  if (b == 0) return cudaSuccess;
  return with_dpad(bg.g.dpad, [&](auto d) {
    return BuildShape<decltype(d)::value>::launch(bg, cfg, ids, first, b, mode, bb, wpb, bm, s);
  });
}

cudaError_t build_beam_warps(const BuildGraph& bg, const WalkCfg& cfg, int sms, uint32_t* warps) {
  return with_dpad(bg.g.dpad, [&](auto d) { return BuildBeamShape<decltype(d)::value>::warps(bg, cfg, sms, warps); });
}

}  // namespace ehb
