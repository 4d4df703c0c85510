// K2b — the wide-beam walk (ef 513 .. 4096): kernel template + launcher (included by search_inst_beam_*.cu).
//
// The one-warp walk (search_impl.cuh) keeps its result set in registers (UList, at most 16 keys per lane: ef <= 512)
// and its visited table in shared memory (2 M0 ef + 64 entries: 1 MB at ef = 4096, M0 = 32).  This form keeps the
// result set in the warp's shared-memory key list (walk.cuh SList) and the visited table in HBM: each warp of a
// persistent grid owns one table slice of the index's scratch and walks the queries q = warp, warp + warps, ...,
// so the scratch is bounded by the resident warps, not by the batch.  The walk itself is beam_search, the descent
// greedy_descent and the rows eval_candidates, exactly as in the one-warp walk: the same expansions, distances and
// counters whenever the visited table does not overflow.
#pragma once
#include "kernels.h"

namespace ehb {

// One warp per block; `vtab` holds gridDim.x slices of `vsize` entries (cfg.hash_size itself is 0: no table in the
// shared-memory slice).  RowT = __nv_bfloat16 walks the bf16 shadow and writes the key sink (k = ef).
// minBlocksPerSM = 1, as for the bf16 one-warp walk: ptxas' default heuristics leave a few bytes of spills in some
// shapes, and shared memory, not registers, sets the resident warps.
template <int LPV, int NQ, bool HASDEL, class RowT>
__global__ void __launch_bounds__(32, 1)
    hnsw_search_beam_kernel(GraphView g, WalkCfg cfg, const float* __restrict__ queries, uint32_t nq, uint32_t k,
                            uint32_t ef, const __grid_constant__ ResultSink sink, uint32_t* __restrict__ out_counts,
                            uint32_t* __restrict__ stats, uint32_t vsize, uint32_t* __restrict__ vtab) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr bool kKeys = !std::is_same<RowT, float>::value;
  WarpCtx c;
  ctx_init(c, smem, cfg, g.dpad, (uint32_t)sizeof(RowT));
  c.hash = vtab + (size_t)blockIdx.x * vsize;
  c.hsize = vsize;
  SList u;
  sl_init(u, c);
  for (uint32_t q = blockIdx.x; q < nq; q += gridDim.x) {
    float4 qr[NQ];  // (unused by the wide shapes: their query is in shared memory)
    if constexpr (wide_shape(LPV, NQ))
      load_query_smem<NQ, RowT>(c, queries + (size_t)q * g.dim, g.dim);
    else
      load_query_regs<LPV, NQ, RowT>(qr, queries + (size_t)q * g.dim, g.dim, c.lane);
    WalkCounters wc = {0, 0, 0, 0};
    ul_clear(u, ef, c.lane);
    if (g.n != 0) {
      uint32_t cur = g.entry;
      if (c.lane == 0) c.cand_id[0] = cur;
      __syncwarp();
      eval_candidates<LPV, NQ, 1, RowT>(c, walk_rows<RowT>(g), qr, 1, g.metric);
      float curdist = c.cand_dist[0];
      __syncwarp();
      wc.evals = 1;
      greedy_descent<LPV, NQ, 1, RowT>(c, g, qr, cur, curdist, g.max_level, 0, wc);
      beam_search<LPV, NQ, 0, true, HASDEL, 1, RowT, false, SList>(c, g, qr, u, cur, curdist, 0, ef, kInvalid, wc);
    }
    // nearest-first output, 32 keys per round: key base + j goes to lane j, then one coalesced store per round
    sl_begin_extract(u, c.lane);
    uint32_t found = 0;
    for (uint32_t base = 0; base < k; base += 32) {
      uint64_t rk = kMaxKey;
      for (uint32_t j = 0; j < 32 && base + j < k && found == base + j; ++j) {
        const uint64_t key = sl_take_min(u, true, c.lane);
        if (key == kMaxKey) break;
        if (c.lane == j) rk = key;
        found++;
      }
      const uint32_t idx = base + c.lane;
      if (idx < k) {
        if constexpr (kKeys) {
          sink.keys[(size_t)q * k + idx] = rk;
        } else {
          const bool ok = rk != kMaxKey;
          sink_store(sink, (size_t)q * k + idx, ok ? g.labels[key_id(rk)] : 0xFFFFFFFFFFFFFFFFull,
                     ok ? key_dist(rk) : INFINITY);
        }
      }
    }
    // the exchange's slice flags (walk.cuh): the persistent grid finishes queries [i W, (i + 1) W) in round i, so the
    // contiguous slices still complete roughly in order
    if constexpr (!kKeys) sink_query_done(sink, q, nq, c.lane);
    if (c.lane == 0) {
      if (out_counts) out_counts[q] = found;
      if (stats) {
        ((uint4*)stats)[2 * q] = make_uint4(wc.hops_upper, wc.hops_base, wc.evals, wc.overflow);
        ((uint4*)stats)[2 * q + 1] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
}

using BeamKernel = void (*)(GraphView, WalkCfg, const float*, uint32_t, uint32_t, uint32_t, const ResultSink,
                            uint32_t*, uint32_t*, uint32_t, uint32_t*);

template <uint32_t DPAD, class RowT>
static BeamKernel beam_kernel(const WalkPlan& p, uint32_t* smem) {
  constexpr int LPV = row_lpv(DPAD * sizeof(RowT)), NQ = row_nq(DPAD, DPAD * sizeof(RowT));
  *smem = warp_smem_bytes(p.cfg, DPAD, (uint32_t)sizeof(RowT));
  if (p.form != WalkForm::beam || p.lpv != LPV || p.nq != NQ) return nullptr;
  return p.hasdel ? hnsw_search_beam_kernel<LPV, NQ, true, RowT> : hnsw_search_beam_kernel<LPV, NQ, false, RowT>;
}

template <uint32_t DPAD, class RowT>
cudaError_t BeamShape<DPAD, RowT>::warps(const WalkPlan& p, int sms, uint64_t nq, uint32_t* out) {
  uint32_t smem = 0;
  const BeamKernel kern = beam_kernel<DPAD, RowT>(p, &smem);
  if (!kern) return cudaErrorInvalidValue;
  uint32_t resident = 0;
  const cudaError_t e = resident_warps((const void*)kern, smem, sms, &resident);
  if (e == cudaSuccess) *out = (uint32_t)std::min<uint64_t>(nq, resident);
  return e;
}

template <uint32_t DPAD, class RowT>
cudaError_t BeamShape<DPAD, RowT>::launch(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq,
                                          uint32_t k, uint32_t ef, const ResultSink& sink, uint32_t* out_counts,
                                          uint32_t* stats, uint32_t* vtab, uint32_t warps, cudaStream_t s) {
  uint32_t smem = 0;
  const BeamKernel kern = beam_kernel<DPAD, RowT>(p, &smem);
  if (!kern || warps == 0) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<warps, 32, smem, s>>>(g, p.cfg, queries, nq, k, ef, sink, out_counts, stats, p.vtab, vtab);
  return cudaGetLastError();
}

}  // namespace ehb
