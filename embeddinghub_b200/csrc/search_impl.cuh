// K2 kernel template + launcher (included by the per-shape translation units).
#pragma once
#include "kernels.h"

namespace ehb {

// One warp walks one query (device body shared by the two kernels below).  RowT = __nv_bfloat16 walks the bf16
// shadow (g.vecs16) and writes the key sink (sink.keys, k = ef: the whole retained set) for the fp32 re-rank.
template <int LPV, int NQ, int KPL, bool HASDEL, int UDIV, class RowT>
__device__ __forceinline__ void search_body(const GraphView& g, const WalkCfg& cfg, const float* __restrict__ queries,
                                            uint32_t nq, uint32_t k, uint32_t ef, const ResultSink& sink,
                                            uint32_t* __restrict__ out_counts, uint32_t* __restrict__ stats,
                                            uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t q = blockIdx.x * (blockDim.x >> 5) + w;
  if (q >= nq) return;
  constexpr bool kKeys = !std::is_same<RowT, float>::value;
  constexpr bool kScreen = !kKeys && screen_shape(LPV, NQ);  // can run a screened plan (no ring)
  WarpCtx c;
  ctx_init(c, smem + (size_t)w * warp_smem, cfg, g.dpad, (uint32_t)sizeof(RowT));
  float4 qr[NQ];  // (unused by the wide shapes: their query is in shared memory)
  if constexpr (wide_shape(LPV, NQ))
    load_query_smem<NQ, RowT>(c, queries + (size_t)q * g.dim, g.dim);
  else
    load_query_regs<LPV, NQ, RowT>(qr, queries + (size_t)q * g.dim, g.dim, c.lane);
  WalkCounters wc = {0, 0, 0, 0};
  UList<KPL> ul;
  ul_clear<KPL>(ul, ef, c.lane);
  if (g.n != 0) {
    QueryPlanes<NQ> qp;  // a screened walk's integer query, for the descent and the base layer
    if constexpr (kScreen)
      if (walk_screens(g)) screen_setup<NQ>(c, g, qr, qp);
    uint32_t cur = g.entry;
    if (c.lane == 0) c.cand_id[0] = cur;
    __syncwarp();
    eval_candidates<LPV, NQ, UDIV, RowT, kScreen>(c, walk_rows<RowT>(g), qr, 1, g.metric);
    float curdist = c.cand_dist[0];
    __syncwarp();
    wc.evals = 1;
    greedy_descent<LPV, NQ, UDIV, RowT, kScreen>(c, g, qr, cur, curdist, g.max_level, 0, wc, &qp);
    beam_search<LPV, NQ, KPL, true, HASDEL, UDIV, RowT, kScreen>(c, g, qr, ul, cur, curdist, 0, ef, kInvalid, wc, &qp);
  }
  // nearest-first output: extract the k closest in ascending order into registers (element i -> lane i & 31,
  // slot i >> 5), then store them to every destination of the sink with coalesced stores
  uint64_t rk[KPL];
#pragma unroll
  for (int s = 0; s < KPL; ++s) rk[s] = kMaxKey;
  uint32_t found = 0;
  for (uint32_t i = 0; i < k; ++i) {
    uint64_t key = ul_extract_min<KPL>(ul, c.lane);
    if (key == kMaxKey) break;
#pragma unroll
    for (int s = 0; s < KPL; ++s)
      if ((i >> 5) == (uint32_t)s && (i & 31u) == c.lane) rk[s] = key;
    found++;
  }
  if constexpr (kKeys) {  // the key sink: raw keys, no labels, no peers
#pragma unroll
    for (int s = 0; s < KPL; ++s) {
      const uint32_t idx = (uint32_t)s * 32u + c.lane;
      if ((uint32_t)s * 32u < k && idx < k) sink.keys[(size_t)q * k + idx] = rk[s];
    }
  } else {
#pragma unroll
    for (int s = 0; s < KPL; ++s) {
      const uint32_t idx = (uint32_t)s * 32u + c.lane;
      if ((uint32_t)s * 32u < k && idx < k) {
        const bool ok = rk[s] != kMaxKey;
        const uint64_t lab = ok ? g.labels[key_id(rk[s])] : 0xFFFFFFFFFFFFFFFFull;
        const float dist = ok ? key_dist(rk[s]) : INFINITY;
        sink_store(sink, (size_t)q * k + idx, lab, dist);
      }
    }
    sink_query_done(sink, q, nq, c.lane);
  }
  if (c.lane == 0) {
    if (out_counts) out_counts[q] = found;
    if (stats) {
      ((uint4*)stats)[2 * q] = make_uint4(wc.hops_upper, wc.hops_base, wc.evals, wc.overflow);
      ((uint4*)stats)[2 * q + 1] = make_uint4(wc.screened, wc.survivors, wc.screened_upper, 0u);
    }
  }
}

// Register budget of the default form: ptxas chooses (16 vectors in flight per warp).  An explicit
// minBlocksPerSM changes its heuristics, and a register cap below what the 16 loads in flight need serialises
// the load batches — so none is given for fp32 rows.  Over bf16 rows the default heuristics leave a few bytes of
// spills in some shapes; minBlocksPerSM = 1 lets ptxas take the registers instead (a staged walk's occupancy is set by
// its shared memory, a few warps per SM, not by registers).  The fp32 shapes that can screen launch
// hnsw_search_screen_kernel instead.
template <class RowT>
constexpr int kWalkMinBlocks = std::is_same<RowT, float>::value ? 0 : 1;
template <int LPV, int NQ, int KPL, bool HASDEL, class RowT>
__global__ void __launch_bounds__(128, (kWalkMinBlocks<RowT>))
    hnsw_search_kernel(GraphView g, WalkCfg cfg, const float* __restrict__ queries, uint32_t nq, uint32_t k, uint32_t ef,
                       const __grid_constant__ ResultSink sink, uint32_t* __restrict__ out_counts,
                       uint32_t* __restrict__ stats, uint32_t warp_smem) {
  search_body<LPV, NQ, KPL, HASDEL, 1, RowT>(g, cfg, queries, nq, k, ef, sink, out_counts, stats, warp_smem);
}

// The one-warp walk over fp32 rows of the shapes that can screen (screen_shape).  A screened plan has no ring, so
// registers, not shared memory, set its occupancy: 200 registers allow ten one-warp blocks per SM, and no
// instantiation up to dpad 768 with KPL <= 8 spills with them (ptxas left alone takes 255, eight blocks; a 168-register
// cap, twelve, spills hundreds of bytes).  Wider rows (48 query registers at dpad 1536) and KPL = 16 keep 255.
template <int NQ, int KPL>
constexpr int kScreenWalkRegs = NQ <= 6 && KPL <= 8 ? 200 : 255;
template <int LPV, int NQ, int KPL, bool HASDEL>
__global__ void __maxnreg__((kScreenWalkRegs<NQ, KPL>))
    hnsw_search_screen_kernel(GraphView g, WalkCfg cfg, const float* __restrict__ queries, uint32_t nq, uint32_t k,
                              uint32_t ef, const __grid_constant__ ResultSink sink, uint32_t* __restrict__ out_counts,
                              uint32_t* __restrict__ stats, uint32_t warp_smem) {
  search_body<LPV, NQ, KPL, HASDEL, 1, float>(g, cfg, queries, nq, k, ef, sink, out_counts, stats, warp_smem);
}

// "Dense" form for big batches of short rows (LPV = 8, d <= 128): 8 vectors in flight per warp instead of 16
// and a 96-register budget -> 20 resident warps per SM instead of 16 (the visited table shrinks to match,
// api.cu walk_cfg): with many queries in flight, more warps hide more of each hop's memory latency.  Only the
// shapes of kernels.h dense_form have one.
template <int LPV, int NQ, int KPL, class RowT>
__global__ void __launch_bounds__(128, 5) hnsw_search_dense_kernel(GraphView g, WalkCfg cfg,
                                                                   const float* __restrict__ queries, uint32_t nq,
                                                                   uint32_t k, uint32_t ef,
                                                                   const __grid_constant__ ResultSink sink,
                                                                   uint32_t* __restrict__ out_counts,
                                                                   uint32_t* __restrict__ stats, uint32_t warp_smem) {
  search_body<LPV, NQ, KPL, false, 2, RowT>(g, cfg, queries, nq, k, ef, sink, out_counts, stats, warp_smem);
}

// The one-warp walk over wide rows (dpad 3072, 4096; walk.cuh eval_wide), fp32 rows or the bf16 shadow.  Shared
// memory, not registers, sets its occupancy (the query slice and the visited table: api.cu walk_cfg aims at eight
// warps per SM, which leave ptxas the full 255 registers; over bf16 rows minBlocksPerSM = 1 again keeps it from
// spilling).
template <int NQ, int KPL, bool HASDEL, class RowT>
__global__ void __launch_bounds__(128, (kWalkMinBlocks<RowT>))
    hnsw_search_wide_kernel(GraphView g, WalkCfg cfg, const float* __restrict__ queries, uint32_t nq, uint32_t k,
                            uint32_t ef, const __grid_constant__ ResultSink sink, uint32_t* __restrict__ out_counts,
                            uint32_t* __restrict__ stats, uint32_t warp_smem) {
  search_body<32, NQ, KPL, HASDEL, 1, RowT>(g, cfg, queries, nq, k, ef, sink, out_counts, stats, warp_smem);
}

using WalkKernel = void (*)(GraphView, WalkCfg, const float*, uint32_t, uint32_t, uint32_t, const ResultSink,
                           uint32_t*, uint32_t*, uint32_t);
// the kernel the plan launches (nullptr: the plan asks for a form the shape does not have)
template <int LPV, int NQ, int KPL, class RowT>
WalkKernel walk_kernel(const WalkPlan& p) {
  constexpr bool kBf16 = !std::is_same<RowT, float>::value;
  if constexpr (wide_shape(LPV, NQ)) {
    if (p.form != WalkForm::wide) return nullptr;
    return p.hasdel ? hnsw_search_wide_kernel<NQ, KPL, true, RowT> : hnsw_search_wide_kernel<NQ, KPL, false, RowT>;
  } else {
    if (p.form == WalkForm::wide) return nullptr;
    if (p.form == WalkForm::dense) {
      if constexpr (dense_form(kBf16, LPV, NQ, KPL, false))
        if (!p.hasdel) return hnsw_search_dense_kernel<LPV, NQ, KPL, RowT>;
      return nullptr;
    }
    if constexpr (std::is_same<RowT, float>::value && screen_shape(LPV, NQ))
      return p.hasdel ? hnsw_search_screen_kernel<LPV, NQ, KPL, true> : hnsw_search_screen_kernel<LPV, NQ, KPL, false>;
    else
      return p.hasdel ? hnsw_search_kernel<LPV, NQ, KPL, true, RowT> : hnsw_search_kernel<LPV, NQ, KPL, false, RowT>;
  }
}

template <int LPV, int NQ, int KPL, class RowT>
cudaError_t launch_search_t(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                            uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats,
                            cudaStream_t s) {
  const uint32_t wpb = p.wpb;
  uint32_t wsm = warp_smem_bytes(p.cfg, g.dpad, (uint32_t)sizeof(RowT));
  size_t smem = (size_t)wsm * wpb;
  dim3 grid((nq + wpb - 1) / wpb), block(32 * wpb);
  const WalkKernel kern = walk_kernel<LPV, NQ, KPL, RowT>(p);
  if (!kern) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, block, smem, s>>>(g, p.cfg, queries, nq, k, ef, sink, out_counts, stats, wsm);
  return cudaGetLastError();
}

template <uint32_t DPAD, class RowT>
cudaError_t SearchShape<DPAD, RowT>::launch(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq,
                                            uint32_t k, uint32_t ef, const ResultSink& sink, uint32_t* out_counts,
                                            uint32_t* stats, cudaStream_t s) {
  constexpr int LPV = row_lpv(DPAD * sizeof(RowT)), NQ = row_nq(DPAD, DPAD * sizeof(RowT));
  if (p.lpv != LPV || p.nq != NQ || p.form == WalkForm::team) return cudaErrorInvalidValue;
  // (Keeping a whole 2M-neighbour hop in flight per batch needs about 168 registers, which costs occupancy;
  //  batches stay at 16 vectors.)
  switch (p.kpl) {
    case 2: return launch_search_t<LPV, NQ, 2, RowT>(p, g, queries, nq, k, ef, sink, out_counts, stats, s);
    case 4: return launch_search_t<LPV, NQ, 4, RowT>(p, g, queries, nq, k, ef, sink, out_counts, stats, s);
    case 8: return launch_search_t<LPV, NQ, 8, RowT>(p, g, queries, nq, k, ef, sink, out_counts, stats, s);
    case 16: return launch_search_t<LPV, NQ, 16, RowT>(p, g, queries, nq, k, ef, sink, out_counts, stats, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ehb
