// K2t — team variant of the graph walk: T warps (one CTA) per query.
//
// When a batch has fewer queries than the machine has warp slots (C2: 1000
// queries on 132 SMs = 7.6 warps per SM) the warp-per-query walk is bound by one
// warp's serial chain of memory round trips.  Here the T warps of a CTA expand
// the T closest unexpanded entries of the result set concurrently:
//   * every warp keeps an identical replica of the unordered result set (ulist)
//     in registers; all replicas apply the same operations in the same order, so
//     they never need to be exchanged;
//   * round: every warp pops the same T closest unexpanded entries, warp w
//     expands the w-th one (adjacency row -> shared visited table, atomicCAS
//     arbitrates between warps -> distance evaluation), publishes its
//     qualifying (distance, id) pairs to a double-buffered shared array,
//     ONE block barrier, then every warp applies all published pairs to its
//     replica.
// With T = 1 this is exactly hnswlib's expansion order; with T > 1 up to T-1
// expansions per round are speculative: recall >= the sequential walk's at the
// same ef, a few per cent more distance evaluations (both are counted).
// Upper-layer descent is done by warp 0 alone.  LPV = 8 row shapes only.
#pragma once
#include "kernels.h"

namespace ehb {

__host__ __device__ inline uint32_t team_smem_bytes(uint32_t hash_size, uint32_t T) {
  uint32_t b = 0;
  b += align_up(hash_size * 4u, 128);        // visited table
  b += 2 * align_up(T * 32u * 8u, 128);      // published pairs, double buffered
  b += 128;                                  // published counts [2][T]
  b += 2 * align_up(T * 32u * 4u, 128);      // cand_id, cand_dist
  b += 128;                                  // misc
  return b;
}

template <int NQ, int KPL, int T, int U>
__global__ void __launch_bounds__(T * 32, (T == 4 && U * NQ >= 16) ? 3 : 7) hnsw_search_team_kernel(GraphView g, uint32_t hash_size,
                                                                     const float* __restrict__ queries, uint32_t nq,
                                                                     uint32_t k, uint32_t ef,
                                                                     uint64_t* __restrict__ out_labels,
                                                                     float* __restrict__ out_dists,
                                                                     uint32_t* __restrict__ out_counts,
                                                                     uint32_t* __restrict__ stats) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t q = blockIdx.x;
  const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  unsigned char* p = smem;
  uint32_t* hash = (uint32_t*)p; p += align_up(hash_size * 4u, 128);
  uint64_t* pub = (uint64_t*)p; p += 2 * align_up(T * 32u * 8u, 128);   // [2][T][32]
  uint32_t* pubcnt = (uint32_t*)p; p += 128;                             // [2][T]
  uint32_t* cand_id = (uint32_t*)p; p += align_up(T * 32u * 4u, 128);
  float* cand_dist = (float*)p; p += align_up(T * 32u * 4u, 128);
  uint32_t* misc = (uint32_t*)p;  // 0 entry id, 1 entry dist bits, 2 hops_upper, 3 hops_base, 4 evals
  const uint32_t pub_stride = align_up(T * 32u * 8u, 128) / 8u;

  WarpCtx c;  // per-warp view used by the shared evaluation / hashing helpers
  c.lane = lane;
  c.dpad = g.dpad;
  c.vbytes = g.dpad * 4u;
  c.hash = hash;
  c.hsize = hash_size;
  c.cand_id = cand_id + w * 32;
  c.cand_dist = cand_dist + w * 32;
  c.keys = nullptr;
  c.cnt = 0;
  c.dcap = 0;
  c.prefetch = 0;

  for (uint32_t i = tid; i < hash_size; i += T * 32) hash[i] = kInvalid;
  if (tid < 8) misc[tid] = 0;
  float4 qr[NQ];
  load_query_regs<8, NQ>(qr, queries + (size_t)q * g.dim, g.dim, lane);
  WalkCounters wc = {0, 0, 0, 0};
  __syncthreads();

  // ---- entry point + upper layers: warp 0 ----------------------------------------
  if (g.n != 0 && w == 0) {
    uint32_t cur = g.entry;
    if (lane == 0) c.cand_id[0] = cur;
    __syncwarp();
    eval_direct<NQ>(c, g.vecs, qr, 1, g.metric);
    float curdist = c.cand_dist[0];
    __syncwarp();
    wc.evals = 1;
    greedy_descent<8, NQ>(c, g, qr, cur, curdist, g.max_level, 0, wc);
    if (lane == 0) {
      misc[0] = cur;
      misc[1] = f2ord(curdist);
      uint32_t o = 0;
      hash_insert(c, cur, o);
    }
  }
  __syncthreads();

  UList<KPL> u;
  ul_clear<KPL>(u, ef, lane);
  uint32_t cnt = 0, worst_hi = 0xFFFFFFFFu;
  uint32_t ovf = 0;
  bool ovf_any = false;
  if (g.n != 0) ul_insert<KPL>(u, misc[1], misc[0], ef, cnt, worst_hi, lane);
  uint32_t par = 0;
  while (cnt != 0) {
    // -- every warp pops the same T closest unexpanded entries ----------------------------------
    uint32_t mynode = kInvalid, nsel = 0;
#pragma unroll
    for (int t = 0; t < T; ++t) {
      uint32_t nd = ul_min_unexpanded<KPL>(u, true, lane);
      if (nd != kInvalid) nsel++;
      if ((uint32_t)t == w) mynode = nd;
    }
    if (nsel == 0) break;  // identical in every warp
    // -- expansion of my entry --------------------------------------------------------------------
    uint32_t nq_mine = 0;
    uint64_t* mypub = pub + par * pub_stride + w * 32;
    if (mynode != kInvalid) {
      wc.hops_base++;
      uint32_t nb = load_row(g, mynode, 0, lane);
      bool is_new = false;
      if (nb != kInvalid) is_new = hash_insert(c, nb, ovf);
      __syncwarp();
      uint32_t mask = __ballot_sync(0xffffffffu, is_new);
      uint32_t m = __popc(mask);
      if (m) {
        if (is_new) c.cand_id[__popc(mask & lanemask_lt())] = nb;
        __syncwarp();
        wc.evals += m;
        eval_direct<NQ, U>(c, g.vecs, qr, m, g.metric);
        uint32_t myhi = 0xFFFFFFFFu, myid = kInvalid;
        if (lane < m) myhi = f2ord(c.cand_dist[lane]), myid = c.cand_id[lane];
        __syncwarp();
        bool okq = lane < m && (cnt < ef || myhi < worst_hi);
        uint32_t qual = __ballot_sync(0xffffffffu, okq);
        nq_mine = __popc(qual);
        if (okq) mypub[__popc(qual & lanemask_lt())] = ((uint64_t)myhi << 32) | myid;
      }
    }
    if (lane == 0) pubcnt[par * T + w] = nq_mine;
    ovf_any = __syncthreads_or(ovf != 0) || ovf_any;  // the round's only barrier (also publishes the pairs)
    // -- every warp applies every published pair, in the same order --------------------------------
#pragma unroll
    for (int t = 0; t < T; ++t) {
      const uint32_t n_t = pubcnt[par * T + t];
      const uint64_t* src = pub + par * pub_stride + t * 32;
      for (uint32_t j = 0; j < n_t; ++j) {
        uint64_t pr = src[j];
        uint32_t hj = (uint32_t)(pr >> 32), ij = (uint32_t)pr;
        if (cnt >= ef && hj >= worst_hi) continue;
        if (ovf_any && ul_contains<KPL>(u, ij)) continue;
        ul_insert<KPL>(u, hj, ij, ef, cnt, worst_hi, lane);
        if ((uint32_t)t == w && lane == 0) prefetch_l2(g.links0 + (size_t)ij * g.M0);
      }
    }
    par ^= 1;
  }

  // ---- results: warp 0 extracts the k closest in ascending order ------------------------------------
  if (lane == 0) {
    atomicAdd(&misc[2], wc.hops_upper);
    atomicAdd(&misc[3], wc.hops_base);
    atomicAdd(&misc[4], wc.evals);
  }
  __syncthreads();
  if (w == 0) {
    uint32_t found = 0;
    for (uint32_t i = 0; i < k; ++i) {
      uint64_t key = ul_extract_min<KPL>(u, lane);
      if (key == kMaxKey) break;
      if (lane == 0) {
        out_labels[(size_t)q * k + i] = g.labels[key_id(key)];
        if (out_dists) out_dists[(size_t)q * k + i] = key_dist(key);
      }
      found++;
    }
    for (uint32_t i = found + lane; i < k; i += 32) {
      out_labels[(size_t)q * k + i] = 0xFFFFFFFFFFFFFFFFull;
      if (out_dists) out_dists[(size_t)q * k + i] = INFINITY;
    }
    if (lane == 0) {
      if (out_counts) out_counts[q] = found;
      if (stats) {  // (the team walk does not screen)
        ((uint4*)stats)[2 * q] = make_uint4(misc[2], misc[3], misc[4], ovf_any ? 1u : 0u);
        ((uint4*)stats)[2 * q + 1] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
}

template <int NQ, int KPL, int T, int U>
cudaError_t launch_team_t(const GraphView& g, uint32_t hash_size, const float* queries, uint32_t nq, uint32_t k,
                          uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts, uint32_t* stats,
                          cudaStream_t s) {
  size_t smem = team_smem_bytes(hash_size, T);
  auto kern = hnsw_search_team_kernel<NQ, KPL, T, U>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<nq, T * 32, smem, s>>>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats);
  return cudaGetLastError();
}

}  // namespace ehb
