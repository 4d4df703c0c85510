// K1 — exact fp32 brute-force k-NN with canonical arithmetic, and K4 — the
// top-k merge that follows the shard all-gather.
//
// Replaces hnswlib::BruteforceSearch<float> semantics (named by the north star
// as the exact path; the reference itself only instantiates HierarchicalNSW,
// embeddinghub/embeddingstore/index.cc:12-15).  Every distance is one fp32 FMA
// chain over k ascending — acc = fmaf(q_k - x_k, q_k - x_k, acc) for L2,
// acc = fmaf(q_k, x_k, acc) and 1 - acc for IP/cosine — which the oracle
// (oracle/hnsw_oracle.cpp: canon_l2 / canon_dot) restates on the CPU, so ids
// are comparable bit-for-bit under the total order (distance asc, index asc).
#include "kernels.h"
#include "merge.cuh"

namespace ehb {

constexpr int TQ = 64, TN = 64, KC = 16;

// dist[(qi - q0) * nc + (ni - n0)] for a 64 x 64 tile per block.
template <int METRIC>
__global__ void __launch_bounds__(256) bf_dist_kernel(const float* __restrict__ qpad, const float* __restrict__ vecs,
                                                      uint32_t dpad, uint64_t q0, uint64_t qn, uint64_t n0,
                                                      uint64_t nn, float* __restrict__ dist, uint64_t nc) {
  __shared__ float As[KC][TQ + 4];
  __shared__ float Bs[KC][TN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const uint64_t qt = (uint64_t)blockIdx.y * TQ, nt = (uint64_t)blockIdx.x * TN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int lrow = threadIdx.x >> 2, lk = (threadIdx.x & 3) * 4;
  for (uint32_t k0 = 0; k0 < dpad; k0 += KC) {
    float4 a = make_float4(0, 0, 0, 0), b = make_float4(0, 0, 0, 0);
    if (qt + lrow < qn && k0 + lk < dpad) a = *(const float4*)(qpad + (q0 + qt + lrow) * dpad + k0 + lk);
    if (nt + lrow < nn && k0 + lk < dpad) b = *(const float4*)(vecs + (n0 + nt + lrow) * dpad + k0 + lk);
    __syncthreads();
    As[lk + 0][lrow] = a.x, As[lk + 1][lrow] = a.y, As[lk + 2][lrow] = a.z, As[lk + 3][lrow] = a.w;
    Bs[lk + 0][lrow] = b.x, Bs[lk + 1][lrow] = b.y, Bs[lk + 2][lrow] = b.z, Bs[lk + 3][lrow] = b.w;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[kk][ty * 4 + i], bv[i] = Bs[kk][tx * 4 + i];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (METRIC == 0) {
            float t = av[i] - bv[j];
            acc[i][j] = fmaf(t, t, acc[i][j]);
          } else {
            acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
          }
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint64_t qi = qt + ty * 4 + i;
    if (qi >= qn) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint64_t ni = nt + tx * 4 + j;
      if (ni >= nn) continue;
      float d = METRIC == 0 ? acc[i][j] : 1.0f - acc[i][j];
      dist[qi * nc + ni] = d;
    }
  }
}

// One warp per (query, slice): sorted top-k of its slice of the distance row.
// Keys that cannot beat the query's running k-th best (run_keys, from the chunks already merged) are
// dropped before they cost an insert.
__global__ void bf_select_kernel(const float* __restrict__ dist, uint64_t nc, uint64_t nn, uint64_t n0, uint64_t qn,
                                 uint32_t slices, uint32_t k, uint64_t* __restrict__ part_keys,
                                 const uint64_t* __restrict__ run_keys, uint64_t q0,
                                 const uint8_t* __restrict__ deleted) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const uint64_t job = (uint64_t)blockIdx.x * wpb + w;
  if (job >= qn * slices) return;
  const uint64_t q = job / slices;
  const uint32_t sl = (uint32_t)(job % slices);
  WarpCtx c;
  c.lane = lane_id();
  c.keys = (uint64_t*)smem + (size_t)w * align_up(k, 32);
  c.cnt = 0;
  const uint64_t per = (nn + slices - 1) / slices;
  const uint64_t lo = (uint64_t)sl * per, hi = min(nn, lo + per);
  const float* row = dist + q * nc;
  const uint64_t thr = run_keys[(q0 + q) * k + (k - 1)];  // kMaxKey until k results exist
  for (uint64_t i0 = lo; i0 < hi; i0 += 32) {
    uint64_t i = i0 + c.lane;
    uint64_t key = kMaxKey;
    if (i < hi && !(deleted && deleted[n0 + i])) key = make_key(row[i], (uint32_t)(n0 + i));
    uint32_t worst_hi = c.cnt >= k ? key_hi(c.keys[k - 1]) : 0xFFFFFFFFu;
    uint32_t qual = __ballot_sync(0xffffffffu, key != kMaxKey && key < thr && (c.cnt < k || key_hi(key) < worst_hi));
    while (qual) {
      int j = __ffs(qual) - 1;
      qual &= qual - 1;
      uint64_t kj = __shfl_sync(0xffffffffu, key, j);
      if (c.cnt >= k && kj >= c.keys[k - 1]) continue;
      list_insert(c, kj, k);
    }
  }
  uint64_t* out = part_keys + (q * slices + sl) * k;
  for (uint32_t i = c.lane; i < k; i += 32) out[i] = i < c.cnt ? c.keys[i] : kMaxKey;
}

// One warp per query: merge the running list with `slices` sorted partial lists.
__global__ void bf_merge_kernel(uint64_t* __restrict__ run_keys, const uint64_t* __restrict__ part_keys, uint64_t q0,
                                uint64_t qn, uint32_t slices, uint32_t k) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const uint64_t q = (uint64_t)blockIdx.x * wpb + w;
  if (q >= qn) return;
  WarpCtx c;
  c.lane = lane_id();
  c.keys = (uint64_t*)smem + (size_t)w * align_up(k, 32);
  c.cnt = 0;
  uint64_t* run = run_keys + (q0 + q) * k;
  for (uint32_t s = 0; s <= slices; ++s) {
    const uint64_t* src = s == 0 ? run : part_keys + (q * slices + (s - 1)) * k;
    bool done = false;
    for (uint32_t i0 = 0; i0 < k && !done; i0 += 32) {
      uint32_t i = i0 + c.lane;
      uint64_t key = i < k ? src[i] : kMaxKey;
      uint32_t valid = __ballot_sync(0xffffffffu, key != kMaxKey);
      uint32_t qual = valid;
      while (qual) {
        int j = __ffs(qual) - 1;
        qual &= qual - 1;
        uint64_t kj = __shfl_sync(0xffffffffu, key, j);
        if (c.cnt >= k && kj >= c.keys[k - 1]) {
          done = true;  // source is sorted: nothing later can qualify
          break;
        }
        list_insert(c, kj, k);
      }
      if (valid != 0xffffffffu) done = true;
    }
  }
  __syncwarp();
  for (uint32_t i = c.lane; i < k; i += 32) run[i] = i < c.cnt ? c.keys[i] : kMaxKey;
}

__global__ void bf_fill_keys_kernel(uint64_t* keys, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = kMaxKey;
}

__global__ void bf_finalize_kernel(const uint64_t* __restrict__ run_keys, const uint64_t* __restrict__ labels,
                                   uint64_t nq, uint32_t k, uint64_t* __restrict__ out_labels,
                                   float* __restrict__ out_dists, uint32_t* __restrict__ out_counts) {
  uint64_t q = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  uint32_t lane = threadIdx.x & 31;
  if (q >= nq) return;
  uint32_t cnt = 0;
  for (uint32_t i0 = 0; i0 < k; i0 += 32) {
    uint32_t i = i0 + lane;
    uint64_t key = i < k ? run_keys[q * k + i] : kMaxKey;
    bool ok = key != kMaxKey;
    if (i < k) {
      out_labels[q * k + i] = ok ? labels[(uint32_t)key] : 0xFFFFFFFFFFFFFFFFull;
      if (out_dists) out_dists[q * k + i] = ok ? key_dist(key) : INFINITY;
    }
    cnt += __popc(__ballot_sync(0xffffffffu, ok));
  }
  if (lane == 0 && out_counts) out_counts[q] = cnt;
}

cudaError_t launch_bruteforce_exact(const float* vecs, uint32_t dpad, uint32_t dim, uint64_t n, const uint64_t* labels,
                                    int metric, const float* qpad /*[nq][dpad]*/, uint64_t nq, uint32_t k,
                                    BruteScratch& sc, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                                    cudaStream_t s) {
  return launch_bruteforce(vecs, dpad, dim, n, labels, metric, qpad, nq, k, sc, nullptr, out_labels, out_dists,
                           out_counts, s);
}

// Shared driver of the exact path (bf == nullptr: fp32 distance tiles, keys are final) and of the
// tensor-core path (bf != nullptr: bf16 GEMM tiles select bf->kc >= k candidates per query, then an
// fp32 re-rank with the canonical arithmetic picks the k results).
cudaError_t launch_bruteforce(const float* vecs, uint32_t dpad, uint32_t dim, uint64_t n, const uint64_t* labels,
                              int metric, const float* qpad, uint64_t nq, uint32_t k, BruteScratch& sc,
                              const Bf16Ctx* bf, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                              cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  const uint32_t ksel = bf ? bf->kc : k;
  const uint32_t kpad = align_up(ksel, 32);
  const uint32_t wpb = 4;
  size_t smem = (size_t)wpb * kpad * 8;
  cudaError_t e;
  if (smem > 48 * 1024) {
    e = cudaFuncSetAttribute(bf_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(bf_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  {
    uint64_t tot = nq * ksel;
    bf_fill_keys_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(sc.run_keys, tot);
  }
  // distance tiles -> HBM -> per-slice select -> merge into run_keys, over base rows [nb, ne)
  auto unfused_range = [&](uint64_t nb, uint64_t ne) -> cudaError_t {
    for (uint64_t q0 = 0; q0 < nq; q0 += sc.qb) {
      uint64_t qn = sc.qb < nq - q0 ? sc.qb : nq - q0;
      for (uint64_t n0 = nb; n0 < ne; n0 += sc.nc) {
        uint64_t nn = sc.nc < ne - n0 ? sc.nc : ne - n0;
        if (bf) {
          cudaError_t e2 = launch_bf16_dist_tile(bf->q_bf16, nq, bf->x_bf16, n, dpad, metric, bf->qnorm, bf->xnorm, q0,
                                                 qn, n0, nn, sc.dist, sc.nc, s);
          if (e2 != cudaSuccess) return e2;
        } else {
          dim3 grid((unsigned)((nn + TN - 1) / TN), (unsigned)((qn + TQ - 1) / TQ));
          if (metric == 0)
            bf_dist_kernel<0><<<grid, 256, 0, s>>>(qpad, vecs, dpad, q0, qn, n0, nn, sc.dist, sc.nc);
          else
            bf_dist_kernel<1><<<grid, 256, 0, s>>>(qpad, vecs, dpad, q0, qn, n0, nn, sc.dist, sc.nc);
        }
        // one warp per (query, slice): as few slices as still fill the machine (~4096 warps) — every slice
        // sorts its own top-k from scratch, so slices multiply the insert work
        uint64_t want_sl = (4096 + qn - 1) / qn;
        if (want_sl > nn / 1024) want_sl = nn / 1024 ? nn / 1024 : 1;
        uint32_t slices = (uint32_t)(want_sl < sc.slices ? want_sl : sc.slices);
        if (slices == 0) slices = 1;
        uint64_t jobs = qn * slices;
        bf_select_kernel<<<(unsigned)((jobs + wpb - 1) / wpb), 32 * wpb, smem, s>>>(
            sc.dist, sc.nc, nn, n0, qn, slices, ksel, sc.part_keys, sc.run_keys, q0, sc.deleted);
        bf_merge_kernel<<<(unsigned)((qn + wpb - 1) / wpb), 32 * wpb, smem, s>>>(sc.run_keys, sc.part_keys, q0, qn,
                                                                                slices, ksel);
      }
    }
    return cudaGetLastError();
  };
  if (bf && bf->fused && n > 8192) {
    // bootstrap thresholds on the first rows, then fused chunks that double in size: a chunk as large as
    // everything seen so far admits about kc survivors per query
    const uint64_t s0 = 8192;
    if ((e = cudaMemsetAsync(bf->ccount, 0, nq * 4, s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(bf->overflow, 0, 4, s)) != cudaSuccess) return e;
    if ((e = unfused_range(0, s0)) != cudaSuccess) return e;
    // compaction with empty buffers publishes thr[q] from the bootstrap lists
    e = launch_bf16_topk_chunk(bf->q_bf16, nq, bf->x_bf16, n, dpad, metric, bf->qnorm, bf->xnorm, 0, 0, bf->thr,
                               bf->cbuf, bf->ccount, bf->ccap, sc.run_keys, ksel, bf->overflow, bf->sms, s);
    if (e != cudaSuccess) return e;
    uint64_t seen = s0;
    while (seen < n) {
      uint64_t chunk = n - seen < seen ? n - seen : seen;
      e = launch_bf16_topk_chunk(bf->q_bf16, nq, bf->x_bf16, n, dpad, metric, bf->qnorm, bf->xnorm, seen,
                                 seen + chunk, bf->thr, bf->cbuf, bf->ccount, bf->ccap, sc.run_keys, ksel,
                                 bf->overflow, bf->sms, s);
      if (e != cudaSuccess) return e;
      uint32_t ovf = 0;
      if ((e = cudaMemcpyAsync(&ovf, bf->overflow, 4, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
      if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
      if (ovf) {  // a candidate buffer filled up: redo this chunk through the unfused path (always exact)
        if ((e = cudaMemsetAsync(bf->overflow, 0, 4, s)) != cudaSuccess) return e;
        if ((e = unfused_range(seen, seen + chunk)) != cudaSuccess) return e;
        e = launch_bf16_topk_chunk(bf->q_bf16, nq, bf->x_bf16, n, dpad, metric, bf->qnorm, bf->xnorm, 0, 0, bf->thr,
                                   bf->cbuf, bf->ccount, bf->ccap, sc.run_keys, ksel, bf->overflow, bf->sms, s);
        if (e != cudaSuccess) return e;
      }
      seen += chunk;
    }
  } else {
    if ((e = unfused_range(0, n)) != cudaSuccess) return e;
  }
  if (bf)
    return launch_rerank(sc.run_keys, ksel, qpad, vecs, dpad, dim, metric, labels, nq, k, out_labels, out_dists,
                         out_counts, s);
  bf_finalize_kernel<<<(unsigned)((nq + 3) / 4), 128, 0, s>>>(sc.run_keys, labels, nq, k, out_labels, out_dists,
                                                            out_counts);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// K4: per query, G sorted lists of (dist, label) -> global top-k.  One warp per
// query, lane g walks list g; each step a warp arg-min on (distance, label).
// ---------------------------------------------------------------------------
// (device part: merge.cuh)
__global__ void merge_topk_kernel(uint32_t G, uint64_t nq, uint32_t k, const float* __restrict__ dists,
                                  const uint64_t* __restrict__ labels, uint64_t stride_d, uint64_t stride_l,
                                  float* __restrict__ out_dists, uint64_t* __restrict__ out_labels,
                                  uint32_t* __restrict__ out_counts) {
  uint64_t q = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= nq) return;
  merge_one_query(G, q, threadIdx.x & 31, k, dists, labels, stride_d, stride_l, out_dists, out_labels, out_counts);
}

cudaError_t launch_merge_topk(uint32_t G, uint64_t nq, uint32_t k, const float* dists, const uint64_t* labels,
                              uint64_t stride_d, uint64_t stride_l, float* out_dists, uint64_t* out_labels,
                              uint32_t* out_counts, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  merge_topk_kernel<<<(unsigned)((nq + 3) / 4), 128, 0, s>>>(G, nq, k, dists, labels, stride_d, stride_l, out_dists,
                                                           out_labels, out_counts);
  return cudaGetLastError();
}

}  // namespace ehb
