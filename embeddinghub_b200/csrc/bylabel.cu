// K7 — searches whose queries are stored points, named by label (ehb_index_search_by_label_ex, the neighbour table,
// ehb_index_get_batch): copy stored rows into a query buffer, list the live ids, and remove each query's own label
// from a k + 1 result list.  The graph walk itself is the existing one (launch_search), fed from the gathered rows.
#include <cmath>

#include "kernels.h"

namespace ehb {

// out[dst ? dst[j] : j][0:dim] = in[src ? src[j] : j][0:dim]; one warp per row, 16-byte moves when both strides and
// dim allow them.
static __global__ void gather_rows_kernel(const float* __restrict__ in, uint32_t in_stride,
                                          const uint32_t* __restrict__ src, float* __restrict__ out,
                                          uint32_t out_stride, const uint32_t* __restrict__ dst, uint64_t n,
                                          uint32_t dim, bool vec4) {
  const uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (j >= n) return;
  const float* a = in + (uint64_t)(src ? src[j] : j) * in_stride;
  float* b = out + (uint64_t)(dst ? dst[j] : j) * out_stride;
  if (vec4) {
    for (uint32_t c = lane; c < dim / 4; c += 32) reinterpret_cast<float4*>(b)[c] = reinterpret_cast<const float4*>(a)[c];
  } else {
    for (uint32_t c = lane; c < dim; c += 32) b[c] = a[c];
  }
}

cudaError_t launch_gather_rows(const float* in, uint32_t in_stride, const uint32_t* src, float* out,
                               uint32_t out_stride, const uint32_t* dst, uint64_t n, uint32_t dim, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const bool vec4 = dim % 4 == 0 && in_stride % 4 == 0 && out_stride % 4 == 0 && ((uintptr_t)in & 15) == 0 &&
                    ((uintptr_t)out & 15) == 0;
  const uint32_t wpb = 8;
  gather_rows_kernel<<<(unsigned)((n + wpb - 1) / wpb), wpb * 32, 0, s>>>(in, in_stride, src, out, out_stride, dst, n,
                                                                         dim, vec4);
  return cudaGetLastError();
}

// One warp per query.  The own label is looked for among the first c entries with a ballot per 32; the output row
// skips it (or, when absent, ends one entry early if c > k: server.cc:204-207) and is padded with
// EHB_NO_LABEL / +inf.
static __global__ void drop_self_kernel(const uint64_t* __restrict__ self, const uint64_t* __restrict__ in_labels,
                                        const float* __restrict__ in_dists, const uint32_t* __restrict__ in_counts,
                                        uint64_t nq, uint32_t k, uint64_t* __restrict__ out_labels,
                                        float* __restrict__ out_dists, uint32_t* __restrict__ out_counts) {
  const uint64_t q = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (q >= nq) return;
  const uint32_t k1 = k + 1;
  const uint64_t* il = in_labels + q * k1;
  const float* id = in_dists + q * k1;
  const uint64_t L = self[q];
  const uint32_t c = min(in_counts[q], k1);
  uint32_t pos = k1;  // position of L in the list, k1 when absent
  for (uint32_t b = 0; b < c && pos == k1; b += 32) {
    const uint32_t j = b + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, j < c && il[j] == L);
    if (hit) pos = b + __ffs(hit) - 1;
  }
  const uint32_t cn = pos < k1 ? c - 1 : min(c, k);
  for (uint32_t j = lane; j < k; j += 32) {
    const uint32_t from = j < pos ? j : j + 1;
    const bool live = j < cn;
    out_labels[q * k + j] = live ? il[from] : ~0ull;
    out_dists[q * k + j] = live ? id[from] : INFINITY;
  }
  if (lane == 0) out_counts[q] = cn;
}

cudaError_t launch_drop_self(const uint64_t* self, const uint64_t* in_labels, const float* in_dists,
                             const uint32_t* in_counts, uint64_t nq, uint32_t k, uint64_t* out_labels,
                             float* out_dists, uint32_t* out_counts, cudaStream_t s) {
  if (nq == 0 || k == 0) return cudaSuccess;
  const uint32_t wpb = 8;
  drop_self_kernel<<<(unsigned)((nq + wpb - 1) / wpb), wpb * 32, 0, s>>>(self, in_labels, in_dists, in_counts, nq, k,
                                                                        out_labels, out_dists, out_counts);
  return cudaGetLastError();
}

cudaError_t load_drop_self() {
  cudaFuncAttributes a;
  return cudaFuncGetAttributes(&a, drop_self_kernel);
}

// One block walks deleted[0..n) in tiles of 16 flags per thread; a block-wide exclusive scan of the live counts
// places each live id, so ids come out ascending in a single pass.
constexpr uint32_t kLiveThreads = 1024;
static __global__ void __launch_bounds__(kLiveThreads) live_ids_kernel(const uint8_t* __restrict__ deleted, uint64_t n,
                                                                       uint32_t* __restrict__ ids,
                                                                       uint32_t* __restrict__ count) {
  __shared__ uint32_t warp_sum[kLiveThreads / 32];
  __shared__ uint32_t base;
  const uint32_t t = threadIdx.x, lane = t & 31, w = t >> 5;
  if (t == 0) base = 0;
  __syncthreads();
  for (uint64_t tile = 0; tile < n; tile += 16ull * kLiveThreads) {
    const uint64_t first = tile + 16ull * t;
    uint32_t mask = 0;  // bit i: id first + i is live
    for (uint32_t i = 0; i < 16; ++i)
      if (first + i < n && !deleted[first + i]) mask |= 1u << i;
    const uint32_t mine = __popc(mask);
    uint32_t incl = mine;
    for (uint32_t o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) warp_sum[w] = incl;
    __syncthreads();
    if (w == 0) {
      uint32_t v = warp_sum[lane], x = v;
      for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += u;
      }
      warp_sum[lane] = x - v;  // exclusive prefix of the warps
    }
    __syncthreads();
    uint32_t at = base + warp_sum[w] + incl - mine;
    for (uint32_t i = 0; i < 16; ++i)
      if (mask >> i & 1u) ids[at++] = (uint32_t)(first + i);
    __syncthreads();
    if (t == kLiveThreads - 1) base = at;
    __syncthreads();
  }
  if (t == 0) *count = base;
}

cudaError_t launch_live_ids(const uint8_t* deleted, uint64_t n, uint32_t* ids, uint32_t* count, cudaStream_t s) {
  live_ids_kernel<<<1, kLiveThreads, 0, s>>>(deleted, n, ids, count);
  return cudaGetLastError();
}

}  // namespace ehb
