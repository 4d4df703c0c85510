// K2 — batched k-NN over the HNSW graph, one warp per query.
// Replaces hnswlib::HierarchicalNSW<float>::searchKnn as called from
// ANNIndex::approx_nearest (embeddinghub/embeddingstore/index.cc:39-52).
// The kernel template lives in search_impl.cuh; one translation unit per group
// of row shapes (search_inst_*.cu) keeps the build parallel.
#include "search_impl.cuh"

namespace ehb {

cudaError_t launch_search(EHB_SEARCH_ARGS) {
  if (nq == 0) return cudaSuccess;
  switch (g.dpad) {
    case 32: return launch_search_d32(EHB_SEARCH_PASS);
    case 64: return launch_search_d64(EHB_SEARCH_PASS);
    case 128: return launch_search_d128(EHB_SEARCH_PASS);
    case 256: return launch_search_d256(EHB_SEARCH_PASS);
    case 384: return launch_search_d384(EHB_SEARCH_PASS);
    case 512: return launch_search_d512(EHB_SEARCH_PASS);
    case 768: return launch_search_d768(EHB_SEARCH_PASS);
    case 1024: return launch_search_d1024(EHB_SEARCH_PASS);
    case 1536: return launch_search_d1536(EHB_SEARCH_PASS);
    case 2048: return launch_search_d2048(EHB_SEARCH_PASS);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_search_bf16(EHB_SEARCH_ARGS) {
  if (nq == 0) return cudaSuccess;
  if (!g.vecs16 || !sink.keys) return cudaErrorInvalidValue;
  switch (g.dpad) {
    case 32: return launch_search_bf16_d32(EHB_SEARCH_PASS);
    case 64: return launch_search_bf16_d64(EHB_SEARCH_PASS);
    case 128: return launch_search_bf16_d128(EHB_SEARCH_PASS);
    case 256: return launch_search_bf16_d256(EHB_SEARCH_PASS);
    case 384: return launch_search_bf16_d384(EHB_SEARCH_PASS);
    case 512: return launch_search_bf16_d512(EHB_SEARCH_PASS);
    case 768: return launch_search_bf16_d768(EHB_SEARCH_PASS);
    case 1024: return launch_search_bf16_d1024(EHB_SEARCH_PASS);
    case 1536: return launch_search_bf16_d1536(EHB_SEARCH_PASS);
    case 2048: return launch_search_bf16_d2048(EHB_SEARCH_PASS);
    default: return cudaErrorInvalidValue;
  }
}

// ---------------------------------------------------------------------------
// Row utilities.  Normalisation follows hnswlib's Python binding
// (normalize_vector): inv = 1 / (sqrt(sum x^2) + 1e-30), one sequential fp32 FMA
// chain per row so that the exact path is reproducible bit-for-bit.
// ---------------------------------------------------------------------------
__global__ void pad_rows_kernel(const float* __restrict__ in, float* __restrict__ out, uint64_t n, uint32_t dim,
                                uint32_t dpad, int normalize) {
  // one warp per row: lanes cooperate on the copy; lane 0 owns the canonical norm chain
  uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  uint32_t lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* src = in + row * dim;
  float* dst = out + row * dpad;
  float inv = 1.0f;
  if (normalize) {
    float acc = 0.f;
    if (lane == 0) {
      for (uint32_t i = 0; i < dim; ++i) acc = fmaf(src[i], src[i], acc);
      inv = 1.0f / (sqrtf(acc) + 1e-30f);
    }
    inv = __shfl_sync(0xffffffffu, inv, 0);
  }
  for (uint32_t i = lane; i < dpad; i += 32) dst[i] = i < dim ? (normalize ? src[i] * inv : src[i]) : 0.f;
}

cudaError_t launch_pad_rows(const float* in, float* out, uint64_t n, uint32_t dim, uint32_t dpad, bool normalize,
                            cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  uint32_t wpb = 8;
  pad_rows_kernel<<<(unsigned)((n + wpb - 1) / wpb), 32 * wpb, 0, s>>>(in, out, n, dim, dpad, normalize ? 1 : 0);
  return cudaGetLastError();
}

cudaError_t launch_normalize(const float* in, uint32_t in_stride, float* out, uint32_t out_stride, uint64_t n,
                             uint32_t dim, cudaStream_t s) {
  (void)in_stride;
  return launch_pad_rows(in, out, n, dim, out_stride, true, s);
}

// per query: hops_upper, hops_base, evals, overflow flag, screened, survivors, 0, 0 -> sums (overflow: queries)
__global__ void sum_stats_kernel(const uint32_t* __restrict__ stats, uint32_t nq, unsigned long long* out) {
  unsigned long long a[kStatWords] = {};
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
    const uint4 s = ((const uint4*)stats)[2 * i], t = ((const uint4*)stats)[2 * i + 1];
    a[0] += s.x, a[1] += s.y, a[2] += s.z, a[3] += s.w ? 1 : 0, a[4] += t.x, a[5] += t.y;
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    for (int o = 16; o > 0; o >>= 1) a[j] += __shfl_xor_sync(0xffffffffu, a[j], o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&out[j], a[j]);
  }
}

cudaError_t launch_sum_stats(const uint32_t* stats, uint32_t nq, unsigned long long* out, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(out, 0, kStatWords * sizeof(unsigned long long), s);
  if (e != cudaSuccess) return e;
  if (nq) sum_stats_kernel<<<64, 256, 0, s>>>(stats, nq, out);
  return cudaGetLastError();
}

}  // namespace ehb
