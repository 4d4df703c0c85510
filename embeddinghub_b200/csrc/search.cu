// K2 — batched k-NN over the HNSW graph, one warp per query.
// Replaces hnswlib::HierarchicalNSW<float>::searchKnn as called from
// ANNIndex::approx_nearest (embeddinghub/embeddingstore/index.cc:39-52).
// The kernel template lives in search_impl.cuh; one translation unit per group
// of row shapes (search_inst_*.cu) keeps the build parallel.
#include <cstdio>

#include "kernels.h"

namespace ehb {

cudaError_t launch_search(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                          uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  if (p.bf16 && (!g.vecs16 || !sink.keys)) return cudaErrorInvalidValue;
  return with_dpad(g.dpad, [&](auto d) {
    constexpr uint32_t D = decltype(d)::value;
    return p.bf16 ? SearchShape<D, __nv_bfloat16>::launch(p, g, queries, nq, k, ef, sink, out_counts, stats, s)
                  : SearchShape<D, float>::launch(p, g, queries, nq, k, ef, sink, out_counts, stats, s);
  });
}

cudaError_t beam_warps(const WalkPlan& p, const GraphView& g, int sms, uint64_t nq, uint32_t* warps) {
  return with_dpad(g.dpad, [&](auto d) {
    constexpr uint32_t D = decltype(d)::value;
    return p.bf16 ? BeamShape<D, __nv_bfloat16>::warps(p, sms, nq, warps) : BeamShape<D, float>::warps(p, sms, nq, warps);
  });
}

cudaError_t resident_warps(const void* kern, uint32_t smem, int sms, uint32_t* out) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int per_sm = 0;
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorInvalidConfiguration;
  *out = (uint32_t)per_sm * (uint32_t)sms;
  return cudaSuccess;
}

cudaError_t launch_search_beam(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                               uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats,
                               uint32_t* vtab, uint32_t warps, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  if (p.bf16 && (!g.vecs16 || !sink.keys)) return cudaErrorInvalidValue;
  return with_dpad(g.dpad, [&](auto d) {
    constexpr uint32_t D = decltype(d)::value;
    return p.bf16 ? BeamShape<D, __nv_bfloat16>::launch(p, g, queries, nq, k, ef, sink, out_counts, stats, vtab, warps, s)
                  : BeamShape<D, float>::launch(p, g, queries, nq, k, ef, sink, out_counts, stats, vtab, warps, s);
  });
}

// (HASDEL and ROW are named only when set, so the common instantiations keep their short names)
void walk_kernel_name(const WalkPlan& p, char* out, size_t out_bytes) {
  if (p.form == WalkForm::team)
    std::snprintf(out, out_bytes, "hnsw_search_team_kernel<NQ=%d,KPL=%d,T=%u,U=%u>", p.nq, p.kpl, p.T, p.U);
  else if (p.form == WalkForm::beam)
    std::snprintf(out, out_bytes, "hnsw_search_beam_kernel<LPV=%d,NQ=%d%s%s>", p.lpv, p.nq,
                  p.hasdel ? ",HASDEL=1" : "", p.bf16 ? ",ROW=bf16" : "");
  else
    std::snprintf(out, out_bytes, "%s<LPV=%d,NQ=%d,KPL=%d%s%s>",
                  p.form == WalkForm::dense  ? "hnsw_search_dense_kernel"
                  : p.form == WalkForm::wide ? "hnsw_search_wide_kernel"
                                             : "hnsw_search_kernel",
                  p.lpv, p.nq, p.kpl, p.hasdel ? ",HASDEL=1" : "", p.bf16 ? ",ROW=bf16" : "");
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

// One warp per row.  The residual r = x - s c is exact in double (s has 24 significant bits, c 7, and x and s c are
// within 31 binades of each other whenever c != 0), so max |r| is exact; the sums of squares are rounded up by far
// more than their double rounding error before they are rounded up to fp32.
__global__ void to_i8_rows_kernel(const float* __restrict__ in, uint32_t dpad, int8_t* __restrict__ codes,
                                  float4* __restrict__ terms, uint64_t n) {
  const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint32_t lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* src = in + row * dpad;
  float mx = 0.f;
  bool finite = true;
  for (uint32_t i = 4 * lane; i < dpad; i += 128) {
    const float4 v = *(const float4*)(src + i);
    finite = finite && isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w);
    mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  finite = __all_sync(0xffffffffu, finite);
  mx = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(mx)));  // >= 0: ordered as its bits
  const float s = (float)((double)mx / 127.0);
  const bool bad = !finite || (s != 0.f && s < 0x1p-126f);  // never rejected: NaN terms
  const double sd = s;
  double rinf = 0.0, r2 = 0.0, x2 = 0.0;
  for (uint32_t i = 4 * lane; i < dpad; i += 128) {
    const float4 v = *(const float4*)(src + i);
    const float xv[4] = {v.x, v.y, v.z, v.w};
    uint32_t packed = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double x = xv[j];
      const double c = bad || s == 0.f ? 0.0 : fmin(fmax(rint(x / sd), -127.0), 127.0);
      const double r = x - sd * c;
      rinf = fmax(rinf, fabs(r));
      r2 = fma(r, r, r2);
      x2 = fma(x, x, x2);
      packed |= (uint32_t)(uint8_t)(int8_t)c << (8 * j);
    }
    *(uint32_t*)(codes + row * dpad + i) = packed;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    rinf = fmax(rinf, __shfl_xor_sync(0xffffffffu, rinf, o));
    r2 += __shfl_xor_sync(0xffffffffu, r2, o);
    x2 += __shfl_xor_sync(0xffffffffu, x2, o);
  }
  if (lane == 0) {
    const double up = 1.0 + 0x1p-30;
    terms[row] = bad ? make_float4(NAN, NAN, NAN, NAN)
                     : make_float4(s, __double2float_ru(rinf), __double2float_ru(sqrt(r2) * up),
                                   __double2float_ru(sqrt(x2) * up));
  }
}

cudaError_t launch_to_i8(const float* in, uint32_t dpad, int8_t* codes, float4* terms, uint64_t n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  to_i8_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, s>>>(in, dpad, codes, terms, n);
  return cudaGetLastError();
}

// per query: hops_upper, hops_base, evals, overflow flag, screened, survivors, screened_upper, 0 -> sums (overflow:
// queries)
__global__ void sum_stats_kernel(const uint32_t* __restrict__ stats, uint32_t nq, unsigned long long* out) {
  unsigned long long a[kStatWords] = {};
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
    const uint4 s = ((const uint4*)stats)[2 * i], t = ((const uint4*)stats)[2 * i + 1];
    a[0] += s.x, a[1] += s.y, a[2] += s.z, a[3] += s.w ? 1 : 0, a[4] += t.x, a[5] += t.y, a[6] += t.z;
  }
#pragma unroll
  for (int j = 0; j < 7; ++j) {
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
