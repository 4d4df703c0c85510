// K3 — brute-force distances as a bf16 tensor-core GEMM (Hopper wgmma + TMA).
//
// The batched exact scan is a genuine dense contraction: D[q][n] = <Q[q], X[n]> over
// d, Q x N x d multiply-adds (C4: 4096 x 10M x 768 = 3.1e13 MACs).  These kernels
// compute 128 x 256 tiles of it on the sm_90a warpgroup tensor cores:
//   warpgroup 0   : TMA producer — one thread issues cp.async.bulk.tensor.2d of a 128 x 64 bf16
//                   query box and a 256 x 64 bf16 base box per k-block, 128B-swizzled, into a
//                   4-stage shared-memory ring (48 KB a stage), completion on mbarriers;
//   warpgroups 1-2: consumers — each issues wgmma.mma_async m64n256k16 (bf16 in, fp32 out) for its
//                   64 query rows of the tile straight from the swizzled stages, with the 64 x 256
//                   fp32 accumulator in registers (128 a thread; setmaxnreg moves registers from the
//                   producer), releases each stage once the wgmma that read it has retired, then turns
//                   the dot products into distances (1 - dot, or |q|^2 + |x|^2 - 2 dot).
// The candidate selection (top-k' per query over the tile rows), and the fp32
// re-rank that restores exact ids, reuse the K1 select / merge kernels
// (bruteforce.cu) and rerank_kernel below.
//
// Replaces: hnswlib::BruteforceSearch semantics on the "bf16 tensor-core GEMM path"
// named by BASELINE.json (configs[3]); the reference itself has no such path.
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdlib>

#include "kernels.h"

namespace ehb {

constexpr int GM = 128, GN = 256, GK = 64, GSTAGES = 4;
constexpr int kGemmThreads = 384;  // producer warpgroup + two consumer warpgroups
constexpr uint32_t kStageBytesA = GM * GK * 2, kStageBytesB = GN * GK * 2;
constexpr uint32_t kGemmSmem = GSTAGES * (kStageBytesA + kStageBytesB) + 1024 /*align*/ + 256 /*barriers*/;

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
__device__ __forceinline__ void fence_acc(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, both operands K-major bf16 in shared memory, fp32 accumulate
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(1u));
}

// K-major, 128B-swizzled operand tile (rows of 64 bf16 = 128 B, 8-row swizzle atoms of 1024 B):
// start address >> 4, SBO = 1024 B >> 4, layout type SWIZZLE_128B (1 in the sm_90 encoding).
__device__ __forceinline__ uint64_t make_smem_desc(const void* smem_tile) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_u32(smem_tile) & 0x3FFFFu) >> 4);  // bits [0,14)
  d |= (uint64_t)1 << 16;                                   // leading byte offset: unused for swizzled K-major
  d |= (uint64_t)(1024u >> 4) << 32;                        // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                                   // SWIZZLE_128B
  return d;
}

// The operand ring shared by both GEMM kernels: full[s] completes on the TMA bytes, empty[s] on one arrival
// from each consumer warpgroup.
struct GemmRing {
  unsigned char* sA;  // [stage][128 x 64] query rows
  unsigned char* sB;  // [stage][256 x 64] base rows
  uint64_t* full;
  uint64_t* empty;
};

__device__ __forceinline__ GemmRing gemm_ring_setup(unsigned char* smem_raw, const CUtensorMap* mq,
                                                    const CUtensorMap* mx) {
  unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);  // 128B swizzle: 1 KB align
  GemmRing r;
  r.sA = smem;
  r.sB = smem + GSTAGES * kStageBytesA;
  r.full = (uint64_t*)(smem + GSTAGES * (kStageBytesA + kStageBytesB));
  r.empty = r.full + GSTAGES;
  if (threadIdx.x == 0) {
    for (int s = 0; s < GSTAGES; ++s) mbar_init(&r.full[s], 1), mbar_init(&r.empty[s], 2);
    fence_mbar_init();
    asm volatile("prefetch.tensormap [%0];" ::"l"(mq) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(mx) : "memory");
  }
  __syncthreads();
  return r;
}

// producer: the k-blocks of one (query rows qr, base rows nr) tile; `it` counts ring slots across tiles
__device__ __forceinline__ void gemm_produce(const GemmRing& r, const CUtensorMap* mq, const CUtensorMap* mx,
                                             uint32_t kblocks, int qr, int nr, uint32_t& it) {
  for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
    uint32_t s = it % GSTAGES, ph = (it / GSTAGES) & 1u;
    mbar_wait(&r.empty[s], ph ^ 1u);  // first pass through the ring passes immediately
    mbar_arrive_expect_tx(&r.full[s], kStageBytesA + kStageBytesB);
    tma_load_2d(r.sA + s * kStageBytesA, mq, (int)(kb * GK), qr, &r.full[s]);
    tma_load_2d(r.sB + s * kStageBytesB, mx, (int)(kb * GK), nr, &r.full[s]);
  }
}

// consumer warpgroup wg (0, 1): acc = rows [64 wg, 64 wg + 64) of the 128 x 256 tile.  One wgmma group stays in
// flight: the stage a k-block read is released once the next k-block's group has been issued and the older one
// has retired.
__device__ __forceinline__ void gemm_consume(const GemmRing& r, uint32_t kblocks, uint32_t wg, float (&acc)[128],
                                             uint32_t& it) {
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  const bool signal = (threadIdx.x & 127u) == 0;
  for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
    uint32_t s = it % GSTAGES, ph = (it / GSTAGES) & 1u;
    mbar_wait(&r.full[s], ph);
    uint64_t da = make_smem_desc(r.sA + s * kStageBytesA + wg * (64u * GK * 2)), db = make_smem_desc(r.sB + s * kStageBytesB);
    fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (uint32_t k4 = 0; k4 < GK / 16; ++k4)  // K = 16 bf16 = 32 B = +2 in the (>>4) start address
      wgmma_m64n256k16(acc, da + 2 * k4, db + 2 * k4);
    wgmma_commit();
    wgmma_wait<1>();
    fence_acc(acc);
    if (kb > 0 && signal) mbar_arrive(&r.empty[(it - 1) % GSTAGES]);
  }
  wgmma_wait<0>();
  fence_acc(acc);
  if (kblocks > 0 && signal) mbar_arrive(&r.empty[(it - 1) % GSTAGES]);
}

// Accumulator fragment of thread (warp w, lane l) of a consumer warpgroup: acc[4 j + 2 h + e] holds row
// 16 w + l / 4 + 8 h of the warpgroup's 64 rows, column 8 j + 2 (l % 4) + e of the tile's 256.

// dist[(q - q0) * ldd + (n - n0)], q in [q0, q0 + qn), n in [n0, n0 + nn).
// metric 0: qnorm[q] + xnorm[n] - 2 dot;  metric 1: 1 - dot.
__global__ void __launch_bounds__(kGemmThreads, 1)
    bf16_dist_gemm_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x,
                          uint32_t kblocks, int metric, const float* __restrict__ qnorm,
                          const float* __restrict__ xnorm, uint64_t q0, uint64_t qn, uint64_t n0, uint64_t nn,
                          float* __restrict__ dist, uint64_t ldd) {
  extern __shared__ unsigned char smem_raw[];
  const GemmRing r = gemm_ring_setup(smem_raw, &map_q, &map_x);
  // query tiles vary fastest: the CTAs that share one 256-row base tile run together, so the base set is
  // read from HBM about once per chunk
  const uint32_t tile_q = blockIdx.x, tile_n = blockIdx.y;
  const uint32_t wg = threadIdx.x >> 7;
  uint32_t it = 0;
  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0)
      gemm_produce(r, &map_q, &map_x, kblocks, (int)(q0 + (uint64_t)tile_q * GM), (int)(n0 + (uint64_t)tile_n * GN), it);
    return;
  }
  setmaxnreg_inc<232>();
  float acc[128];
  gemm_consume(r, kblocks, wg - 1, acc, it);
  const uint32_t t = threadIdx.x & 127u, w = t >> 5, l = t & 31u;
  const uint64_t row0 = (uint64_t)tile_q * GM + (wg - 1) * 64u + w * 16u + (l >> 2);  // relative to q0
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint64_t qrow = row0 + 8u * h;
    if (qrow >= qn) continue;
    const float qn2 = metric == 0 ? qnorm[q0 + qrow] : 0.f;
    float* out = dist + qrow * ldd;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const uint64_t ncol = (uint64_t)tile_n * GN + 8u * j + 2u * (l & 3u);  // relative to n0
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float dot = acc[4 * j + 2 * h + e];
        float xn = (metric == 0 && ncol + e < nn) ? xnorm[n0 + ncol + e] : 0.f;
        v[e] = metric == 0 ? fmaxf(qn2 + xn - 2.0f * dot, 0.f) : 1.0f - dot;
      }
      if (ncol + 2 <= nn && (ldd & 1u) == 0) {
        *(float2*)(out + ncol) = make_float2(v[0], v[1]);
      } else {
        if (ncol < nn) out[ncol] = v[0];
        if (ncol + 1 < nn) out[ncol + 1] = v[1];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Persistent variant with the selection fused into the epilogue: the Q x N distance tile never goes to HBM.
// One CTA per SM walks the (query tile, base tile) list (query tile fastest, so the CTAs that share a base
// tile run together); the producer runs up to four k-blocks ahead, so the loads of tile i+1 overlap the
// epilogue of tile i.  The epilogue compares every distance with the query's current threshold thr[q] (its
// kc-th best bf16 distance so far) and appends the survivors (ordered distance | row index) to the query's
// candidate buffer with one global atomic each; compact_candidates_kernel folds the buffer into the running
// top-kc and tightens thr between chunks.  With chunk sizes that double, a chunk admits about kc candidates
// per query, so the buffer (capacity 2 kc + 64) practically never overflows; if it does the driver re-runs
// that chunk through the unfused path.
// ---------------------------------------------------------------------------------------------------
static cudaError_t make_map(CUtensorMap* map, const void* base, uint64_t rows, uint32_t dpad, uint32_t box_rows);

__global__ void __launch_bounds__(kGemmThreads, 1)
    bf16_topk_gemm_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x,
                          uint32_t kblocks, int metric, const float* __restrict__ qnorm,
                          const float* __restrict__ xnorm, uint64_t nq, uint64_t n_lo, uint64_t n_hi,
                          const float* __restrict__ thr, uint64_t* __restrict__ cbuf, uint32_t* __restrict__ ccount,
                          uint32_t ccap) {
  extern __shared__ unsigned char smem_raw[];
  const GemmRing r = gemm_ring_setup(smem_raw, &map_q, &map_x);
  const uint64_t q_tiles = (nq + GM - 1) / GM, n_tiles = (n_hi - n_lo + GN - 1) / GN;
  const uint64_t tiles = q_tiles * n_tiles;
  const uint32_t wg = threadIdx.x >> 7;
  uint32_t it = 0;
  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0)
      for (uint64_t t = blockIdx.x; t < tiles; t += gridDim.x)
        gemm_produce(r, &map_q, &map_x, kblocks, (int)((t % q_tiles) * GM), (int)(n_lo + (t / q_tiles) * GN), it);
    return;
  }
  setmaxnreg_inc<232>();
  const uint32_t t_ = threadIdx.x & 127u, w = t_ >> 5, l = t_ & 31u;
  float acc[128];
  for (uint64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint64_t tq = t % q_tiles, tn = t / q_tiles;
    gemm_consume(r, kblocks, wg - 1, acc, it);
    uint64_t q[2];
    float tau[2], qn2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      q[h] = tq * GM + (wg - 1) * 64u + w * 16u + (l >> 2) + 8u * h;
      const bool qok = q[h] < nq;
      tau[h] = qok ? thr[q[h]] : -INFINITY;
      qn2[h] = (metric == 0 && qok) ? qnorm[q[h]] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const uint64_t nb = n_lo + tn * GN + 8u * j + 2u * (l & 3u);
      float xn[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) xn[e] = (metric == 0 && nb + e < n_hi) ? xnorm[nb + e] : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float dot = acc[4 * j + 2 * h + e];
          float d = metric == 0 ? fmaxf(qn2[h] + xn[e] - 2.0f * dot, 0.f) : 1.0f - dot;
          if (d < tau[h] && nb + e < n_hi) {
            uint32_t pos = atomicAdd(&ccount[q[h]], 1u);
            if (pos < ccap) cbuf[q[h] * ccap + pos] = make_key(d, (uint32_t)(nb + e));
          }
        }
      }
    }
  }
}

// One warp per query: fold the candidate buffer into the running top-kc, publish the new threshold, reset
// the counter; overflow[0] != 0 tells the driver the buffer was too small.  The (<= kc + ccap) keys are
// sorted with a warp-wide bitonic network in shared memory (P = next power of two; ~20 k instructions per
// query for P = 2048, 4x cheaper than ~kc sorted inserts into a kc-long list).
__global__ void compact_candidates_kernel(uint64_t* __restrict__ run_keys, uint64_t* __restrict__ cbuf,
                                          uint32_t* __restrict__ ccount, uint32_t ccap, uint32_t kc, uint32_t P,
                                          uint64_t nq, float* __restrict__ thr, uint32_t* __restrict__ overflow) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5, wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  const uint64_t q = (uint64_t)blockIdx.x * wpb + w;
  if (q >= nq) return;
  uint64_t* keys = (uint64_t*)smem + (size_t)w * P;
  uint64_t* run = run_keys + q * kc;
  uint32_t m = ccount[q];
  if (m > ccap) {
    if (lane == 0) atomicExch(overflow, 1u);
    m = ccap;
  }
  for (uint32_t i = lane; i < P; i += 32) {
    uint64_t key = kMaxKey;
    if (i < kc) key = run[i];
    else if (i - kc < m) key = cbuf[q * ccap + (i - kc)];
    keys[i] = key;
  }
  __syncwarp();
  for (uint32_t size = 2; size <= P; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = lane; t < (P >> 1); t += 32) {
        uint32_t i = 2 * t - (t & (stride - 1));     // lower index of the pair
        uint32_t j = i + stride;
        bool up = (i & size) == 0;                   // ascending blocks
        uint64_t a = keys[i], b = keys[j];
        if ((a > b) == up) keys[i] = b, keys[j] = a;
      }
      __syncwarp();
    }
  }
  for (uint32_t i = lane; i < kc; i += 32) run[i] = keys[i];
  if (lane == 0) {
    thr[q] = keys[kc - 1] != kMaxKey ? key_dist(keys[kc - 1]) : INFINITY;
    ccount[q] = 0;
  }
}

cudaError_t launch_bf16_topk_chunk(const void* q_bf16, uint64_t nq, const void* x_bf16, uint64_t x_rows, uint32_t dpad,
                                   int metric, const float* qnorm, const float* xnorm, uint64_t n_lo, uint64_t n_hi,
                                   float* thr, uint64_t* cbuf, uint32_t* ccount, uint32_t ccap, uint64_t* run_keys,
                                   uint32_t kc, uint32_t* overflow, int sms, cudaStream_t s) {
  if (dpad % GK != 0) return cudaErrorInvalidValue;
  CUtensorMap mq, mx;
  cudaError_t e;
  if ((e = make_map(&mq, q_bf16, nq, dpad, GM)) != cudaSuccess) return e;
  if ((e = make_map(&mx, x_bf16, x_rows, dpad, GN)) != cudaSuccess) return e;
  e = cudaFuncSetAttribute(bf16_topk_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmem);
  if (e != cudaSuccess) return e;
  if (n_hi > n_lo) {
    uint64_t tiles = ((nq + GM - 1) / GM) * ((n_hi - n_lo + GN - 1) / GN);
    unsigned grid = (unsigned)(tiles < (uint64_t)sms ? tiles : (uint64_t)sms);
    bf16_topk_gemm_kernel<<<grid, kGemmThreads, kGemmSmem, s>>>(mq, mx, dpad / GK, metric == 0 ? 0 : 1, qnorm, xnorm,
                                                                nq, n_lo, n_hi, thr, cbuf, ccount, ccap);
  }
  // fold the survivors into the running top-kc
  uint32_t P = 64;
  while (P < kc + ccap) P <<= 1;
  uint32_t wpb = (uint32_t)(65536u / (P * 8u));
  wpb = wpb < 1 ? 1 : (wpb > 8 ? 8 : wpb);
  size_t smem = (size_t)wpb * P * 8;
  e = cudaFuncSetAttribute(compact_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  compact_candidates_kernel<<<(unsigned)((nq + wpb - 1) / wpb), 32 * wpb, smem, s>>>(run_keys, cbuf, ccount, ccap, kc,
                                                                                     P, nq, thr, overflow);
  return cudaGetLastError();
}

// ---- fp32 -> bf16 rows (+ squared norms of the rounded values) ------------------------------------
__global__ void to_bf16_rows_kernel(const float* __restrict__ in, uint32_t in_stride, __nv_bfloat16* __restrict__ out,
                                    float* __restrict__ norms, uint64_t n, uint32_t dpad) {
  uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  uint32_t lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* src = in + row * in_stride;
  float acc = 0.f;
  for (uint32_t i = lane; i < dpad; i += 32) {
    __nv_bfloat16 b = __float2bfloat16_rn(src[i]);
    out[row * dpad + i] = b;
    float f = __bfloat162float(b);
    acc = fmaf(f, f, acc);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0 && norms) norms[row] = acc;
}

cudaError_t launch_to_bf16(const float* in, uint32_t in_stride, void* out_bf16, float* norms, uint64_t n, uint32_t dpad,
                           cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  to_bf16_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, s>>>(in, in_stride, (__nv_bfloat16*)out_bf16, norms, n, dpad);
  return cudaGetLastError();
}

// ---- tensor maps -------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static cudaError_t make_map(CUtensorMap* map, const void* base, uint64_t rows, uint32_t dpad, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess) return e;
    if (qres != cudaDriverEntryPointSuccess || !p) return cudaErrorNotSupported;
    fn = (EncodeTiledFn)p;
  }
  cuuint64_t dims[2] = {dpad, rows};
  cuuint64_t strides[1] = {(cuuint64_t)dpad * 2};
  cuuint32_t box[2] = {(cuuint32_t)GK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// distances of queries [q0, q0+qn) x base rows [n0, n0+nn) into dist (row stride ldd)
cudaError_t launch_bf16_dist_tile(const void* q_bf16, uint64_t q_rows, const void* x_bf16, uint64_t x_rows,
                                  uint32_t dpad, int metric, const float* qnorm, const float* xnorm, uint64_t q0,
                                  uint64_t qn, uint64_t n0, uint64_t nn, float* dist, uint64_t ldd, cudaStream_t s) {
  if (dpad % GK != 0) return cudaErrorInvalidValue;
  CUtensorMap mq, mx;
  cudaError_t e;
  if ((e = make_map(&mq, q_bf16, q_rows, dpad, GM)) != cudaSuccess) return e;
  if ((e = make_map(&mx, x_bf16, x_rows, dpad, GN)) != cudaSuccess) return e;
  e = cudaFuncSetAttribute(bf16_dist_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmem);
  if (e != cudaSuccess) return e;
  dim3 grid((unsigned)((qn + GM - 1) / GM), (unsigned)((nn + GN - 1) / GN));
  bf16_dist_gemm_kernel<<<grid, kGemmThreads, kGemmSmem, s>>>(mq, mx, dpad / GK, metric == 0 ? 0 : 1, qnorm, xnorm, q0, qn, n0,
                                                    nn, dist, ldd);
  return cudaGetLastError();
}

// ---- fp32 re-rank of the bf16 candidates (canonical arithmetic, total order (dist, index)) ----------------
// One warp per query: candidates cand[q][kc] (keys from the select pass: low 32 bits = row index), exact
// distance per candidate by lane-strided loop over candidates (each lane runs the sequential FMA chain),
// then the k best by repeated warp arg-min.  kSink: the results go to every destination of `sink` (sink_store and
// sink_query_done, walk.cuh) instead of out_labels / out_dists: the k selected keys are collected in shared memory
// first (the row tile is free by then), then every lane stores its elements of the list to each destination,
// coalesced.
template <bool kSink>
__device__ __forceinline__ void rerank_body(const uint64_t* __restrict__ cand, uint32_t kc, const float* __restrict__ qpad,
                                            const float* __restrict__ vecs, uint32_t dpad, uint32_t dim, int metric,
                                            const uint64_t* __restrict__ labels, uint64_t nq, uint32_t k,
                                            uint64_t* __restrict__ out_labels, float* __restrict__ out_dists,
                                            const ResultSink& sink, uint32_t* __restrict__ out_counts) {
  extern __shared__ uint64_t skeys[];  // [wpb][kc] keys, then [wpb][32][33] row tile, [wpb][32] query segment
  const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const uint64_t q = (uint64_t)blockIdx.x * wpb + w;
  if (q >= nq) return;
  uint64_t* keys = skeys + (size_t)w * kc;
  float* tile = (float*)(skeys + (size_t)wpb * kc) + (size_t)w * (32 * 33 + 32);
  float* qseg = tile + 32 * 33;
  uint64_t* sel = (uint64_t*)tile;  // kSink: the selected keys (the tile and query segment hold 544 >= kMaxEf)
  const float* qv = qpad + q * dpad;
  // 32 candidates at a time: rows are staged 32 floats per row per step with coalesced loads, then every
  // lane advances the canonical (k ascending, single accumulator) chain of ITS candidate by 32 terms
  for (uint32_t c0 = 0; c0 < kc; c0 += 32) {
    uint32_t c = c0 + lane;
    uint64_t ck = c < kc ? cand[q * kc + c] : kMaxKey;
    uint32_t idx = ck != kMaxKey ? (uint32_t)ck : 0u;
    float acc = 0.f;
    for (uint32_t s0 = 0; s0 < dim; s0 += 32) {
      __syncwarp();
#pragma unroll 8
      for (uint32_t r = 0; r < 32; ++r) {
        uint32_t ridx = __shfl_sync(0xffffffffu, idx, r);
        tile[r * 33 + lane] = s0 + lane < dim ? vecs[(size_t)ridx * dpad + s0 + lane] : 0.f;
      }
      qseg[lane] = s0 + lane < dim ? qv[s0 + lane] : 0.f;
      __syncwarp();
      const uint32_t lim = min(32u, dim - s0);
      if (metric == 0) {
        for (uint32_t i = 0; i < lim; ++i) {
          float t = qseg[i] - tile[lane * 33 + i];
          acc = fmaf(t, t, acc);
        }
      } else {
        for (uint32_t i = 0; i < lim; ++i) acc = fmaf(qseg[i], tile[lane * 33 + i], acc);
      }
    }
    if (c < kc) keys[c] = ck != kMaxKey ? make_key(metric == 0 ? acc : 1.0f - acc, idx) : kMaxKey;
  }
  __syncwarp();
  uint32_t found = 0;
  for (uint32_t i = 0; i < k; ++i) {
    uint64_t best = kMaxKey;
    uint32_t bpos = 0;
    for (uint32_t c = lane; c < kc; c += 32)
      if (keys[c] < best) best = keys[c], bpos = c;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      uint64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
      uint32_t op = __shfl_xor_sync(0xffffffffu, bpos, o);
      if (ob < best) best = ob, bpos = op;
    }
    if (best == kMaxKey) break;
    if (lane == 0) {
      if constexpr (kSink) {
        sel[i] = best;
      } else {
        out_labels[q * k + i] = labels[(uint32_t)best];
        if (out_dists) out_dists[q * k + i] = key_dist(best);
      }
      keys[bpos] = kMaxKey;
    }
    __syncwarp();
    found++;
  }
  if constexpr (kSink) {
    for (uint32_t i = found + lane; i < k; i += 32) sel[i] = kMaxKey;
    __syncwarp();
    for (uint32_t i = lane; i < k; i += 32) {
      const uint64_t key = sel[i];
      const bool ok = key != kMaxKey;
      sink_store(sink, (size_t)q * k + i, ok ? labels[(uint32_t)key] : 0xFFFFFFFFFFFFFFFFull,
                 ok ? key_dist(key) : INFINITY);
    }
    sink_query_done(sink, (uint32_t)q, (uint32_t)nq, lane);
  } else {
    for (uint32_t i = found + lane; i < k; i += 32) {
      out_labels[q * k + i] = 0xFFFFFFFFFFFFFFFFull;
      if (out_dists) out_dists[q * k + i] = INFINITY;
    }
  }
  if (lane == 0 && out_counts) out_counts[q] = found;
}

__global__ void rerank_kernel(const uint64_t* __restrict__ cand, uint32_t kc, const float* __restrict__ qpad,
                              const float* __restrict__ vecs, uint32_t dpad, uint32_t dim, int metric,
                              const uint64_t* __restrict__ labels, uint64_t nq, uint32_t k,
                              uint64_t* __restrict__ out_labels, float* __restrict__ out_dists,
                              uint32_t* __restrict__ out_counts) {
  rerank_body<false>(cand, kc, qpad, vecs, dpad, dim, metric, labels, nq, k, out_labels, out_dists, ResultSink{},
                     out_counts);
}

// The re-rank of a bf16 graph walk that is the last kernel of a sharded search step: destination 0 is this shard's
// block, the others are its block in every peer's receive buffer, and the slice flags rise as queries finish.
__global__ void rerank_sink_kernel(const uint64_t* __restrict__ cand, uint32_t kc, const float* __restrict__ qpad,
                                   const float* __restrict__ vecs, uint32_t dpad, uint32_t dim, int metric,
                                   const uint64_t* __restrict__ labels, uint64_t nq, uint32_t k,
                                   const __grid_constant__ ResultSink sink, uint32_t* __restrict__ out_counts) {
  rerank_body<true>(cand, kc, qpad, vecs, dpad, dim, metric, labels, nq, k, nullptr, nullptr, sink, out_counts);
}

constexpr uint32_t kRerankWarps = 4;
static size_t rerank_smem(uint32_t kc) {
  return (size_t)kRerankWarps * kc * 8 + (size_t)kRerankWarps * (32 * 33 + 32) * 4;
}

cudaError_t launch_rerank(const uint64_t* cand, uint32_t kc, const float* qpad, const float* vecs, uint32_t dpad,
                          uint32_t dim, int metric, const uint64_t* labels, uint64_t nq, uint32_t k,
                          uint64_t* out_labels, float* out_dists, uint32_t* out_counts, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  const uint32_t wpb = kRerankWarps;
  const size_t smem = rerank_smem(kc);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(rerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  rerank_kernel<<<(unsigned)((nq + wpb - 1) / wpb), 32 * wpb, smem, s>>>(cand, kc, qpad, vecs, dpad, dim, metric,
                                                                         labels, nq, k, out_labels, out_dists,
                                                                         out_counts);
  return cudaGetLastError();
}

cudaError_t launch_rerank_sink(const uint64_t* cand, uint32_t kc, const float* qpad, const float* vecs, uint32_t dpad,
                               uint32_t dim, int metric, const uint64_t* labels, uint64_t nq, uint32_t k,
                               const ResultSink& sink, uint32_t* out_counts, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  if (k > kMaxEf || nq > 0xFFFFFFFFull || !sink.n) return cudaErrorInvalidValue;
  const uint32_t wpb = kRerankWarps;
  const size_t smem = rerank_smem(kc);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(rerank_sink_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  rerank_sink_kernel<<<(unsigned)((nq + wpb - 1) / wpb), 32 * wpb, smem, s>>>(cand, kc, qpad, vecs, dpad, dim, metric,
                                                                              labels, nq, k, sink, out_counts);
  return cudaGetLastError();
}

}  // namespace ehb
