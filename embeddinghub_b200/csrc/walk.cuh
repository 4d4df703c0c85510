// Warp-per-query HNSW graph walk machinery (device side).
//
// Replaces hnswlib's searchKnn / searchBaseLayerST / searchBaseLayer hot loops
// (called from embeddinghub/embeddingstore/index.cc:36,41) with a design that
// fits the H100 memory system:
//   * one warp owns one query (or one point being inserted);
//   * an adjacency row is one 128 B line (2M = 32 u32, padded with kInvalid);
//   * hnswlib's ef-bounded result heap and its candidate heap are ONE unordered
//     array of (ordered distance, id | expanded flag) held in registers, KPL
//     entries per lane; the heap tops are warp reductions (redux.sync);
//   * the visited set is a per-warp open-addressing table in shared memory;
//   * distances of the unvisited neighbours of a node are evaluated together:
//       - rows up to 1 KB (LPV = 8 lanes per vector): every lane issues its
//         128-bit loads for up to 16 vectors before the first use, so a hop
//         has 8 KB..16 KB in flight per warp straight into registers;
//       - larger rows (LPV = 32): the TMA engine pulls whole rows HBM -> shared
//         memory (cp.async.bulk, one bulk copy per vector, completion counted
//         on an mbarrier) in a ring of groups, and the math on group r overlaps
//         the copies of the following groups.
//     (Staging every row through TMA makes the walk issue-bound on the
//      per-lane bulk-copy issue loops at d=128.)
//   * rows are padded to an exact multiple of the per-lane tile, so the inner
//     loops carry no bounds checks;
//   * the walk reads either the fp32 rows or their bf16 shadow (RowT = __nv_bfloat16: the bf16 graph
//     search, re-ranked in fp32 afterwards).  The query stays fp32 in registers either way and the same
//     "rows <= 1 KB direct, larger rows TMA" rule applies to the row's bytes;
//   * rows wider than 2048 floats (dpad 3072, 4096: the wide form, eval_wide) keep the fp32 query in the
//     warp's shared-memory slice instead and read the rows straight into registers in d-slices.
#pragma once
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"

namespace ehb {

struct GraphView {
  const float* vecs;         // [n][dpad] fp32, rows 16 B aligned, zero padded
  const uint32_t* links0;    // [n][M0]
  const uint32_t* up_off;    // [n] first upper row of node i, kInvalid if level 0
  const uint32_t* links_up;  // [rows][M]
  const uint64_t* labels;    // [n]
  const uint8_t* deleted;    // [n] tombstones (hnswlib markDelete), nullptr when the index has none
  uint32_t n, dim, dpad, M, M0, entry;
  int32_t max_level;
  int32_t metric;            // 0 = squared L2, 1 = 1 - dot (IP and cosine)
  // [n][dpad] bf16 shadow of vecs, else nullptr.  The bf16 graph search walks it.
  const __nv_bfloat16* vecs16;
  // The int8 screen copy of vecs (launch_to_i8), else nullptr: the fp32 walk (metric 1, staged rows) screens
  // candidates on it when it is set (beam_search).  codes8: [n][dpad] c = RN(x / s) in [-127, 127];
  // terms8: [n] (s, >= max |r_i|, >= |r|_2, >= |x|_2) with r = x - s c (all NaN: the row is never rejected).
  const int8_t* codes8;
  const float4* terms8;
};

struct WalkCfg {
  uint32_t lcap;       // shared-memory key list capacity (0 = none; cold paths only)
  uint32_t hash_size;  // entries of the visited table (multiple of 4), 0 = none
  uint32_t G;          // vectors per TMA staging group (<= 32), LPV = 32 only
  uint32_t NG;         // staging groups (ring depth, <= 8)
  uint32_t staged;     // 1 when the TMA staging ring is allocated
  uint32_t dense;      // 1: launch the low-register form of the walk (more resident warps; rows <= 512 B only)
  uint32_t prefetch;   // 1: pull the speculated next hop's vectors towards L2 (rows <= 1 KB)
  uint32_t dcap;       // capacity of the side queue of admitted-but-deleted candidates (0 = index has no tombstones)
};

// Where a walk writes its [nq][k] results.  Destination 0 is local; in a sharded deployment the others are
// THIS rank's block inside every peer's receive buffer (CUDA-IPC / peer mappings): the walk's epilogue stores
// the results of each query to all of them with coalesced stores over NVLink, and the warp that completes a
// slice of `qs` queries raises that slice's flag on every peer (st.release.sys) — the transfer overlaps the
// rest of the walk, and the merge kernel (exchange.cu) only waits on flags.
constexpr uint32_t kMaxSinks = 16;
struct ResultSink {
  uint64_t* labels[kMaxSinks];
  float* dists[kMaxSinks];     // all null or none
  uint32_t* flags[kMaxSinks];  // [slices] of (parity, this rank) on destination t; unused for t = 0
  uint32_t* slice_count;       // local [slices], zero between steps
  uint32_t n, qs, epoch;       // destinations; queries per slice (0: no flags); value the flags take
  // bf16 walk only (the "key" sink): [nq][k] retained (ordered distance, internal id) keys, nearest-first,
  // kMaxKey past the retained count; launch_rerank turns them into results.  Nothing above is written then.
  uint64_t* keys;
};

// The epilogue of every kernel that ends a graph search in a result sink (the fp32 walk, the re-rank after a bf16
// walk).  sink_store: element `at` of the [nq][k] results to every destination; the lanes of a warp store
// consecutive elements, so each destination gets coalesced stores.  sink_query_done, after all of query q's stores,
// with the whole warp: when the sink has slices, the warp fences its stores system-wide and counts its query in, and
// the warp that completes the slice resets the counter and raises the slice's flag on every peer (t >= 1).
__device__ __forceinline__ void sink_store(const ResultSink& sink, size_t at, uint64_t lab, float dist) {
  for (uint32_t t = 0; t < sink.n; ++t) {
    sink.labels[t][at] = lab;
    if (sink.dists[t]) sink.dists[t][at] = dist;
  }
}
__device__ __forceinline__ void sink_query_done(const ResultSink& sink, uint32_t q, uint32_t nq, uint32_t lane) {
  if (sink.qs) {  // sharded: the warp that completes a slice raises its flag on every peer
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
      const uint32_t slice = q / sink.qs;
      const uint32_t size = min(sink.qs, nq - slice * sink.qs);
      if (atomicAdd(&sink.slice_count[slice], 1u) + 1u == size) {
        sink.slice_count[slice] = 0;  // ready for the next step (which starts after this kernel)
        __threadfence_system();       // the other warps fenced before their atomicAdd: fence-fence ordering
        for (uint32_t t = 1; t < sink.n; ++t) st_release_sys(sink.flags[t] + slice, sink.epoch);
      }
    }
  }
}

__host__ __device__ inline uint32_t align_up(uint32_t x, uint32_t a) { return (x + a - 1) / a * a; }

// ---- Row shapes ------------------------------------------------------------------------------------------
// The padded row lengths (floats) the walk supports, ascending.  A row of `row_bytes` as the walk reads it
// (dpad * 4 for fp32 rows, dpad * 2 for the bf16 shadow) is loaded directly by LPV = 8 lanes per vector up to
// 1 KB, and staged through the TMA ring and read by LPV = 32 lanes above; a lane holds NQ float4 chunks of the
// fp32 query (dpad == 4 * LPV * NQ).  The wide shapes (wide_shape: dpad 3072 and 4096, NQ 24 and 32) hold those
// chunks in shared memory instead, and have no ring (eval_wide).
constexpr uint32_t kPadDims[] = {32, 64, 128, 256, 384, 512, 768, 1024, 1536, 2048, 3072, 4096};
constexpr uint32_t kNumPadDims = sizeof(kPadDims) / sizeof(kPadDims[0]);
__host__ __device__ constexpr int row_lpv(uint32_t row_bytes) { return row_bytes > 1024 ? 32 : 8; }
__host__ __device__ constexpr int row_nq(uint32_t dpad, uint32_t row_bytes) {
  return (int)(dpad / (4u * (uint32_t)row_lpv(row_bytes)));
}
__host__ __device__ constexpr bool wide_shape(int LPV, int NQ) { return LPV == 32 && NQ > 16; }
// register-resident result set entries per lane for a beam of ef (<= 512)
constexpr int kpl_for(uint32_t ef) { return ef <= 64 ? 2 : (ef <= 128 ? 4 : (ef <= 256 ? 8 : 16)); }

inline uint32_t pad_dim(uint32_t dim) {
  for (uint32_t d : kPadDims)
    if (dim <= d) return d;
  return 0;
}

// Calls f(std::integral_constant<uint32_t, DPAD>{}) for the padded row length DPAD == dpad; any other dpad, or one
// above MaxDpad, is cudaErrorInvalidValue.
template <uint32_t MaxDpad = 4096, uint32_t I = 0, class F>
cudaError_t with_dpad(uint32_t dpad, F&& f) {
  if constexpr (I == kNumPadDims || kPadDims[I] > MaxDpad)
    return cudaErrorInvalidValue;
  else
    return dpad == kPadDims[I] ? f(std::integral_constant<uint32_t, kPadDims[I]>{})
                               : with_dpad<MaxDpad, I + 1>(dpad, f);
}

// The fp32 walk's screen applies to staged fp32 rows of dpad 384 .. 1536 (dpad 2048: DESIGN.md §9).
__host__ __device__ constexpr bool screen_shape(int LPV, int NQ) { return LPV == 32 && NQ <= 12; }

// Per-warp shared-memory slice; every region offset is a multiple of 128 B.  esize: bytes per row element as the
// walk reads it (4 for fp32 rows, 2 for the bf16 shadow); dpad * esize sizes the TMA staging ring.  The wide shapes
// have the fp32 query (dpad * 4 bytes) where the ring would be.
__host__ __device__ inline uint32_t warp_smem_bytes(const WalkCfg& c, uint32_t dpad, uint32_t esize) {
  const uint32_t vbytes = dpad * esize;
  uint32_t b = 0;
  if (wide_shape(row_lpv(vbytes), row_nq(dpad, vbytes))) b += dpad * 4u;
  b += align_up(c.lcap * 8u, 128);
  b += align_up(c.hash_size * 4u, 128);
  b += 128;  // cand_id[32]
  b += 128;  // cand_dist[32]
  b += 128;  // mbarriers (<= 8) + the fp32 screen's per-query terms (ScreenQuery)
  b += align_up(c.dcap * 8u, 128);  // deleted-candidate queue: hi[dcap] | id[dcap]
  b += c.staged ? align_up(c.G * c.NG * vbytes, 128) : 0u;
  return b;
}

struct WarpCtx {
  uint64_t* keys;
  uint32_t* hash;
  uint32_t* cand_id;
  float* cand_dist;
  uint64_t* mbar;
  uint32_t* dq_hi;   // deleted-candidate queue (unordered), see beam_search
  uint32_t* dq_id;
  float* stage;
  uint32_t lcap, hsize, G, NG, dpad, vbytes, dcap, prefetch;
  uint32_t staged;  // the TMA staging ring is allocated (else LPV = 32 rows are read straight into registers)
  uint32_t phases;  // one parity bit per staging group
  uint32_t cnt;     // live entries in keys[] (shared-memory list only)
  uint32_t lane;
};

// esize: bytes per row element (4 = fp32 rows, 2 = bf16 shadow)
__device__ __forceinline__ void ctx_init(WarpCtx& c, unsigned char* base, const WalkCfg& cfg, uint32_t dpad,
                                         uint32_t esize = 4u) {
  c.lane = lane_id();
  c.lcap = cfg.lcap;
  c.G = cfg.G;
  c.NG = cfg.NG;
  c.dpad = dpad;
  c.vbytes = dpad * esize;
  c.hsize = cfg.hash_size;
  unsigned char* p = base;
  c.keys = (uint64_t*)p;
  p += align_up(cfg.lcap * 8u, 128);
  c.hash = (uint32_t*)p;
  p += align_up(cfg.hash_size * 4u, 128);
  c.cand_id = (uint32_t*)p;
  p += 128;
  c.cand_dist = (float*)p;
  p += 128;
  c.mbar = (uint64_t*)p;
  p += 128;
  c.dcap = cfg.dcap;
  c.prefetch = cfg.prefetch;
  c.staged = cfg.staged;
  c.dq_hi = (uint32_t*)p;
  c.dq_id = c.dq_hi + cfg.dcap;
  p += align_up(cfg.dcap * 8u, 128);
  c.stage = (float*)p;
  c.phases = 0;
  c.cnt = 0;
  if (cfg.staged) {
    if (c.lane < cfg.NG) mbar_init(&c.mbar[c.lane], 1);
    fence_mbar_init();
  }
  __syncwarp();
}

__device__ __forceinline__ void hash_clear(WarpCtx& c) {
  uint4* h4 = (uint4*)c.hash;
  uint32_t n4 = c.hsize >> 2;
  for (uint32_t i = c.lane; i < n4; i += 32) h4[i] = make_uint4(kInvalid, kInvalid, kInvalid, kInvalid);
  __syncwarp();
}

// Lane-parallel "test and set".  Returns true when id was not in the table
// (and is now, unless the probe budget ran out -> overflow).
__device__ __forceinline__ bool hash_insert(WarpCtx& c, uint32_t id, uint32_t& overflow) {
  uint32_t h = __umulhi(id * 0x9E3779B1u, c.hsize);  // fast range reduction: any table size
#pragma unroll 1
  for (int probe = 0; probe < 8; ++probe) {  // bounded: a crowded table costs re-evaluations, never long probes
    uint32_t old = atomicCAS(&c.hash[h], kInvalid, id);
    if (old == kInvalid) return true;
    if (old == id) return false;
    h = h + 1u == c.hsize ? 0u : h + 1u;
  }
  overflow = 1;
  return true;
}

// ---------------------------------------------------------------------------
// Lane chunks: how a lane holds its share of a row.  Lane `sub = lane % LPV`
// holds the fp32 query as NQ float4 registers (dpad == 4 * LPV * NQ exactly)
// and reads a row of RowT in chunks of W consecutive values: chunk j covers
// elements W * (sub + LPV * j) .. + W - 1 and pairs with the V = W / 4 query
// registers qr[j * V] .. qr[j * V + V - 1].  The chunk kinds:
//   fp32 rows, W = 4: float4;
//   bf16 rows, W = 8: uint4 (the walk, NQ >= 2);
//   bf16 rows, W = 4: uint2 (the walk at NQ = 1).
// (The fp32 walk's int8 screen reads its codes in the same layout, a u32 of four codes per chunk: screen_regs.)
// ---------------------------------------------------------------------------
template <class RowT, int NQ, int W = (std::is_same<RowT, __nv_bfloat16>::value && NQ > 1) ? 8 : 4>
struct LaneChunks {
  static_assert(W == 4 || (W == 8 && std::is_same<RowT, __nv_bfloat16>::value), "no such chunk");
  using T = std::conditional_t<std::is_same<RowT, float>::value, float4, std::conditional_t<W == 8, uint4, uint2>>;
  static constexpr int V = W / 4;   // query registers per chunk
  static constexpr int N = NQ / V;  // chunks per lane
};
__device__ __forceinline__ float4 ld_chunk(const float4* p) { return ld_nc_f4(p); }
__device__ __forceinline__ uint4 ld_chunk(const uint4* p) { return ld_nc_u4(p); }
__device__ __forceinline__ uint2 ld_chunk(const uint2* p) { return ld_nc_u2(p); }
// two packed bf16 pairs -> four floats (exact: bf16 is the top half of an fp32)
__device__ __forceinline__ float4 bf16x4_to_f4(uint32_t a, uint32_t b) {
  return make_float4(__uint_as_float(a << 16), __uint_as_float(a & 0xFFFF0000u), __uint_as_float(b << 16),
                     __uint_as_float(b & 0xFFFF0000u));
}
// chunk -> its V float4s of row values
__device__ __forceinline__ void widen(const float4& v, float4* x) { x[0] = v; }
__device__ __forceinline__ void widen(const uint4& v, float4* x) {
  x[0] = bf16x4_to_f4(v.x, v.y);
  x[1] = bf16x4_to_f4(v.z, v.w);
}
__device__ __forceinline__ void widen(const uint2& v, float4* x) { x[0] = bf16x4_to_f4(v.x, v.y); }

// the fp32 query in the lane layout of RowT rows (zero past dim)
template <int LPV, int NQ, class RowT = float>
__device__ __forceinline__ void load_query_regs(float4 (&qr)[NQ], const float* __restrict__ src, uint32_t dim,
                                                uint32_t lane) {
  constexpr int V = LaneChunks<RowT, NQ>::V;
  uint32_t sub = lane % LPV;
#pragma unroll
  for (int t = 0; t < NQ; ++t) {
    uint32_t e = (sub + LPV * (t / V)) * 4u * V + 4u * (t % V);
    float4 v;
    v.x = e + 0 < dim ? src[e + 0] : 0.f;
    v.y = e + 1 < dim ? src[e + 1] : 0.f;
    v.z = e + 2 < dim ? src[e + 2] : 0.f;
    v.w = e + 3 < dim ? src[e + 3] : 0.f;
    qr[t] = v;
  }
}
// a lane's chunks of one row (fp32 rows: the row's values, which the build kernels also use as a query)
template <int LPV, int NQ, class RowT, class C = LaneChunks<RowT, NQ>>
__device__ __forceinline__ void load_vec_regs(typename C::T (&r)[C::N], const RowT* __restrict__ row,
                                              uint32_t lane) {
  const typename C::T* p = (const typename C::T*)row + (lane % LPV);
#pragma unroll
  for (int t = 0; t < C::N; ++t) r[t] = p[LPV * t];
}

template <int NQ>
__device__ __forceinline__ float partial_dist(const float4 (&v)[NQ], const float4 (&qr)[NQ], int metric) {
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (metric == 0) {
#pragma unroll
    for (int t = 0; t < NQ; ++t) {
      float dx = qr[t].x - v[t].x, dy = qr[t].y - v[t].y, dz = qr[t].z - v[t].z, dw = qr[t].w - v[t].w;
      a0 = fmaf(dx, dx, a0);
      a1 = fmaf(dy, dy, a1);
      a2 = fmaf(dz, dz, a2);
      a3 = fmaf(dw, dw, a3);
    }
  } else {
#pragma unroll
    for (int t = 0; t < NQ; ++t) {
      a0 = fmaf(qr[t].x, v[t].x, a0);
      a1 = fmaf(qr[t].y, v[t].y, a1);
      a2 = fmaf(qr[t].z, v[t].z, a2);
      a3 = fmaf(qr[t].w, v[t].w, a3);
    }
  }
  return (a0 + a1) + (a2 + a3);
}
template <int LPV>
__device__ __forceinline__ float group_reduce(float acc) {
#pragma unroll
  for (int o = LPV / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// a lane's chunks of a row widened to fp32, then the fp32 chain (fp32 products and accumulation)
template <int NQ, class RowT, class C = LaneChunks<RowT, NQ>>
__device__ __forceinline__ float chunk_dist(const typename C::T (&v)[C::N], const float4 (&qr)[NQ], int metric) {
  float4 x[NQ];
#pragma unroll
  for (int j = 0; j < C::N; ++j) widen(v[j], x + j * C::V);
  return partial_dist<NQ>(x, qr, metric);
}
template <class RowT>
__device__ __forceinline__ const RowT* walk_rows(const GraphView& g) {
  if constexpr (std::is_same<RowT, float>::value)
    return g.vecs;
  else
    return g.vecs16;
}

// ---- LPV = 8: direct loads, U steps (4 vectors each) in flight --------------
// U for N chunks per lane: 64 registers of loads in flight (16 vectors of fp32 rows at d <= 128; a bf16 chunk
// carries twice the values, so the same registers hold twice the vectors, capped at the 32 candidates of a hop).
// UDIV > 1 divides it (the dense walk and the team walk's narrow form).
__host__ __device__ constexpr int eval_u(int N, int UDIV) {
  return ((N <= 2 ? 8 : (N <= 4 ? 4 : 2)) / UDIV) > 0 ? (N <= 2 ? 8 : (N <= 4 ? 4 : 2)) / UDIV : 1;
}
// (the default U is the one of fp32 rows)
template <int NQ, int U = eval_u(NQ, 1), class RowT = float>
__device__ __forceinline__ void eval_direct(WarpCtx& c, const RowT* __restrict__ rows, const float4 (&qr)[NQ],
                                            uint32_t m, int metric) {
  using C = LaneChunks<RowT, NQ>;
  const uint32_t sub = c.lane & 7u, grp = c.lane >> 3;
  __syncwarp();
#pragma unroll 1
  for (uint32_t j0 = 0; j0 < m; j0 += 4 * U) {
    typename C::T v[U][C::N];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (j0 + 4u * u < m) {                          // warp-uniform
        uint32_t j = min(j0 + 4u * u + grp, m - 1u);  // clamped lanes re-read the last row (same lines)
        const typename C::T* p = (const typename C::T*)(rows + (size_t)c.cand_id[j] * c.dpad) + sub;
#pragma unroll
        for (int t = 0; t < C::N; ++t) v[u][t] = ld_chunk(p + 8 * t);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (j0 + 4u * u < m) {
        uint32_t j = j0 + 4u * u + grp;
        float acc = group_reduce<8>(chunk_dist<NQ, RowT>(v[u], qr, metric));
        if (sub == 0 && j < m) c.cand_dist[j] = metric == 0 ? acc : 1.0f - acc;
      }
    }
  }
  __syncwarp();
}

// ---- LPV = 32: TMA bulk staging ring ----------------------------------------
// group r of G rows (vbytes each) of cand_id[0..m) -> ring buffer r % NG
template <class RowT>
__device__ __forceinline__ void issue_rows(WarpCtx& c, const RowT* __restrict__ vecs, uint32_t r, uint32_t m,
                                           uint32_t G, uint32_t vbytes) {
  uint32_t buf = r % c.NG;
  uint32_t first = r * G;
  uint32_t cnt = min(G, m - first);
  if (c.lane == 0) mbar_arrive_expect_tx(&c.mbar[buf], cnt * vbytes);
  __syncwarp();
  if (c.lane < cnt) {
    uint32_t id = c.cand_id[first + c.lane];
    bulk_g2s((RowT*)c.stage + (size_t)(buf * G + c.lane) * c.dpad, vecs + (size_t)id * c.dpad, vbytes, &c.mbar[buf]);
  }
}
template <class RowT>
__device__ __forceinline__ void issue_group(WarpCtx& c, const RowT* __restrict__ vecs, uint32_t r, uint32_t m) {
  issue_rows(c, vecs, r, m, c.G, c.vbytes);
}
template <int NQ, class RowT>
__device__ __forceinline__ void eval_staged(WarpCtx& c, const RowT* __restrict__ vecs, const float4 (&qr)[NQ],
                                            uint32_t m, int metric) {
  const uint32_t rounds = (m + c.G - 1) / c.G;
  const uint32_t pre = min(rounds, c.NG);
  for (uint32_t r = 0; r < pre; ++r) issue_group(c, vecs, r, m);
#pragma unroll 1
  for (uint32_t r = 0; r < rounds; ++r) {
    uint32_t buf = r % c.NG;
    mbar_wait(&c.mbar[buf], (c.phases >> buf) & 1u);
    c.phases ^= (1u << buf);
    uint32_t first = r * c.G;
    uint32_t cnt = min(c.G, m - first);
    // four staged vectors per step: their shuffle reductions are independent and overlap
#pragma unroll 1
    for (uint32_t v0 = 0; v0 < cnt; v0 += 4) {
      float acc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t v = min(v0 + (uint32_t)i, cnt - 1u);  // clamped repeats are discarded below
        typename LaneChunks<RowT, NQ>::T x[LaneChunks<RowT, NQ>::N];
        load_vec_regs<32, NQ>(x, (const RowT*)c.stage + (size_t)(buf * c.G + v) * c.dpad, c.lane);
        acc[i] = chunk_dist<NQ, RowT>(x, qr, metric);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
      }
      if (c.lane < 4 && v0 + c.lane < cnt) {
        float a = c.lane == 0 ? acc[0] : (c.lane == 1 ? acc[1] : (c.lane == 2 ? acc[2] : acc[3]));
        c.cand_dist[first + v0 + c.lane] = metric == 0 ? a : 1.0f - a;
      }
    }
    __syncwarp();
    if (r + c.NG < rounds) {
      fence_proxy_async();
      issue_group(c, vecs, r + c.NG, m);
    }
  }
  __syncwarp();
}

// ---- LPV = 32 without the ring: rows straight into registers ----------------------------------------------
// The walks that screen (WalkCfg::staged == 0) read fp32 rows this way, SB rows per batch (24 float4 registers per
// lane: eight rows at dpad 384 down to two at 1536; loading the next batch during this one's math would double them,
// and the kernel would spill at its 200-register budget).  A lane holds the chunks eval_staged reads from the ring
// (lane l: chunks l, l + 32, ...), and the fp32 chain and the shuffle reduction are eval_staged's, so the distances
// have the same bits.
template <int NQ>
__device__ __forceinline__ void eval_regs(WarpCtx& c, const float* __restrict__ vecs, const float4 (&qr)[NQ],
                                          uint32_t m, int metric) {
  constexpr int SB = NQ <= 24 ? 24 / NQ : 1;
#pragma unroll 1
  for (uint32_t v0 = 0; v0 < m; v0 += SB) {
    float4 x[SB][NQ];
#pragma unroll
    for (int i = 0; i < SB; ++i) {
      const uint32_t v = min(v0 + (uint32_t)i, m - 1u);  // clamped repeats are discarded below
      const float4* p = (const float4*)(vecs + (size_t)c.cand_id[v] * c.dpad) + c.lane;
#pragma unroll
      for (int t = 0; t < NQ; ++t) x[i][t] = ld_nc_f4(p + 32 * t);
    }
    float acc[SB];
#pragma unroll
    for (int i = 0; i < SB; ++i) acc[i] = chunk_dist<NQ, float>(x[i], qr, metric);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < SB; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    }
    if (c.lane < (uint32_t)SB && v0 + c.lane < m) {
      float a = acc[0];
#pragma unroll
      for (int i = 1; i < SB; ++i)
        if (c.lane == (uint32_t)i) a = acc[i];
      c.cand_dist[v0 + c.lane] = metric == 0 ? a : 1.0f - a;
    }
  }
  __syncwarp();
}

// ---- Wide rows (dpad 3072, 4096): the query in shared memory ---------------------------------------------
// 24 or 32 float4 of query per lane beside a row's chunks leave no registers (a register query spills kilobytes at
// dpad 4096), and a TMA ring of 12 or 16 KB rows would leave one warp per SM.  The wide form keeps the fp32 query in
// the warp's shared-memory slice where the ring would be (c.stage, dpad * 4 bytes), in the register layout of
// load_query_regs: float4 t of lane l at stage[32 t + l], so that the warp's 128-bit reads are free of bank
// conflicts.  The query of a walk, or a stored row that the build uses as one (first element past dim: dpad).
template <int NQ, class RowT>
__device__ __forceinline__ void load_query_smem(WarpCtx& c, const float* __restrict__ src, uint32_t dim) {
  constexpr int V = LaneChunks<RowT, NQ>::V;
  float4* qs = (float4*)c.stage + c.lane;
  __syncwarp();  // the previous query's readers are done
#pragma unroll 4
  for (int t = 0; t < NQ; ++t) {
    const uint32_t e = (c.lane + 32u * (t / V)) * 4u * V + 4u * (t % V);  // load_query_regs' element of (lane, t)
    float4 v;
    v.x = e + 0 < dim ? src[e + 0] : 0.f;
    v.y = e + 1 < dim ? src[e + 1] : 0.f;
    v.z = e + 2 < dim ? src[e + 2] : 0.f;
    v.w = e + 3 < dim ? src[e + 3] : 0.f;
    qs[32 * t] = v;
  }
  __syncwarp();
}
// cand_id[0..m) -> cand_dist[0..m) from the shared-memory query.  Per batch of kWideRows candidates a lane reads its
// chunks (lane l: chunks l, l + 32, ..., as eval_staged) straight into registers one d-slice of 1024 elements at a
// time (32 values per lane: 8 fp32 chunks or 4 bf16 ones, 64 load registers per lane for the batch), and folds each
// d-slice into the four accumulators of partial_dist in ascending chunk order, with the query slice read once from
// shared memory for all the batch's rows.  (a0 + a1) + (a2 + a3) and the shuffle tree of eval_staged follow, so the
// distances have the bits of the register-query walk's chain.  Loading the next d-slice during this one's math would
// double the load registers (ptxas then spills); the other resident warps overlap the round trips instead.
constexpr int kWideRows = 4;
template <int NQ, class RowT>
__device__ __forceinline__ void eval_wide(WarpCtx& c, const RowT* __restrict__ vecs, uint32_t m, int metric) {
  using C = LaneChunks<RowT, NQ>;
  constexpr int V = C::V, SB = kWideRows, NS = 8 / V;
  static_assert(C::N % NS == 0, "the d-slices tile the row");
  const float4* qs = (const float4*)c.stage + c.lane;
#pragma unroll 1
  for (uint32_t v0 = 0; v0 < m; v0 += SB) {
    const typename C::T* p[SB];
#pragma unroll
    for (int i = 0; i < SB; ++i)  // clamped repeats are discarded below
      p[i] = (const typename C::T*)(vecs + (size_t)c.cand_id[min(v0 + (uint32_t)i, m - 1u)] * c.dpad) + c.lane;
    float a[SB][4];
#pragma unroll
    for (int i = 0; i < SB; ++i) a[i][0] = a[i][1] = a[i][2] = a[i][3] = 0.f;
#pragma unroll 1
    for (int j0 = 0; j0 < C::N; j0 += NS) {
      typename C::T x[SB][NS];
#pragma unroll
      for (int i = 0; i < SB; ++i)
#pragma unroll
        for (int j = 0; j < NS; ++j) x[i][j] = ld_chunk(p[i] + 32 * (j0 + j));
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        float4 q[V];
#pragma unroll
        for (int v = 0; v < V; ++v) q[v] = qs[32 * ((j0 + j) * V + v)];
#pragma unroll
        for (int i = 0; i < SB; ++i) {
          float4 r[V];
          widen(x[i][j], r);
#pragma unroll
          for (int v = 0; v < V; ++v) {
            if (metric == 0) {
              const float dx = q[v].x - r[v].x, dy = q[v].y - r[v].y, dz = q[v].z - r[v].z, dw = q[v].w - r[v].w;
              a[i][0] = fmaf(dx, dx, a[i][0]);
              a[i][1] = fmaf(dy, dy, a[i][1]);
              a[i][2] = fmaf(dz, dz, a[i][2]);
              a[i][3] = fmaf(dw, dw, a[i][3]);
            } else {
              a[i][0] = fmaf(q[v].x, r[v].x, a[i][0]);
              a[i][1] = fmaf(q[v].y, r[v].y, a[i][1]);
              a[i][2] = fmaf(q[v].z, r[v].z, a[i][2]);
              a[i][3] = fmaf(q[v].w, r[v].w, a[i][3]);
            }
          }
        }
      }
    }
    float acc[SB];
#pragma unroll
    for (int i = 0; i < SB; ++i) acc[i] = (a[i][0] + a[i][1]) + (a[i][2] + a[i][3]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int i = 0; i < SB; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    }
    if (c.lane < (uint32_t)SB && v0 + c.lane < m) {
      float d = acc[0];
#pragma unroll
      for (int i = 1; i < SB; ++i)
        if (c.lane == (uint32_t)i) d = acc[i];
      c.cand_dist[v0 + c.lane] = metric == 0 ? d : 1.0f - d;
    }
  }
  __syncwarp();
}

// cand_id[0..m) -> cand_dist[0..m): distances from the register-held query (the wide shapes: from the shared-memory
// query, eval_wide; qr is then unused).  UDIV > 1 halves (…) the
// load batches kept in flight per warp: fewer registers, more resident warps (the "dense" walk).  SCREEN: the
// instantiation can run a screened plan, which has no ring (c.staged == 0) and reads its rows into registers.
template <int LPV, int NQ, int UDIV = 1, class RowT = float, bool SCREEN = false>
__device__ __forceinline__ void eval_candidates(WarpCtx& c, const RowT* __restrict__ vecs, const float4 (&qr)[NQ],
                                                uint32_t m, int metric) {
  if constexpr (wide_shape(LPV, NQ)) {
    eval_wide<NQ, RowT>(c, vecs, m, metric);
    return;
  }
  if (LPV == 8) {
    eval_direct<NQ, eval_u(LaneChunks<RowT, NQ>::N, UDIV)>(c, vecs, qr, m, metric);
  } else {
    if constexpr (SCREEN) {
      if (!c.staged) {  // warp-uniform
        eval_regs<NQ>(c, vecs, qr, m, metric);
        return;
      }
    }
    eval_staged<NQ>(c, vecs, qr, m, metric);
  }
}

// ---- fp32 walk: the int8 screen (LPV = 32, metric 1, no ring) ---------------------------------------------
// The query as integers k = RN(q / sq) with |k| <= kQMax, packed in two signed byte planes k = 128 h + l
// (h in [-64, 64], l in [-64, 63]) in the codes' lane layout.  kQMax keeps every partial sum of K = sum k_i c_i inside
// int32 at dpad 1536: kQMax * 127 * 1536 < 2^31.
constexpr int kQMax = 8191;
// Per-query terms of the screen's bound (screen_setup): l1 >= |q|_1, l2 >= |q|_2, a: the walk chain's subnormal term,
// en >= |e|_2 for e = q - sq k, and sq.  They live in shared memory behind the mbarriers: held in registers through
// the walk, they cost spills.
struct ScreenQuery {
  float l1, l2, a, en, sq;
};
__device__ __forceinline__ ScreenQuery* screen_query(const WarpCtx& c) { return (ScreenQuery*)(c.mbar + 8); }
// The integer query planes k = 128 h + l, in the codes' lane layout (a u32 of four signed bytes per chunk).
template <int NQ>
struct QueryPlanes {
  uint32_t h[NQ], l[NQ];
};
// the walk screens its fp32 candidates (the plan set the int8 copy, which it does only for metric 1 and no ring)
__device__ __forceinline__ bool walk_screens(const GraphView& g) { return g.codes8 && g.metric == 1; }
// Once per query, before the upper-layer descent: the integer planes of the query (registers, kept through the whole
// walk) and its ScreenQuery terms (shared memory).
template <int NQ>
__device__ __forceinline__ void screen_setup(WarpCtx& c, const GraphView& g, const float4 (&qr)[NQ],
                                             QueryPlanes<NQ>& qp) {
  float mx = 0.f, l1 = 0.f, l2 = 0.f;
#pragma unroll
  for (int t = 0; t < NQ; ++t) {
    const float v[4] = {qr[t].x, qr[t].y, qr[t].z, qr[t].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mx = fmaxf(mx, fabsf(v[j]));
      l1 = __fadd_ru(l1, fabsf(v[j]));
      l2 = __fmaf_ru(v[j], v[j], l2);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // sums of non-negative terms rounded up: upper bounds
    l1 = __fadd_ru(l1, __shfl_xor_sync(0xffffffffu, l1, o));
    l2 = __fadd_ru(l2, __shfl_xor_sync(0xffffffffu, l2, o));
  }
  mx = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(mx)));  // >= 0: ordered as its bits
  // k = RN(q / sq) clamped to +-kQMax, and e = q - sq k, exact in double (sq k has at most 38 significant bits and
  // lies within 14 binades of q when k != 0).  A zero, tiny or non-finite max |q| gets sq = 0: k = 0 and e = q (a
  // NaN or infinite element then makes en non-finite, and every candidate is kept).
  float sq = mx / (float)kQMax;
  if (!(sq >= 0x1p-126f && sq <= 0x1.fffffep127f)) sq = 0.f;
  double e2 = 0.0;
#pragma unroll
  for (int t = 0; t < NQ; ++t) {
    const float v[4] = {qr[t].x, qr[t].y, qr[t].z, qr[t].w};
    uint32_t h = 0, l = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = sq != 0.f ? max(-kQMax, min(kQMax, __float2int_rn(v[j] / sq))) : 0;
      const double e = (double)v[j] - (double)sq * (double)k;
      e2 = __fma_ru(e, e, e2);
      const int kh = (k + 64) >> 7;  // floor: k - 128 kh in [-64, 63]
      h |= (uint32_t)(kh & 0xFF) << (8 * j);
      l |= (uint32_t)((k - 128 * kh) & 0xFF) << (8 * j);
    }
    qp.h[t] = h;
    qp.l[t] = l;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) e2 = __dadd_ru(e2, __shfl_xor_sync(0xffffffffu, e2, o));
  // the walk chain's subnormal inputs and products, flushed or not: d (2^-125 max|q| + 2^-124)
  if (c.lane == 0)
    *screen_query(c) = {l1, __fsqrt_ru(l2), __fmul_ru((float)g.dpad, __fmaf_ru(mx, 0x1p-125f, 0x1p-124f)),
                        __double2float_ru(__dsqrt_ru(e2)), sq};
  __syncwarp();
}
// Per candidate of cand_id[0..m) the warp loads the codes straight into registers (RB rows per batch: 96 registers
// of codes per lane, 32 rows at dpad 384 down to 8 at 1536; loading the next batch during this one's math would
// double them, and the kernel would spill at its 200-register budget)
// and computes K = sum k_i c_i exactly, with two dp4a per u32 of codes and one int32 warp reduction.  With the row's
// terms (s, rinf, r2, nx) it forms L = RD(RD(1 - RU(s sq K)) - M'),
//   M' = RU(gam l2 nx + min(l1 rinf, l2 r2) + en (nx + r2) + a),  gam = dpad 2^-24 / (1 - dpad 2^-24):
// a lower bound on the distance RN(1 - P^) of the fp32 pass (DESIGN.md §9).  A candidate with f2ord(L) >= worst_hi
// cannot be chosen and is dropped (beam_search: the hop-start worst of a full result set, which only shrinks within
// the hop; greedy_descent: the current node's distance, which a move must beat); a non-finite L keeps it.  The
// survivors move to the front of cand_id in their order, and their count is returned.  `unsure` (a bit per cand_id
// position) moves with them.
template <int NQ>
__device__ __forceinline__ uint32_t screen_regs(WarpCtx& c, const GraphView& g, const QueryPlanes<NQ>& qp, uint32_t m,
                                                uint32_t worst_hi, uint32_t& unsure) {
  constexpr int RB = 96 / NQ;
  const bool in = c.lane < m;
  const uint32_t id = in ? c.cand_id[c.lane] : kInvalid;
  // lane j's candidate's row terms, loaded together with the codes
  float4 tm = make_float4(0.f, 0.f, 0.f, 0.f);
  if (in) tm = ld_nc_f4(g.terms8 + id);
  int K = 0;  // lane j: K of candidate j
#pragma unroll 1
  for (uint32_t v0 = 0; v0 < m; v0 += RB) {
    uint32_t x[RB][NQ];
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      const uint32_t* p = (const uint32_t*)(g.codes8 + (size_t)c.cand_id[min(v0 + (uint32_t)i, m - 1u)] * c.dpad) +
                          c.lane;  // clamped repeats are discarded below
#pragma unroll
      for (int t = 0; t < NQ; ++t) x[i][t] = ld_nc_u32(p + 32 * t);
    }
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      int h = 0, l = 0;
#pragma unroll
      for (int t = 0; t < NQ; ++t) {
        h = __dp4a((int)x[i][t], (int)qp.h[t], h);
        l = __dp4a((int)x[i][t], (int)qp.l[t], l);
      }
      const int kv = __reduce_add_sync(0xffffffffu, 128 * h + l);
      if (c.lane == v0 + (uint32_t)i) K = kv;
    }
  }
  float L = 0.f;
  if (in) {
    const ScreenQuery sq = *screen_query(c);
    const float e = (float)c.dpad * 0x1p-24f;  // exact, and so is 1 - e (dpad <= 2048)
    const float gam = __fdiv_ru(e, 1.0f - e);
    // s, sq >= 0: RU(RU(s RU(K)) sq) >= s sq K whatever the sign of K
    const float se = __fmul_ru(__fmul_ru(tm.x, __int2float_ru(K)), sq.sq);
    float mg = __fmul_ru(__fmul_ru(gam, sq.l2), tm.w);
    mg = __fadd_ru(mg, fminf(__fmul_ru(sq.l1, tm.y), __fmul_ru(sq.l2, tm.z)));
    mg = __fadd_ru(mg, __fmaf_ru(sq.en, __fadd_ru(tm.w, tm.z), sq.a));
    L = __fsub_rd(__fsub_rd(1.0f, se), mg);
  }
  const bool keep = in && !(isfinite(L) && f2ord(L) >= worst_hi);
  const uint32_t mask = __ballot_sync(0xffffffffu, keep);
  const uint32_t pos = __popc(mask & lanemask_lt());
  __syncwarp();
  if (keep) c.cand_id[pos] = id;
  if (unsure) unsure = __reduce_or_sync(0xffffffffu, (keep && ((unsure >> c.lane) & 1u)) ? (1u << pos) : 0u);
  __syncwarp();
  return __popc(mask);
}

// ---------------------------------------------------------------------------
// Unsorted register-resident result set ("ulist"): position p = slot*32 + lane,
// valid iff p < ef.  hnswlib keeps a max-heap (results) and a min-heap
// (candidates); here both are one unordered array and the two heap tops are
// found with warp reductions (redux.sync min / max on the ordered 32-bit
// distance): insert-or-replace-worst and pop-closest-unexpanded cost ~10
// instructions each instead of a ~70-instruction sorted insert.
//   hi[s]: ordered distance; empty valid position = 0xFFFFFFFF; dead (p >= ef) = 0
//   id[s]: node id | expanded flag; empty / dead = kInvalid (flag set -> never popped)
// ---------------------------------------------------------------------------
template <int KPL>
struct UList {
  uint32_t hi[KPL];
  uint32_t id[KPL];
};
template <int KPL>
__device__ __forceinline__ void ul_clear(UList<KPL>& u, uint32_t ef, uint32_t lane) {
#pragma unroll
  for (int s = 0; s < KPL; ++s) {
    u.hi[s] = ((uint32_t)s * 32u + lane) < ef ? 0xFFFFFFFFu : 0u;
    u.id[s] = kInvalid;
  }
}
// worst (largest) ordered distance over the valid positions; meaningful when the set is full
template <int KPL>
__device__ __forceinline__ uint32_t ul_worst(const UList<KPL>& u) {
  uint32_t m = u.hi[0];
#pragma unroll
  for (int s = 1; s < KPL; ++s) m = max(m, u.hi[s]);
  return __reduce_max_sync(0xffffffffu, m);
}
// Insert (hi, id) [warp-uniform]; cnt/worst_hi are maintained by the caller's copies.
// Precondition when cnt == ef: hi < worst_hi.
// (Round 2 tried a per-lane form — every lane reduces over its own KPL slots, then ONE ballot elects the
//  lane, predicated writes select the slot — to cut the ~KPL dependent ballots per insert.  It needs more
//  registers than the slot-walking form below (136 vs 128 at KPL = 8), which costs the walk its occupancy.)
template <int KPL>
__device__ __forceinline__ void ul_insert(UList<KPL>& u, uint32_t hi, uint32_t id, uint32_t ef, uint32_t& cnt,
                                          uint32_t& worst_hi, uint32_t lane) {
  bool done = false;
  if (cnt < ef) {
#pragma unroll
    for (int s = 0; s < KPL; ++s) {
      if (!done) {
        uint32_t b = __ballot_sync(0xffffffffu, u.id[s] == kInvalid && u.hi[s] == 0xFFFFFFFFu);
        if (b) {
          if ((int)lane == __ffs(b) - 1) u.hi[s] = hi, u.id[s] = id;
          done = true;
        }
      }
    }
    cnt++;
    if (cnt == ef) worst_hi = ul_worst<KPL>(u);
  } else {
#pragma unroll
    for (int s = 0; s < KPL; ++s) {
      if (!done) {
        uint32_t b = __ballot_sync(0xffffffffu, u.hi[s] == worst_hi && u.id[s] != kInvalid);
        if (b) {
          if ((int)lane == __ffs(b) - 1) u.hi[s] = hi, u.id[s] = id;
          done = true;
        }
      }
    }
    worst_hi = ul_worst<KPL>(u);
  }
}
// closest unexpanded entry: returns its id (flag clear) or kInvalid; mark=true sets its expanded flag
template <int KPL>
__device__ __forceinline__ uint32_t ul_min_unexpanded(UList<KPL>& u, bool mark, uint32_t lane) {
  uint32_t m = 0xFFFFFFFFu;
#pragma unroll
  for (int s = 0; s < KPL; ++s)
    if (!(u.id[s] & kExpandedFlag)) m = min(m, u.hi[s]);
  m = __reduce_min_sync(0xffffffffu, m);
  uint32_t node = kInvalid;
  bool done = false;
#pragma unroll
  for (int s = 0; s < KPL; ++s) {
    if (!done) {
      uint32_t b = __ballot_sync(0xffffffffu, !(u.id[s] & kExpandedFlag) && u.hi[s] == m);
      if (b) {
        int l = __ffs(b) - 1;
        node = __shfl_sync(0xffffffffu, u.id[s], l);
        if (mark && (int)lane == l) u.id[s] |= kExpandedFlag;
        done = true;
      }
    }
  }
  return node;
}
// ordered distance of the closest unexpanded entry (0xFFFFFFFF when there is none)
template <int KPL>
__device__ __forceinline__ uint32_t ul_min_unexpanded_hi(const UList<KPL>& u) {
  uint32_t m = 0xFFFFFFFFu;
#pragma unroll
  for (int s = 0; s < KPL; ++s)
    if (!(u.id[s] & kExpandedFlag)) m = min(m, u.hi[s]);
  return __reduce_min_sync(0xffffffffu, m);
}
template <int KPL>
__device__ __forceinline__ bool ul_contains(const UList<KPL>& u, uint32_t id) {
  bool hit = false;
#pragma unroll
  for (int s = 0; s < KPL; ++s) hit |= u.id[s] != kInvalid && (u.id[s] & kIdMask) == id;
  return __any_sync(0xffffffffu, hit);
}
// Destructive extraction in ascending order: returns the next (hi, id) or id == kInvalid when empty.
template <int KPL>
__device__ __forceinline__ uint64_t ul_extract_min(UList<KPL>& u, uint32_t lane) {
  uint32_t m = 0xFFFFFFFFu;
#pragma unroll
  for (int s = 0; s < KPL; ++s)
    if (u.id[s] != kInvalid) m = min(m, u.hi[s]);
  m = __reduce_min_sync(0xffffffffu, m);
  uint64_t out = kMaxKey;
  bool done = false;
#pragma unroll
  for (int s = 0; s < KPL; ++s) {
    if (!done) {
      uint32_t b = __ballot_sync(0xffffffffu, u.id[s] != kInvalid && u.hi[s] == m);
      if (b) {
        int l = __ffs(b) - 1;
        uint32_t id = __shfl_sync(0xffffffffu, u.id[s], l);
        out = ((uint64_t)m << 32) | (id & kIdMask);
        if ((int)lane == l) u.id[s] = kInvalid, u.hi[s] = 0xFFFFFFFFu;
        done = true;
      }
    }
  }
  return out;
}
// Empties the set into the shared-memory key list c.keys[0..c.cnt) in ascending order.
template <int KPL>
__device__ __forceinline__ void ul_extract_all(WarpCtx& c, UList<KPL>& u) {
  c.cnt = 0;
  for (;;) {
    uint64_t key = ul_extract_min<KPL>(u, c.lane);
    if (key == kMaxKey) break;
    if (c.lane == 0) c.keys[c.cnt] = key;
    c.cnt++;
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------
// Shared-memory result set of the wide-beam walk (ef 513 .. 4096; hnsw_search_beam_kernel): the same unordered set
// as UList, with the same entry encoding (hi: ordered distance; id: node id | expanded flag; an unused entry is hi 0,
// id kInvalid), in the warp's key list c.keys, which holds lcap = align_up(ef, 32) 8-byte keys: the hi words
// hi[0..lcap) and then the id words.  The set is 32 columns of C = lcap / 32 entries, column l at [l C, l C + C);
// the set's n-th entry goes to row n / 32 of column n % 32, so a column's entries are its first rows.  Lane l keeps
// its column's summary in registers: the worst (largest) entry and the closest unexpanded one, with their rows.
// The set's worst entry and its closest unexpanded entry are then one warp reduction each; an insert into a set that
// is not full tightens one column's summary; replacing the worst entry, or marking an entry expanded, rescans that
// one column cooperatively (C / 32 shared loads per lane and two reductions: sl_scan).
// ---------------------------------------------------------------------------
struct SList {
  uint32_t* hi;  // [lcap] column-major
  uint32_t* id;  // [lcap]
  uint32_t C;    // entries per column
  uint32_t whi, wrow;  // this lane's column: worst entry (wrow kInvalid: the column is empty)
  uint32_t uhi, urow;  // this lane's column: closest unexpanded entry (urow kInvalid: none)
};
__device__ __forceinline__ void sl_init(SList& u, const WarpCtx& c) {
  u.hi = (uint32_t*)c.keys;
  u.id = u.hi + c.lcap;
  u.C = c.lcap / 32u;
}
// Recomputes column col's summary (worst too, when `worst`), held by lane col.  Ties go to the lower row.
__device__ __forceinline__ void sl_scan(SList& u, uint32_t col, bool worst, uint32_t lane) {
  __syncwarp();  // the writer of the column is done
  const uint32_t* hc = u.hi + col * u.C;
  const uint32_t* ic = u.id + col * u.C;
  uint32_t wh = 0, wr = kInvalid, uh = 0xFFFFFFFFu, ur = kInvalid;
  for (uint32_t r = lane; r < u.C; r += 32) {
    const uint32_t h = hc[r], d = ic[r];
    if (d != kInvalid && (wr == kInvalid || h > wh)) wh = h, wr = r;
    if (!(d & kExpandedFlag) && (ur == kInvalid || h < uh)) uh = h, ur = r;
  }
  const uint32_t um = __reduce_min_sync(0xffffffffu, ur != kInvalid ? uh : 0xFFFFFFFFu);
  const uint32_t ub = __ballot_sync(0xffffffffu, ur != kInvalid && uh == um);
  const uint32_t urow = ub ? __shfl_sync(0xffffffffu, ur, __ffs(ub) - 1) : kInvalid;
  if (lane == col) u.uhi = um, u.urow = urow;
  if (worst) {
    const uint32_t wm = __reduce_max_sync(0xffffffffu, wr != kInvalid ? wh : 0u);
    const uint32_t wb = __ballot_sync(0xffffffffu, wr != kInvalid && wh == wm);
    const uint32_t wrow = wb ? __shfl_sync(0xffffffffu, wr, __ffs(wb) - 1) : kInvalid;
    if (lane == col) u.whi = wm, u.wrow = wrow;
  }
}
__device__ __forceinline__ void ul_clear(SList& u, uint32_t ef, uint32_t lane) {
  (void)ef;
  __syncwarp();  // the previous query's readers are done
  for (uint32_t i = lane; i < 32u * u.C; i += 32) u.hi[i] = 0, u.id[i] = kInvalid;
  u.whi = 0, u.wrow = kInvalid, u.uhi = 0xFFFFFFFFu, u.urow = kInvalid;
  __syncwarp();
}
// UList's ul_insert contract: warp-uniform; precondition when cnt == ef: hi < worst_hi.
__device__ __forceinline__ void ul_insert(SList& u, uint32_t hi, uint32_t id, uint32_t ef, uint32_t& cnt,
                                          uint32_t& worst_hi, uint32_t lane) {
  if (cnt < ef) {
    const uint32_t col = cnt & 31u, row = cnt >> 5;
    if (lane == col) {
      u.hi[col * u.C + row] = hi, u.id[col * u.C + row] = id;
      if (u.wrow == kInvalid || hi > u.whi) u.whi = hi, u.wrow = row;
      if (u.urow == kInvalid || hi < u.uhi) u.uhi = hi, u.urow = row;
    }
    __syncwarp();
    cnt++;
    if (cnt == ef) worst_hi = __reduce_max_sync(0xffffffffu, u.wrow != kInvalid ? u.whi : 0u);
  } else {
    const uint32_t b = __ballot_sync(0xffffffffu, u.wrow != kInvalid && u.whi == worst_hi);
    const uint32_t col = __ffs(b) - 1;
    const uint32_t row = __shfl_sync(0xffffffffu, u.wrow, col);
    if (lane == col) u.hi[col * u.C + row] = hi, u.id[col * u.C + row] = id;
    sl_scan(u, col, true, lane);
    worst_hi = __reduce_max_sync(0xffffffffu, u.wrow != kInvalid ? u.whi : 0u);
  }
}
// closest unexpanded entry: its key (flag clear) or kMaxKey; mark sets its expanded flag
__device__ __forceinline__ uint64_t sl_take_min(SList& u, bool mark, uint32_t lane) {
  const uint32_t m = __reduce_min_sync(0xffffffffu, u.urow != kInvalid ? u.uhi : 0xFFFFFFFFu);
  const uint32_t b = __ballot_sync(0xffffffffu, u.urow != kInvalid && u.uhi == m);
  if (!b) return kMaxKey;
  const uint32_t col = __ffs(b) - 1;
  const uint32_t at = col * u.C + __shfl_sync(0xffffffffu, u.urow, col);
  const uint32_t node = u.id[at];
  if (mark) {
    __syncwarp();
    if (lane == col) u.id[at] = node | kExpandedFlag;
    sl_scan(u, col, false, lane);
  }
  return ((uint64_t)m << 32) | node;
}
__device__ __forceinline__ uint32_t ul_min_unexpanded(SList& u, bool mark, uint32_t lane) {
  const uint64_t key = sl_take_min(u, mark, lane);
  return key == kMaxKey ? kInvalid : (uint32_t)key;
}
__device__ __forceinline__ uint32_t ul_min_unexpanded_hi(const SList& u) {
  return __reduce_min_sync(0xffffffffu, u.urow != kInvalid ? u.uhi : 0xFFFFFFFFu);
}
__device__ __forceinline__ bool ul_contains(const SList& u, uint32_t id) {
  bool hit = false;
  for (uint32_t i = (uint32_t)threadIdx.x & 31u; i < 32u * u.C; i += 32) hit |= u.id[i] != kInvalid && (u.id[i] & kIdMask) == id;
  return __any_sync(0xffffffffu, hit);
}
// After the walk: clears every expanded flag, so that sl_take_min(u, true, lane) then takes the entries in ascending
// order (UList's ul_extract_min).
__device__ __forceinline__ void sl_begin_extract(SList& u, uint32_t lane) {
  __syncwarp();
  for (uint32_t i = lane; i < 32u * u.C; i += 32)
    if (u.id[i] != kInvalid) u.id[i] &= kIdMask;
  for (uint32_t col = 0; col < 32; ++col) sl_scan(u, col, false, lane);
}

// ---------------------------------------------------------------------------
// Shared-memory sorted key list (cold paths: brute-force select, row merge).
// Returns the insert position, or kInvalid when rejected (duplicate id or
// beyond the limit).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t list_insert(WarpCtx& c, uint64_t key, uint32_t limit) {
  const uint32_t id = key_id(key);
  uint32_t pos = 0;
  uint32_t dup = 0;
  for (uint32_t base = 0; base < c.cnt; base += 32) {
    uint32_t i = base + c.lane;
    uint64_t k = i < c.cnt ? c.keys[i] : kMaxKey;
    pos += __popc(__ballot_sync(0xffffffffu, k < key));
    dup |= __ballot_sync(0xffffffffu, i < c.cnt && key_id(k) == id);
  }
  if (dup || pos >= limit) return kInvalid;
  const uint32_t newcnt = min(c.cnt + 1u, limit);
  for (int base = (int)((newcnt - 1u) & ~31u); base >= (int)(pos & ~31u); base -= 32) {
    uint32_t i = (uint32_t)base + c.lane;
    bool in = i >= pos && i < newcnt;
    uint64_t v = key;
    if (in && i > pos) v = c.keys[i - 1];
    __syncwarp();
    if (in) c.keys[i] = v;
  }
  __syncwarp();
  c.cnt = newcnt;
  return pos;
}

// screened: evaluations made on the int8 screen copy first (fp32 screen); survivors: those of them whose fp32 row
// was then read.  An fp32 walk reads evals - screened + survivors fp32 rows.  screened_upper: the screened evaluations
// of the upper-layer descent (part of screened).
struct WalkCounters {
  uint32_t hops_upper, hops_base, evals, overflow, screened, survivors, screened_upper;
};

// Adjacency row of `node` at `level` -> one id per lane (kInvalid beyond the row).
// Branch-free (clamped index + select) so the warp never splits here.
__device__ __forceinline__ uint32_t load_row(const GraphView& g, uint32_t node, int level, uint32_t lane) {
  const uint32_t* row;
  uint32_t width;
  if (level == 0) {  // warp-uniform
    row = g.links0 + (size_t)node * g.M0;
    width = g.M0;
  } else {
    row = g.links_up + (size_t)(g.up_off[node] + (uint32_t)(level - 1)) * g.M;
    width = g.M;
  }
  uint32_t v = row[min(lane, width - 1u)];
  return lane < width ? v : kInvalid;
}

// hnswlib searchKnn's upper-layer descent: at each level move to the closest
// neighbour until no neighbour improves.
// A screened walk (SCREEN, walk_screens(g); *qp from screen_setup) screens each hop's neighbours on the int8 copy
// against the current distance first and evaluates only the survivors in fp32.  The descent moves only to a
// neighbour with d < curdist, and L <= d, so a neighbour with L >= curdist is never chosen; the survivors keep their
// order, so a tie among them still goes to the earliest position, and the descent takes the same path.
template <int LPV, int NQ, int UDIV = 1, class RowT = float, bool SCREEN = false>
__device__ __forceinline__ void greedy_descent(WarpCtx& c, const GraphView& g, const float4 (&qr)[NQ], uint32_t& cur,
                                               float& curdist, int from_level, int to_level_excl,
                                               WalkCounters& wc, const QueryPlanes<NQ>* qp = nullptr) {
  const bool screen = SCREEN && walk_screens(g);  // warp-uniform
  for (int level = from_level; level > to_level_excl; --level) {
    bool changed = true;
    while (changed) {
      changed = false;
      __syncwarp();
      uint32_t nb = load_row(g, cur, level, c.lane);
      uint32_t mask = __ballot_sync(0xffffffffu, nb != kInvalid);
      uint32_t m = __popc(mask);
      wc.hops_upper++;
      if (!m) break;
      if (nb != kInvalid) c.cand_id[__popc(mask & lanemask_lt())] = nb;
      __syncwarp();
      wc.evals += m;
      if (SCREEN && screen) {
        uint32_t unsure = 0;
        wc.screened += m;
        wc.screened_upper += m;
        m = screen_regs<NQ>(c, g, *qp, m, f2ord(curdist), unsure);
        wc.survivors += m;
        eval_regs<NQ>(c, g.vecs, qr, m, 1);
      } else {
        eval_candidates<LPV, NQ, UDIV, RowT, SCREEN>(c, walk_rows<RowT>(g), qr, m, g.metric);
      }
      float bd = c.lane < m ? c.cand_dist[c.lane] : INFINITY;
      uint32_t bl = c.lane;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float od = __shfl_xor_sync(0xffffffffu, bd, o);
        uint32_t ol = __shfl_xor_sync(0xffffffffu, bl, o);
        if (od < bd || (od == bd && ol < bl)) bd = od, bl = ol;
      }
      if (bd < curdist) {
        curdist = bd;
        cur = c.cand_id[bl];
        changed = true;
      }
      __syncwarp();
    }
  }
}

// hnswlib searchBaseLayer(ST): best-first beam search with an ef-bounded
// result set.  On return `u` holds the (<= ef) closest visited nodes (unordered).
//
// Why one array replaces hnswlib's two heaps (same expansion order, same result):
//   hnswlib keeps `top_candidates` (max-heap, <= ef results) and `candidate_set` (min-heap of everything
//   ever admitted).  A node enters both at the same moment (when top is not full or it beats the worst
//   result) and is only ever removed from top by eviction of the worst.  The loop pops the closest
//   unexpanded admitted node c and stops when dist(c) > worst result and top is full.  An admitted node
//   that is no longer in top was evicted, i.e. is not closer than the current worst; every node still in
//   top is.  Hence "closest unexpanded admitted node" is in top whenever top holds any unexpanded node, and
//   when it does not, the pop would hit the stop condition (or the queue is empty).  So the walk is:
//   repeatedly expand the closest entry of the result set whose expanded flag is clear, until none is
//   left — which needs only the result set itself plus one flag per entry.  Admission is the same test
//   (`cnt < ef || d < worst`); the tests check id-for-id equality with the oracle on identical graphs.
// `exclude` (kInvalid = none) is never admitted (used when re-linking an updated
// node).  The adjacency row of the likely next node (the closest unexpanded entry
// before this hop's candidates are known) is requested ahead of the distance
// evaluation, so its latency overlaps the vector loads.
// Side queue of admitted-but-deleted candidates (only when g.deleted != nullptr).  hnswlib's
// searchBaseLayerST<has_deletions=true> puts a tombstoned node into candidate_set (it is traversed) but never
// into top_candidates (it is not a result and does not move lowerBound).  Such nodes cannot live in the
// result set, so they wait here, unordered, until they are the closest unexpanded candidate.
// bound: the worst result once the result set is full, else 0xFFFFFFFF.  An entry beyond it can never be expanded
// (the set stays full and its worst only shrinks: the walk stops before reaching it), so dropping one is exact.
__device__ __forceinline__ void dq_push(WarpCtx& c, uint32_t& dn, uint32_t hi, uint32_t id, uint32_t bound,
                                        uint32_t& overflow) {
  if (dn < c.dcap) {
    if (c.lane == 0) c.dq_hi[dn] = hi, c.dq_id[dn] = id;
    dn++;
  } else {  // full: keep the closest dcap entries (the farthest is the least likely to be expanded)
    uint32_t w = 0, wp = 0;
    for (uint32_t i = c.lane; i < dn; i += 32)
      if (c.dq_hi[i] >= w) w = c.dq_hi[i], wp = i;
    uint32_t wm = __reduce_max_sync(0xffffffffu, w);
    uint32_t b = __ballot_sync(0xffffffffu, w == wm);
    uint32_t pos = __shfl_sync(0xffffffffu, wp, __ffs(b) - 1);
    if (hi < wm && c.lane == 0) c.dq_hi[pos] = hi, c.dq_id[pos] = id;
    if (max(hi, wm) <= bound) overflow = 1;  // the dropped entry could still have been expanded
  }
  __syncwarp();
}
// closest queued entry: returns its position (kInvalid when empty) and ordered distance
__device__ __forceinline__ uint32_t dq_min(const WarpCtx& c, uint32_t dn, uint32_t& hi_out) {
  uint32_t m = 0xFFFFFFFFu, mp = kInvalid;
  for (uint32_t i = c.lane; i < dn; i += 32)
    if (c.dq_hi[i] < m) m = c.dq_hi[i], mp = i;
  uint32_t mm = __reduce_min_sync(0xffffffffu, m);
  uint32_t b = __ballot_sync(0xffffffffu, m == mm && mp != kInvalid);
  hi_out = mm;
  return b ? __shfl_sync(0xffffffffu, mp, __ffs(b) - 1) : kInvalid;
}

// HASDEL = false compiles every trace of the tombstone machinery out (an index without tombstones runs
// exactly the plain loop: the extra live registers would cost the 16-vector load batches their overlap).
// The fp32 screen (SCREEN instantiations: fp32 rows of dpad 384 .. 1536; metric 1, g.codes8 set, no ring): at a hop
// that starts with a full result set the hop's candidates are screened on the int8 copy first (screen_regs), and only
// the survivors are evaluated in fp32 and offered for admission.  A dropped candidate's fp32 distance is >= the
// hop-start worst result, so it would not have been admitted (nor queued, if tombstoned): the walk, its results and
// its counters stay the same.
template <int LPV, int NQ, int KPL, bool PREFETCH, bool HASDEL, int UDIV = 1, class RowT = float, bool SCREEN = false,
          class Set = UList<KPL>>
__device__ __forceinline__ void beam_search(WarpCtx& c, const GraphView& g, const float4 (&qr)[NQ], Set& u,
                                            uint32_t ep, float epdist, int level, uint32_t ef, uint32_t exclude,
                                            WalkCounters& wc, const QueryPlanes<NQ>* qp = nullptr) {
  static_assert(!SCREEN || (screen_shape(LPV, NQ) && std::is_same<RowT, float>::value), "no screen for this shape");
  const bool screen = SCREEN && walk_screens(g);  // warp-uniform; *qp from screen_setup
  hash_clear(c);
  ul_clear(u, ef, c.lane);
  const uint8_t* __restrict__ del = (HASDEL && c.dcap) ? g.deleted : nullptr;  // warp-uniform
  uint32_t dn = 0;                                                  // entries in the deleted-candidate queue
  uint32_t ovf = 0;
  if (c.lane == 0) {
    hash_insert(c, ep, ovf);
    if (exclude != kInvalid) hash_insert(c, exclude, ovf);
  }
  __syncwarp();
  uint32_t cnt = 0;
  uint32_t worst_hi = 0xFFFFFFFFu;  // ordered distance of the worst entry once the set is full
  bool ovf_any = false;
  // a tombstoned (or excluded) entry point is expanded once but never becomes a result
  const bool ep_result = ep != exclude && !(del && del[ep]);
  if (ep_result) ul_insert(u, f2ord(epdist), ep, ef, cnt, worst_hi, c.lane);
  uint32_t node = ep;
  if (ep_result) node = ul_min_unexpanded(u, true, c.lane);
  uint32_t nb = load_row(g, node, level, c.lane);
  for (;;) {
    if (level == 0) wc.hops_base++; else wc.hops_upper++;
    // a walk expands each admitted node once; the bound only guards against a corrupt graph
    if (HASDEL && wc.hops_base + wc.hops_upper > 64u * ef + 65536u) break;
    __syncwarp();
    // speculative: the row of the closest entry still unexpanded
    const uint32_t spec = ul_min_unexpanded(u, false, c.lane);
    uint32_t spec_row = kInvalid;
    if (spec != kInvalid) spec_row = load_row(g, spec & kIdMask, level, c.lane);
    bool is_new = false;
    uint32_t o = 0;  // this insert ran out of probes: "new" is then only a guess
    if (nb != kInvalid && nb != exclude) is_new = hash_insert(c, nb, o);
    ovf |= o;
    __syncwarp();  // hash probing diverges; reconverge before the collective section
    uint32_t mask = __ballot_sync(0xffffffffu, is_new);
    uint32_t m = __popc(mask);
    if (m) {
      const uint32_t pos = __popc(mask & lanemask_lt());
      if (is_new) c.cand_id[pos] = nb;
      // tombstones only: candidates (compacted positions) whose visited status is a guess
      uint32_t unsure = (HASDEL && del) ? __reduce_or_sync(0xffffffffu, (is_new && o) ? (1u << pos) : 0u) : 0u;
      __syncwarp();
      wc.evals += m;
      if (SCREEN && screen && cnt >= ef) {
        wc.screened += m;
        m = screen_regs<NQ>(c, g, *qp, m, worst_hi, unsure);
        wc.survivors += m;
        eval_regs<NQ>(c, g.vecs, qr, m, 1);
      } else {
        eval_candidates<LPV, NQ, UDIV, RowT, SCREEN>(c, walk_rows<RowT>(g), qr, m, g.metric);
      }
      // the speculative row has arrived by now: pull its neighbours' vectors towards L2 while this hop's
      // candidates are inserted (rows <= 1 KB only; a wrong guess costs bandwidth, not correctness)
      if (PREFETCH && LPV == 8 && c.prefetch && spec_row != kInvalid) {
        const char* pv = (const char*)(walk_rows<RowT>(g) + (size_t)spec_row * g.dpad);
#pragma unroll
        for (int b = 0; b < NQ * 8 * 16 * (int)sizeof(RowT) / 4; b += 128) prefetch_l2(pv + b);
      }
      uint32_t myhi = 0xFFFFFFFFu, myid = kInvalid;
      if (c.lane < m) myhi = f2ord(c.cand_dist[c.lane]), myid = c.cand_id[c.lane];
      const bool mydel = HASDEL && del && c.lane < m && del[myid];
      __syncwarp();
      ovf_any = ovf_any || __any_sync(0xffffffffu, ovf);
      uint32_t qual = __ballot_sync(0xffffffffu, c.lane < m && (cnt < ef || myhi < worst_hi));
      const uint32_t delmask = (HASDEL && del) ? __ballot_sync(0xffffffffu, mydel) : 0u;
      // A screened walk is bound by DRAM bandwidth, and most admitted candidates are evicted before they are
      // expanded: it pulls a candidate's adjacency row towards L2 only when the candidate is closer than every
      // unexpanded entry so far this hop, i.e. when it would be the next node expanded (hint only).
      uint32_t next_hi = (SCREEN && screen) ? ul_min_unexpanded_hi(u) : 0xFFFFFFFFu;
      while (qual) {
        int j = __ffs(qual) - 1;
        qual &= qual - 1;
        uint32_t hj = __shfl_sync(0xffffffffu, myhi, j);
        uint32_t ij = __shfl_sync(0xffffffffu, myid, j);
        if (cnt >= ef && hj >= worst_hi) continue;
        if (HASDEL && ((delmask >> j) & 1u)) {  // admitted like any candidate, but queued instead of becoming a result
          // (a tombstone whose visited status is only a guess is dropped: nothing else would keep it from
          //  being queued and expanded again and again once the visited table is full)
          if (!((unsure >> j) & 1u)) dq_push(c, dn, hj, ij, cnt >= ef ? worst_hi : 0xFFFFFFFFu, ovf);
          continue;
        }
        if (ovf_any && ul_contains(u, ij)) continue;
        ul_insert(u, hj, ij, ef, cnt, worst_hi, c.lane);
        if (PREFETCH && (!(SCREEN && screen) || hj < next_hi)) {
          next_hi = hj;
          if (c.lane == 0) prefetch_l2(g.links0 + (size_t)ij * g.M0);
        }
      }
    }
    if (HASDEL && dn) {
      // candidate_set.top(): the closer of (closest unexpanded result, closest queued tombstone)
      uint32_t dhi;
      const uint32_t dpos = dq_min(c, dn, dhi);
      if (dhi < ul_min_unexpanded_hi(u)) {
        if (cnt >= ef && dhi > worst_hi) break;  // hnswlib: dist > lowerBound && top_candidates.size() == ef
        node = c.dq_id[dpos];
        __syncwarp();
        if (c.lane == 0) c.dq_hi[dpos] = c.dq_hi[dn - 1], c.dq_id[dpos] = c.dq_id[dn - 1];
        dn--;
        __syncwarp();
        nb = load_row(g, node, level, c.lane);
        continue;
      }
    }
    node = ul_min_unexpanded(u, true, c.lane);
    if (node == kInvalid) break;
    nb = (node == spec) ? spec_row : load_row(g, node, level, c.lane);
  }
  // ovf_any is folded before a hop's candidates are admitted; a side-queue overflow raised while admitting them
  // (dq_push) in the walk's last hop is only in ovf
  wc.overflow |= (ovf_any || __any_sync(0xffffffffu, ovf)) ? 1u : 0u;
}

}  // namespace ehb
