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
#pragma once
#include "kernels.h"

namespace ehb {

struct Aux {
  uint32_t* sel_id;   // [32]
  float* sel_dist;    // [32]
};

// Aux arrays live in the tail of the 128 B mbarrier region + an extra 256 B.
__device__ __forceinline__ Aux aux_of(const WarpCtx& c) {
  Aux a;
  // cand_id (128 B) | cand_dist (128 B) | mbar (128 B) | stage ...
  // the build kernels reserve 256 extra bytes in front of keys (see build_warp_smem)
  a.sel_id = (uint32_t*)((unsigned char*)c.keys - 256);
  a.sel_dist = (float*)((unsigned char*)c.keys - 128);
  return a;
}
__host__ __device__ inline uint32_t build_warp_smem(const WalkCfg& cfg, uint32_t dpad) {
  return 256u + warp_smem_bytes(cfg, dpad, 4u);
}

// The query of a build walk is a stored row: into registers, or into the warp's query slice for the wide shapes
// (walk.cuh load_query_smem; qr is then unused).
template <int LPV, int NQ>
__device__ __forceinline__ void load_row_query(WarpCtx& c, float4 (&qr)[NQ], const GraphView& g, uint32_t id) {
  if constexpr (wide_shape(LPV, NQ))
    load_query_smem<NQ, float>(c, g.vecs + (size_t)id * g.dpad, g.dpad);
  else
    load_vec_regs<LPV, NQ>(qr, g.vecs + (size_t)id * g.dpad, c.lane);
}

// hnswlib getNeighborsByHeuristic2 over keys[0..cnt) (ascending distance to
// the point being linked): keep a candidate iff it is not closer to an already
// kept neighbour than to the point.  Returns the number kept (<= Msel).
template <int LPV, int NQ>
__device__ __forceinline__ uint32_t heuristic_select(WarpCtx& c, const GraphView& g, uint32_t Msel, const Aux& a) {
  if (c.cnt < Msel) {
    for (uint32_t i = c.lane; i < c.cnt; i += 32) {
      a.sel_id[i] = key_id(c.keys[i]);
      a.sel_dist[i] = key_dist(c.keys[i]);
    }
    __syncwarp();
    return c.cnt;
  }
  uint32_t nsel = 0;
  for (uint32_t i = 0; i < c.cnt && nsel < Msel; ++i) {
    uint64_t key = c.keys[i];
    uint32_t cid = key_id(key);
    float dq = key_dist(key);
    bool good = true;
    if (nsel > 0) {
      float4 cr[NQ];
      load_row_query<LPV, NQ>(c, cr, g, cid);  // (the wide shapes: this replaces the caller's query)
      if (c.lane < nsel) c.cand_id[c.lane] = a.sel_id[c.lane];
      __syncwarp();
      eval_candidates<LPV, NQ>(c, g.vecs, cr, nsel, g.metric);
      bool bad = c.lane < nsel && c.cand_dist[c.lane] < dq;
      good = !__any_sync(0xffffffffu, bad);
    }
    if (good) {
      if (c.lane == 0) {
        a.sel_id[nsel] = cid;
        a.sel_dist[nsel] = dq;
      }
      nsel++;
    }
    __syncwarp();
  }
  return nsel;
}

// Drops `id` from the sorted key list c.keys[0..cnt) if it is there.  hnswlib's repairConnectionsForUpdate walks
// and admits the moved point like any other node and removes it from the result list afterwards.
__device__ __forceinline__ void list_remove_id(WarpCtx& c, uint32_t id) {
  uint32_t pos = kInvalid;
  for (uint32_t base = 0; base < c.cnt && pos == kInvalid; base += 32) {
    const uint32_t i = base + c.lane;
    const uint32_t m = __ballot_sync(0xffffffffu, i < c.cnt && key_id(c.keys[i]) == id);
    if (m) pos = base + __ffs(m) - 1;
  }
  if (pos == kInvalid) return;
  for (uint32_t base = pos & ~31u; base < c.cnt; base += 32) {
    const uint32_t i = base + c.lane;
    const uint64_t v = i + 1 < c.cnt ? c.keys[i + 1] : kMaxKey;
    __syncwarp();
    if (i >= pos && i + 1 < c.cnt) c.keys[i] = v;
    __syncwarp();
  }
  c.cnt--;
}

// The update path never rewrites a row in place while other warps of the wave may read it: a new row is staged in
// bb.side_out (one slot of M0 entries per row, bb.side_row names the row) and copied back by apply_staged_kernel
// once every warp has read the graph.  Returns the slot the calling warp writes (lanes < row width); slot side_cap
// is a sink that is never copied back (the build then reports an overflow).
__device__ __forceinline__ uint32_t* stage_row(const BuildBuffers& bb, uint32_t rid, uint32_t M0, uint32_t lane) {
  uint32_t slot = 0;
  if (lane == 0) {
    slot = atomicAdd(bb.side_count, 1u);
    if (slot < bb.side_cap) bb.side_row[slot] = rid;
    else atomicExch(bb.error_flag, 1u);
  }
  slot = __shfl_sync(0xffffffffu, slot, 0);
  return bb.side_out + (size_t)min(slot, bb.side_cap) * M0;
}

// Copies the staged rows back (one thread per entry) and clears the rows' update tags (bb.row_fill).
static __global__ void apply_staged_kernel(BuildBuffers bb, uint32_t* links0, uint32_t* links_up, uint32_t cap,
                                           uint32_t M0, uint32_t M) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t slot = (uint32_t)(t / M0), j = (uint32_t)(t % M0);
  if (slot >= min(*bb.side_count, bb.side_cap)) return;
  const uint32_t rid = bb.side_row[slot];
  const uint32_t v = bb.side_out[(size_t)slot * M0 + j];
  if (rid < cap) {
    links0[(size_t)rid * M0 + j] = v;
  } else if (j < M) {
    links_up[(size_t)(rid - cap) * M + j] = v;
  }
  if (j == 0) bb.row_fill[rid] = 0u;
}

// The wide form's result sets are the shared-memory SList of the wide-beam walk (walk.cuh).  Its key list holds
// 2 L keys (cfg.lcap = 2 L, L = align_up(set capacity, 32)): the ordered list that heuristic_select and
// list_remove_id read in keys[0, L), the set in keys[L, 2 L).
__device__ __forceinline__ void set_init(SList& u, const WarpCtx& c) {
  const uint32_t L = c.lcap / 2u;
  u.hi = (uint32_t*)(c.keys + L);
  u.id = u.hi + L;
  u.C = L / 32u;
}
// Readies a freshly declared set: the register form's needs nothing, the wide form's points into the key list.
template <int KPL>
__device__ __forceinline__ void set_begin(UList<KPL>&, const WarpCtx&) {}
__device__ __forceinline__ void set_begin(SList& u, const WarpCtx& c) { set_init(u, c); }
// Empties the set (UList: the register form; SList: the wide form, set_init) into c.keys[0..c.cnt) in ascending
// (distance, id) order: the list the selection heuristic walks.
template <int KPL>
__device__ __forceinline__ void set_to_list(WarpCtx& c, UList<KPL>& u) {
  ul_extract_all<KPL>(c, u);
}
__device__ __forceinline__ void set_to_list(WarpCtx& c, SList& u) {
  sl_begin_extract(u, c.lane);
  c.cnt = 0;
  for (;;) {
    const uint64_t key = sl_take_min(u, true, c.lane);
    if (key == kMaxKey) break;
    if (c.lane == 0) c.keys[c.cnt] = key;
    c.cnt++;
  }
  __syncwarp();
}

// Phase A for one point p: search, select, write p's own rows, emit the reverse-edge records.  Set is the result set:
// UList<KPL> in the register form, the shared-memory SList (KPL = 0) in the wide form.
template <int LPV, int NQ, int KPL, bool HASDEL, class Set>
__device__ __forceinline__ void link_point(WarpCtx& c, const Aux& a, const BuildGraph& bg, uint32_t p, int is_update,
                                           const BuildBuffers& bb) {
  const GraphView& g = bg.g;
  float4 qr[NQ];
  load_row_query<LPV, NQ>(c, qr, g, p);
  Set ul;
  set_begin(ul, c);
  WalkCounters wc = {0, 0, 0, 0};
  const int level_p = bg.levels[p];
  const int top = g.max_level;
  uint32_t cur = g.entry;
  if (c.lane == 0) c.cand_id[0] = cur;
  __syncwarp();
  eval_candidates<LPV, NQ>(c, g.vecs, qr, 1, g.metric);
  float curdist = c.cand_dist[0];
  __syncwarp();
  if (level_p < top) greedy_descent<LPV, NQ>(c, g, qr, cur, curdist, top, level_p, wc);
  uint32_t* links0 = const_cast<uint32_t*>(g.links0);
  uint32_t* links_up = const_cast<uint32_t*>(g.links_up);
  for (int level = min(level_p, top); level >= 0; --level) {
    beam_search<LPV, NQ, KPL, false, HASDEL, 1, float, false, Set>(c, g, qr, ul, cur, curdist, level, bg.efc, kInvalid,
                                                                   wc);
    set_to_list(c, ul);
    if (is_update) list_remove_id(c, p);
    if (c.cnt == 0) continue;
    uint32_t nsel = heuristic_select<LPV, NQ>(c, g, g.M, a);
    if constexpr (wide_shape(LPV, NQ))
      if (level > 0) load_row_query<LPV, NQ>(c, qr, g, p);  // the selection replaced the shared-memory query
    uint32_t width = level == 0 ? g.M0 : g.M;
    uint32_t* row = level == 0 ? links0 + (size_t)p * g.M0 : links_up + (size_t)(g.up_off[p] + level - 1) * g.M;
    if (is_update) {
      // other warps of the wave may still walk this row: stage it, it lands before phase C
      const uint32_t rid = level == 0 ? p : bg.cap + g.up_off[p] + (uint32_t)(level - 1);
      row = stage_row(bb, rid, g.M0, c.lane);
    }
    if (c.lane < width) row[c.lane] = c.lane < nsel ? a.sel_id[c.lane] : kInvalid;
    uint32_t base = 0;
    if (c.lane == 0) base = atomicAdd(bb.edge_count, nsel);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base + nsel > bb.edge_cap) {
      if (c.lane == 0) atomicExch(bb.error_flag, 1u);
    } else if (c.lane < nsel) {
      uint32_t t = a.sel_id[c.lane];
      bb.edge_row[base + c.lane] = level == 0 ? t : bg.cap + g.up_off[t] + (uint32_t)(level - 1);
      bb.edge_src[base + c.lane] = p;
      bb.edge_dist[base + c.lane] = a.sel_dist[c.lane];
    }
    cur = key_id(c.keys[0]);
    curdist = key_dist(c.keys[0]);
    __syncwarp();
  }
}

// The register form of phase A (efc <= kMaxRegEfc): one warp per point of the wave.
template <int LPV, int NQ, int KPL, bool HASDEL>
__global__ void __launch_bounds__(128) build_search_kernel(BuildGraph bg, WalkCfg cfg, const uint32_t* __restrict__ ids,
                                                           uint32_t first, uint32_t b, int is_update, BuildBuffers bb,
                                                           uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  const GraphView& g = bg.g;
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t pi = blockIdx.x * (blockDim.x >> 5) + w;
  if (pi >= b) return;
  const uint32_t p = ids ? ids[pi] : first + pi;
  WarpCtx c;
  ctx_init(c, smem + (size_t)w * warp_smem + 256, cfg, g.dpad);
  Aux a = aux_of(c);
  link_point<LPV, NQ, KPL, HASDEL, UList<KPL>>(c, a, bg, p, is_update, bb);
}

// The wide form of phase A (efc > kMaxRegEfc): a persistent grid of one-warp blocks; warp w links points w, w + W, ...
// of the wave, so the scratch depends on the resident warps, not on the wave (up to 16384 points).  The result set is
// the shared-memory SList of the wide-beam walk (L = align_up(efc, 32) keys, the ordered list beside it: set_init), the
// visited table warp w's slice of vsize entries of vtab in HBM.  Every point reads the pre-wave graph and its edge
// records go through phases B and C as in the register form, so the schedule cannot change the result.
template <int LPV, int NQ, bool HASDEL>
__global__ void __launch_bounds__(32, 1)
    build_search_beam_kernel(BuildGraph bg, WalkCfg cfg, const uint32_t* __restrict__ ids, uint32_t first, uint32_t b,
                             int is_update, BuildBuffers bb, uint32_t vsize, uint32_t* __restrict__ vtab) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx c;
  ctx_init(c, smem + 256, cfg, bg.g.dpad);
  c.hash = vtab + (size_t)blockIdx.x * vsize;
  c.hsize = vsize;
  Aux a = aux_of(c);
  for (uint32_t pi = blockIdx.x; pi < b; pi += gridDim.x)
    link_point<LPV, NQ, 0, HASDEL, SList>(c, a, bg, ids ? ids[pi] : first + pi, is_update, bb);
}

// Adds one id per lane (kInvalid = none; the ids of one call are distinct) to the candidate set cand[0..ncand),
// deduplicated through the visited table.  A probe-budget overflow falls back to a linear scan of what is
// stored, so the set is exact.
__device__ __forceinline__ void cand_add(WarpCtx& c, uint32_t* cand, uint32_t& ncand, uint32_t id) {
  uint32_t o = 0;
  bool is_new = id != kInvalid && hash_insert(c, id, o);
  __syncwarp();
  if (__any_sync(0xffffffffu, o != 0)) {
    if (o)
      for (uint32_t i = 0; i < ncand && is_new; ++i) is_new = cand[i] != id;
    __syncwarp();
  }
  const uint32_t mask = __ballot_sync(0xffffffffu, is_new);
  if (is_new) cand[ncand + __popc(mask & lanemask_lt())] = id;
  ncand += __popc(mask);
  __syncwarp();
}

// The keep-then-select step of hnswlib updatePoint for one row: the `keep` members of cand[0..ncand) closest
// to `owner` (owner itself skipped), ordered by (distance, id), then the heuristic with Mmax.  The selected
// ids are left in a.sel_id; returns their number.  u holds the `keep`: UList<8> in the register form, the
// shared-memory SList (up to kUpdCandCap - 1) in the wide form.
template <int LPV, int NQ, class Set>
__device__ __forceinline__ uint32_t reselect_row(WarpCtx& c, const GraphView& g, const Aux& a, Set& u,
                                                 const uint32_t* cand, uint32_t ncand, uint32_t owner, uint32_t keep,
                                                 uint32_t Mmax) {
  float4 qr[NQ];
  load_row_query<LPV, NQ>(c, qr, g, owner);
  ul_clear(u, keep, c.lane);
  uint32_t cnt = 0, worst_hi = 0xFFFFFFFFu;
  for (uint32_t b0 = 0; b0 < ncand; b0 += 32) {
    uint32_t id = b0 + c.lane < ncand ? cand[b0 + c.lane] : kInvalid;
    if (id == owner) id = kInvalid;
    uint32_t mask = __ballot_sync(0xffffffffu, id != kInvalid);
    uint32_t m = __popc(mask);
    if (!m) continue;
    if (id != kInvalid) c.cand_id[__popc(mask & lanemask_lt())] = id;
    __syncwarp();
    eval_candidates<LPV, NQ>(c, g.vecs, qr, m, g.metric);
    uint32_t myhi = 0xFFFFFFFFu, myid = kInvalid;
    if (c.lane < m) myhi = f2ord(c.cand_dist[c.lane]), myid = c.cand_id[c.lane];
    __syncwarp();
    uint32_t qual = __ballot_sync(0xffffffffu, c.lane < m && (cnt < keep || myhi < worst_hi));
    while (qual) {
      int l = __ffs(qual) - 1;
      qual &= qual - 1;
      uint32_t hj = __shfl_sync(0xffffffffu, myhi, l);
      uint32_t ij = __shfl_sync(0xffffffffu, myid, l);
      if (cnt >= keep && hj >= worst_hi) continue;
      ul_insert(u, hj, ij, keep, cnt, worst_hi, c.lane);
    }
  }
  set_to_list(c, u);
  return heuristic_select<LPV, NQ>(c, g, Mmax, a);
}

// hnswlib updatePoint, first half (the part before repairConnectionsForUpdate): when the vector of an
// already linked point p changes, every one-hop neighbour nb of p (per layer) gets its adjacency row
// re-selected by the heuristic over the closest ef_construction members of
//   sCand = {p} U one-hop(p) U two-hop(p)   (minus nb itself),
// distances measured from nb.  One warp per updated point; sCand (<= 1 + 2M + 2M*2M ids) is gathered
// into `upd_cand`.  Every warp reads the pre-wave graph.  When several moved points of one wave share a
// neighbour, the latest in arrival order re-selects its row: update_tag_kernel leaves 1 + that wave index in
// bb.row_fill (idle in this phase), only the winner computes the row, and it is staged (stage_row), so the
// result does not depend on scheduling.
static __global__ void update_tag_kernel(GraphView g, const uint8_t* __restrict__ levels, uint32_t cap,
                                         const uint32_t* __restrict__ ids, uint32_t b, uint32_t* tag) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t pi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pi >= b) return;
  const uint32_t p = ids[pi];
  const int level_p = min((int)levels[p], g.max_level);
  for (int layer = 0; layer <= level_p; ++layer) {
    const uint32_t nb = load_row(g, p, layer, lane);
    if (nb != kInvalid) atomicMax(&tag[layer == 0 ? nb : cap + g.up_off[nb] + (uint32_t)(layer - 1)], pi + 1u);
  }
}

// One moved point pi (= ids[pi] in the wave) with the warp's context; u holds the keep list (set_begin done).
template <int LPV, int NQ, class Set>
__device__ __forceinline__ void update_point(WarpCtx& c, const Aux& a, Set& u, const BuildGraph& bg, uint32_t pi,
                                             uint32_t p, const BuildBuffers& bb) {
  const GraphView& g = bg.g;
  uint32_t* cand = bb.upd_cand + (size_t)pi * kUpdCandCap;
  const int level_p = min((int)bg.levels[p], g.max_level);
  for (int layer = 0; layer <= level_p; ++layer) {
    const uint32_t one = load_row(g, p, layer, c.lane);
    const uint32_t n1 = __popc(__ballot_sync(0xffffffffu, one != kInvalid));
    if (n1 == 0) continue;
    // ---- sCand ----------------------------------------------------------------------------------
    hash_clear(c);
    uint32_t ncand = 0;
    cand_add(c, cand, ncand, c.lane == 0 ? p : kInvalid);
    cand_add(c, cand, ncand, one);
    for (uint32_t j = 0; j < n1; ++j) {
      const uint32_t e1 = __shfl_sync(0xffffffffu, one, j);
      cand_add(c, cand, ncand, load_row(g, e1, layer, c.lane));
    }
    // ---- re-select the row of every one-hop neighbour ----------------------------------------------
    const uint32_t Mmax = layer == 0 ? g.M0 : g.M;
    for (uint32_t j = 0; j < n1; ++j) {
      const uint32_t nbid = __shfl_sync(0xffffffffu, one, j);
      const uint32_t rid = layer == 0 ? nbid : bg.cap + g.up_off[nbid] + (uint32_t)(layer - 1);
      if (bb.row_fill[rid] != pi + 1u) continue;  // a later moved point of this wave re-selects this row
      // nb is always a member of sCand
      const uint32_t nsel = reselect_row<LPV, NQ>(c, g, a, u, cand, ncand, nbid, min(bg.efc, ncand - 1u), Mmax);
      uint32_t* row = stage_row(bb, rid, g.M0, c.lane);
      if (c.lane < Mmax) row[c.lane] = c.lane < nsel ? a.sel_id[c.lane] : kInvalid;
      __syncwarp();
    }
  }
}

template <int LPV, int NQ, int KPL>
__global__ void __launch_bounds__(128) update_neighbors_kernel(BuildGraph bg, WalkCfg cfg,
                                                               const uint32_t* __restrict__ ids, uint32_t b,
                                                               BuildBuffers bb, uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t pi = blockIdx.x * (blockDim.x >> 5) + w;
  if (pi >= b) return;
  const uint32_t p = ids[pi];
  WarpCtx c;
  ctx_init(c, smem + (size_t)w * warp_smem + 256, cfg, bg.g.dpad);
  Aux a = aux_of(c);
  UList<KPL> u;
  update_point<LPV, NQ>(c, a, u, bg, pi, p, bb);
}

// The wide form's update re-selection (efc > kMaxRegEfc): the keep list (up to kUpdCandCap - 1) in an SList of
// cfg.lcap / 2 keys beside its ordered list (set_init).  One warp per block and per moved point.
template <int LPV, int NQ>
__global__ void __launch_bounds__(32, 1) update_neighbors_wide_kernel(BuildGraph bg, WalkCfg cfg,
                                                                      const uint32_t* __restrict__ ids, uint32_t b,
                                                                      BuildBuffers bb, uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  (void)warp_smem;
  const uint32_t pi = blockIdx.x;
  if (pi >= b) return;
  WarpCtx c;
  ctx_init(c, smem + 256, cfg, bg.g.dpad);
  Aux a = aux_of(c);
  SList u;
  set_begin(u, c);
  update_point<LPV, NQ>(c, a, u, bg, pi, ids[pi], bb);
}

// Compaction repair (ehb_index_compact): the row of a live node p at layer l that names deleted points is
// re-selected over
//   C = {live ids of row_l(p)} U {live ids of row_l(v) : v in row_l(p), v deleted}   (minus p),
// keeping the efc closest to p and then the heuristic with Mmax -- the step updatePoint applies to a
// neighbour's row.  Every warp reads the pre-compaction graph and writes its result to bb.repair_out
// ([b][M0], kInvalid padded), so the outcome does not depend on scheduling.  rows[] holds row ids in the
// edge_row convention (< cap: level-0 row of that node; >= cap: upper row - cap).  One warp per row.
template <int LPV, int NQ, class Set>
__device__ __forceinline__ void repair_row(WarpCtx& c, const Aux& a, Set& u, const BuildGraph& bg, uint32_t pi,
                                           uint32_t r, const BuildBuffers& bb) {
  const GraphView& g = bg.g;
  uint32_t* cand = bb.upd_cand + (size_t)pi * kUpdCandCap;
  uint32_t p = r, layer = 0;
  if (r >= bg.cap) {
    p = bg.up_owner[r - bg.cap];
    layer = r - bg.cap - g.up_off[p] + 1u;
  }
  const uint32_t one = load_row(g, p, (int)layer, c.lane);
  const bool dead = one != kInvalid && g.deleted[one];
  hash_clear(c);
  uint32_t ncand = 0;
  cand_add(c, cand, ncand, dead ? kInvalid : one);
  for (uint32_t dm = __ballot_sync(0xffffffffu, dead); dm; dm &= dm - 1) {
    const uint32_t v = __shfl_sync(0xffffffffu, one, __ffs(dm) - 1);
    const uint32_t two = load_row(g, v, (int)layer, c.lane);
    cand_add(c, cand, ncand, two == kInvalid || two == p || g.deleted[two] ? kInvalid : two);
  }
  const uint32_t nsel =
      ncand ? reselect_row<LPV, NQ>(c, g, a, u, cand, ncand, p, min(bg.efc, ncand), layer ? g.M : g.M0) : 0u;
  uint32_t* out = bb.repair_out + (size_t)pi * g.M0;
  if (c.lane < g.M0) out[c.lane] = c.lane < nsel ? a.sel_id[c.lane] : kInvalid;
}

template <int LPV, int NQ, int KPL>
__global__ void __launch_bounds__(128) repair_rows_kernel(BuildGraph bg, WalkCfg cfg, const uint32_t* __restrict__ rows,
                                                          uint32_t b, BuildBuffers bb, uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t pi = blockIdx.x * (blockDim.x >> 5) + w;
  if (pi >= b) return;
  WarpCtx c;
  ctx_init(c, smem + (size_t)w * warp_smem + 256, cfg, bg.g.dpad);
  Aux a = aux_of(c);
  UList<KPL> u;
  repair_row<LPV, NQ>(c, a, u, bg, pi, rows[pi], bb);
}

// The wide form's compaction repair: keep min(efc, |C|) in an SList, as update_neighbors_wide_kernel.
template <int LPV, int NQ>
__global__ void __launch_bounds__(32, 1) repair_rows_wide_kernel(BuildGraph bg, WalkCfg cfg,
                                                                 const uint32_t* __restrict__ rows, uint32_t b,
                                                                 BuildBuffers bb, uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  (void)warp_smem;
  const uint32_t pi = blockIdx.x;
  if (pi >= b) return;
  WarpCtx c;
  ctx_init(c, smem + 256, cfg, bg.g.dpad);
  Aux a = aux_of(c);
  SList u;
  set_begin(u, c);
  repair_row<LPV, NQ>(c, a, u, bg, pi, rows[pi], bb);
}

static __global__ void edge_count_kernel(BuildBuffers bb) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t n = min(*bb.edge_count, bb.edge_cap);
  if (e >= n) return;
  uint32_t r = bb.edge_row[e];
  if (atomicAdd(&bb.row_cnt[r], 1u) == 0u) bb.touched[atomicAdd(bb.touched_count, 1u)] = r;
}
static __global__ void edge_alloc_kernel(BuildBuffers bb) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= *bb.touched_count) return;
  uint32_t r = bb.touched[t];
  bb.row_start[r] = atomicAdd(bb.seg_cursor, bb.row_cnt[r]);
}
static __global__ void edge_scatter_kernel(BuildBuffers bb) {
  uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t n = min(*bb.edge_count, bb.edge_cap);
  if (e >= n) return;
  uint32_t r = bb.edge_row[e];
  uint32_t pos = bb.row_start[r] + atomicAdd(&bb.row_fill[r], 1u);
  bb.seg_src[pos] = bb.edge_src[e];
  bb.seg_dist[pos] = bb.edge_dist[e];
}

// Phase C.  Incoming links are applied in source-id (= insertion) order, one at
// a time, exactly like hnswlib's mutuallyConnectNewElement: append while the row
// has room; when it is full re-select the row with the heuristic over
// (existing + the one new link).  Only after kMaxSeqPrunes such re-selections
// in one wave (hub rows) is the remainder -- every record of the row with a higher
// source id, however many -- folded into a single re-selection.
constexpr uint32_t kMaxSeqPrunes = 3;

template <int LPV, int NQ>
__global__ void __launch_bounds__(128) merge_rows_kernel(BuildGraph bg, WalkCfg cfg, BuildBuffers bb,
                                                         uint32_t warp_smem) {
  extern __shared__ __align__(128) unsigned char smem[];
  const GraphView& g = bg.g;
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t t = blockIdx.x * (blockDim.x >> 5) + w;
  if (t >= *bb.touched_count) return;
  const uint32_t r = bb.touched[t];
  const uint32_t ninc_all = bb.row_cnt[r], start = bb.row_start[r];
  WarpCtx c;
  ctx_init(c, smem + (size_t)w * warp_smem + 256, cfg, g.dpad);
  Aux a = aux_of(c);
  uint32_t node, W;
  uint32_t* row;
  if (r < bg.cap) {
    node = r;
    W = g.M0;
    row = const_cast<uint32_t*>(g.links0) + (size_t)r * g.M0;
  } else {
    uint32_t ur = r - bg.cap;
    node = bg.up_owner[ur];
    W = g.M;
    row = const_cast<uint32_t*>(g.links_up) + (size_t)ur * g.M;
  }
  const uint32_t limit = cfg.lcap;  // 128
  // 1. order the incoming links by source id (deterministic, = insertion order)
  c.cnt = 0;
  for (uint32_t j = 0; j < ninc_all; ++j)
    list_insert(c, ((uint64_t)bb.seg_src[start + j] << 32) | (j & kIdMask), limit);
  const uint32_t ninc = c.cnt;
  uint32_t in_src[4], in_j[4];
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    uint32_t i = (uint32_t)s * 32u + c.lane;
    uint64_t key = i < ninc ? c.keys[i] : kMaxKey;
    in_src[s] = (uint32_t)(key >> 32);
    in_j[s] = (uint32_t)key & kIdMask;
  }
  __syncwarp();
  // 2. the row, one entry per lane (compact: valid ids first)
  uint32_t e = c.lane < W ? row[c.lane] : kInvalid;
  float ed = 0.f;
  uint32_t ne = __popc(__ballot_sync(0xffffffffu, e != kInvalid));
  bool have_dists = false;
  uint32_t prunes = 0;
  float4 qr[NQ];
  for (uint32_t i = 0; i < ninc; ++i) {
    uint32_t sv = in_src[0], jv = in_j[0];
#pragma unroll
    for (int s = 1; s < 4; ++s)
      if ((i >> 5) == (uint32_t)s) sv = in_src[s], jv = in_j[s];
    const uint32_t sid = __shfl_sync(0xffffffffu, sv, i & 31);
    const uint32_t sj = __shfl_sync(0xffffffffu, jv, i & 31);
    if (__any_sync(0xffffffffu, e == sid)) continue;  // already linked (update path)
    const float sd = bb.seg_dist[start + sj];
    if (ne < W) {
      if (c.lane == ne) e = sid, ed = sd;
      ne++;
      continue;
    }
    // row full: distances of the existing entries to the row's owner are needed once
    if (!have_dists) {
      load_row_query<LPV, NQ>(c, qr, g, node);
      if (c.lane < ne) c.cand_id[c.lane] = e;
      __syncwarp();
      eval_candidates<LPV, NQ>(c, g.vecs, qr, ne, g.metric);
      if (c.lane < ne) ed = c.cand_dist[c.lane];
      __syncwarp();
      have_dists = true;
    }
    c.cnt = 0;
    uint64_t mykey = c.lane < ne ? make_key(ed, e) : kMaxKey;
    for (uint32_t j = 0; j < ne; ++j) list_insert(c, __shfl_sync(0xffffffffu, mykey, j), limit);
    list_insert(c, make_key(sd, sid), limit);
    bool fold_rest = ++prunes > kMaxSeqPrunes;
    if (fold_rest) {
      // every record not applied yet (source id above sid), read from the whole segment: a hub row can receive
      // more records than the `limit` lowest source ids ordered above.  The list keeps the `limit` closest by
      // (distance, id) whatever the insertion order; list_insert drops duplicate ids.
      for (uint32_t j0 = 0; j0 < ninc_all; j0 += 32) {
        const uint32_t j = j0 + c.lane;
        const uint32_t s2 = j < ninc_all ? bb.seg_src[start + j] : 0u;
        const uint64_t key = j < ninc_all && s2 > sid ? make_key(bb.seg_dist[start + j], s2) : kMaxKey;
        for (uint32_t q = __ballot_sync(0xffffffffu, key != kMaxKey); q; q &= q - 1)
          list_insert(c, __shfl_sync(0xffffffffu, key, __ffs(q) - 1), limit);
      }
    }
    uint32_t nsel = heuristic_select<LPV, NQ>(c, g, W, a);
    e = c.lane < nsel ? a.sel_id[c.lane] : kInvalid;
    ed = c.lane < nsel ? a.sel_dist[c.lane] : 0.f;
    ne = nsel;
    __syncwarp();
    if (fold_rest) break;
  }
  if (c.lane < W) row[c.lane] = e;
  if (c.lane == 0) {
    bb.row_cnt[r] = 0;
    bb.row_fill[r] = 0;
  }
}

static cudaError_t apply_staged(const BuildGraph& bg, const BuildBuffers& bb, cudaStream_t s) {
  const uint64_t threads = (uint64_t)bb.side_cap * bg.g.M0;
  apply_staged_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(
      bb, const_cast<uint32_t*>(bg.g.links0), const_cast<uint32_t*>(bg.g.links_up), bg.cap, bg.g.M0, bg.g.M);
  return cudaGetLastError();
}

template <uint32_t DPAD>
cudaError_t BuildShape<DPAD>::launch(const BuildGraph& bg, const WalkCfg& cfg, const uint32_t* ids, uint32_t first,
                                     uint32_t b, int mode, BuildBuffers& bb, uint32_t wpb, const BuildBeam& bm,
                                     cudaStream_t s) {
  constexpr int LPV = row_lpv(DPAD * 4u), NQ = row_nq(DPAD, DPAD * 4u);
  constexpr int KPL = 8;  // the register form: ef_construction <= kMaxRegEfc
  // the wide form (efc > kMaxRegEfc): shared-memory sets, the search's visited tables in bm.vtab
  const bool beam = bg.efc > kMaxRegEfc;
  if (beam && (!bm.vtab || bm.warps == 0 || bm.vsize == 0)) return cudaErrorInvalidValue;
  cudaError_t e;
  const bool is_update = mode == kBuildUpdate;
  if (mode == kBuildUpdate || mode == kBuildRepair) {
    if (!ids || !bb.upd_cand || (mode == kBuildRepair && (!bb.repair_out || !bg.g.deleted))) return cudaErrorInvalidValue;
    // the two-hop candidate sets are deduplicated through a visited table of >= 4096 entries
    WalkCfg ucfg = cfg;
    if (ucfg.hash_size < 4096) ucfg.hash_size = 4096;
    // the wide form keeps up to min(efc, kUpdCandCap - 1) candidates in an SList beside their ordered list
    if (beam) ucfg.lcap = 2u * align_up(min(bg.efc, kUpdCandCap), 32);
    uint32_t uwsm = build_warp_smem(ucfg, bg.g.dpad), uwpb = beam ? 1u : wpb;  // the wide kernels: one warp per block
    while (uwpb > 1 && (size_t)uwsm * uwpb > 200 * 1024) uwpb >>= 1;
    auto ku = beam ? BuildBeamShape<DPAD>::rows(mode)
                   : (mode == kBuildUpdate ? update_neighbors_kernel<LPV, NQ, KPL> : repair_rows_kernel<LPV, NQ, KPL>);
    if ((e = cudaFuncSetAttribute(ku, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)uwsm * uwpb))) !=
        cudaSuccess)
      return e;
    if (mode == kBuildUpdate) {
      if (!bb.side_row || !bb.side_out || !bb.side_count) return cudaErrorInvalidValue;
      if ((e = cudaMemsetAsync(bb.side_count, 0, 4, s)) != cudaSuccess) return e;
      update_tag_kernel<<<(b + 3) / 4, 128, 0, s>>>(bg.g, bg.levels, bg.cap, ids, b, bb.row_fill);
    }
    // one warp per moved point / repaired row; repairs go in launches of <= kRepairWarps rows (upd_cand slots)
    const uint32_t chunk = mode == kBuildUpdate ? b : kRepairWarps;
    for (uint32_t off = 0; off < b; off += chunk) {
      const uint32_t m = min(chunk, b - off);
      BuildBuffers cb = bb;
      if (mode == kBuildRepair) cb.repair_out += (size_t)off * bg.g.M0;
      ku<<<(m + uwpb - 1) / uwpb, 32 * uwpb, (size_t)uwsm * uwpb, s>>>(bg, ucfg, ids + off, m, cb, uwsm);
    }
    // updatePoint's neighbour re-selection runs before the moved points are re-linked
    if (mode == kBuildRepair) return cudaGetLastError();
    if ((e = apply_staged(bg, bb, s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(bb.side_count, 0, 4, s)) != cudaSuccess) return e;
  }
  if ((e = cudaMemsetAsync(bb.edge_count, 0, 4, s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(bb.touched_count, 0, 4, s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(bb.seg_cursor, 0, 4, s)) != cudaSuccess) return e;
  uint32_t wsm = build_warp_smem(cfg, bg.g.dpad);
  size_t smem = (size_t)wsm * wpb;
  // the merge pass needs no visited table
  WalkCfg mcfg = cfg;
  mcfg.hash_size = 0;
  mcfg.lcap = 128;
  uint32_t mwsm = build_warp_smem(mcfg, bg.g.dpad);
  uint32_t mwpb = 4;
  size_t msmem = (size_t)mwsm * mwpb;
  while (msmem > 200 * 1024 && mwpb > 1) mwpb >>= 1, msmem = (size_t)mwsm * mwpb;
  dim3 grid((b + wpb - 1) / wpb), block(32 * wpb);
  uint32_t ethreads = bb.edge_cap;
  auto km = merge_rows_kernel<LPV, NQ>;
  if ((e = cudaFuncSetAttribute(km, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msmem)) != cudaSuccess) return e;
  if (beam) {
    // one warp per block, at most one per visited-table slice
    const BuildSearchBeamKernel kb = BuildBeamShape<DPAD>::search(bg.g.deleted != nullptr);
    if ((e = cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsm)) != cudaSuccess) return e;
    kb<<<min(b, bm.warps), 32, wsm, s>>>(bg, cfg, ids, first, b, is_update ? 1 : 0, bb, bm.vsize, bm.vtab);
  } else {
    auto ks = bg.g.deleted ? build_search_kernel<LPV, NQ, KPL, true> : build_search_kernel<LPV, NQ, KPL, false>;
    if ((e = cudaFuncSetAttribute(ks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    ks<<<grid, block, smem, s>>>(bg, cfg, ids, first, b, is_update ? 1 : 0, bb, wsm);
  }
  edge_count_kernel<<<(ethreads + 255) / 256, 256, 0, s>>>(bb);
  edge_alloc_kernel<<<(ethreads + 255) / 256, 256, 0, s>>>(bb);
  edge_scatter_kernel<<<(ethreads + 255) / 256, 256, 0, s>>>(bb);
  if (is_update && (e = apply_staged(bg, bb, s)) != cudaSuccess) return e;  // the moved points' own rows
  km<<<(ethreads + mwpb - 1) / mwpb, 32 * mwpb, msmem, s>>>(bg, mcfg, bb, mwsm);
  return cudaGetLastError();
}

}  // namespace ehb
