// Host side of the ehb200 C ABI (include/ehb200.h): index state in HBM, batched construction driver,
// tombstones, re-entrant search entry points with a combining queue.  Mirrors the responsibilities of
// featureform::embedding::ANNIndex + hnswlib::HierarchicalNSW as used in
// embeddinghub/embeddingstore/index.cc:10-52.  (Persistence: io.cu; sharding / shard exchange: exchange.cu.)
#include "index_impl.h"

namespace ehb {
thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
const std::string& last_error_text() { return g_err; }
}  // namespace ehb
using ehb::fail;

// ============================================================================================
// index state
// ============================================================================================
ehb_index::~ehb_index() {
  slots.clear();
  if (bf_ev0) cudaEventDestroy(bf_ev0);
  if (bf_ev1) cudaEventDestroy(bf_ev1);
  if (beam_done) cudaEventDestroy(beam_done);
  if (stream) cudaStreamDestroy(stream);
}

ehb::GraphView ehb_index::view() const {
  ehb::GraphView g;
  g.vecs = vecs.p;
  g.links0 = links0.p;
  g.up_off = up_off.p;
  g.links_up = links_up.p;
  g.labels = labels.p;
  g.deleted = n_deleted ? deleted.p : nullptr;
  g.n = (uint32_t)n_linked;
  g.dim = dim;
  g.dpad = dpad;
  g.M = M;
  g.M0 = M0;
  g.entry = entry;
  g.max_level = max_level;
  g.metric = metric == EHB_L2 ? 0 : 1;
  g.vecs16 = nullptr;
  g.codes8 = nullptr;
  g.terms8 = nullptr;
  return g;
}

// The fp32 walk's int8 screen (walk.cuh beam_search) applies to staged rows (> 1 KB, dpad <= 1536) under 1 - dot.
// By default it runs for batches of at least kScreenMinBatchPerSm queries per SM: those keep the walk bound by DRAM
// bandwidth, which the screen relieves; a smaller batch is bound by each warp's chain of memory round trips, to
// which the screen adds one per hop.
bool ehb_index::walk_screens(uint64_t nq) const {
  if (o_walk_screen == 0 || metric == EHB_L2) return false;
  if (!ehb::screen_shape(ehb::row_lpv(dpad * 4u), ehb::row_nq(dpad, dpad * 4u))) return false;
  return o_walk_screen > 0 || nq >= (uint64_t)ehb::kScreenMinBatchPerSm * sms;
}

// The screen is an optimisation: when its copy does not fit next to the index, the walk runs unscreened.
int ehb_index::try_screen_copy() {
  size_t fr = 0, tot = 0;
  const uint64_t need = std::max<uint64_t>(cap, 1) * (dpad + sizeof(float4)) + (256ull << 20);
  bool ok = cudaMemGetInfo(&fr, &tot) == cudaSuccess && fr >= need;
  if (ok) {
    cudaError_t e = x_i8.grow(std::max<uint64_t>(cap, 1) * dpad, 0, -1, stream);
    if (e == cudaSuccess) e = x_i8t.grow(std::max<uint64_t>(cap, 1), 0, -1, stream);
    if (e == cudaSuccess) e = ehb::launch_to_i8(vecs.p, dpad, x_i8.p, x_i8t.p, n, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    screen_copy = e == cudaSuccess;
    if (!screen_copy) {
      x_i8.release();
      x_i8t.release();
      ok = false;
    }
  }
  if (!ok) {
    (void)cudaGetLastError();
    ehb::g_err.clear();
    screen_no_room = true;
  }
  return EHB_OK;
}

// ef_eff: beam width; smem_list: capacity of the shared-memory key list (0 for plain searches);
// jobs: warps (queries or points) of the launch; team: warps sharing one visited table; dense: the launch runs
// the dense form of the walk (walk_plan); screen: the launch runs a screened fp32 walk, which reads its rows straight
// into registers and has no TMA ring (its G and NG are unused).
ehb::WalkCfg ehb_index::walk_cfg(uint32_t ef_eff, uint32_t smem_list, uint64_t jobs, uint32_t team, bool bf16,
                                 bool dense, bool screen) const {
  ehb::WalkCfg c;
  const uint32_t esize = bf16 ? 2u : 4u, vbytes = dpad * esize;  // bytes of a row as the walk reads it
  // the wide shapes keep the query in shared memory and have no ring (walk.cuh eval_wide)
  const bool wide = ehb::wide_shape(ehb::row_lpv(vbytes), ehb::row_nq(dpad, vbytes));
  c.lcap = smem_list;
  c.staged = ehb::row_lpv(vbytes) == 32 && !wide ? 1 : 0;  // rows above 1 KB go through the TMA staging ring
  c.dcap = n_deleted ? ehb::kDeletedQueue : 0;
  c.prefetch = o_walk_prefetch ? 1 : 0;
  c.dense = dense ? 1 : 0;
  // resident warps per SM the visited-table sizing aims at; the wide walk's ~220 registers allow eight
  const uint32_t warp_target = c.dense ? 20u : (wide ? 8u : 16u);
  uint32_t nslots = std::max(4u, std::min(32u, 24576u / vbytes));
  uint32_t ng = 2;                      // two groups: math on one overlaps the copies of the other
  uint32_t g = std::max(4u, nslots / ng / 4 * 4);  // vectors per group, multiple of the 4-vector math step
  if (t_slots) g = std::min(32u, t_slots);
  if (t_groups) ng = std::min(8u, t_groups);
  c.G = std::max(1u, g);
  c.NG = std::max(1u, ng);
  // Visited table.  A hop admits at most 2M new ids and the walk makes about ef hops.  "roomy" keeps
  // the final load near 0.5 even on iid Gaussian data (~29 new ids per hop); but every KB of table
  // costs occupancy, and a crowded table only costs re-evaluations (probes are bounded; duplicates
  // are filtered against the result set), so a table smaller than the visited count adds only a few
  // re-evaluations while the occupancy it buys speeds up the memory-bound walk.  So: as roomy as the
  // occupancy target allows, never below a quarter of the worst case.
  const uint32_t roomy = 2u * M0 * ef_eff + 64u, tight = std::max(256u, M0 * ef_eff / 4u);
  uint32_t hs = roomy;
  if (t_hash_bits) {
    hs = 1u << t_hash_bits;
  } else {
    uint64_t ctas = (jobs + team - 1) / std::max(team, 1u);
    uint32_t want = (uint32_t)std::min<uint64_t>((ctas + sms - 1) / sms, c.staged ? 5u : warp_target / team);
    want = std::max(want, 4u);
    c.hash_size = 0;
    uint32_t fixed = ehb::warp_smem_bytes(c, dpad, esize) * team + 1024u + (smem_list ? 256u : 0u);
    uint32_t per_cta = (227u * 1024u) / want;
    uint32_t avail = per_cta > fixed + 1024u ? (per_cta - fixed) / 4u : 256u;
    hs = std::min(roomy, std::max(tight, avail));
    if (n_deleted) hs = roomy;  // tombstoned candidates rely on the visited table alone (no result-set filter)
  }
  c.hash_size = ehb::align_up(std::max(hs, 256u), 32);
  // stay inside the 227 KB per-block limit
  while (ehb::warp_smem_bytes(c, dpad, esize) + 256 > 200 * 1024 && c.hash_size > 512)
    c.hash_size = ehb::align_up(c.hash_size / 2, 32);
  // A screened walk keeps the visited table sized as above, for five staged warps per SM, so that it revisits and
  // counts exactly what the unscreened walk does; without the ring that table still leaves room for the ten warps its
  // 200 registers allow at dpad <= 768 (search_impl.cuh; at C3: 5,152 entries, 21 KB per warp).
  if (screen) c.staged = 0;
  return c;
}

ehb::WalkCfg ehb_index::beam_cfg(uint32_t ef, uint32_t smem_list, uint64_t jobs, bool bf16) const {
  ehb::WalkCfg c = walk_cfg(ef, smem_list, jobs, 1, bf16);
  c.hash_size = 0;
  // tombstoned candidates wait in the side queue; a wider beam keeps proportionally more of them pending
  if (n_deleted) c.dcap = std::max(ehb::kDeletedQueue, ehb::align_up(ef / 4, 32));
  return c;
}

uint32_t ehb_index::wpb_for(const ehb::WalkCfg& c, uint32_t extra, bool bf16) const {
  uint32_t w = t_wpb ? t_wpb : 1;
  while (w > 1 && (size_t)(ehb::warp_smem_bytes(c, dpad, bf16 ? 2u : 4u) + extra) * w > 220 * 1024) w >>= 1;
  return w;
}

// Largest batch for which the T = 4 team walk keeps its wide U: registers are no constraint while <= 3 CTAs of 128
// threads (~125 registers each) sit on each SM of the H100's 132.
constexpr uint64_t kTeamWideMaxQueries = 132u * 3u;

ehb::WalkPlan ehb_index::walk_plan(uint64_t nq, uint32_t ef_eff, bool bf16) const {
  ehb::WalkPlan p;
  p.bf16 = bf16;
  const uint32_t row_bytes = dpad * (bf16 ? 2u : 4u);
  p.lpv = ehb::row_lpv(row_bytes);
  p.nq = ehb::row_nq(dpad, row_bytes);
  p.kpl = ehb::kpl_for(ef_eff);
  p.hasdel = n_deleted != 0;
  // Warps per query (rows <= 1 KB, ef <= 256): four while 3 CTAs of 128 threads per SM hold every query (small
  // online batches, where one warp's serial chain of memory round trips is the bound), two while 7 CTAs of 64
  // threads do (C2, Q=1000), else one warp per query: once the batch alone fills the SMs, the team walk's
  // speculative expansions only add work (C5 shape, Q=10k).
  if (ef_eff > ehb::kMaxEf) {  // the wide-beam walk: result set in shared memory, visited table in HBM
    p.kpl = 0;
    p.T = 1;
    p.U = 0;
    p.form = ehb::WalkForm::beam;
    p.screen = false;
    p.cfg = beam_cfg(ef_eff, ehb::align_up(ef_eff, 32), nq, bf16);
    p.vtab = beam_vtab_size(ef_eff);
    p.wpb = 1;
    return p;
  }
  p.vtab = 0;
  uint32_t team = t_team;
  if (team == 0) team = nq <= (uint64_t)sms * 3 ? 4 : (nq <= (uint64_t)sms * 7 ? 2 : 1);
  if (dpad > 256 || ef_eff > 256 || n_deleted) team = 1;  // tombstones: the one-warp walk carries the side queue
  if (bf16) team = 1;                                       // the team walk reads fp32 rows only
  p.T = team;
  // Vector-load steps (4 vectors each) a team warp keeps in flight.  Registers of loads in flight per lane are
  // sized so that 7 CTAs fit an SM (T = 2: 64, T = 3 and 4: 32), except that T = 4 keeps the full 16-vector
  // batches when the batch is so small that registers are no constraint.
  const bool wide = team == 2 || (team == 4 && nq <= kTeamWideMaxQueries);
  p.U = team == 1 ? 0 : (uint32_t)ehb::eval_u(p.nq, wide ? 1 : 2);
  // dense walk (search_impl.cuh): batches big enough to fill 20 warps per SM, on the shapes that have one
  if (team > 1)
    p.form = ehb::WalkForm::team;
  else if (ehb::wide_shape(p.lpv, p.nq))
    p.form = ehb::WalkForm::wide;
  else if (nq >= 20ull * (uint64_t)sms && ehb::dense_form(bf16, p.lpv, p.nq, p.kpl, p.hasdel))
    p.form = ehb::WalkForm::dense;
  else
    p.form = ehb::WalkForm::plain;
  p.screen = !bf16 && team == 1 && screen_copy && walk_screens(nq);
  p.cfg = walk_cfg(ef_eff, 0, nq * team, team, bf16, p.form == ehb::WalkForm::dense, p.screen);
  p.wpb = wpb_for(p.cfg, 0, bf16);
  return p;
}

int ehb_index::ensure_capacity(uint64_t want) {
  if (want <= cap) return EHB_OK;
  uint64_t nc = std::max<uint64_t>(cap ? cap : 1, 1);
  while (nc < want) nc *= 2;  // index.cc:29-32 doubles
  if (nc >= 0x7FFFFFFFull) return fail(EHB_ERR_INVALID, "capacity must stay below 2^31 vectors per index");
  CU(vecs.grow(nc * dpad, n * dpad, -1, stream));
  CU(labels.grow(nc, n, -1, stream));
  CU(levels.grow(nc, n, 0, stream));
  CU(deleted.grow(nc, n, 0, stream));
  CU(links0.grow(nc * M0, n * M0, 0xFF, stream));
  CU(up_off.grow(nc, n, 0xFF, stream));
  if (shadow) {
    CU(x_bf16.grow(nc * dpad, n * dpad, -1, stream));
    CU(x_norm.grow(nc, n, -1, stream));
  }
  if (screen_copy) {
    CU(x_i8.grow(nc * dpad, n * dpad, -1, stream));
    CU(x_i8t.grow(nc, n, -1, stream));
  }
  cap = nc;
  return EHB_OK;
}

// ---- copies derived from the rows (index_impl.h) -----------------------------------------------------------
// Writer side.  Sized like vecs (capacity rows), so adds within the capacity never reallocate them.
int ehb_index::create_shadow() {
  if (shadow) return EHB_OK;
  CU(x_bf16.grow(std::max<uint64_t>(cap, 1) * dpad, 0, -1, stream));
  CU(x_norm.grow(std::max<uint64_t>(cap, 1), 0, -1, stream));
  CU(ehb::launch_to_bf16(vecs.p, dpad, x_bf16.p, x_norm.p, n, dpad, stream));
  CU(cudaStreamSynchronize(stream));
  shadow = true;
  return EHB_OK;
}

void ehb_index::drop_derived() {
  x_bf16.release();
  x_norm.release();
  shadow = false;
  x_i8.release();
  x_i8t.release();
  screen_copy = false;
}

int ehb_index::derive_rows(uint64_t first, uint64_t cnt) {
  if (cnt == 0) return EHB_OK;
  if (shadow)
    CU(ehb::launch_to_bf16(vecs.p + first * dpad, dpad, x_bf16.p + first * dpad, x_norm.p + first, cnt, dpad, stream));
  if (screen_copy) CU(ehb::launch_to_i8(vecs.p + first * dpad, dpad, x_i8.p + first * dpad, x_i8t.p + first, cnt, stream));
  return EHB_OK;
}

int ehb_index::ensure_upper(uint64_t want_rows) {
  if (want_rows <= links_up.n / M && links_up.n) return EHB_OK;
  uint64_t nr = std::max<uint64_t>(links_up.n / M, 64);
  while (nr < want_rows) nr *= 2;
  CU(links_up.grow(nr * M, up_rows * M, 0xFF, stream));
  CU(up_owner.grow(nr, up_rows, 0, stream));
  return EHB_OK;
}

// hnswlib getRandomLevel: (int)(-log(U(0,1)) * 1/ln(M)) drawn from std::default_random_engine(seed), one
// draw per new point in insertion order — the same generator classes upstream uses, so levels match an
// hnswlib built against the same C++ standard library.  Levels are stored in a byte and upper rows are laid
// out per level, so a draw above 31 (probability M^-32) is clamped.
int ehb_index::draw_level() {
  std::uniform_real_distribution<double> u(0.0, 1.0);
  double r = -std::log(u(level_rng)) * (1.0 / std::log((double)M));
  return std::min((int)r, 31);
}

bool ehb_index::find_id(uint64_t label, uint32_t* id) const {
  if (identity_labels) {
    if (label >= n) return false;
    *id = (uint32_t)label;
    return true;
  }
  auto it = lookup.find(label);
  if (it == lookup.end()) return false;
  *id = it->second;
  return true;
}

void ehb_index::reset_content() {
  n = n_linked = up_rows = n_deleted = n_removed = 0;
  entry = 0;
  max_level = -1;
  lookup.clear();
  h_labels.clear();
  h_levels.clear();
  h_deleted.clear();
  pending_updates.clear();
  identity_labels = true;
  drop_derived();
}

// ---- ingest ---------------------------------------------------------------------------------------
// Insert-or-update (ANNIndex::set, index.cc:20-37).  Host-side maps are committed only after every device
// operation of the chunk succeeded, so a failed add (OOM while doubling) leaves the index unchanged.
int ehb_index::add_rows(uint64_t cnt, const float* src, bool src_is_device, const uint64_t* lab) {
  if (cnt == 0) return EHB_OK;
  const uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / (dim * 4));
  for (uint64_t off = 0; off < cnt; off += chunk) {
    const uint64_t m = std::min(chunk, cnt - off);
    std::vector<uint32_t> dst(m);
    std::vector<uint64_t> new_labels;
    std::vector<uint32_t> relink, undelete;
    std::unordered_map<uint64_t, uint32_t> new_map;  // labels first seen in this chunk (non-identity mode)
    const uint64_t first_new = n;
    bool contiguous_new = true;
    uint64_t nn = n;
    for (uint64_t i = 0; i < m; ++i) {
      const uint64_t l = lab ? lab[off + i] : nn + n_removed;  // labels removed by compact() are not reused
      bool exists = false;
      uint32_t id = 0;
      if (identity_labels) {
        if (l < nn) {
          exists = true, id = (uint32_t)l;
        } else if (l != nn) {
          // leave identity mode: materialise the map (a consistent state on its own)
          lookup.reserve(std::max<uint64_t>(nn * 2, 1024));
          for (uint64_t j = 0; j < n; ++j) lookup[j] = (uint32_t)j;
          for (uint64_t j = n; j < nn; ++j) new_map[j] = (uint32_t)j;
          identity_labels = false;
        }
      }
      if (!identity_labels && !exists) {
        auto it = lookup.find(l);
        if (it != lookup.end()) {
          exists = true, id = it->second;
        } else {
          auto it2 = new_map.find(l);
          if (it2 != new_map.end()) exists = true, id = it2->second;
        }
      }
      if (exists) {
        dst[i] = id;
        contiguous_new = false;
        if (id < n_linked) relink.push_back(id);  // already in the graph: updatePoint at the next build
        if (id < n && h_deleted[id]) undelete.push_back(id);  // hnswlib addPoint un-deletes a re-added label
      } else {
        dst[i] = (uint32_t)nn;
        if (!identity_labels) new_map[l] = (uint32_t)nn;
        new_labels.push_back(l);
        nn++;
      }
    }
    RET(ensure_capacity(nn));
    // levels + upper rows for the new ids (the generator only advances on commit)
    const uint64_t new_cnt = nn - first_new;
    std::default_random_engine rng_backup = level_rng;
    std::vector<uint8_t> lv(new_cnt);
    std::vector<uint32_t> uo(new_cnt), owners;
    uint64_t rows = up_rows;
    for (uint64_t j = 0; j < new_cnt; ++j) {
      int l = draw_level();
      lv[j] = (uint8_t)l;
      uo[j] = l ? (uint32_t)rows : ehb::kInvalid;
      for (int t = 0; t < l; ++t) owners.push_back((uint32_t)(first_new + j));
      rows += l;
    }
    auto device_part = [&]() -> int {
      RET(ensure_upper(rows));
      if (new_cnt) {
        CU(cudaMemcpyAsync(levels.p + first_new, lv.data(), new_cnt, cudaMemcpyHostToDevice, stream));
        CU(cudaMemcpyAsync(up_off.p + first_new, uo.data(), new_cnt * 4, cudaMemcpyHostToDevice, stream));
        CU(cudaMemcpyAsync(labels.p + first_new, new_labels.data(), new_cnt * 8, cudaMemcpyHostToDevice, stream));
        CU(cudaMemsetAsync(deleted.p + first_new, 0, new_cnt, stream));
        if (!owners.empty())
          CU(cudaMemcpyAsync(up_owner.p + up_rows, owners.data(), owners.size() * 4, cudaMemcpyHostToDevice, stream));
      }
      for (uint32_t id : undelete) CU(cudaMemsetAsync(deleted.p + id, 0, 1, stream));
      // stage the rows and scatter/pad/normalise them into place
      const float* dsrc;
      if (src_is_device) {
        dsrc = src + off * dim;
      } else {
        CU(b_stage_in.grow(m * dim, 0, -1, stream));
        CU(cudaMemcpyAsync(b_stage_in.p, src + off * dim, m * dim * 4, cudaMemcpyHostToDevice, stream));
        dsrc = b_stage_in.p;
      }
      if (contiguous_new) {
        CU(ehb::launch_pad_rows(dsrc, vecs.p + first_new * dpad, m, dim, dpad, metric == EHB_COSINE, stream));
        RET(derive_rows(first_new, m));
      } else {
        // rows go to arbitrary ids: one launch per run of consecutive destinations
        uint64_t i = 0;
        while (i < m) {
          uint64_t j = i + 1;
          while (j < m && dst[j] == dst[j - 1] + 1) ++j;
          CU(ehb::launch_pad_rows(dsrc + i * dim, vecs.p + (uint64_t)dst[i] * dpad, j - i, dim, dpad,
                                  metric == EHB_COSINE, stream));
          RET(derive_rows(dst[i], j - i));
          i = j;
        }
      }
      CU(cudaStreamSynchronize(stream));  // host staging vectors go out of scope
      return EHB_OK;
    };
    int rc = device_part();
    if (rc != EHB_OK) {
      level_rng = rng_backup;
      return rc;
    }
    // ---- commit ----
    if (!identity_labels)
      for (auto& kv : new_map) lookup[kv.first] = kv.second;
    h_labels.insert(h_labels.end(), new_labels.begin(), new_labels.end());
    h_levels.insert(h_levels.end(), lv.begin(), lv.end());
    h_deleted.resize(nn, 0);
    for (uint32_t id : undelete)
      if (h_deleted[id]) h_deleted[id] = 0, n_deleted--;
    pending_updates.insert(pending_updates.end(), relink.begin(), relink.end());
    n = nn;
    up_rows = rows;
  }
  return EHB_OK;
}

// hnswlib markDelete (promised by embeddinghub/docs/reading_and_writing_embeddings.md:49-66): the point
// stays in the graph as a tombstone — still traversed, never returned.
int ehb_index::remove_labels(uint64_t cnt, const uint64_t* lab) {
  std::vector<uint32_t> ids(cnt);
  for (uint64_t i = 0; i < cnt; ++i) {
    if (!find_id(lab[i], &ids[i])) return fail(EHB_ERR_NOT_FOUND, "label not found");
    if (h_deleted[ids[i]]) return fail(EHB_ERR_STATE, "the requested to delete element is already deleted");
  }
  {
    std::vector<uint32_t> s = ids;
    std::sort(s.begin(), s.end());
    if (std::adjacent_find(s.begin(), s.end()) != s.end()) return fail(EHB_ERR_INVALID, "label listed twice");
  }
  for (uint32_t id : ids) CU(cudaMemsetAsync(deleted.p + id, 1, 1, stream));
  CU(cudaStreamSynchronize(stream));
  for (uint32_t id : ids) h_deleted[id] = 1;
  n_deleted += cnt;
  return EHB_OK;
}

// ---- construction ------------------------------------------------------------------------------------
int ehb_index::ensure_build_scratch(uint64_t edges, uint32_t batch, bool updates) {
  const uint64_t ecap = edges + 1024;
  CU(b_edge_row.grow(ecap, 0, -1, stream));
  CU(b_edge_src.grow(ecap, 0, -1, stream));
  CU(b_edge_dist.grow(ecap, 0, -1, stream));
  CU(b_touched.grow(ecap, 0, -1, stream));
  CU(b_seg_src.grow(ecap, 0, -1, stream));
  CU(b_seg_dist.grow(ecap, 0, -1, stream));
  CU(b_counters.grow(8, 0, 0, stream));
  if (updates) CU(b_upd_cand.grow((uint64_t)batch * ehb::kUpdCandCap, 0, -1, stream));
  uint64_t rowspace = cap + links_up.n / M;
  if (b_row_cnt.n < rowspace) {
    b_row_cnt.release();
    b_row_fill.release();
    b_row_start.release();
    CU(b_row_cnt.grow(rowspace, 0, 0, stream));
    CU(b_row_fill.grow(rowspace, 0, 0, stream));
    CU(b_row_start.grow(rowspace, 0, 0, stream));
  }
  return EHB_OK;
}

ehb::BuildBuffers ehb_index::build_buffers(uint64_t edges) {
  ehb::BuildBuffers bb;
  bb.edge_row = b_edge_row.p;
  bb.edge_src = b_edge_src.p;
  bb.edge_dist = b_edge_dist.p;
  bb.edge_count = b_counters.p + 0;
  bb.edge_cap = (uint32_t)std::min<uint64_t>(b_edge_row.n, edges + 1024);
  bb.row_cnt = b_row_cnt.p;
  bb.row_fill = b_row_fill.p;
  bb.row_start = b_row_start.p;
  bb.touched = b_touched.p;
  bb.touched_count = b_counters.p + 1;
  bb.seg_cursor = b_counters.p + 2;
  bb.seg_src = b_seg_src.p;
  bb.seg_dist = b_seg_dist.p;
  bb.error_flag = b_counters.p + 3;
  bb.upd_cand = b_upd_cand.p;
  bb.repair_out = nullptr;
  bb.side_row = b_side_row.p;
  bb.side_out = b_side_out.p;
  bb.side_count = b_counters.p + 6;
  bb.side_cap = (uint32_t)b_side_row.n;
  return bb;
}

ehb::BuildGraph ehb_index::build_graph() const {
  ehb::BuildGraph bg;
  bg.g = view();
  bg.levels = levels.p;
  bg.up_owner = up_owner.p;
  bg.cap = (uint32_t)cap;
  bg.efc = std::max(prm.ef_construction, M);
  return bg;
}

ehb::WalkCfg ehb_index::build_cfg(uint64_t jobs) const {
  const uint32_t efc = std::max(prm.ef_construction, M);
  if (efc <= ehb::kMaxRegEfc) return walk_cfg(efc, 256, jobs, 1);
  return beam_cfg(efc, 2u * ehb::align_up(efc, 32), jobs);  // the set and the ordered list the heuristic walks
}

int ehb_index::reserve_build_beam(ehb::BuildBeam* bm) {
  *bm = ehb::BuildBeam{nullptr, 0, 0};
  const uint32_t efc = std::max(prm.ef_construction, M);
  if (efc <= ehb::kMaxRegEfc) return EHB_OK;
  bm->vsize = beam_vtab_size(efc);
  // Sized for the form without tombstones, whose footprint is the smaller one, so that the size does not depend on the
  // tombstones of the moment (a compaction's re-links run after it has dropped them); a launch never uses more warps
  // than the tables here hold.
  ehb::BuildGraph bg = build_graph();
  bg.g.deleted = nullptr;
  ehb::WalkCfg cfg = build_cfg(1);
  cfg.dcap = 0;
  uint32_t warps = 0;
  CU(ehb::build_beam_warps(bg, cfg, sms, &warps));
  CU(b_vtab.grow((size_t)warps * bm->vsize, 0, -1, stream));
  bm->vtab = b_vtab.p;
  bm->warps = (uint32_t)(b_vtab.n / bm->vsize);
  return EHB_OK;
}

int ehb_index::build() {
  if (!needs_build()) return EHB_OK;
  const uint32_t maxb = prm.build_batch ? prm.build_batch : 16384;
  // a point of level l emits at most M reverse-edge records on each of its l+1 layers
  auto edges_of = [&](uint64_t lo, uint64_t hi) {
    uint64_t e = 0;
    for (uint64_t i = lo; i < hi; ++i) e += (uint64_t)M * (h_levels[i] + 1u);
    return e;
  };
  RET(ensure_build_scratch((uint64_t)std::min<uint64_t>(maxb, std::max<uint64_t>(n, 1)) * M * 2, 1, false));
  ehb::BuildBeam bm;
  RET(reserve_build_beam(&bm));
  CU(cudaMemsetAsync(b_counters.p + 3, 0, 4, stream));  // error flag of earlier builds
  ehb::WalkCfg cfg = build_cfg(std::min<uint64_t>(maxb, n));
  uint32_t wpb = wpb_for(cfg, 256);
  while (n_linked < n) {
    if (n_linked == 0) {
      entry = 0;
      max_level = h_levels[0];
      n_linked = 1;
      continue;
    }
    // a wave never exceeds 1/64 of the linked graph: points of one wave cannot see each other
    // (recall stays within the seed-to-seed noise of the sequential build; tests/test_gpu_parity.py checks it)
    const uint64_t frac = o_build_frac ? o_build_frac : 64;
    uint64_t b = std::min<uint64_t>(maxb, std::max<uint64_t>(1, n_linked / frac));
    b = std::min<uint64_t>(b, n - n_linked);
    const uint64_t edges = edges_of(n_linked, n_linked + b);
    RET(ensure_build_scratch(edges, 1, false));
    ehb::BuildGraph bg = build_graph();
    ehb::BuildBuffers bb = build_buffers(edges);
    CU(ehb::launch_build_batch(bg, cfg, nullptr, (uint32_t)n_linked, (uint32_t)b, ehb::kBuildInsert, bb, wpb, bm,
                               stream));
    for (uint64_t i = n_linked; i < n_linked + b; ++i)
      if ((int)h_levels[i] > max_level) max_level = h_levels[i], entry = (uint32_t)i;
    n_linked += b;
  }
  if (!pending_updates.empty()) {
    // hnswlib updatePoint: neighbour re-selection over the two-hop set, then repairConnectionsForUpdate.
    // Up to o_seq_updates moved points are processed one at a time, which is exactly the reference's
    // sequential semantics (index_test.cc:39-49); larger bulks go in waves.  Within a wave every
    // re-selection reads the pre-wave graph (a row shared by several moved points takes the re-selection
    // of the latest in arrival order), every re-link reads the graph after all re-selections, and the
    // moved points' own new rows land together before the reverse links are merged: moved points of one
    // wave never see each other's new links, whatever the scheduling.
    std::vector<uint32_t> ups;
    {
      std::vector<uint32_t> sorted_ids = pending_updates;
      std::sort(sorted_ids.begin(), sorted_ids.end());
      sorted_ids.erase(std::unique(sorted_ids.begin(), sorted_ids.end()), sorted_ids.end());
      std::vector<bool> done(sorted_ids.size(), false);  // keep first-occurrence (arrival) order
      for (uint32_t id : pending_updates) {
        size_t pos = std::lower_bound(sorted_ids.begin(), sorted_ids.end(), id) - sorted_ids.begin();
        if (!done[pos]) done[pos] = true, ups.push_back(id);
      }
    }
    const uint32_t ub = ups.size() <= o_seq_updates ? 1u : (prm.build_batch ? prm.build_batch : 1024u);
    if (n_linked > 1) {
      for (size_t off = 0; off < ups.size(); off += ub) {
        uint32_t b = (uint32_t)std::min<size_t>(ub, ups.size() - off);
        uint64_t edges = 0, staged = 0;  // staged: rows a wave may rewrite (re-selections or own rows)
        for (uint32_t i = 0; i < b; ++i) {
          edges += (uint64_t)M * (h_levels[ups[off + i]] + 1u);
          staged += M0 + (uint64_t)M * h_levels[ups[off + i]];
        }
        RET(ensure_build_scratch(edges, b, true));
        CU(b_side_row.grow(staged, 0, -1, stream));
        CU(b_side_out.grow((b_side_row.n + 1) * M0, 0, -1, stream));
        CU(b_ids.grow(std::max<uint32_t>(b, 64), 0, -1, stream));
        CU(cudaMemcpyAsync(b_ids.p, ups.data() + off, (size_t)b * 4, cudaMemcpyHostToDevice, stream));
        ehb::BuildGraph bg = build_graph();
        ehb::BuildBuffers bb = build_buffers(edges);
        CU(ehb::launch_build_batch(bg, cfg, b_ids.p, 0, b, ehb::kBuildUpdate, bb, wpb, bm, stream));
      }
      CU(cudaStreamSynchronize(stream));
    }
    pending_updates.clear();
  }
  uint32_t err = 0;
  CU(cudaMemcpyAsync(&err, b_counters.p + 3, 4, cudaMemcpyDeviceToHost, stream));
  CU(cudaStreamSynchronize(stream));
  if (err) return fail(EHB_ERR_STATE, "build: edge buffer overflow");
  return EHB_OK;
}

// ---- compaction -------------------------------------------------------------------------------------------
// Removes every tombstone.  All passes read the pre-compaction graph, so the result does not depend on
// scheduling:
//   1. rows of live nodes that name deleted ids are found (and level-0 in-degrees counted);
//   2. each such row is re-selected over its live ids and the live ids of its deleted members' rows
//      (repair_rows_kernel), into a side buffer that is copied back once every repair has read the old graph;
//   3. the entry point stays if it is live, else the live node of highest level (smallest id) takes over;
//   4. survivors are renumbered densely in insertion order (new id = live ids below the old id): adjacency is
//      gathered into new arrays, vectors are moved down in place through a bounded staging buffer;
//   5. survivors left with an empty level-0 row, or with level-0 in-links before and none after, are
//      re-linked by the updatePoint path (ascending new id);
//   6. host tables follow.  Capacity is kept; later adds reuse the freed rows.
int ehb_index::compact() {
  RET(build());
  if (n_deleted == 0) return EHB_OK;
  cudaStream_t s = stream;
  const uint64_t n_old = n;
  std::vector<uint32_t> remap(n_old, ehb::kInvalid), inv;
  inv.reserve(n_old - n_deleted);
  for (uint64_t i = 0; i < n_old; ++i)
    if (!h_deleted[i]) remap[i] = (uint32_t)inv.size(), inv.push_back((uint32_t)i);
  const uint64_t nn = inv.size();
  if (nn == 0) {  // everything deleted: an empty index, later adds start a fresh graph
    const uint64_t removed = n_removed + n_old;
    CU(cudaMemsetAsync(links0.p, 0xFF, links0.bytes(), s));
    CU(cudaMemsetAsync(up_off.p, 0xFF, up_off.bytes(), s));
    CU(cudaMemsetAsync(deleted.p, 0, deleted.bytes(), s));
    CU(cudaMemsetAsync(links_up.p, 0xFF, links_up.bytes(), s));
    CU(cudaStreamSynchronize(s));
    reset_content();
    n_removed = removed;
    return EHB_OK;
  }
  // host side of the renumbering: old upper rows are laid out consecutively in id order
  std::vector<uint64_t> labels_new(nn);
  std::vector<uint8_t> levels_new(nn);
  std::vector<uint32_t> up_off_new(nn), owner_new, src_up;
  {
    std::vector<uint32_t> up_off_old(n_old);
    uint32_t r = 0;
    for (uint64_t i = 0; i < n_old; ++i) up_off_old[i] = r, r += h_levels[i];
    for (uint64_t i = 0; i < nn; ++i) {
      const uint32_t o = inv[i];
      labels_new[i] = h_labels[o];
      levels_new[i] = h_levels[o];
      up_off_new[i] = h_levels[o] ? (uint32_t)owner_new.size() : ehb::kInvalid;
      for (uint32_t l = 0; l < h_levels[o]; ++l) owner_new.push_back((uint32_t)i), src_up.push_back(up_off_old[o] + l);
    }
  }
  const uint64_t rows_new = owner_new.size();
  uint32_t entry_new;
  int32_t max_level_new = max_level;
  if (!h_deleted[entry]) {
    entry_new = remap[entry];
  } else {
    entry_new = 0;
    for (uint64_t i = 1; i < nn; ++i)
      if (levels_new[i] > levels_new[entry_new]) entry_new = (uint32_t)i;
    max_level_new = levels_new[entry_new];
  }
  // 1. affected rows + level-0 in-degrees of the old graph
  ehb::DevBuf<uint32_t> rows, indeg_old, indeg_new, d_remap, d_inv, d_src_up, repaired, nl0, nlu;
  ehb::DevBuf<uint8_t> orphan;
  ehb::DevBuf<float> stage;
  CU(rows.grow(n_old + up_rows, 0, -1, s));
  CU(indeg_old.grow(n_old, 0, 0, s));
  CU(b_counters.grow(8, 0, 0, s));
  CU(cudaMemsetAsync(b_counters.p + 5, 0, 4, s));
  CU(ehb::launch_compact_mark(links0.p, links_up.p, up_owner.p, deleted.p, n_old, up_rows, M0, M, (uint32_t)cap,
                              rows.p, b_counters.p + 5, indeg_old.p, s));
  uint32_t nrows = 0;
  CU(cudaMemcpyAsync(&nrows, b_counters.p + 5, 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  // every allocation before the graph changes, so running out of memory leaves the index as it was
  const uint64_t stage_rows = std::max<uint64_t>(1, std::min<uint64_t>(nn, (256ull << 20) / (dpad * 4ull)));
  const uint32_t warps = std::min<uint32_t>(std::max<uint32_t>(nrows, 1), ehb::kRepairWarps);
  RET(ensure_build_scratch(0, warps, true));
  ehb::BuildBeam bm;  // (the re-links of step 5)
  RET(reserve_build_beam(&bm));
  CU(repaired.grow(std::max<uint64_t>(nrows, 1) * M0, 0, -1, s));
  CU(d_remap.grow(n_old, 0, -1, s));
  CU(d_inv.grow(nn, 0, -1, s));
  CU(d_src_up.grow(std::max<uint64_t>(rows_new, 1), 0, -1, s));
  CU(indeg_new.grow(nn, 0, -1, s));
  CU(orphan.grow(nn, 0, -1, s));
  CU(nl0.grow(cap * M0, 0, 0xFF, s));
  CU(nlu.grow(links_up.n, 0, 0xFF, s));
  CU(stage.grow(stage_rows * dpad, 0, -1, s));
  // 2. repair, then copy the rows back
  if (nrows) {
    ehb::BuildGraph bg = build_graph();
    ehb::BuildBuffers bb = build_buffers(0);
    bb.repair_out = repaired.p;
    const ehb::WalkCfg cfg = build_cfg(warps);
    CU(ehb::launch_build_batch(bg, cfg, rows.p, 0, nrows, ehb::kBuildRepair, bb, wpb_for(cfg, 256), bm, s));
    CU(ehb::launch_compact_apply(rows.p, nrows, repaired.p, links0.p, links_up.p, M0, M, (uint32_t)cap, s));
  }
  // 4. renumber the adjacency into the new arrays, find the orphans, move the vectors
  CU(cudaMemcpyAsync(d_remap.p, remap.data(), n_old * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(d_inv.p, inv.data(), nn * 4, cudaMemcpyHostToDevice, s));
  if (rows_new) CU(cudaMemcpyAsync(d_src_up.p, src_up.data(), rows_new * 4, cudaMemcpyHostToDevice, s));
  CU(ehb::launch_compact_remap_rows(links0.p, d_inv.p, nn, M0, d_remap.p, nl0.p, s));
  CU(ehb::launch_compact_remap_rows(links_up.p, d_src_up.p, rows_new, M, d_remap.p, nlu.p, s));
  CU(ehb::launch_compact_orphans(nl0.p, nn, M0, d_inv.p, indeg_old.p, indeg_new.p, orphan.p, s));
  uint64_t lo = 0;
  while (lo < nn && inv[lo] == lo) ++lo;  // rows below the first tombstone stay where they are
  CU(ehb::launch_compact_move_rows(vecs.p, dpad, d_inv.p, lo, nn, stage.p, stage_rows, s));
  RET(derive_rows(lo, nn - lo));  // the survivors' rows moved: re-derive them in their new places
  CU(cudaMemcpyAsync(labels.p, labels_new.data(), nn * 8, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(levels.p, levels_new.data(), nn, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(up_off.p, up_off_new.data(), nn * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(up_off.p + nn, 0xFF, (cap - nn) * 4, s));
  if (rows_new) CU(cudaMemcpyAsync(up_owner.p, owner_new.data(), rows_new * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(deleted.p, 0, deleted.bytes(), s));
  std::vector<uint8_t> is_orphan(nn);
  CU(cudaMemcpyAsync(is_orphan.data(), orphan.p, nn, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  std::swap(links0.p, nl0.p);
  std::swap(links_up.p, nlu.p);
  // 6. host tables
  identity_labels = true;
  for (uint64_t i = 0; i < nn && identity_labels; ++i) identity_labels = labels_new[i] == i;
  lookup.clear();
  if (!identity_labels) {
    lookup.reserve(nn * 2);
    for (uint64_t i = 0; i < nn; ++i) lookup[labels_new[i]] = (uint32_t)i;
  }
  h_labels = std::move(labels_new);
  h_levels = std::move(levels_new);
  h_deleted.assign(nn, 0);
  n_removed += n_old - nn;
  n = n_linked = nn;
  up_rows = rows_new;
  n_deleted = 0;
  entry = entry_new;
  max_level = max_level_new;
  // 5. re-link the orphans (updatePoint: a beam search from the entry point, then mutual links)
  for (uint64_t i = 0; i < nn; ++i)
    if (is_orphan[i]) pending_updates.push_back((uint32_t)i);
  return build();
}

// Searches link pending points lazily, the first bf16 search creates the bf16 shadow and the first screened search
// the int8 screen copy; all need the writer side of the lock.  Another writer may run between the unlock and the
// lock, so the state is checked again.
int ehb_index::ensure_built(std::shared_lock<ehb::RwLock>& lk, bool bf16, bool screen) {
  auto screen_wants_copy = [&] { return screen && !screen_copy && !screen_no_room; };
  while (needs_build() || (bf16 && !shadow) || screen_wants_copy()) {
    lk.unlock();
    int rc;
    {
      std::unique_lock<ehb::RwLock> x(rw);
      rc = build();
      if (rc == EHB_OK && bf16) rc = create_shadow();
      if (rc == EHB_OK && screen_wants_copy()) rc = try_screen_copy();
    }
    lk.lock();
    if (rc != EHB_OK) return rc;
  }
  return EHB_OK;
}

int ehb_index::ensure_shadow(std::shared_lock<ehb::RwLock>& lk) {
  while (!shadow) {
    lk.unlock();
    int rc;
    {
      std::unique_lock<ehb::RwLock> x(rw);
      rc = create_shadow();
    }
    lk.lock();
    if (rc != EHB_OK) return rc;
  }
  return EHB_OK;
}

int ehb_index::prepare(std::shared_lock<ehb::RwLock>& lk, bool brute, int precision, uint64_t nq) {
  const bool bf16 = precision == EHB_BF16;
  if (brute) return bf16 ? ensure_shadow(lk) : EHB_OK;
  return ensure_built(lk, bf16, !bf16 && walk_screens(nq));
}

// ---- search slots ------------------------------------------------------------------------------------
int ehb::SlotLease::take(cudaStream_t stream) {
  {
    std::unique_lock<std::mutex> g(ix_->slot_mu);
    while (!sl) {
      if (!ix_->free_slots.empty()) {
        sl = ix_->free_slots.back();  // LIFO: a single-threaded caller keeps reusing one slot (stream-ordered scratch)
        ix_->free_slots.pop_back();
      } else if (ix_->slots.size() < kMaxSlots) {
        std::unique_ptr<SearchSlot> ns(new (std::nothrow) SearchSlot());
        if (!ns) return fail(EHB_ERR_OOM, "host allocation failed");
        cudaError_t e = cudaStreamCreateWithFlags(&ns->stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreate(&ns->ev0);
        if (e == cudaSuccess) e = cudaEventCreate(&ns->ev1);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ns->busy, cudaEventDisableTiming);
        if (e != cudaSuccess) return fail(EHB_ERR_CUDA, cudaGetErrorString(e));
        sl = ns.get();
        ix_->slots.push_back(std::move(ns));
      } else {
        ix_->slot_cv.wait(g);
      }
    }
  }
  s = stream ? stream : sl->stream;
  if (sl->busy_valid) CU(cudaStreamWaitEvent(s, sl->busy, 0));
  return EHB_OK;
}

ehb::SlotLease::~SlotLease() {
  if (!sl) return;
  // the scratch stays in use until the work queued on `s` is done: the next user orders itself after it
  sl->busy_valid = cudaEventRecord(sl->busy, s) == cudaSuccess;
  {
    std::lock_guard<std::mutex> g(ix_->slot_mu);
    ix_->free_slots.push_back(sl);
  }
  ix_->slot_cv.notify_one();
}

// ---- search --------------------------------------------------------------------------------------------
int ehb::check_request(const ehb_index* ix, bool brute, int precision, bool null_buf, uint64_t nq, uint32_t k,
                       uint64_t k_walk, uint32_t* ef, bool* none, uint32_t max_beam) {
  *none = false;
  if (precision != EHB_FP32 && precision != EHB_BF16) return fail(EHB_ERR_INVALID, "unknown precision");
  if (null_buf) return fail(EHB_ERR_INVALID, "null buffer");
  *none = k == 0 || nq == 0;
  if (*none) return EHB_OK;
  if (brute) {
    if (k_walk > 2048) return fail(EHB_ERR_INVALID, "k (k + 1 by label) must be <= 2048 for brute force");
    if (precision == EHB_BF16 && ix->dpad % 64 != 0)
      return fail(EHB_ERR_INVALID, "bf16 brute force needs dim > 32 (64-wide k-blocks)");
  } else {
    if (*ef == 0) *ef = ix->ef;
    if (std::max<uint64_t>(*ef, k_walk) > max_beam)
      return fail(EHB_ERR_INVALID, "max(ef, k) (k + 1 by label) must be <= " + std::to_string(max_beam));
  }
  return EHB_OK;
}

int ehb::copy_results(uint64_t nq, uint32_t k, const uint64_t* dl, const float* dd, const uint32_t* dc, uint64_t* ol,
                      float* od, uint32_t* oc, cudaStream_t s) {
  CU(cudaMemcpyAsync(ol, dl, nq * k * 8, cudaMemcpyDeviceToHost, s));
  if (od) CU(cudaMemcpyAsync(od, dd, nq * k * 4, cudaMemcpyDeviceToHost, s));
  if (oc) CU(cudaMemcpyAsync(oc, dc, nq * 4, cudaMemcpyDeviceToHost, s));
  return EHB_OK;
}

int ehb_index::grow_beam(const ehb::WalkPlan& plan, uint64_t nq, uint32_t ef_eff, cudaStream_t s, uint32_t* warps) {
  if (!beam_done) CU(cudaEventCreateWithFlags(&beam_done, cudaEventDisableTiming));
  CU(cudaStreamWaitEvent(s, beam_done, 0));
  CU(ehb::beam_warps(plan, view(), sms, nq, warps));
  CU(beam_vtab.grow((size_t)*warps * plan.vtab, 0, -1, s));
  if (plan.bf16) CU(beam_keys.grow(nq * ef_eff, 0, -1, s));
  return EHB_OK;
}

int ehb_index::reserve_beam(uint64_t nq, uint32_t ef_eff, int precision, cudaStream_t s) {
  const ehb::WalkPlan plan = walk_plan(nq, ef_eff, precision == EHB_BF16);
  if (plan.form != ehb::WalkForm::beam) return EHB_OK;
  std::lock_guard<std::mutex> bl(beam_mu);
  uint32_t warps = 0;
  return grow_beam(plan, nq, ef_eff, s, &warps);
}

int ehb_index::search_dev(ehb::SearchSlot* sl, uint64_t nq, const float* dq, uint32_t k, uint32_t ef_in, uint64_t* dl,
                          float* dd, uint32_t* dc, cudaStream_t s, const ehb::ResultSink* sink, bool* pushed,
                          int precision) {
  if (pushed) *pushed = false;
  const uint32_t ef_eff = std::max(ef_in, k);
  const bool bf16 = precision == EHB_BF16;
  if (bf16 && !shadow) return fail(EHB_ERR_STATE, "bf16 shadow missing");
  const ehb::WalkPlan plan = walk_plan(nq, ef_eff, bf16);
  const bool beam = plan.form == ehb::WalkForm::beam;
  // the wide-beam walk's scratch: after the previous wide-beam search on the device, allocated before anything runs
  std::unique_lock<std::mutex> bl(beam_mu, std::defer_lock);
  uint32_t warps = 0;
  if (beam) {
    bl.lock();
    RET(grow_beam(plan, nq, ef_eff, s, &warps));
  }
  // the team walk writes destination 0 only (a bf16 search never plans one: its re-rank stores to every destination),
  // and so does the re-rank of more than kMaxEf results (its sink form collects at most that many keys in shared
  // memory): the exchange's merge kernel then pushes the block
  const bool rerank_sink = sink && bf16 && k <= ehb::kMaxEf;
  if (pushed) *pushed = sink && plan.form != ehb::WalkForm::team && (!bf16 || rerank_sink);
  const float* q = dq;
  if (metric == EHB_COSINE) {
    CU(sl->q_norm.grow(nq * dim, 0, -1, s));
    CU(ehb::launch_pad_rows(dq, sl->q_norm.p, nq, dim, dim, true, s));
    q = sl->q_norm.p;
  }
  CU(sl->stats.grow(nq * ehb::kStatWords, 0, -1, s));
  CU(sl->stat_sum.grow(ehb::kStatWords, 0, 0, s));
  if (bf16) {
    CU(sl->q_pad.grow(nq * dpad, 0, -1, s));
    if (!beam) CU(sl->walk_keys.grow(nq * ef_eff, 0, -1, s));
    CU(sl->walk_counts.grow(nq, 0, -1, s));
    CU(ehb::launch_pad_rows(dq, sl->q_pad.p, nq, dim, dpad, metric == EHB_COSINE, s));
  }
  CU(cudaEventRecord(sl->ev0, s));
  if (bf16) {
    // walk the bf16 rows keeping the whole retained set, then re-rank it with the canonical fp32 chain (with a
    // sink, the re-rank stores into every destination and raises the slice flags, as the fp32 walk's epilogue does)
    ehb::ResultSink ks;
    std::memset(&ks, 0, sizeof(ks));
    ks.keys = beam ? beam_keys.p : sl->walk_keys.p;
    ehb::GraphView g = view();
    g.vecs16 = (const __nv_bfloat16*)x_bf16.p;
    if (beam)
      CU(ehb::launch_search_beam(plan, g, q, (uint32_t)nq, ef_eff, ef_eff, ks, sl->walk_counts.p, sl->stats.p,
                                 beam_vtab.p, warps, s));
    else
      CU(ehb::launch_search(plan, g, q, (uint32_t)nq, ef_eff, ef_eff, ks, sl->walk_counts.p, sl->stats.p, s));
    if (rerank_sink)
      CU(ehb::launch_rerank_sink(ks.keys, ef_eff, sl->q_pad.p, vecs.p, dpad, dim, metric == EHB_L2 ? 0 : 1,
                                 labels.p, nq, k, *sink, dc, s));
    else
      CU(ehb::launch_rerank(ks.keys, ef_eff, sl->q_pad.p, vecs.p, dpad, dim, metric == EHB_L2 ? 0 : 1,
                            labels.p, nq, k, dl, dd, dc, s));
  } else if (plan.form == ehb::WalkForm::team) {
    CU(ehb::launch_search_team(plan, view(), q, (uint32_t)nq, k, ef_eff, dl, dd, dc, sl->stats.p, s));
  } else {
    ehb::ResultSink one;
    if (!sink) {
      std::memset(&one, 0, sizeof(one));
      one.labels[0] = dl;
      one.dists[0] = dd;
      one.n = 1;
      sink = &one;
    }
    ehb::GraphView g = view();
    if (plan.screen) {
      g.codes8 = x_i8.p;
      g.terms8 = x_i8t.p;
    }
    if (beam)
      CU(ehb::launch_search_beam(plan, g, q, (uint32_t)nq, k, ef_eff, *sink, dc, sl->stats.p, beam_vtab.p, warps, s));
    else
      CU(ehb::launch_search(plan, g, q, (uint32_t)nq, k, ef_eff, *sink, dc, sl->stats.p, s));
  }
  if (beam) CU(cudaEventRecord(beam_done, s));
  CU(cudaEventRecord(sl->ev1, s));
  sl->last_nq = nq;
  sl->last_bf16 = bf16;
  ehb::walk_kernel_name(plan, sl->last_kernel, sizeof(sl->last_kernel));
  {
    std::lock_guard<std::mutex> g(last_mu);
    last_slot = sl;
    last_was_brute = false;
    timed = true;
    last_sum_valid = false;
  }
  return EHB_OK;
}

// Caller holds the shared lock and bf_mu, and has checked the request (ehb::check_request).
int ehb_index::bruteforce_dev(uint64_t nq, const float* dq, uint32_t k, int precision, uint64_t* dl, float* dd,
                              uint32_t* dc, cudaStream_t s) {
  const bool bf16 = precision == EHB_BF16;
  // candidates kept by the bf16 pass: bf16 rounding perturbs each dot product by ~|q||x| 2^-9 / sqrt(d),
  // comparable to the spacing of the best matches, so 4x (>= k + 64) of them go to the fp32 re-rank
  const uint32_t kc = bf16 ? (uint32_t)std::min<uint64_t>(std::min<uint64_t>(2048, std::max<uint64_t>(n, 1)),
                                                          std::max<uint64_t>(4ull * k, k + 64ull)) : k;
  ehb::BruteScratch sc;
  sc.qb = std::min<uint64_t>(nq, bf16 ? 2048 : 1024);
  sc.nc = std::min<uint64_t>(std::max<uint64_t>(n, 1), 131072);
  sc.slices = 32;
  CU(bf_dist.grow(sc.qb * sc.nc, 0, -1, s));
  CU(bf_part.grow(sc.qb * sc.slices * std::max(kc, k), 0, -1, s));
  CU(bf_run.grow(nq * std::max(kc, k), 0, -1, s));
  CU(bf_qpad.grow(nq * dpad, 0, -1, s));
  CU(ehb::launch_pad_rows(dq, bf_qpad.p, nq, dim, dpad, metric == EHB_COSINE, s));
  sc.dist = bf_dist.p;
  sc.part_keys = bf_part.p;
  sc.run_keys = bf_run.p;
  sc.deleted = n_deleted ? deleted.p : nullptr;
  ehb::Bf16Ctx bctx;
  if (bf16) {
    // the bf16 shadow of the base rows (+ squared norms): the caller made sure it exists (ensure_shadow), and
    // the mutations keep it current
    if (!shadow) return fail(EHB_ERR_STATE, "bf16 shadow missing");
    CU(q_bf16.grow(nq * dpad, 0, -1, s));
    CU(q_norm2.grow(nq, 0, -1, s));
    CU(ehb::launch_to_bf16(bf_qpad.p, dpad, q_bf16.p, q_norm2.p, nq, dpad, s));
    bctx.q_bf16 = q_bf16.p;
    bctx.x_bf16 = x_bf16.p;
    bctx.qnorm = q_norm2.p;
    bctx.xnorm = x_norm.p;
    bctx.kc = kc;
    // fused selection state (option "bf16_unfused" keeps the distance tiles in HBM: A/B switch); tombstones
    // are filtered where keys are formed, which only the unfused selection does
    bctx.fused = !o_bf16_unfused && !n_deleted;
    bctx.ccap = 2 * kc + 64;
    CU(bf_thr.grow(nq, 0, -1, s));
    CU(bf_cbuf.grow(nq * bctx.ccap, 0, -1, s));
    CU(bf_ccount.grow(nq + 1, 0, 0, s));
    bctx.thr = bf_thr.p;
    bctx.cbuf = bf_cbuf.p;
    bctx.ccount = bf_ccount.p;
    bctx.overflow = bf_ccount.p + nq;
    bctx.sms = sms;
  }
  CU(cudaEventRecord(bf_ev0, s));
  CU(ehb::launch_bruteforce(vecs.p, dpad, dim, n, labels.p, metric == EHB_L2 ? 0 : 1, bf_qpad.p, nq, k, sc,
                            bf16 ? &bctx : nullptr, dl, dd, dc, s));
  CU(cudaEventRecord(bf_ev1, s));
  {
    std::lock_guard<std::mutex> g(last_mu);
    last_was_brute = true;
    timed = true;
  }
  return EHB_OK;
}

// ============================================================================================
// C ABI
// ============================================================================================
#define ENTER_X(ix)                                                    \
  if (!(ix)) return fail(EHB_ERR_INVALID, "null index handle");        \
  std::unique_lock<ehb::RwLock> _g((ix)->rw);                    \
  CU(cudaSetDevice((ix)->device))
#define ENTER_S(ix)                                                    \
  if (!(ix)) return fail(EHB_ERR_INVALID, "null index handle");        \
  std::shared_lock<ehb::RwLock> _g((ix)->rw);                    \
  CU(cudaSetDevice((ix)->device))

namespace {

// The leader's part of the combining queue: all taken requests share (k, ef, precision) and go out as one launch.
// (Every queued caller holds the shared lock and has seen the graph built, so no mutation can intervene.)
int run_combined(ehb_index* ix, std::vector<ehb::CombineReq*>& batch) {
  uint64_t tot = 0;
  for (auto* r : batch) tot += r->nq;
  const uint32_t k = batch[0]->k, ef = batch[0]->ef, dim = ix->dim;
  const int precision = batch[0]->precision;
  ehb::SlotLease ls(ix);
  RET(ls.take());
  ix->combined_batches++;
  ix->combined_queries += tot;
  ehb::SearchSlot* sl = ls.sl;
  const cudaStream_t s = ls.s;
  CU(sl->h_q.reserve(tot * dim * 4));
  CU(sl->h_l.reserve(tot * k * 8));
  CU(sl->h_d.reserve(tot * k * 4));
  CU(sl->h_c.reserve(tot * 4));
  CU(sl->q_in.grow(tot * dim, 0, -1, s));
  CU(sl->o_labels.grow(tot * k, 0, -1, s));
  CU(sl->o_dists.grow(tot * k, 0, -1, s));
  CU(sl->o_counts.grow(tot, 0, -1, s));
  uint64_t off = 0;
  for (auto* r : batch) {
    std::memcpy(sl->h_q.p + off * dim * 4, r->q, r->nq * dim * 4);
    off += r->nq;
  }
  CU(cudaMemcpyAsync(sl->q_in.p, sl->h_q.p, tot * dim * 4, cudaMemcpyHostToDevice, s));
  RET(ix->search_dev(sl, tot, sl->q_in.p, k, ef, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, s, nullptr, nullptr,
                     precision));
  RET(ehb::copy_results(tot, k, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, (uint64_t*)sl->h_l.p,
                        (float*)sl->h_d.p, (uint32_t*)sl->h_c.p, s));
  CU(cudaStreamSynchronize(s));
  off = 0;
  for (auto* r : batch) {
    std::memcpy(r->ol, sl->h_l.p + off * k * 8, r->nq * k * 8);
    if (r->od) std::memcpy(r->od, sl->h_d.p + off * k * 4, r->nq * k * 4);
    if (r->oc) std::memcpy(r->oc, sl->h_c.p + off * 4, r->nq * 4);
    off += r->nq;
  }
  return EHB_OK;
}

// Combining queue ("group commit"): a caller queues its request; whoever finds a free leader seat takes
// every queued request with its own (k, ef, precision) and runs them as ONE batched search.  Nobody ever waits on a
// timer: requests pile up only while earlier batches occupy the leader seats, which is exactly when
// batching pays.  A lone caller becomes its own leader at once.
int search_host_combined(ehb_index* ix, uint64_t nq, const float* q, uint32_t k, uint32_t ef, int precision,
                         uint64_t* ol, float* od, uint32_t* oc) {
  ehb::CombineReq me{q, nq, k, ef, precision, ol, od, oc};
  std::unique_lock<std::mutex> g(ix->cq_mu);
  ix->cq.push_back(&me);
  for (;;) {
    if (me.done) break;
    if (!me.taken && ix->cq_leaders < ehb::kCombineLeaders) {
      std::vector<ehb::CombineReq*> batch;
      uint64_t tot = 0;
      for (auto it = ix->cq.begin(); it != ix->cq.end();) {
        ehb::CombineReq* r = *it;
        if (r->k == k && r->ef == ef && r->precision == precision && (r == &me || tot + r->nq <= ehb::kCombineMaxBatch)) {
          r->taken = true;
          tot += r->nq;
          batch.push_back(r);
          it = ix->cq.erase(it);
        } else {
          ++it;
        }
      }
      ix->cq_leaders++;
      g.unlock();
      int rc = run_combined(ix, batch);
      const std::string err = rc == EHB_OK ? std::string() : ehb::last_error_text();
      g.lock();
      ix->cq_leaders--;
      for (auto* r : batch) r->rc = rc, r->err = err, r->done = true;
      ix->cq_cv.notify_all();
      continue;
    }
    ix->cq_cv.wait(g);
  }
  if (me.rc != EHB_OK) return fail(me.rc, me.err);
  return EHB_OK;
}

// ---- queries that are stored points (bylabel.cu) ---------------------------------------------------------------
// Caller holds the shared lock.  hnswlib getDataByLabel: a tombstoned label reads as not found.
int resolve_labels(const ehb_index* ix, uint64_t n, const uint64_t* labels, std::vector<uint32_t>& ids) {
  ids.resize(n);
  for (uint64_t i = 0; i < n; ++i)
    if (!ix->find_id(labels[i], &ids[i]) || ix->h_deleted[ids[i]]) return fail(EHB_ERR_NOT_FOUND, "label not found");
  return EHB_OK;
}

// Caller holds the shared lock and `sl`: the rows of ids into out ([n][dim]) on s, exactly as ehb_index_get reads them.
int gather_ids(ehb_index* ix, ehb::SearchSlot* sl, const std::vector<uint32_t>& ids, float* out, cudaStream_t s) {
  const uint64_t n = ids.size();
  CU(sl->q_ids.grow(n, 0, -1, s));
  CU(cudaMemcpyAsync(sl->q_ids.p, ids.data(), n * 4, cudaMemcpyHostToDevice, s));
  CU(ehb::launch_gather_rows(ix->vecs.p, ix->dpad, sl->q_ids.p, out, ix->dim, nullptr, n, ix->dim, s));
  return EHB_OK;
}

// Every host search entry point: queries are the host rows q, or (by_label) the stored rows of `labels`, searched at
// k + 1, then the reference's self-removal (server.cc:190-207) on the device; brute: the exact / bf16 brute force on
// ix->stream under bf_mu instead of the graph walk.  Small host-row graph searches go through the combining queue;
// every other call stages, searches and copies out on one leased slot with one synchronisation.
int search_host(ehb_index* ix, std::shared_lock<ehb::RwLock>& lk, bool brute, bool by_label, uint64_t nq,
                const float* q, const uint64_t* labels, uint32_t k, uint32_t ef, int precision, uint64_t* ol, float* od,
                uint32_t* oc, uint32_t max_beam = ehb::kMaxEf) {
  const uint64_t k_walk = k + (uint64_t)by_label;
  const bool null_q = by_label ? !labels : !q;
  bool none;
  RET(ehb::check_request(ix, brute, precision, nq && (null_q || !ol), nq, k, k_walk, brute ? nullptr : &ef, &none,
                         max_beam));
  if (none) return EHB_OK;
  const uint32_t kw = (uint32_t)k_walk;  // checked: <= 4096
  // before queueing or bf_mu: a waiting follower must never block a writer the leader needs, and the upgrade waits
  // for the other readers
  RET(ix->prepare(lk, brute, precision, nq));
  if (!brute && !by_label && ix->o_combine && nq <= ehb::kCombineMaxCall && std::max(ef, kw) <= ehb::kMaxEf)
    return search_host_combined(ix, nq, q, k, ef, precision, ol, od, oc);
  std::vector<uint32_t> ids;
  if (by_label) RET(resolve_labels(ix, nq, labels, ids));
  std::unique_lock<std::mutex> bg(ix->bf_mu, std::defer_lock);
  if (brute) bg.lock();  // brute-force scratch and stream
  ehb::SlotLease ls(ix);
  RET(ls.take(brute ? ix->stream : nullptr));
  ehb::SearchSlot* sl = ls.sl;
  const cudaStream_t s = ls.s;
  CU(sl->q_in.grow(nq * ix->dim, 0, -1, s));
  CU(sl->o_labels.grow(nq * kw, 0, -1, s));
  CU(sl->o_dists.grow(nq * kw, 0, -1, s));
  CU(sl->o_counts.grow(nq, 0, -1, s));
  if (by_label) {
    CU(sl->q_labels.grow(nq, 0, -1, s));
    CU(sl->s_labels.grow(nq * k, 0, -1, s));
    CU(sl->s_dists.grow(nq * k, 0, -1, s));
    CU(sl->s_counts.grow(nq, 0, -1, s));
    RET(gather_ids(ix, sl, ids, sl->q_in.p, s));
    CU(cudaMemcpyAsync(sl->q_labels.p, labels, nq * 8, cudaMemcpyHostToDevice, s));
  } else {
    CU(cudaMemcpyAsync(sl->q_in.p, q, nq * ix->dim * 4, cudaMemcpyHostToDevice, s));
  }
  if (brute)
    RET(ix->bruteforce_dev(nq, sl->q_in.p, kw, precision, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, s));
  else
    RET(ix->search_dev(sl, nq, sl->q_in.p, kw, ef, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, s, nullptr, nullptr,
                       precision));
  if (by_label) {
    CU(ehb::launch_drop_self(sl->q_labels.p, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, nq, k, sl->s_labels.p,
                             sl->s_dists.p, sl->s_counts.p, s));
    RET(ehb::copy_results(nq, k, sl->s_labels.p, sl->s_dists.p, sl->s_counts.p, ol, od, oc, s));
  } else {
    RET(ehb::copy_results(nq, k, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, ol, od, oc, s));
  }
  CU(cudaStreamSynchronize(s));
  return EHB_OK;
}

// Stream and events of the neighbour table's result copies; released on every return.
struct TableCopies {
  cudaStream_t s = nullptr;
  cudaEvent_t ready[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};
  ~TableCopies() {
    if (s) cudaStreamSynchronize(s);
    for (int b = 0; b < 2; ++b) {
      if (ready[b]) cudaEventDestroy(ready[b]);
      if (copied[b]) cudaEventDestroy(copied[b]);
    }
    if (s) cudaStreamDestroy(s);
  }
};

}  // namespace

extern "C" {

const char* ehb_last_error(void) { return ehb::g_err.c_str(); }
uint32_t ehb_abi_version(void) { return 2; }

int ehb_device_count(int32_t* out) {
  if (!out) return fail(EHB_ERR_INVALID, "null out");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    *out = 0;
    return fail(EHB_ERR_CUDA, std::string("no CUDA device (ehb200 has no CPU fallback): ") + cudaGetErrorString(e));
  }
  *out = n;
  return EHB_OK;
}

void ehb_params_default(ehb_params* p, uint32_t dim) {
  std::memset(p, 0, sizeof(*p));
  p->dim = dim;
  p->metric = EHB_L2;
  p->capacity = 128;        // index.h:21
  p->M = 16;                // hnswlib default used by index.cc:14-15
  p->ef_construction = 200;
  p->ef_search = 10;        // hnswlib ef_ default; the reference never calls setEf
  p->seed = 100;
  p->device = 0;
}

int ehb_index_create(const ehb_params* p, ehb_index** out) {
  if (!p || !out) return fail(EHB_ERR_INVALID, "null argument");
  if (p->dim == 0 || p->dim > ehb::kMaxDim) return fail(EHB_ERR_INVALID, "dim must be in 1..4096");
  if (p->M < 2 || p->M > 16) return fail(EHB_ERR_INVALID, "M must be in 2..16");
  if (p->ef_construction > ehb::kMaxBeam) return fail(EHB_ERR_INVALID, "ef_construction must be <= 4096");
  if (p->metric < 0 || p->metric > 2) return fail(EHB_ERR_INVALID, "unknown metric");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(EHB_ERR_CUDA, std::string("no CUDA device (ehb200 has no CPU fallback): ") + cudaGetErrorString(e));
  if (p->device < 0 || p->device >= ndev) return fail(EHB_ERR_INVALID, "bad device ordinal");
  CU(cudaSetDevice(p->device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, p->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(EHB_ERR_CUDA, "ehb200 kernels are built for sm_90a (compute capability 9.0) only");
  ehb_index* ix = new (std::nothrow) ehb_index();
  if (!ix) return fail(EHB_ERR_OOM, "host allocation failed");
  ix->prm = *p;
  ix->dim = p->dim;
  ix->dpad = ehb::pad_dim(p->dim);
  ix->M = p->M;
  ix->M0 = 2 * p->M;
  ix->metric = p->metric;
  ix->device = p->device;
  ix->sms = prop.multiProcessorCount;
  ix->ef = p->ef_search ? p->ef_search : 10;
  ix->level_rng.seed((unsigned)p->seed);
  if (ix->prm.ef_construction == 0) ix->prm.ef_construction = 200;
  cudaError_t ce = cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking);
  if (ce == cudaSuccess) ce = cudaEventCreate(&ix->bf_ev0);
  if (ce == cudaSuccess) ce = cudaEventCreate(&ix->bf_ev1);
  if (ce != cudaSuccess) {
    delete ix;
    return fail(EHB_ERR_CUDA, cudaGetErrorString(ce));
  }
  int rc = ix->ensure_capacity(std::max<uint64_t>(p->capacity, 1));
  if (rc != EHB_OK) {
    delete ix;
    return rc;
  }
  *out = ix;
  return EHB_OK;
}

int ehb_index_destroy(ehb_index* ix) {
  if (!ix) return EHB_OK;
  cudaSetDevice(ix->device);
  cudaDeviceSynchronize();
  delete ix;
  return EHB_OK;
}

int ehb_index_add(ehb_index* ix, uint64_t n, const float* vecs, const uint64_t* labels) {
  ENTER_X(ix);
  if (n && !vecs) return fail(EHB_ERR_INVALID, "null vectors");
  return ix->add_rows(n, vecs, false, labels);
}
int ehb_index_add_dev(ehb_index* ix, uint64_t n, const float* vecs_dev, const uint64_t* labels) {
  ENTER_X(ix);
  if (n && !vecs_dev) return fail(EHB_ERR_INVALID, "null vectors");
  return ix->add_rows(n, vecs_dev, true, labels);
}
int ehb_index_remove(ehb_index* ix, uint64_t n, const uint64_t* labels) {
  ENTER_X(ix);
  if (n && !labels) return fail(EHB_ERR_INVALID, "null labels");
  return ix->remove_labels(n, labels);
}
int ehb_index_build(ehb_index* ix) {
  ENTER_X(ix);
  RET(ix->build());
  CU(cudaStreamSynchronize(ix->stream));
  return EHB_OK;
}
int ehb_index_compact(ehb_index* ix) {
  ENTER_X(ix);
  RET(ix->compact());
  CU(cudaStreamSynchronize(ix->stream));
  return EHB_OK;
}
int ehb_index_set_ef(ehb_index* ix, uint32_t ef) {
  ENTER_X(ix);
  if (ef == 0) return fail(EHB_ERR_INVALID, "ef must be > 0");
  ix->ef = ef;
  return EHB_OK;
}
int ehb_index_size(ehb_index* ix, uint64_t* out) {
  ENTER_S(ix);
  if (!out) return fail(EHB_ERR_INVALID, "null out");
  *out = ix->n;
  return EHB_OK;
}

int ehb_index_get(ehb_index* ix, uint64_t label, float* out) {
  ENTER_S(ix);
  if (!out) return fail(EHB_ERR_INVALID, "null out");
  uint32_t id;
  // hnswlib getDataByLabel: a tombstoned label reads as "Label not found"
  if (!ix->find_id(label, &id) || ix->h_deleted[id]) return fail(EHB_ERR_NOT_FOUND, "label not found");
  CU(cudaMemcpy(out, ix->vecs.p + (uint64_t)id * ix->dpad, ix->dim * 4, cudaMemcpyDeviceToHost));
  return EHB_OK;
}

int ehb_index_get_batch(ehb_index* ix, uint64_t n, const uint64_t* labels, float* out) {
  ENTER_S(ix);
  if (n && (!labels || !out)) return fail(EHB_ERR_INVALID, "null buffer");
  if (n == 0) return EHB_OK;
  std::vector<uint32_t> ids;
  RET(resolve_labels(ix, n, labels, ids));
  ehb::SlotLease ls(ix);
  RET(ls.take());
  CU(ls.sl->q_in.grow(n * ix->dim, 0, -1, ls.s));
  RET(gather_ids(ix, ls.sl, ids, ls.sl->q_in.p, ls.s));
  CU(cudaMemcpyAsync(out, ls.sl->q_in.p, n * ix->dim * 4, cudaMemcpyDeviceToHost, ls.s));
  CU(cudaStreamSynchronize(ls.s));
  return EHB_OK;
}

int ehb_index_search_by_label_ex(ehb_index* ix, uint64_t nq, const uint64_t* labels, uint32_t k, uint32_t ef,
                                 int precision, uint64_t* ol, float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, false, true, nq, nullptr, labels, k, ef, precision, ol, od, oc);
}

int ehb_index_search_bruteforce_by_label(ehb_index* ix, uint64_t nq, const uint64_t* labels, uint32_t k, int precision,
                                         uint64_t* ol, float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, true, true, nq, nullptr, labels, k, 0, precision, ol, od, oc);
}

// Chunks of C live points in internal-id order.  Chunk j + 1 is gathered and walked while the results of chunk j
// are copied out (two result buffers).  The shared lock is held throughout: the table is one snapshot.
int ehb_index_neighbor_table(ehb_index* ix, uint32_t k, uint32_t ef, int precision, uint64_t* oq, uint64_t* ol,
                             float* od, uint32_t* oc, uint64_t* out_rows) {
  ENTER_S(ix);
  bool none;  // (nq = 1: the table's rows are not an argument)
  RET(ehb::check_request(ix, false, precision, !oq || !ol || !out_rows, 1, k, k + 1ull, &ef, &none));
  if (none) return EHB_OK;
  const uint32_t k1 = k + 1;
  const uint64_t C = ix->o_table_chunk;
  RET(ix->prepare(_g, false, precision, std::min<uint64_t>(C, ix->n - ix->n_deleted)));
  const uint64_t n = ix->n, live = n - ix->n_deleted;
  if (live > *out_rows) {
    const uint64_t room = *out_rows;
    *out_rows = live;
    return fail(EHB_ERR_INVALID, "the buffers hold " + std::to_string(room) + " rows, the table has " +
                                     std::to_string(live));
  }
  if (live == 0) {
    *out_rows = 0;
    return EHB_OK;
  }
  TableCopies tc;
  CU(cudaStreamCreateWithFlags(&tc.s, cudaStreamNonBlocking));
  for (int b = 0; b < 2; ++b) {
    CU(cudaEventCreateWithFlags(&tc.ready[b], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&tc.copied[b], cudaEventDisableTiming));
  }
  const uint64_t cmax = std::min(C, live);
  ehb::DevBuf<uint64_t> rl[2];
  ehb::DevBuf<float> rd[2];
  ehb::DevBuf<uint32_t> rc_[2];
  ehb::SlotLease ls(ix);
  RET(ls.take());
  ehb::SearchSlot* sl = ls.sl;
  const cudaStream_t s = ls.s;
  for (int b = 0; b < 2; ++b) {
    CU(rl[b].grow(cmax * k, 0, -1, s));
    CU(rd[b].grow(cmax * k, 0, -1, s));
    CU(rc_[b].grow(cmax, 0, -1, s));
  }
  CU(sl->q_in.grow(cmax * ix->dim, 0, -1, s));
  CU(sl->q_labels.grow(live, 0, -1, s));
  CU(sl->o_labels.grow(cmax * k1, 0, -1, s));
  CU(sl->o_dists.grow(cmax * k1, 0, -1, s));
  CU(sl->o_counts.grow(cmax, 0, -1, s));
  // the live ids (none to list without tombstones: chunk rows are then consecutive ids)
  const bool listed = ix->n_deleted != 0;
  if (listed) {
    CU(sl->q_ids.grow(n + 1, 0, -1, s));
    CU(ehb::launch_live_ids(ix->deleted.p, n, sl->q_ids.p, sl->q_ids.p + n, s));
    std::vector<uint32_t> ids(live);
    CU(cudaMemcpyAsync(ids.data(), sl->q_ids.p, live * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    for (uint64_t r = 0; r < live; ++r) oq[r] = ix->h_labels[ids[r]];
  } else {
    std::copy(ix->h_labels.begin(), ix->h_labels.begin() + n, oq);
  }
  CU(cudaMemcpyAsync(sl->q_labels.p, oq, live * 8, cudaMemcpyHostToDevice, s));
  auto copy_out = [&](uint64_t off, uint64_t m, int b) -> int {
    CU(cudaStreamWaitEvent(tc.s, tc.ready[b], 0));
    RET(ehb::copy_results(m, k, rl[b].p, rd[b].p, rc_[b].p, ol + off * k, od ? od + off * k : nullptr,
                          oc ? oc + off : nullptr, tc.s));
    CU(cudaEventRecord(tc.copied[b], tc.s));
    return EHB_OK;
  };
  uint64_t prev_off = 0, prev_m = 0;
  for (uint64_t off = 0, j = 0; off < live; off += C, ++j) {
    const uint64_t m = std::min(C, live - off);
    const int b = (int)(j & 1);
    if (j >= 2) CU(cudaStreamWaitEvent(s, tc.copied[b], 0));  // chunk j - 2's results have left buffer b
    if (listed)
      CU(ehb::launch_gather_rows(ix->vecs.p, ix->dpad, sl->q_ids.p + off, sl->q_in.p, ix->dim, nullptr, m, ix->dim, s));
    else
      CU(ehb::launch_gather_rows(ix->vecs.p + off * ix->dpad, ix->dpad, nullptr, sl->q_in.p, ix->dim, nullptr, m,
                                 ix->dim, s));
    RET(ix->search_dev(sl, m, sl->q_in.p, k1, ef, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, s, nullptr, nullptr,
                       precision));
    CU(ehb::launch_drop_self(sl->q_labels.p + off, sl->o_labels.p, sl->o_dists.p, sl->o_counts.p, m, k, rl[b].p,
                             rd[b].p, rc_[b].p, s));
    CU(cudaEventRecord(tc.ready[b], s));
    // chunk j - 1 is copied out while chunk j runs
    if (j >= 1) RET(copy_out(prev_off, prev_m, 1 - b));
    prev_off = off, prev_m = m;
  }
  RET(copy_out(prev_off, prev_m, (int)(((live + C - 1) / C - 1) & 1)));
  CU(cudaStreamSynchronize(tc.s));
  CU(cudaStreamSynchronize(s));
  *out_rows = live;
  return EHB_OK;
}

int ehb_index_search_ex(ehb_index* ix, uint64_t nq, const float* q, uint32_t k, uint32_t ef, int precision,
                        uint64_t* ol, float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, false, false, nq, q, nullptr, k, ef, precision, ol, od, oc);
}
int ehb_index_search(ehb_index* ix, uint64_t nq, const float* q, uint32_t k, uint32_t ef, uint64_t* ol, float* od,
                     uint32_t* oc) {
  return ehb_index_search_ex(ix, nq, q, k, ef, EHB_FP32, ol, od, oc);
}

int ehb_index_search_ex_dev(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, uint32_t ef, int precision,
                            uint64_t* dl, float* dd, uint32_t* dc, void* stream) {
  ENTER_S(ix);
  bool none;
  RET(ehb::check_request(ix, false, precision, nq && (!dq || !dl), nq, k, k, &ef, &none));
  if (none) return EHB_OK;
  RET(ix->prepare(_g, false, precision, nq));
  ehb::SlotLease ls(ix);
  RET(ls.take((cudaStream_t)stream));
  return ix->search_dev(ls.sl, nq, dq, k, ef, dl, dd, dc, ls.s, nullptr, nullptr, precision);
}
int ehb_index_search_dev(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, uint32_t ef, uint64_t* dl, float* dd,
                         uint32_t* dc, void* stream) {
  return ehb_index_search_ex_dev(ix, nq, dq, k, ef, EHB_FP32, dl, dd, dc, stream);
}

// The wide-beam entry points: the _ex calls with the width limit raised to EHB_MAX_BEAM.  Up to 512 they run exactly
// what the _ex calls run; above, walk_plan picks the wide-beam walk, which never goes through the combining queue.
int ehb_index_search_beam(ehb_index* ix, uint64_t nq, const float* q, uint32_t k, uint32_t ef, int precision,
                          uint64_t* ol, float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, false, false, nq, q, nullptr, k, ef, precision, ol, od, oc, ehb::kMaxBeam);
}
int ehb_index_search_by_label_beam(ehb_index* ix, uint64_t nq, const uint64_t* labels, uint32_t k, uint32_t ef,
                                   int precision, uint64_t* ol, float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, false, true, nq, nullptr, labels, k, ef, precision, ol, od, oc, ehb::kMaxBeam);
}
int ehb_index_search_beam_dev(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, uint32_t ef, int precision,
                              uint64_t* dl, float* dd, uint32_t* dc, void* stream) {
  ENTER_S(ix);
  bool none;
  RET(ehb::check_request(ix, false, precision, nq && (!dq || !dl), nq, k, k, &ef, &none, ehb::kMaxBeam));
  if (none) return EHB_OK;
  RET(ix->prepare(_g, false, precision, nq));
  ehb::SlotLease ls(ix);
  RET(ls.take((cudaStream_t)stream));
  return ix->search_dev(ls.sl, nq, dq, k, ef, dl, dd, dc, ls.s, nullptr, nullptr, precision);
}

}  // extern "C"

int ehb_index_search_dev_sink(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, uint32_t ef, int precision,
                              const ehb::ResultSink* sink, uint32_t* dc, cudaStream_t stream, bool* pushed) {
  ENTER_S(ix);
  return ehb_index_search_dev_sink_held(ix, _g, nq, dq, k, ef, precision, sink, dc, stream, pushed);
}

int ehb_index_search_dev_sink_held(ehb_index* ix, std::shared_lock<ehb::RwLock>& lk, uint64_t nq, const float* dq,
                                   uint32_t k, uint32_t ef, int precision, const ehb::ResultSink* sink, uint32_t* dc,
                                   cudaStream_t stream, bool* pushed, uint32_t max_beam) {
  bool none;
  RET(ehb::check_request(ix, false, precision, !dq || !sink || !sink->n || !sink->labels[0], nq, k, k, &ef, &none,
                         max_beam));
  if (none) return EHB_OK;
  RET(ix->prepare(lk, false, precision, nq));
  ehb::SlotLease ls(ix);
  RET(ls.take(stream));
  return ix->search_dev(ls.sl, nq, dq, k, ef, sink->labels[0], sink->dists[0], dc, ls.s, sink, pushed, precision);
}

int ehb_index_gather_dev(ehb_index* ix, uint64_t n, const uint64_t* labels, float* rows_dev, cudaStream_t stream) {
  ENTER_S(ix);
  if (n && (!labels || !rows_dev)) return fail(EHB_ERR_INVALID, "null buffer");
  if (n == 0) return EHB_OK;
  std::vector<uint32_t> ids;
  RET(resolve_labels(ix, n, labels, ids));
  ehb::SlotLease ls(ix);
  RET(ls.take(stream));
  return gather_ids(ix, ls.sl, ids, rows_dev, ls.s);
}

extern "C" {

int ehb_index_search_bruteforce(ehb_index* ix, uint64_t nq, const float* q, uint32_t k, int precision, uint64_t* ol,
                                float* od, uint32_t* oc) {
  ENTER_S(ix);
  return search_host(ix, _g, true, false, nq, q, nullptr, k, 0, precision, ol, od, oc);
}

int ehb_index_search_bruteforce_dev(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, int precision,
                                    uint64_t* dl, float* dd, uint32_t* dc, void* stream) {
  ENTER_S(ix);
  bool none;
  RET(ehb::check_request(ix, true, precision, nq && (!dq || !dl), nq, k, k, nullptr, &none));
  if (none) return EHB_OK;
  RET(ix->prepare(_g, true, precision, nq));  // before bf_mu: the upgrade waits for other readers
  std::lock_guard<std::mutex> bg(ix->bf_mu);
  return ix->bruteforce_dev(nq, dq, k, precision, dl, dd, dc, stream ? (cudaStream_t)stream : ix->stream);
}

// Caller holds last_mu: the counters of the last graph search, summed once (false when there is none)
static int last_walk_sums(ehb_index* ix, bool* have) {
  ehb::SearchSlot* sl = ix->last_slot;
  *have = sl && !ix->last_was_brute && sl->last_nq;
  if (!*have || ix->last_sum_valid) return EHB_OK;
  CU(cudaEventSynchronize(sl->ev1));
  CU(ehb::launch_sum_stats(sl->stats.p, (uint32_t)sl->last_nq, sl->stat_sum.p, ix->stream));
  CU(cudaMemcpyAsync(ix->last_sum, sl->stat_sum.p, sizeof(ix->last_sum), cudaMemcpyDeviceToHost, ix->stream));
  ix->last_reranked = 0;
  std::vector<uint32_t> cnt(sl->last_bf16 ? sl->last_nq : 0);
  if (sl->last_bf16)
    CU(cudaMemcpyAsync(cnt.data(), sl->walk_counts.p, sl->last_nq * 4, cudaMemcpyDeviceToHost, ix->stream));
  CU(cudaStreamSynchronize(ix->stream));
  for (uint32_t c : cnt) ix->last_reranked += c;
  ix->last_sum_valid = true;
  return EHB_OK;
}
// fp32 rows the last graph walk read: every evaluation but the screened ones, plus the screen's survivors (none
// for a bf16 walk)
static uint64_t last_fp32_rows(const ehb_index* ix) {
  return ix->last_slot->last_bf16 ? 0 : ix->last_sum[2] - ix->last_sum[4] + ix->last_sum[5];
}

int ehb_index_stats(ehb_index* ix, ehb_stats* out) {
  ENTER_S(ix);
  if (!out) return fail(EHB_ERR_INVALID, "null out");
  std::memset(out, 0, sizeof(*out));
  {
    std::lock_guard<std::mutex> g(ix->last_mu);
    bool have = false;
    RET(last_walk_sums(ix, &have));
    if (have) {
      ehb::SearchSlot* sl = ix->last_slot;
      out->queries = sl->last_nq;
      out->hops_upper = ix->last_sum[0];
      out->hops_base = ix->last_sum[1];
      out->dist_evals = ix->last_sum[2];
      out->visited_overflow = ix->last_sum[3];
      // A bf16 walk reads 2 bytes per element, and its re-rank reads the fp32 rows of the retained keys.  A
      // screened fp32 walk reads 1 byte per element and the 16 bytes of per-row terms of every screened candidate,
      // and 4 bytes per element of the fp32 rows it read.
      const uint64_t screened = ix->last_sum[4];
      out->algorithmic_bytes = out->hops_upper * 4ull * ix->M + out->hops_base * 4ull * ix->M0 +
                               (sl->last_bf16 ? out->dist_evals * 2ull * ix->dim
                                              : last_fp32_rows(ix) * 4ull * ix->dim +
                                                    screened * (ix->dim + (uint64_t)sizeof(float4))) +
                               out->queries * 4ull * ix->dim + ix->last_reranked * 4ull * ix->dim;
    }
  }
  out->size = ix->n;
  out->capacity = ix->cap;
  out->upper_rows = ix->up_rows;
  out->dim = ix->dim;
  out->M = ix->M;
  out->max_level = ix->max_level < 0 ? 0 : (uint32_t)ix->max_level;
  out->entry_point = ix->entry;
  out->device_bytes = ix->vecs.bytes() + ix->labels.bytes() + ix->levels.bytes() + ix->deleted.bytes() +
                      ix->links0.bytes() + ix->up_off.bytes() + ix->links_up.bytes() + ix->up_owner.bytes() +
                      ix->x_bf16.bytes() + ix->x_norm.bytes() + ix->x_i8.bytes() + ix->x_i8t.bytes();
  out->deleted = ix->n_deleted;
  out->combined_batches = ix->combined_batches.load();
  out->combined_queries = ix->combined_queries.load();
  out->metric = (uint32_t)ix->metric;
  return EHB_OK;
}

int ehb_index_screen_stats(ehb_index* ix, uint64_t* screened_evals, uint64_t* fp32_row_reads) {
  ENTER_S(ix);
  if (!screened_evals || !fp32_row_reads) return fail(EHB_ERR_INVALID, "null out");
  std::lock_guard<std::mutex> g(ix->last_mu);
  bool have = false;
  RET(last_walk_sums(ix, &have));
  *screened_evals = have ? ix->last_sum[4] : 0;
  *fp32_row_reads = have ? last_fp32_rows(ix) : 0;
  return EHB_OK;
}

int ehb_index_last_kernel_ms(ehb_index* ix, float* out_ms) {
  ENTER_S(ix);
  if (!out_ms) return fail(EHB_ERR_INVALID, "null out");
  std::lock_guard<std::mutex> g(ix->last_mu);
  if (!ix->timed) return fail(EHB_ERR_STATE, "no search has been timed yet");
  cudaEvent_t e0 = ix->last_was_brute ? ix->bf_ev0 : ix->last_slot->ev0;
  cudaEvent_t e1 = ix->last_was_brute ? ix->bf_ev1 : ix->last_slot->ev1;
  CU(cudaEventSynchronize(e1));
  CU(cudaEventElapsedTime(out_ms, e0, e1));
  return EHB_OK;
}

int ehb_index_last_kernel_name(ehb_index* ix, char* out, uint32_t out_bytes) {
  ENTER_S(ix);
  if (!out || !out_bytes) return fail(EHB_ERR_INVALID, "null out");
  std::lock_guard<std::mutex> g(ix->last_mu);
  const char* name = !ix->timed ? "" : (ix->last_was_brute ? "bruteforce" : ix->last_slot->last_kernel);
  std::snprintf(out, out_bytes, "%s", name);
  return EHB_OK;
}

int ehb_index_set_search_width(ehb_index* ix, uint32_t warps_per_query) {
  ENTER_X(ix);
  if (warps_per_query > 4) return fail(EHB_ERR_INVALID, "warps_per_query must be 0 (auto) or 1..4");
  ix->t_team = warps_per_query;
  return EHB_OK;
}

int ehb_index_set_option(ehb_index* ix, const char* name, int64_t value) {
  ENTER_X(ix);
  if (!name) return fail(EHB_ERR_INVALID, "null option name");
  const std::string o(name);
  if (o == "build_frac") {
    if (value < 0 || value > (1 << 20)) return fail(EHB_ERR_INVALID, "build_frac must be in 0..2^20");
    ix->o_build_frac = (uint32_t)value;
  } else if (o == "seq_updates") {
    if (value < 0) return fail(EHB_ERR_INVALID, "seq_updates must be >= 0");
    ix->o_seq_updates = (uint64_t)value;
  } else if (o == "bf16_unfused") {
    ix->o_bf16_unfused = value != 0;
  } else if (o == "walk_prefetch") {
    ix->o_walk_prefetch = value != 0;
  } else if (o == "walk_screen") {
    ix->o_walk_screen = value < 0 ? -1 : (value ? 1 : 0);
    ix->screen_no_room = false;
  } else if (o == "combine") {
    ix->o_combine = value != 0;
  } else if (o == "table_chunk") {
    if (value < 1 || value > (1ll << 31)) return fail(EHB_ERR_INVALID, "table_chunk must be in 1..2^31");
    ix->o_table_chunk = (uint64_t)value;
  } else {
    return fail(EHB_ERR_INVALID, "unknown option: " + o);
  }
  return EHB_OK;
}

int ehb_index_set_tuning(ehb_index* ix, uint32_t slots, uint32_t groups, uint32_t hash_bits, uint32_t wpb) {
  ENTER_X(ix);
  ix->t_slots = slots;
  ix->t_groups = groups;
  ix->t_hash_bits = hash_bits;
  ix->t_wpb = wpb;
  return EHB_OK;
}

int ehb_merge_topk_dev(uint32_t G, uint64_t nq, uint32_t k, const float* dists, const uint64_t* labels,
                       float* out_dists, uint64_t* out_labels, uint32_t* out_counts, int32_t device, void* stream) {
  if (G == 0 || G > 32) return fail(EHB_ERR_INVALID, "G must be in 1..32");
  if (nq && k && (!dists || !labels || !out_labels)) return fail(EHB_ERR_INVALID, "null buffer");
  CU(cudaSetDevice(device));
  CU(ehb::launch_merge_topk(G, nq, k, dists, labels, nq * k * 4ull, nq * k * 8ull, out_dists, out_labels, out_counts,
                            (cudaStream_t)stream));
  return EHB_OK;
}

int ehb_merge_topk_packed_dev(uint32_t G, uint64_t nq, uint32_t k, const void* packed, uint64_t rank_stride_bytes,
                              float* out_dists, uint64_t* out_labels, uint32_t* out_counts, int32_t device,
                              void* stream) {
  if (G == 0 || G > 32) return fail(EHB_ERR_INVALID, "G must be in 1..32");
  if (nq && k && (!packed || !out_labels)) return fail(EHB_ERR_INVALID, "null buffer");
  if (rank_stride_bytes < nq * k * 12ull || (rank_stride_bytes & 7u)) return fail(EHB_ERR_INVALID, "bad rank stride");
  CU(cudaSetDevice(device));
  const unsigned char* base = (const unsigned char*)packed;
  CU(ehb::launch_merge_topk(G, nq, k, (const float*)(base + nq * k * 8ull), (const uint64_t*)base, rank_stride_bytes,
                            rank_stride_bytes, out_dists, out_labels, out_counts, (cudaStream_t)stream));
  return EHB_OK;
}

}  // extern "C"
