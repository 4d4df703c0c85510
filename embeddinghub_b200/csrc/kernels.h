// Host-callable launchers of the ehb200 kernels (internal header).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "walk.cuh"

namespace ehb {

constexpr uint32_t kMaxDim = 4096;  // pad_dim() supports rows up to 4096 floats
constexpr uint32_t kMaxEf = 512;    // register-resident list: 16 keys per lane
constexpr uint32_t kMaxBeam = 4096; // wide-beam walk (WalkForm::beam): shared-memory list, visited table in HBM
constexpr uint32_t kMaxRegEfc = 256;    // construction beam in the register set (UList<8>); wider: K5's wide form
constexpr uint32_t kUpdCandCap = 1088;  // update path: sCand capacity per moved point, >= 1 + 32 + 32*32
constexpr uint32_t kRepairWarps = 8192; // compaction repair: warps of the persistent grid (upd_cand slots)

// Shapes with a dense form of the one-warp walk (search_impl.cuh): LPV = 8, NQ <= 4, no tombstones.  Over bf16 rows
// the dense form's 96-register budget spills at dpad = 128 with KPL >= 8, so those shapes have none.
constexpr bool dense_form(bool bf16, int LPV, int NQ, int KPL, bool HASDEL) {
  return LPV == 8 && NQ <= 4 && !HASDEL && (!bf16 || NQ < 4 || KPL < 8);
}

// Which graph-walk kernel a search runs and how it is launched (ehb_index::walk_plan).  The launchers and the
// reported kernel name read it and decide nothing themselves.
// wide: the form of the wide shapes (walk.cuh wide_shape, dpad 3072 and 4096), and their only one.
// beam: every beam above kMaxEf, any row shape (beam_impl.cuh).
enum class WalkForm { plain, dense, team, wide, beam };
struct WalkPlan {
  bool bf16;           // the walk reads the bf16 shadow g.vecs16 (else the fp32 rows)
  int lpv, nq, kpl;    // row shape (walk.cuh row_lpv / row_nq) and result-set entries per lane (kpl_for)
  bool hasdel;         // the index has tombstones
  WalkForm form;
  uint32_t T, U;       // team form: warps per query (2..4) and load steps in flight; 1 and 0 otherwise
  bool screen;         // the fp32 walk screens candidates on the int8 screen copy (g.codes8 / g.terms8 set by the caller);
                       // its cfg then has no TMA ring (staged = 0): rows go straight into registers
  WalkCfg cfg;
  uint32_t wpb;        // warps per block of the one-warp forms
  uint32_t vtab;       // beam form: entries of each warp's visited table in HBM (cfg.hash_size is 0)
};
// the name of the kernel the plan launches, e.g. hnsw_search_kernel<LPV=32,NQ=6,KPL=4>
void walk_kernel_name(const WalkPlan& p, char* out, size_t out_bytes);

// K2 — batched k-NN graph walk (hnswlib searchKnn), one warp per query, plain, dense or wide form.  ef >= k.
// stats: [nq][kStatWords] u32 = hops_upper, hops_base, evals, overflow, screened, survivors, screened_upper (those
// of the upper-layer descent), 0.  With g.codes8 set (metric 1, rows > 1 KB) the fp32 walk screens candidates on the
// int8 screen copy (walk.cuh greedy_descent, beam_search).
// With p.bf16 the walk reads the bf16 shadow g.vecs16 (fp32 queries, fp32 accumulation) and writes the retained
// set, not results: sink.keys[nq][k] gets the (ordered distance, internal id) keys nearest-first (call with k = ef
// to keep all of them) and out_counts the retained count; launch_rerank then produces the fp32 results.
constexpr uint32_t kStatWords = 8;
cudaError_t launch_search(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                          uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats, cudaStream_t s);
// K2 for rows of DPAD floats of type RowT (search_impl.cuh; instantiated per shape in search_inst_*.cu)
template <uint32_t DPAD, class RowT>
struct SearchShape {
  static cudaError_t launch(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                            uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats,
                            cudaStream_t s);
};

// K2b — the wide-beam walk (p.form == WalkForm::beam, ef <= kMaxBeam): a persistent grid of one-warp blocks, each
// with a visited table of p.vtab entries in vtab.  beam_warps: the warps of the launch for nq queries (resident
// warps, at most nq); vtab must hold warps * p.vtab entries.  Results, key sink and stats as launch_search.
cudaError_t beam_warps(const WalkPlan& p, const GraphView& g, int sms, uint64_t nq, uint32_t* warps);
cudaError_t launch_search_beam(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                               uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats,
                               uint32_t* vtab, uint32_t warps, cudaStream_t s);
// The resident warps of a persistent grid of one-warp blocks of `kern` with smem bytes of dynamic shared memory each,
// on sms SMs (sets the kernel's dynamic shared-memory limit to smem; cudaErrorInvalidConfiguration when not even one
// block fits an SM).
cudaError_t resident_warps(const void* kern, uint32_t smem, int sms, uint32_t* out);
template <uint32_t DPAD, class RowT>
struct BeamShape {
  static cudaError_t warps(const WalkPlan& p, int sms, uint64_t nq, uint32_t* out);
  static cudaError_t launch(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                            uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats, uint32_t* vtab,
                            uint32_t warps, cudaStream_t s);
};

// K2t — team walk (p.T warps per query); fp32 rows <= 1 KB and ef <= 256 only.
cudaError_t launch_search_team(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                               uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                               uint32_t* stats, cudaStream_t s);

// row-wise L2 normalisation (hnswlib cosine convention), canonical arithmetic.
cudaError_t launch_normalize(const float* in, uint32_t in_stride, float* out, uint32_t out_stride, uint64_t n,
                             uint32_t dim, cudaStream_t s);
// copy [n][dim] -> [n][dpad] with zero padding (and optional normalisation)
cudaError_t launch_pad_rows(const float* in, float* out, uint64_t n, uint32_t dim, uint32_t dpad, bool normalize,
                            cudaStream_t s);
// the int8 screen copy of fp32 rows [n][dpad] (GraphView::codes8 / terms8): per row, s = RN(max |x_i| / 127),
// codes RN(x_i / s) clamped to [-127, 127], and terms (s, max |r_i|, |r|_2, |x|_2) rounded up, r = x - s c computed
// in double.  An all-zero row has s = 0 and zero terms; a row with a non-finite value or a subnormal s gets NaN terms.
cudaError_t launch_to_i8(const float* in, uint32_t dpad, int8_t* codes, float4* terms, uint64_t n, cudaStream_t s);
// sums the per-query stats into out[6] (the overflow word counts queries)
cudaError_t launch_sum_stats(const uint32_t* stats, uint32_t nq, unsigned long long* out, cudaStream_t s);

// K1 — exact fp32 brute force with canonical arithmetic.
struct BruteScratch {
  float* dist;          // [qb][nc]
  uint64_t* part_keys;  // [qb][slices][k]
  uint64_t* run_keys;   // [nq][k] running best
  uint64_t qb, nc, slices;
  const uint8_t* deleted = nullptr;  // tombstones: such rows never form a key
};
cudaError_t launch_bruteforce_exact(const float* vecs, uint32_t dpad, uint32_t dim, uint64_t n, const uint64_t* labels,
                                    int metric, const float* queries /*[nq][dim]*/, uint64_t nq, uint32_t k,
                                    BruteScratch& sc, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                                    cudaStream_t s);

// K3 — bf16 tensor-core (wgmma) distance tiles + fp32 re-rank.
struct Bf16Ctx {
  const void* q_bf16;   // [nq][dpad] bf16
  const void* x_bf16;   // [n][dpad] bf16
  const float* qnorm;   // [nq] squared norms of the rounded queries (L2 only)
  const float* xnorm;   // [n]
  uint32_t kc;          // candidates kept per query before the fp32 re-rank (>= k)
  // fused selection (epilogue filter): per-query threshold, candidate buffer [nq][ccap], counters, flag
  float* thr;
  uint64_t* cbuf;
  uint32_t* ccount;
  uint32_t ccap;
  uint32_t* overflow;   // device flag
  int sms;
  bool fused;
};
cudaError_t launch_bf16_topk_chunk(const void* q_bf16, uint64_t nq, const void* x_bf16, uint64_t x_rows, uint32_t dpad,
                                   int metric, const float* qnorm, const float* xnorm, uint64_t n_lo, uint64_t n_hi,
                                   float* thr, uint64_t* cbuf, uint32_t* ccount, uint32_t ccap, uint64_t* run_keys,
                                   uint32_t kc, uint32_t* overflow, int sms, cudaStream_t s);
cudaError_t launch_to_bf16(const float* in, uint32_t in_stride, void* out_bf16, float* norms, uint64_t n, uint32_t dpad,
                           cudaStream_t s);
cudaError_t launch_bf16_dist_tile(const void* q_bf16, uint64_t q_rows, const void* x_bf16, uint64_t x_rows,
                                  uint32_t dpad, int metric, const float* qnorm, const float* xnorm, uint64_t q0,
                                  uint64_t qn, uint64_t n0, uint64_t nn, float* dist, uint64_t ldd, cudaStream_t s);
cudaError_t launch_rerank(const uint64_t* cand, uint32_t kc, const float* qpad, const float* vecs, uint32_t dpad,
                          uint32_t dim, int metric, const uint64_t* labels, uint64_t nq, uint32_t k,
                          uint64_t* out_labels, float* out_dists, uint32_t* out_counts, cudaStream_t s);
// The same re-rank storing into every destination of a result sink and raising its slice flags (walk.cuh):
// the bf16 graph walk's last kernel in a sharded search step.  k <= kMaxEf.
cudaError_t launch_rerank_sink(const uint64_t* cand, uint32_t kc, const float* qpad, const float* vecs, uint32_t dpad,
                               uint32_t dim, int metric, const uint64_t* labels, uint64_t nq, uint32_t k,
                               const ResultSink& sink, uint32_t* out_counts, cudaStream_t s);
cudaError_t launch_bruteforce(const float* vecs, uint32_t dpad, uint32_t dim, uint64_t n, const uint64_t* labels,
                              int metric, const float* qpad, uint64_t nq, uint32_t k, BruteScratch& sc,
                              const Bf16Ctx* bf, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                              cudaStream_t s);

// K4 — merge of G sorted (dist,label) lists per query.
cudaError_t launch_merge_topk(uint32_t G, uint64_t nq, uint32_t k, const float* dists, const uint64_t* labels,
                              uint64_t stride_d_bytes, uint64_t stride_l_bytes, float* out_dists, uint64_t* out_labels,
                              uint32_t* out_counts, cudaStream_t s);

// K5 — batched graph construction.
struct BuildBuffers {
  // per-batch edge list (reverse links to apply)
  uint32_t* edge_row;   // target row id (level-0 rows: node id; upper rows: cap + row)
  uint32_t* edge_src;
  float* edge_dist;
  uint32_t* edge_count; // [1]
  uint32_t edge_cap;
  // per-row scratch, sized row_space = cap + upper_cap
  uint32_t* row_cnt;
  uint32_t* row_fill;
  uint32_t* row_start;
  uint32_t* touched;    // [edge_cap]
  uint32_t* touched_count;  // [1]
  uint32_t* seg_cursor;     // [1]
  uint32_t* seg_src;    // [edge_cap]
  float* seg_dist;      // [edge_cap]
  uint32_t* error_flag; // [1]
  uint32_t* upd_cand;   // [batch][kUpdCandCap] sCand scratch of the update path (nullptr for plain inserts)
  uint32_t* repair_out; // [rows][M0] re-selected rows of the compaction repair (nullptr otherwise)
  // update path: rows staged until every warp of the phase has read the graph (build_impl.cuh stage_row)
  uint32_t* side_row;   // [side_cap] row id (edge_row convention)
  uint32_t* side_out;   // [side_cap + 1][M0] the new rows (+ one sink slot)
  uint32_t* side_count;
  uint32_t side_cap;
};
struct BuildGraph {
  GraphView g;          // links are written through these pointers (const-cast inside)
  const uint8_t* levels;
  const uint32_t* up_owner;  // [upper rows] owning node of each upper row
  uint32_t cap;         // row id space split: rows >= cap are upper rows
  uint32_t efc;
};
enum BuildMode : int {
  kBuildInsert = 0,  // link points ids[0..b) (or first..first+b when ids == nullptr) into the graph
  kBuildUpdate = 1,  // hnswlib updatePoint of the already linked points ids[0..b)
  kBuildRepair = 2,  // compaction: re-select the rows ids[0..b) (row ids as edge_row) into bb.repair_out
};
// The wide form of K5 (bg.efc > kMaxRegEfc): its construction search runs as a persistent grid of one-warp blocks,
// each with a visited table of vsize = align_up(2 M0 efc + 64, 32) entries in vtab, which holds `warps` of them.  The
// launch uses min(b, warps) warps.  Unused (all zero) in the register form.
struct BuildBeam {
  uint32_t* vtab;
  uint32_t vsize;
  uint32_t warps;
};
// cfg: walk_cfg's for the search; in the wide form lcap = 2 align_up(efc, 32) (the set and its ordered list),
// hash_size = 0 and, with tombstones, dcap = max(kDeletedQueue, align_up(efc / 4, 32)).
cudaError_t launch_build_batch(const BuildGraph& bg, const WalkCfg& cfg, const uint32_t* ids, uint32_t first,
                               uint32_t b, int mode, BuildBuffers& bb, uint32_t warps_per_block, const BuildBeam& bm,
                               cudaStream_t s);
// The resident warps of the wide form's construction search for cfg and the tombstone state of bg.g, on sms SMs
// (cudaErrorInvalidConfiguration when not even one fits an SM).
cudaError_t build_beam_warps(const BuildGraph& bg, const WalkCfg& cfg, int sms, uint32_t* warps);
// K5 for rows of DPAD floats (build_impl.cuh; instantiated per shape in build_inst_*.cu)
template <uint32_t DPAD>
struct BuildShape {
  static cudaError_t launch(const BuildGraph& bg, const WalkCfg& cfg, const uint32_t* ids, uint32_t first, uint32_t b,
                            int mode, BuildBuffers& bb, uint32_t wpb, const BuildBeam& bm, cudaStream_t s);
};
// The wide form's kernels for rows of DPAD floats (build_impl.cuh; instantiated per shape in build_inst_beam_*.cu):
// the construction search (with or without tombstones) and the update / repair re-selection (rows(kBuildUpdate) or
// rows(kBuildRepair)) with its keep list in shared memory.
using BuildSearchBeamKernel = void (*)(BuildGraph, WalkCfg, const uint32_t*, uint32_t, uint32_t, int, BuildBuffers,
                                       uint32_t, uint32_t*);
using BuildRowsKernel = void (*)(BuildGraph, WalkCfg, const uint32_t*, uint32_t, BuildBuffers, uint32_t);
template <uint32_t DPAD>
struct BuildBeamShape {
  static BuildSearchBeamKernel search(bool hasdel);
  static BuildRowsKernel rows(int mode);
  static cudaError_t warps(const BuildGraph& bg, const WalkCfg& cfg, int sms, uint32_t* out);
};

// K6 — compaction (ehb_index_compact).  Row ids follow the edge_row convention: < cap a level-0 row, >= cap an
// upper row.
// Appends to rows[] (count in *nrows) every row of a live node that names a deleted id, and counts the level-0
// in-links of every node (indeg, zeroed by the caller).
cudaError_t launch_compact_mark(const uint32_t* links0, const uint32_t* links_up, const uint32_t* up_owner,
                                const uint8_t* deleted, uint64_t n, uint64_t up_rows, uint32_t M0, uint32_t M,
                                uint32_t cap, uint32_t* rows, uint32_t* nrows, uint32_t* indeg, cudaStream_t s);
// Copies the re-selected rows repair_out[i] back over rows[i] (after every repair has read the old graph).
cudaError_t launch_compact_apply(const uint32_t* rows, uint32_t nrows, const uint32_t* repair_out, uint32_t* links0,
                                 uint32_t* links_up, uint32_t M0, uint32_t M, uint32_t cap, cudaStream_t s);
// dst[i][j] = remap[src[src_row[i]][j]] (kInvalid stays kInvalid) for i < rows, j < width.
cudaError_t launch_compact_remap_rows(const uint32_t* src, const uint32_t* src_row, uint64_t rows, uint32_t width,
                                      const uint32_t* remap, uint32_t* dst, cudaStream_t s);
// flag[i] = 1 for a node of the renumbered level-0 graph that must be re-linked: an empty row, or level-0
// in-links before compaction (indeg_old[inv[i]] > 0) and none after.
cudaError_t launch_compact_orphans(const uint32_t* links0, uint64_t n, uint32_t M0, const uint32_t* inv,
                                   const uint32_t* indeg_old, uint32_t* indeg_new, uint8_t* flag, cudaStream_t s);
// Moves vector rows inv[i] -> i for i in [lo, n) in place, through `stage` (stage_rows rows).  Safe because
// inv[i] >= i and the chunks go in increasing i.
cudaError_t launch_compact_move_rows(float* vecs, uint32_t dpad, const uint32_t* inv, uint64_t lo, uint64_t n,
                                     float* stage, uint64_t stage_rows, cudaStream_t s);

// K7 — queries that are stored points (bylabel.cu).
// out[dst ? dst[j] : j][0:dim] = in[src ? src[j] : j][0:dim] for j < n (row strides in floats): the stored rows of
// labels as queries, and the scatter of gathered rows to their query positions on a sharded index.
cudaError_t launch_gather_rows(const float* in, uint32_t in_stride, const uint32_t* src, float* out,
                               uint32_t out_stride, const uint32_t* dst, uint64_t n, uint32_t dim, cudaStream_t s);
// Self-removal of the reference's key mode (server.cc:190-207): from [nq][k + 1] results (nearest-first, counts
// in_counts) to [nq][k]: query q's own label self[q] is removed when present among its hits, else the last hit is
// dropped when there are k + 1; rows are padded with EHB_NO_LABEL / +inf.
cudaError_t launch_drop_self(const uint64_t* self, const uint64_t* in_labels, const float* in_dists,
                             const uint32_t* in_counts, uint64_t nq, uint32_t k, uint64_t* out_labels,
                             float* out_dists, uint32_t* out_counts, cudaStream_t s);
// Loads drop_self_kernel now rather than at its first launch: with lazy module loading a first launch can wait for
// the kernels already running in the context, and in a key-mode exchange step one of those may be a peer's merge
// that waits for this rank (ehb_exchange_create_ex).
cudaError_t load_drop_self();
// The ids i < n with deleted[i] == 0, ascending, into ids[0..*count).
cudaError_t launch_live_ids(const uint8_t* deleted, uint64_t n, uint32_t* ids, uint32_t* count, cudaStream_t s);

}  // namespace ehb
