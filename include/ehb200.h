/* ehb200 — C ABI of the H100-native ANN backend for embeddinghub.
 *
 * This is the drop-in boundary (SURVEY.md §8b, B4): everything the reference's
 * hnswlib-backed ANNIndex does for the k-NN hot path, as plain C entry points a
 * cgo / ctypes / C++ caller can bind.  Each entry point names the reference
 * interface it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - every function returns an ehb_status (0 = OK); no exceptions cross the ABI;
 *     ehb_last_error() returns a thread-local message for the last failure.
 *   - the caller owns every buffer; vectors are row-major contiguous fp32.
 *   - "host" entry points take host pointers and do the H2D/D2H copies
 *     themselves (what a Go slice / std::vector caller binds);  "_dev" entry
 *     points take device pointers + a cudaStream_t (passed as void*) and never
 *     synchronise, for callers that keep queries/results resident in HBM.
 *   - results are nearest-first; rows with fewer than k hits are padded with
 *     EHB_NO_LABEL / +inf and the true count is written to out_counts.
 *   - searches are re-entrant: several host threads may search one index at the
 *     same time (each in-flight search has its own stream and scratch; concurrent
 *     small ehb_index_search calls are coalesced into one batched launch by a
 *     combining queue — the goroutine-per-request pattern of
 *     serving/serving.go:744-771); mutations (add / remove / build / import) are
 *     exclusive.  The reference serialises everything under one service mutex
 *     (embeddinghub/embeddingstore/server.cc:175).
 *   - there is no CPU fallback: every call fails with EHB_ERR_CUDA when no
 *     sm_90 (H100-class) device is usable.
 */
#ifndef EHB200_H
#define EHB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EHB_NO_LABEL UINT64_MAX

typedef enum ehb_status {
  EHB_OK = 0,
  EHB_ERR_INVALID = 1,   /* bad argument                                      */
  EHB_ERR_CUDA = 2,      /* CUDA runtime / launch failure, or no device        */
  EHB_ERR_OOM = 3,       /* device or host allocation failed                   */
  EHB_ERR_STATE = 4,     /* call not valid in the index's current state        */
  EHB_ERR_NOT_FOUND = 5, /* unknown label                                      */
  EHB_ERR_IO = 6         /* save / load failed                                 */
} ehb_status;

/* Distance "space".  Replaces hnswlib::L2Space (embeddinghub/embeddingstore/
 * index.cc:12-13: squared L2, no sqrt), hnswlib::InnerProductSpace (1 - dot) and
 * hnswlib's cosine convention (normalise on insert and on query, then IP) that
 * the Go providers use (provider/redis.go:253, provider/pinecone.go:252). */
typedef enum ehb_metric { EHB_L2 = 0, EHB_IP = 1, EHB_COSINE = 2 } ehb_metric;

typedef enum ehb_precision { EHB_FP32 = 0, EHB_BF16 = 1 } ehb_precision;

typedef struct ehb_index ehb_index; /* opaque */

/* Construction parameters.  Zero-initialise, then set what you need;
 * ehb_params_default() fills the reference's implicit hnswlib defaults
 * (index.cc:14-15: M=16, ef_construction=200, random_seed=100; ef=10 because the
 * reference never calls setEf; init capacity 128, index.h:21). */
typedef struct ehb_params {
  uint32_t dim;             /* 1..4096 (ehb_index_create: EHB_ERR_INVALID above)  */
  int32_t metric;           /* ehb_metric                                      */
  uint64_t capacity;        /* initial capacity in vectors; grows by doubling  */
  uint32_t M;               /* 2..16 (level-0 rows hold 2*M ids)               */
  uint32_t ef_construction; /* 0 (= 200) .. 4096, EHB_ERR_INVALID above; the
                               build searches at max(ef_construction, M)      */
  uint32_t ef_search;       /* default ef of searches (hnswlib ef_)            */
  uint64_t seed;            /* level generator seed                            */
  int32_t device;           /* CUDA device ordinal                             */
  uint32_t build_batch;     /* max points linked per build wave (0 = default)  */
  uint32_t reserved[6];
} ehb_params;

typedef struct ehb_stats {
  /* counters of the most recent graph search (hnswlib metric_hops /
   * metric_distance_computations semantics: one hop per expanded node, one eval
   * per unvisited neighbour + 1 for the entry point) */
  uint64_t queries;
  uint64_t hops_upper;
  uint64_t hops_base;
  uint64_t dist_evals;
  uint64_t visited_overflow; /* queries whose visited table filled up          */
  /* fp32 search: hops_upper*4M + hops_base*8M + fp32_rows*4d + screened*(d+16) + Q*4d, where screened = the
   * evaluations the walk's int8 screen made and fp32_rows = evals - screened + the screen's survivors (both from
   * ehb_index_screen_stats; an unscreened walk has screened = 0 and fp32_rows = evals);
   * bf16 search: hops_upper*4M + hops_base*8M + evals*2d + Q*4d + reranked*4d, reranked = the keys the walk
   * retained and the fp32 re-rank read (min(max(ef, k), reachable live points) per query) */
  uint64_t algorithmic_bytes;
  /* index shape */
  uint64_t size, capacity, upper_rows;
  uint32_t dim, M, max_level, entry_point;
  uint64_t device_bytes;      /* every device array of the index, the bf16 and int8 copies of its rows included */
  uint64_t deleted;           /* tombstones (ehb_index_remove); `size` counts them, like hnswlib   */
  uint64_t combined_batches;  /* batched launches issued by the combining queue of ehb_index_search */
  uint64_t combined_queries;  /* queries those launches carried                                     */
  uint32_t metric;            /* ehb_metric of the index                                            */
  uint32_t reserved_;
} ehb_stats;

const char* ehb_last_error(void);
uint32_t ehb_abi_version(void);

void ehb_params_default(ehb_params* p, uint32_t dim);
/* Number of usable CUDA devices (what a caller sizes device_ids[] from); EHB_ERR_CUDA when there is none. */
int ehb_device_count(int32_t* out);

/* ANNIndex::ANNIndex(dims, init_cap) — index.cc:10-18 (allocates the hnswlib
 * arena); here: device arrays for vectors, labels, levels and adjacency.  dim 1..4096: rows are padded to
 * 32 ... 2048, 3072 or 4096 floats; above 2048 the graph walk and build run their wide form (DESIGN.md §4). */
int ehb_index_create(const ehb_params* p, ehb_index** out);
int ehb_index_destroy(ehb_index* ix);

/* ANNIndex::set -> hnswlib addPoint / resizeIndex — index.cc:20-37.  Insert or
 * update-in-place (existing label).  labels == NULL assigns labels
 * s..s+n-1 with s = size() + the number of points removed by ehb_index_compact
 * so far (= size() on an index that was never compacted).  Points are linked into the graph lazily by the next
 * ehb_index_build / search (batched GPU construction replaces the reference's
 * one-addPoint-per-row loop, version.cc:64-74). */
int ehb_index_add(ehb_index* ix, uint64_t n, const float* vecs_host, const uint64_t* labels_host);
int ehb_index_add_dev(ehb_index* ix, uint64_t n, const float* vecs_dev, const uint64_t* labels_host);
int ehb_index_build(ehb_index* ix);

/* Delete (embeddinghub/docs/reading_and_writing_embeddings.md:49-66 promises delete / multidelete; hnswlib
 * markDelete semantics): the points stay in the graph as tombstones — traversed by searches, never returned,
 * ehb_index_get answers EHB_ERR_NOT_FOUND, size() still counts them.  Unknown label: EHB_ERR_NOT_FOUND;
 * already deleted: EHB_ERR_STATE.  Adding a deleted label again un-deletes it and updates it in place
 * (hnswlib addPoint). */
int ehb_index_remove(ehb_index* ix, uint64_t n, const uint64_t* labels_host);

/* Compaction: removes every tombstone for good.  Pending points are linked first (like ehb_index_save).  Rows
 * of live points that named deleted points are re-selected on the GPU over their live neighbours and the live
 * neighbours of those deleted points (hnswlib's updatePoint selection); the survivors are renumbered densely
 * in insertion order, and survivors left without level-0 in-links (or with an empty row) are re-linked by
 * updatePoint.  If the entry point was deleted, the live point of highest level (smallest internal id on a
 * tie) becomes the entry point.  Afterwards size() counts the survivors only, labels and vectors are kept,
 * internal ids (ehb_index_export_graph) change, capacity is kept (later adds reuse the freed rows) and the
 * tombstone-free search paths apply again.  Deleting everything and compacting gives an empty index.
 * Searches in flight finish first; later ones see the compacted graph.  No deletes: no change.
 * The number of points removed so far is kept (automatic labels, level draws) and saved by ehb_index_save;
 * ehb_index_export_graph / ehb_index_import_graph do not carry it, so an imported index counts from 0. */
int ehb_index_compact(ehb_index* ix);

/* hnswlib setEf (never called by the reference; named by BASELINE configs). */
int ehb_index_set_ef(ehb_index* ix, uint32_t ef);
int ehb_index_size(ehb_index* ix, uint64_t* out);

/* Version::get of the stored vector (version.cc / storage.cc:32-36 serve this
 * from RocksDB; the index keeps the fp32 rows resident so Get needs no KV). */
int ehb_index_get(ehb_index* ix, uint64_t label, float* out_vec_host);

/* ANNIndex::approx_nearest -> hnswlib searchKnn — index.cc:39-52, batched over
 * nq queries.  ef == 0 uses the index default; the walk runs with max(ef, k) like
 * searchKnn.  out_dists / out_counts may be NULL. */
int ehb_index_search(ehb_index* ix, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef,
                     uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_index_search_dev(ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k, uint32_t ef,
                         uint64_t* out_labels_dev, float* out_dists_dev, uint32_t* out_counts_dev, void* stream);
/* The same search at a chosen precision; ehb_index_search(_dev) is exactly the _ex form with EHB_FP32, and an
 * unknown precision fails with EHB_ERR_INVALID.  EHB_BF16 walks the same graph with hnswlib's searchKnn order and
 * stop rule, but evaluates every distance between the fp32 query and the bf16 copy of the row (widened to fp32,
 * fp32 accumulation); the walk keeps its whole result set (max(ef, k) entries), which is re-ranked with the
 * exact path's canonical fp32 arithmetic over the fp32 rows.  So every returned distance is bit-identical to the
 * exact distance of that id, ties go by internal id, and only the set the walk retains can differ from the fp32
 * walk's.  It always runs one warp per query (the multi-warp team walk reads fp32 rows only).  Tombstones,
 * padding, counts and cosine normalisation behave as in the fp32 search.  The first bf16 search (graph or brute
 * force) creates the index's bf16 copy of its rows (2 * dim-padded bytes per vector), which every later add,
 * update and compaction keeps current; an index that never runs one allocates none of it.
 * ehb_index_last_kernel_ms covers the walk and the re-rank. */
int ehb_index_search_ex(ehb_index* ix, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef, int precision,
                        uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_index_search_ex_dev(ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k, uint32_t ef,
                            int precision, uint64_t* out_labels_dev, float* out_dists_dev, uint32_t* out_counts_dev,
                            void* stream);

/* hnswlib BruteforceSearch (not used by the reference; the exact path named by
 * the north star).  EHB_FP32 is exact with a defined total order (distance asc,
 * insertion index asc) and canonical arithmetic (one fp32 FMA chain, k
 * ascending) so ids are reproducible bit-for-bit.  EHB_BF16 is the tensor-core
 * path (bf16 GEMM + fp32 re-rank of an oversampled candidate set).  An unknown
 * precision fails with EHB_ERR_INVALID whatever k and nq are, as in the graph
 * search, and so does ehb_sharded_search_bruteforce. */
int ehb_index_search_bruteforce(ehb_index* ix, uint64_t nq, const float* queries_host, uint32_t k, int precision,
                                uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_index_search_bruteforce_dev(ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k, int precision,
                                    uint64_t* out_labels_dev, float* out_dists_dev, uint32_t* out_counts_dev,
                                    void* stream);

/* Batched Version::get: the stored rows of n labels into out_vecs_host ([n][dim]), each exactly as
 * ehb_index_get returns it (for cosine: the normalised row).  One gather kernel and one copy instead of n
 * synchronous reads.  An unknown or tombstoned label fails with EHB_ERR_NOT_FOUND and nothing is written. */
int ehb_index_get_batch(ehb_index* ix, uint64_t n, const uint64_t* labels_host, float* out_vecs_host);

/* Key mode of the reference's NearestNeighbor (embeddinghub/embeddingstore/server.cc:190-207, also
 * serving/offlinehub.py:110-130): the neighbours of points already stored, named by label.  For each label L the
 * stored row (as ehb_index_get returns it) is the query, prepared like any host query (cosine normalises it
 * again), and searched at k + 1 with the given ef and precision, taking the walk an ehb_index_search_ex of the same
 * nq would take.  From that list R of c hits, nearest-first: if L is in R it is removed; otherwise, if c > k, the
 * last hit is dropped.  The first k remaining entries are written, padded with EHB_NO_LABEL / +inf, and the count
 * is min(c', k).  Labels, distance bits and counts equal the host composition ehb_index_get of every label ->
 * ehb_index_search_ex(rows, k + 1, ef, precision) -> that rule; the queries never leave the device.
 * Checked before anything is written: a null pointer or max(ef, k + 1) > 512 fails with EHB_ERR_INVALID, an
 * unknown or tombstoned label with EHB_ERR_NOT_FOUND.  nq == 0 or k == 0 writes nothing.  The call does not go
 * through the combining queue; ehb_index_last_kernel_ms / _name and ehb_index_stats describe its walk.
 * out_dists / out_counts may be NULL. */
int ehb_index_search_by_label_ex(ehb_index* ix, uint64_t nq, const uint64_t* labels_host, uint32_t k, uint32_t ef,
                                 int precision, uint64_t* out_labels_host, float* out_dists_host,
                                 uint32_t* out_counts_host);
/* Graph search with a beam above 512 (hnswlib searchKnn with num in the hundreds or thousands).
 * - Checks, in the order of every other search: an unknown precision, then a null query / label or out_labels
 *   pointer fail with EHB_ERR_INVALID; then k == 0 or nq == 0 writes nothing and returns EHB_OK; then
 *   max(ef, k_walk) > EHB_MAX_BEAM fails with EHB_ERR_INVALID (k_walk: k, or k + 1 by label; ef == 0: the index
 *   default, which ehb_index_set_ef may set above 512).  By label, an unknown or tombstoned label then fails with
 *   EHB_ERR_NOT_FOUND.  A rejected call leaves every output buffer untouched.
 * - Up to max(ef, k_walk) == 512 each call is exactly ehb_index_search_ex(_dev) / ehb_index_search_by_label_ex:
 *   the same kernel, results and counters.
 * - Above 512 the wide-beam walk runs (hnsw_search_beam_kernel): hnswlib's searchKnn order and stop rule with beam
 *   max(ef, k), one warp per query, its result set in shared memory and its visited table (2 * M0 * beam + 64
 *   entries per walking warp) in device memory.  Labels, distance bits, counts and the hop / evaluation counters
 *   equal hnswlib's on the same graph as long as the visited table does not overflow, as for the other walks.
 *   Tombstones, padding with EHB_NO_LABEL / +inf, cosine normalisation and EHB_BF16 (walk the bf16 copy, re-rank
 *   the whole retained set in fp32) behave as in ehb_index_search_ex; by label is the same k + 1 search followed
 *   by the rule of ehb_index_search_by_label_ex.  The scratch (visited tables of the resident warps; at EHB_BF16
 *   also nq * beam 8-byte keys) belongs to the index: it grows on demand, is freed with the index, and one
 *   wide-beam search at a time uses it (the next waits for it on the device).  An allocation that fails returns
 *   EHB_ERR_OOM before anything is written.
 * - These calls do not go through the combining queue.  ehb_index_stats, ehb_index_last_kernel_ms and
 *   ehb_index_last_kernel_name describe the walk; the kernel name is
 *   hnsw_search_beam_kernel<LPV=..,NQ=..[,HASDEL=1][,ROW=bf16]>.
 * out_dists / out_counts may be NULL. */
#define EHB_MAX_BEAM 4096
int ehb_index_search_beam(ehb_index* ix, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef,
                          int precision, uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_index_search_beam_dev(ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k, uint32_t ef,
                              int precision, uint64_t* out_labels_dev, float* out_dists_dev, uint32_t* out_counts_dev,
                              void* stream);
int ehb_index_search_by_label_beam(ehb_index* ix, uint64_t nq, const uint64_t* labels_host, uint32_t k, uint32_t ef,
                                   int precision, uint64_t* out_labels_host, float* out_dists_host,
                                   uint32_t* out_counts_host);

/* The same rule over ehb_index_search_bruteforce(rows, k + 1, precision); k + 1 must be <= 2048. */
int ehb_index_search_bruteforce_by_label(ehb_index* ix, uint64_t nq, const uint64_t* labels_host, uint32_t k,
                                         int precision, uint64_t* out_labels_host, float* out_dists_host,
                                         uint32_t* out_counts_host);
/* Every live point's k nearest other points: ehb_index_search_by_label_ex (same rule, server.cc:190-207) over
 * all live labels in internal-id order (insertion order, which compaction keeps), in consecutive chunks of
 * "table_chunk" points (ehb_index_set_option, default 65536); each chunk's rows are by definition
 * ehb_index_search_by_label_ex of that chunk's labels.  out_query_labels[r] is row r's label.  *out_rows is in / out:
 * on entry the rows the buffers hold (size them for size - deleted rows, ehb_stats), on return the rows written;
 * when the table has more rows, the call fails with EHB_ERR_INVALID, writes nothing else and stores the row count
 * needed in *out_rows.  The call holds the index's reader side
 * throughout, so the table is one consistent snapshot: searches run alongside it, and mutations (add, remove,
 * build, compact) wait until it returns.  Errors as ehb_index_search_by_label_ex; k == 0 writes nothing.
 * out_dists / out_counts may be NULL. */
int ehb_index_neighbor_table(ehb_index* ix, uint32_t k, uint32_t ef, int precision, uint64_t* out_query_labels_host,
                             uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host,
                             uint64_t* out_rows);

int ehb_index_stats(ehb_index* ix, ehb_stats* out);
/* Counters of the fp32 walk's int8 screen in the most recent graph search (option "walk_screen"):
 * screened_evals = distance evaluations made on the int8 copy first (dim code bytes + 16 bytes of per-row terms each), fp32_row_reads = fp32 rows the walk read
 * (evaluations that were not screened plus the screened ones that could still be admitted).  Both count within
 * ehb_stats.dist_evals; a bf16 search reads no fp32 rows in its walk, and 0, 0 is returned before any graph search. */
int ehb_index_screen_stats(ehb_index* ix, uint64_t* screened_evals, uint64_t* fp32_row_reads);

/* Timing of the most recent search on the index's launch stream, measured with
 * CUDA events recorded around the kernel(s): milliseconds of the graph-walk (or
 * brute-force) kernels alone.  Synchronises on those events. */
int ehb_index_last_kernel_ms(ehb_index* ix, float* out_ms);
/* Name (with template arguments) of the graph-walk kernel that search launched. */
int ehb_index_last_kernel_name(ehb_index* ix, char* out, uint32_t out_bytes);

/* Graph exchange (hnswlib saveIndex/loadIndex are never called by the
 * reference; persistence is a "next" row, SURVEY.md §8f-3).  Layout:
 *   levels[n] u8; links0[n][2M] u32 padded with UINT32_MAX; up_off[n] u32 = first
 *   upper row of node i (UINT32_MAX if level 0); links_up[rows][M] u32.
 * import replaces the whole index content (vectors are taken as stored, i.e.
 * already normalised for cosine). */
int ehb_index_export_graph(ehb_index* ix, float* vectors, uint64_t* labels, uint8_t* levels, uint32_t* links0,
                           uint32_t* up_off, uint32_t* links_up, uint32_t* entry, int32_t* max_level);
int ehb_index_import_graph(ehb_index* ix, uint64_t n, const float* vectors, const uint64_t* labels,
                           const uint8_t* levels, const uint32_t* links0, const uint32_t* up_off,
                           uint64_t upper_rows, const uint32_t* links_up, uint32_t entry, int32_t max_level);
int ehb_index_save(ehb_index* ix, const char* path);
int ehb_index_load(const char* path, int32_t device, ehb_index** out);

/* Final merge of G per-shard top-k lists (each [nq][k], nearest-first, padded
 * with EHB_NO_LABEL/+inf) gathered contiguously as [G][nq][k] — the step after
 * the single NCCL all-gather of the range-sharded index (SURVEY.md §8e). */
int ehb_merge_topk_dev(uint32_t G, uint64_t nq, uint32_t k, const float* dists_dev, const uint64_t* labels_dev,
                       float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev, int32_t device,
                       void* stream);

/* Same merge over ONE packed gather buffer: rank g's block starts at packed + g * rank_stride_bytes and
 * holds [nq*k u64 labels | nq*k f32 distances] — what a single all-gather of each rank's packed
 * (labels, distances) result delivers, merged in place without unpacking. */
int ehb_merge_topk_packed_dev(uint32_t G, uint64_t nq, uint32_t k, const void* packed_dev, uint64_t rank_stride_bytes,
                              float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev, int32_t device,
                              void* stream);

/* Warps cooperating on one query: 1 = the exact hnswlib expansion order (one warp
 * per query); 2 or 4 = that many of the closest unexpanded candidates are expanded
 * concurrently per round (recall >= the sequential walk's at the same ef; used when
 * a batch is too small to fill the GPU with one warp per query); 0 = automatic. */
int ehb_index_set_search_width(ehb_index* ix, uint32_t warps_per_query);

/* Search tuning knobs (advanced; 0 = automatic).  stage_slots: vectors staged
 * per TMA group; stage_groups: groups in flight per warp (neither applies to a
 * screened fp32 walk, which has no TMA ring); hash_bits: log2 of the per-warp
 * visited table. */
int ehb_index_set_tuning(ehb_index* ix, uint32_t stage_slots, uint32_t stage_groups, uint32_t hash_bits,
                         uint32_t warps_per_block);

/* ---------------------------------------------------------------------------------------------------
 * Range-sharded index over several GPUs of one box (SURVEY.md §8b B4 "device_ids[], n_dev"; §8e).
 * One process drives n_dev devices: labels [i*span, (i+1)*span) live on shard i % n_dev (span 0: label %
 * n_dev); every shard owns an independent graph; a search runs on every shard, whose kernels store their
 * top-k straight into device_ids[0]'s gather buffer over NVLink (peer access), and one merge kernel there
 * produces the result.  No collective on either path.  Same conventions as the single-index calls; calls on one
 * ehb_sharded handle are serialised (one gather buffer per handle). */
typedef struct ehb_sharded ehb_sharded; /* opaque */
int ehb_sharded_create(const ehb_params* p /* device ignored; capacity per shard */, const int32_t* device_ids,
                       uint32_t n_dev, uint64_t shard_span, ehb_sharded** out);
int ehb_sharded_destroy(ehb_sharded* sh);
int ehb_sharded_n_shards(ehb_sharded* sh, uint32_t* out);
int ehb_sharded_shard(ehb_sharded* sh, uint32_t i, ehb_index** out /* borrowed */);
int ehb_sharded_add(ehb_sharded* sh, uint64_t n, const float* vecs_host, const uint64_t* labels_host);
int ehb_sharded_remove(ehb_sharded* sh, uint64_t n, const uint64_t* labels_host);
int ehb_sharded_get(ehb_sharded* sh, uint64_t label, float* out_vec_host);
int ehb_sharded_size(ehb_sharded* sh, uint64_t* out);
int ehb_sharded_build(ehb_sharded* sh); /* shards build concurrently */
int ehb_sharded_compact(ehb_sharded* sh); /* ehb_index_compact on every shard, concurrently */
int ehb_sharded_set_ef(ehb_sharded* sh, uint32_t ef);
int ehb_sharded_search(ehb_sharded* sh, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef,
                       uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
/* ehb_index_search_ex on every shard, then the same merge (ehb_sharded_search is the EHB_FP32 form). */
int ehb_sharded_search_ex(ehb_sharded* sh, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef,
                          int precision, uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_sharded_search_bruteforce(ehb_sharded* sh, uint64_t nq, const float* queries_host, uint32_t k, int precision,
                                  uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
/* ehb_index_get_batch routed to each label's shard. */
int ehb_sharded_get_batch(ehb_sharded* sh, uint64_t n, const uint64_t* labels_host, float* out_vecs_host);
/* Key mode (server.cc:190-207, offlinehub.py:110-130) on the sharded index: each label's owning shard copies its
 * row into every shard's query buffer (device-to-device, no round trip through the host), every shard searches at
 * k + 1, the lists are merged on device_ids[0], and the self-removal rule of ehb_index_search_by_label_ex runs
 * there.  Equal to ehb_sharded_get of every label -> ehb_sharded_search_ex(rows, k + 1) -> that rule; errors as
 * ehb_index_search_by_label_ex. */
int ehb_sharded_search_by_label_ex(ehb_sharded* sh, uint64_t nq, const uint64_t* labels_host, uint32_t k, uint32_t ef,
                                   int precision, uint64_t* out_labels_host, float* out_dists_host,
                                   uint32_t* out_counts_host);
/* The sharded searches with a beam above 512: ehb_index_search_beam_dev on every shard, storing into device_ids[0]'s
 * gather buffer, then the same merge; by label, the same row staging, the k + 1 beam search on every shard, the merge
 * and the self-removal rule.  Checks and their order as ehb_index_search_beam / ehb_index_search_by_label_beam
 * (max(ef, k_walk) > EHB_MAX_BEAM fails with EHB_ERR_INVALID).  Up to max(ef, k_walk) == 512 each call is exactly
 * ehb_sharded_search_ex / ehb_sharded_search_by_label_ex.  Above, the result equals ehb_merge_topk_dev over every
 * shard's own ehb_index_search_beam_dev output (labels, distance bits, counts), followed by label by the rule.  The
 * gather buffer on device_ids[0] is n_dev * nq * k_walk * 12 bytes (10k queries at k = 4096 over 8 shards: 3.9 GB),
 * and each shard grows its own wide-beam scratch as ehb_index_search_beam does. */
int ehb_sharded_search_beam(ehb_sharded* sh, uint64_t nq, const float* queries_host, uint32_t k, uint32_t ef,
                            int precision, uint64_t* out_labels_host, float* out_dists_host, uint32_t* out_counts_host);
int ehb_sharded_search_by_label_beam(ehb_sharded* sh, uint64_t nq, const uint64_t* labels_host, uint32_t k,
                                     uint32_t ef, int precision, uint64_t* out_labels_host, float* out_dists_host,
                                     uint32_t* out_counts_host);

/* Shard exchange for one-process-per-GPU deployments (torchrun / MPI): replaces "one ncclAllGather of the
 * per-shard top-k + merge kernel" (SURVEY.md §8e) with ONE kernel per rank that pushes this rank's lists
 * into every peer's receive buffer with stores over NVLink (CUDA IPC mappings), flags them per slice and
 * merges each slice as soon as all peers' flags are up.  Protocol per rank:
 *   create -> ipc_handle -> (exchange the 64-byte handles out of band, e.g. one torch.distributed
 *   all_gather at start-up) -> open;  then per step, in lock step on every rank:
 *   begin(nq, k) -> run the local search with the returned output pointers -> merge_dev(stream). */
#define EHB_IPC_HANDLE_BYTES 64
typedef struct ehb_exchange ehb_exchange; /* opaque */
int ehb_exchange_create(int32_t device, uint32_t world, uint32_t rank, uint64_t max_nq, uint32_t max_k,
                        ehb_exchange** out);
/* ehb_exchange_create is exactly this with max_dim = 0.  max_dim > 0 (at most 4096) also makes room for key-mode
 * steps (ehb_exchange_search_by_label_ex_dev) over indexes of dim <= max_dim: in the exported block, after the
 * receive buffer, a row region of two parts of max_nq * max_dim fp32 each (rounded up to 64 floats), a mark array [2][world][max_nq] bytes and [2][world] 64-bit
 * digests; on this rank only, scratch for one step (the ids and labels of max_nq queries, max_nq * max_k merged
 * entries, a verdict word) and pinned host staging.  Everything is allocated here; no step allocates or frees.
 * Every rank creates its exchange with the same world, max_nq, max_k and max_dim (ehb_exchange_attach_local fails
 * with EHB_ERR_INVALID when the max_dim differ). */
int ehb_exchange_create_ex(int32_t device, uint32_t world, uint32_t rank, uint64_t max_nq, uint32_t max_k,
                           uint32_t max_dim, ehb_exchange** out);
int ehb_exchange_destroy(ehb_exchange* ex);
int ehb_exchange_ipc_handle(ehb_exchange* ex, void* out_handle /* EHB_IPC_HANDLE_BYTES */);
int ehb_exchange_open(ehb_exchange* ex, const void* handles /* [world][EHB_IPC_HANDLE_BYTES], rank order */);
int ehb_exchange_attach_local(ehb_exchange* ex, uint32_t peer_rank, ehb_exchange* peer /* same process */);
int ehb_exchange_begin(ehb_exchange* ex, uint64_t nq, uint32_t k, uint64_t** labels_dev, float** dists_dev);
int ehb_exchange_merge_dev(ehb_exchange* ex, float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev,
                           void* stream);
/* The fused step for graph searches (replaces begin + ehb_index_search_ex_dev + merge_dev): the search's last
 * kernel stores each query's top-k into every peer's receive buffer (coalesced stores over NVLink, overlapping
 * the rest of the search) and raises per-slice flags; one kernel then waits for the peers' flags and merges.
 * With EHB_FP32 that kernel is the walk itself (a batch small enough for the multi-warp team walk is pushed after
 * it instead); with EHB_BF16 it is the fp32 re-rank that follows the bf16 walk, so every rank's results are those
 * of ehb_index_search_ex_dev at EHB_BF16, merged.  The first EHB_BF16 step creates the index's bf16 copy of its
 * rows, as any first bf16 search does.  shard_counts_dev ([nq], this shard's hit counts) may be NULL.  An unknown
 * precision, a null pointer, nq * k above the capacity and max(ef, k) > 512 fail before the step starts, so the
 * next step still pairs with the peers' (call it on every rank, so every rank fails the same way).  These are
 * checked as in any search (precision, then max(ef, k)) before the exchange's own state, so a call that is both too
 * wide and made before the peers are attached fails with EHB_ERR_INVALID, not EHB_ERR_STATE.
 * ehb_exchange_search_dev is exactly the _ex form with EHB_FP32. */
int ehb_exchange_search_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                            uint32_t ef, float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev,
                            uint32_t* shard_counts_dev, void* stream);
int ehb_exchange_search_ex_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                               uint32_t ef, int precision, float* out_dists_dev, uint64_t* out_labels_dev,
                               uint32_t* out_counts_dev, uint32_t* shard_counts_dev, void* stream);
/* Key mode (server.cc:190-207, offlinehub.py:110-130) over the exchange: every rank passes the same nq labels, each
 * stored on exactly one rank, and every rank receives [nq][k] results.  They equal ehb_exchange_search_ex_dev(rows,
 * k + 1, ef, precision) followed by the self-removal rule of ehb_index_search_by_label_ex, where rows[q] is label q's
 * stored row as ehb_index_get returns it on the rank that holds it (cosine rows are normalised again, like any query).
 * A step takes two epochs.  At the first, one kernel per rank copies the rows of the labels this rank holds (a
 * tombstoned label is not held) from its index straight into row q of every rank's row region, writes which queries
 * it holds and a digest of its label list into every rank, raises per-slice flags, waits for the peers' flags and
 * counts each query's holders.  Then ONE 4-byte copy to the host and a synchronisation of `stream`: the call's only
 * host synchronisation.  Every rank has read the same digests and, when those agree, the same marks, so every rank
 * then returns the same status:
 *   EHB_ERR_INVALID    the ranks were given different label lists (of any lengths);
 *   EHB_ERR_NOT_FOUND  otherwise, some label is held by no rank (unknown or tombstoned everywhere);
 *   EHB_ERR_STATE      otherwise, some label is held by more than one rank;
 * and nothing is written; each rank has consumed the first epoch, so the next step still pairs with the peers'.
 * Otherwise the fused k + 1 step runs at the second epoch with this rank's row region as its queries (the walk
 * ehb_exchange_search_ex_dev would take for nq queries), the merge writes into the exchange's scratch, and the
 * self-removal writes the caller's buffers, all queued on `stream` without further synchronisation.
 * Checked before the first epoch, as in the fused step (call it on every rank, so every rank fails the same way):
 * an unknown precision, a null pointer (all three outputs are required), max(ef, k + 1) > 512, nq > max_nq,
 * nq * (k + 1) > max_nq * max_k and an index dim above max_dim (so an exchange created with max_dim = 0) fail with
 * EHB_ERR_INVALID, and a call before the peers are attached with EHB_ERR_STATE.  nq == 0 or k == 0 writes nothing
 * and does not advance the epoch.  A wait that gives up (ehb_exchange_timed_out) fails with EHB_ERR_CUDA. */
int ehb_exchange_search_by_label_ex_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const uint64_t* labels_host,
                                        uint32_t k, uint32_t ef, int precision, float* out_dists_dev,
                                        uint64_t* out_labels_dev, uint32_t* out_counts_dev, void* stream);
/* The exchange steps with a beam above 512 (same arguments as the _ex forms).
 * - ehb_exchange_search_beam_dev is the fused step with each rank's search being ehb_index_search_beam_dev: the
 *   wide-beam walk (or, at EHB_BF16, the re-rank after it) stores each query's top-k into every peer's receive buffer
 *   and raises the slice flags, then the merge (at EHB_BF16 with k_walk > 512 the re-rank writes this rank's block
 *   and the merge kernel pushes it).  ehb_exchange_search_by_label_beam_dev is the row step, then that
 *   fused step at k + 1, the merge and the self-removal rule of ehb_exchange_search_by_label_ex_dev.
 * - Up to max(ef, k_walk) == 512 (k_walk: k, or k + 1 by label) each call is exactly its _ex counterpart: the same
 *   kernels, results and counters.  Above, on every rank the result equals ehb_merge_topk_dev over every rank's own
 *   ehb_index_search_beam_dev output (labels, distance bits, counts), followed by label by the self-removal rule;
 *   shard_counts_dev is this shard's own beam counts.
 * - Checked in the order of every other search, each before the epoch advances and with the output buffers
 *   untouched, so the next step still pairs with the peers': an unknown precision, a null pointer, nq == 0 or
 *   k == 0 (as in the _ex form: the fused step fails with EHB_ERR_INVALID, by label writes nothing), max(ef, k_walk)
 *   > EHB_MAX_BEAM, nq * k_walk above max_nq * max_k (and by label nq > max_nq), by label an index dim above max_dim,
 *   then the peers not attached (EHB_ERR_STATE).
 * - The index's wide-beam scratch (ehb_index_search_beam) is grown for this nq and beam before the epoch advances,
 *   so an allocation failure returns EHB_ERR_OOM with this rank still in phase.  OOM is local to the rank: the
 *   peers' merges of that step still wait for it and time out (ehb_exchange_timed_out).  A step that grows the
 *   scratch synchronises `stream` and frees the old buffer, which waits for the whole device; on a device shared by
 *   several ranks of one process, size the scratch (one ehb_index_search_beam_dev of the largest nq and beam) before
 *   the first fused step, since that wait would include a peer's merge waiting for this rank.
 * - Memory: the receive buffer is 2 * world * max_nq * max_k * 12 bytes per rank (7.9 GB at world 8, max_nq 10k,
 *   max_k 4096). */
int ehb_exchange_search_beam_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                                 uint32_t ef, int precision, float* out_dists_dev, uint64_t* out_labels_dev,
                                 uint32_t* out_counts_dev, uint32_t* shard_counts_dev, void* stream);
int ehb_exchange_search_by_label_beam_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const uint64_t* labels_host,
                                          uint32_t k, uint32_t ef, int precision, float* out_dists_dev,
                                          uint64_t* out_labels_dev, uint32_t* out_counts_dev, void* stream);
int ehb_exchange_timed_out(ehb_exchange* ex, uint32_t* out /* 1: a wait for a peer gave up (~20 s) */);

/* Named integer options (A/B switches and construction knobs that are not part of
 * the reference's surface).  Unknown names fail with EHB_ERR_INVALID.
 *   "build_frac"    a construction wave links at most size/build_frac points (0 = default 64)
 *   "seq_updates"   up to this many pending moves of existing labels are re-linked one point at a time at a
 *                   build (default 4096, hnswlib's sequential updatePoint); more go in waves of build_batch
 *                   (default 1024)
 *   "bf16_unfused"  bf16 brute force keeps the distance tiles in HBM (A/B of the fused epilogue)
 *   "combine"       1 (default): concurrent host searches of <= 256 queries share batched launches
 *   "table_chunk"   live points per batch of ehb_index_neighbor_table (default 65536, 1..2^31)
 *   "walk_prefetch" 1: L2-prefetch the speculated next hop's vectors (default 0: it also fetches rows the walk
 *                   never evaluates, extra DRAM traffic for a DRAM-bound walk)
 *   "walk_screen"   the fp32 walk's int8 screen, for inner product and cosine with 256 < dim <= 1536: once the
 *                   result set is full, a hop's candidates are first evaluated on a per-row-scaled int8
 *                   copy of their rows with a rigorous error bound, and only those that could still be admitted
 *                   are read in fp32.  Results, counts and the hop / evaluation counters are exactly those of the
 *                   unscreened walk.  -1 (default): on for batches of at least 4 queries per SM; 0: off; 1: on for
 *                   every batch.  The screen needs the int8 copy of the rows (dim-padded + 16 bytes per vector): a
 *                   search it applies to creates it when it fits in free device memory, else the walk runs
 *                   unscreened.
 * ABI change with the sm_90a build: "gemm_2cta" (a two-SM cta_group::2 form of the bf16 GEMM that only
 * Blackwell has) is no longer accepted and fails with EHB_ERR_INVALID like any unknown name. */
int ehb_index_set_option(ehb_index* ix, const char* name, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* EHB200_H */
