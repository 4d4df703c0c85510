// Internal state of an ehb_index (shared by api.cu, io.cu and exchange.cu).  Mirrors the
// responsibilities of featureform::embedding::ANNIndex + hnswlib::HierarchicalNSW as used in
// embeddinghub/embeddingstore/index.cc:10-52.
//
// Concurrency (SURVEY.md §8b B4: "searches re-entrant ... mutations exclusive").  The reference
// serialises every RPC under one service mutex (embeddinghub/embeddingstore/server.cc:175); here
//   * `rw` is a reader/writer lock: searches share it, mutations (add / remove / build / compact / import) own
//     it, so a compaction waits for the searches in flight and later searches see the compacted graph;
//   * every in-flight graph search works on a SearchSlot (own stream, own device scratch, own pinned
//     staging) taken from a small pool, so host threads never share scratch;
//   * concurrent small host searches are coalesced into one batched launch by the combining queue
//     (api.cu) — the cgo pattern of serving/serving.go:744-771: one goroutine, one query, per request.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <random>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/ehb200.h"
#include "kernels.h"

namespace ehb {

int fail(int code, const std::string& msg);  // sets the thread-local error text, returns code
const std::string& last_error_text();
extern thread_local std::string g_err;

#define CU(expr)                                                                                         \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess)                                                                               \
      return ehb::fail(_e == cudaErrorMemoryAllocation ? EHB_ERR_OOM : EHB_ERR_CUDA,                     \
                       std::string(#expr) + ": " + cudaGetErrorString(_e));                              \
  } while (0)
#define RET(expr)                \
  do {                           \
    int _r = (expr);             \
    if (_r != EHB_OK) return _r; \
  } while (0)

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  // grow to >= want elements, preserving the first `keep` elements; fill new tail with byte `fill` if fill >= 0
  cudaError_t grow(size_t want, size_t keep, int fill, cudaStream_t s) {
    if (want <= n) return cudaSuccess;
    T* np = nullptr;
    cudaError_t e = cudaMalloc(&np, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (keep && p) e = cudaMemcpyAsync(np, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess && fill >= 0) e = cudaMemsetAsync(np + keep, fill, (want - keep) * sizeof(T), s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
      cudaFree(np);  // the old buffer stays valid
      return e;
    }
    if (p) cudaFree(p);
    p = np;
    n = want;
    return cudaSuccess;
  }
  size_t bytes() const { return n * sizeof(T); }
};

// page-locked host staging
struct PinBuf {
  unsigned char* p = nullptr;
  size_t n = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() {
    if (p) cudaFreeHost(p);
  }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= n) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
    size_t want = std::max<size_t>(bytes, 4096);
    cudaError_t e = cudaMallocHost((void**)&p, want);
    if (e == cudaSuccess) n = want;
    return e;
  }
};

// Reader/writer lock that prefers writers: once a mutation waits, new searches queue behind it, so a stream
// of overlapping searches can never starve an add (glibc's rwlock, which std::shared_mutex wraps, prefers
// readers by default).  Meets the SharedMutex requirements used by std::shared_lock / std::unique_lock.
class RwLock {
 public:
  void lock() {
    std::unique_lock<std::mutex> g(mu_);
    ++writers_waiting_;
    cv_.wait(g, [&] { return !writer_ && readers_ == 0; });
    --writers_waiting_;
    writer_ = true;
  }
  void unlock() {
    {
      std::lock_guard<std::mutex> g(mu_);
      writer_ = false;
    }
    cv_.notify_all();
  }
  void lock_shared() {
    std::unique_lock<std::mutex> g(mu_);
    cv_.wait(g, [&] { return !writer_ && writers_waiting_ == 0; });
    ++readers_;
  }
  void unlock_shared() {
    bool wake;
    {
      std::lock_guard<std::mutex> g(mu_);
      wake = --readers_ == 0;
    }
    if (wake) cv_.notify_all();
  }

 private:
  std::mutex mu_;
  std::condition_variable cv_;
  uint32_t readers_ = 0, writers_waiting_ = 0;
  bool writer_ = false;
};

// Everything one in-flight graph search needs.
struct SearchSlot {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, busy = nullptr;
  bool busy_valid = false;
  DevBuf<float> q_in, q_norm, o_dists;
  DevBuf<uint64_t> o_labels;
  DevBuf<uint32_t> o_counts, stats;
  DevBuf<float> q_pad;          // bf16 graph search: padded (cosine: normalised) queries for the fp32 re-rank
  DevBuf<uint64_t> walk_keys;   // bf16 graph search: [nq][ef] retained keys of the walk
  DevBuf<uint32_t> walk_counts; // bf16 graph search: [nq] retained count (the keys re-ranked)
  bool last_bf16 = false;       // the most recent search on this slot walked the bf16 shadow
  DevBuf<unsigned long long> stat_sum;
  // by-label searches (bylabel.cu): the queries' internal ids and labels, and the results after self-removal
  DevBuf<uint32_t> q_ids;
  DevBuf<uint64_t> q_labels;
  DevBuf<uint64_t> s_labels;
  DevBuf<float> s_dists;
  DevBuf<uint32_t> s_counts;
  PinBuf h_q, h_l, h_d, h_c;
  uint64_t last_nq = 0;
  char last_kernel[96] = {0};  // name of the graph-walk kernel of the most recent search on this slot
  ~SearchSlot() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (busy) cudaEventDestroy(busy);
    if (stream) cudaStreamDestroy(stream);
  }
};

// One pending host search in the combining queue.
struct CombineReq {
  const float* q;
  uint64_t nq;
  uint32_t k, ef;
  int precision;
  uint64_t* ol;
  float* od;
  uint32_t* oc;
  int rc = EHB_OK;
  std::string err;
  bool taken = false, done = false;
};

constexpr uint32_t kMaxSlots = 4;          // graph searches in flight per index
constexpr uint32_t kCombineMaxCall = 256;  // host searches up to this many queries go through the combining queue
constexpr uint32_t kCombineMaxBatch = 8192;
constexpr uint32_t kCombineLeaders = 2;    // batches in flight (copies of one overlap the walk of the other)
constexpr uint32_t kDeletedQueue = 64;     // side queue of tombstoned candidates per walking warp
constexpr uint32_t kScreenMinBatchPerSm = 4;  // default fp32 walk screen: batches of >= 4 queries per SM
static_assert(EHB_MAX_BEAM == kMaxBeam, "the header's beam limit is the wide-beam walk's");

class SlotLease;

// The checks every search entry point makes before it touches the index, in this order: the precision, the buffers
// (null_buf: the entry point found a pointer it needs null), then k == 0 or nq == 0, which sets *none (the call does
// nothing and returns EHB_OK), then the width: max(*ef, k_walk) <= max_beam for the graph walk (512, or kMaxBeam on the
// wide-beam entry points); k_walk <= 2048 and, at bf16, a dim padded to whole 64-wide blocks for the brute force.  k_walk is k + 1 for the by-label searches, k otherwise.
// ef (graph walk; nullptr for the brute force): in, the requested beam, 0 for the index default; out, the beam that was
// checked, which the search must use: the default can change while ensure_built drops the lock.  Caller holds the
// reader side of ix->rw.
int check_request(const ehb_index* ix, bool brute, int precision, bool null_buf, uint64_t nq, uint32_t k,
                  uint64_t k_walk, uint32_t* ef, bool* none, uint32_t max_beam = kMaxEf);
// Queues the copies of nq result rows of k to the host on s: labels, and dists / counts where the host asked for them.
int copy_results(uint64_t nq, uint32_t k, const uint64_t* dl, const float* dd, const uint32_t* dc, uint64_t* ol,
                 float* od, uint32_t* oc, cudaStream_t s);

}  // namespace ehb

// ehb_index_search_dev with a result sink (exchange.cu)
int ehb_index_search_dev_sink(ehb_index* ix, uint64_t nq, const float* dq, uint32_t k, uint32_t ef, int precision,
                              const ehb::ResultSink* sink, uint32_t* dc, cudaStream_t stream, bool* pushed);
// The same for a caller that already holds the reader side of ix->rw as `lk` (a second shared acquire would deadlock
// behind a queued writer) and has made the device current.  max_beam: the width limit of ehb::check_request (512, or
// kMaxBeam for the wide-beam exchange steps)
int ehb_index_search_dev_sink_held(ehb_index* ix, std::shared_lock<ehb::RwLock>& lk, uint64_t nq, const float* dq,
                                   uint32_t k, uint32_t ef, int precision, const ehb::ResultSink* sink, uint32_t* dc,
                                   cudaStream_t stream, bool* pushed, uint32_t max_beam = ehb::kMaxEf);
// The stored rows of n live labels into rows_dev ([n][dim] on the index's device), queued on `stream`; an unknown or
// tombstoned label fails with EHB_ERR_NOT_FOUND before anything is queued (exchange.cu: by-label sharded searches)
int ehb_index_gather_dev(ehb_index* ix, uint64_t n, const uint64_t* labels_host, float* rows_dev, cudaStream_t stream);

struct ehb_index {
  ehb_params prm;
  uint32_t dim, dpad, M, M0;
  int metric;
  int device;
  int sms = 132;
  cudaStream_t stream = nullptr;  // mutation / construction / brute-force stream
  cudaEvent_t bf_ev0 = nullptr, bf_ev1 = nullptr;
  ehb::RwLock rw;

  uint64_t cap = 0;        // vector capacity
  uint64_t n = 0;          // stored vectors (tombstones included, like hnswlib cur_element_count)
  uint64_t n_linked = 0;   // vectors linked into the graph
  uint64_t up_rows = 0;    // used upper rows
  uint64_t n_deleted = 0;  // tombstones
  // points removed by compact() so far: automatic labels continue at n + n_removed, and the level generator has
  // made n + n_removed draws (saved in the file header so a loaded index continues both sequences)
  uint64_t n_removed = 0;
  uint32_t entry = 0;
  int32_t max_level = -1;
  uint32_t ef;

  ehb::DevBuf<float> vecs;
  ehb::DevBuf<uint64_t> labels;
  ehb::DevBuf<uint8_t> levels, deleted;
  ehb::DevBuf<uint32_t> links0, up_off, links_up, up_owner;

  std::vector<uint8_t> h_levels, h_deleted;
  std::vector<uint64_t> h_labels;
  bool identity_labels = true;
  std::unordered_map<uint64_t, uint32_t> lookup;
  std::vector<uint32_t> pending_updates;

  // search slots
  std::mutex slot_mu;
  std::condition_variable slot_cv;
  std::vector<std::unique_ptr<ehb::SearchSlot>> slots;
  std::vector<ehb::SearchSlot*> free_slots;
  // what ehb_index_stats / ehb_index_last_kernel_ms report: the most recently issued search
  std::mutex last_mu;
  ehb::SearchSlot* last_slot = nullptr;  // graph search (counters + events)
  bool last_was_brute = false, timed = false;
  unsigned long long last_sum[ehb::kStatWords] = {};
  unsigned long long last_reranked = 0;  // keys the bf16 re-rank read (0 for an fp32 search)
  bool last_sum_valid = false;

  // combining queue of small host searches
  std::mutex cq_mu;
  std::condition_variable cq_cv;
  std::deque<ehb::CombineReq*> cq;
  uint32_t cq_leaders = 0;
  std::atomic<uint64_t> combined_batches{0}, combined_queries{0};

  // brute-force scratch (one brute-force search at a time: bf_mu; a host call stages in a search slot)
  std::mutex bf_mu;
  ehb::DevBuf<float> bf_dist, bf_qpad;
  ehb::DevBuf<uint64_t> bf_part, bf_run;
  ehb::DevBuf<uint16_t> q_bf16;
  ehb::DevBuf<float> q_norm2, bf_thr;
  ehb::DevBuf<uint64_t> bf_cbuf;
  ehb::DevBuf<uint32_t> bf_ccount;
  // wide-beam walk scratch (WalkForm::beam): the persistent grid's visited tables and, at bf16, the [nq][ef] key sink.
  // One wide-beam search at a time owns them (beam_mu); beam_done, recorded after its last kernel, orders the next
  // one's use after it on the device.
  std::mutex beam_mu;
  ehb::DevBuf<uint32_t> beam_vtab;
  ehb::DevBuf<uint64_t> beam_keys;
  cudaEvent_t beam_done = nullptr;
  // Copies derived from the base rows, sized like vecs (capacity rows).  Each is created on the writer side of `rw`
  // by the first search that needs it, and from then on every mutation keeps rows [0, n) equal to a function of
  // vecs under the writer lock: add_rows and compact call derive_rows for the rows they wrote or moved,
  // ensure_capacity grows the copies with vecs, load / import / reset call drop_derived.  An index allocates only the
  // copies its searches used.
  //  - The bf16 shadow ([cap][dpad] bf16 + squared norms of the rounded rows): the bf16 graph walk and the bf16 brute
  //    force.  Created by the first bf16 search.
  //  - The int8 screen copy ([cap][dpad] int8 codes + [cap] per-row terms, launch_to_i8): the fp32 walk's screen.
  //    Created by the first screened search when it fits (try_screen_copy).
  ehb::DevBuf<uint16_t> x_bf16;
  ehb::DevBuf<float> x_norm;
  bool shadow = false;
  ehb::DevBuf<int8_t> x_i8;
  ehb::DevBuf<float4> x_i8t;
  bool screen_copy = false;

  // build scratch
  ehb::DevBuf<uint32_t> b_edge_row, b_edge_src, b_row_cnt, b_row_fill, b_row_start, b_touched, b_seg_src, b_counters,
      b_ids, b_upd_cand, b_side_row, b_side_out;
  ehb::DevBuf<float> b_edge_dist, b_seg_dist, b_stage_in;
  // the wide construction form's visited tables (ef_construction > 256): one HBM slice per resident warp of its
  // persistent grid (reserve_build_beam)
  ehb::DevBuf<uint32_t> b_vtab;

  // tuning (0 = auto)
  uint32_t t_slots = 0, t_groups = 0, t_hash_bits = 0, t_wpb = 0, t_team = 0;
  // options (ehb_index_set_option)
  uint32_t o_build_frac = 0;     // a wave links at most n_linked / build_frac points (0 = 64)
  uint64_t o_seq_updates = 4096; // up to this many pending moves are re-linked one point per wave
  bool o_bf16_unfused = false;   // bf16 brute force: keep the distance tiles in HBM (A/B)
  bool o_combine = true;         // coalesce concurrent small host searches
  // L2 prefetch of the speculated next hop's vectors (rows <= 1 KB).  Off: already-visited neighbours and wrong
  // guesses are fetched too, which adds DRAM traffic to a walk that is bound by DRAM traffic.
  bool o_walk_prefetch = false;
  // fp32 walk screen (walk.cuh beam_search): -1 = automatic (walk_screens), 0 = off, 1 = on for every batch it applies
  // to.  It needs the int8 screen copy; when there was no room for it the walk runs unscreened (screen_no_room,
  // cleared when the option is set again).
  int o_walk_screen = -1;
  bool screen_no_room = false;
  uint64_t o_table_chunk = 65536;  // ehb_index_neighbor_table: live points searched per batch

  std::default_random_engine level_rng;

  ~ehb_index();

  ehb::GraphView view() const;
  // bf16: the walk reads the bf16 shadow (rows of dpad * 2 bytes); screen: a screened fp32 walk (no TMA ring)
  ehb::WalkCfg walk_cfg(uint32_t ef_eff, uint32_t smem_list, uint64_t jobs, uint32_t team, bool bf16 = false,
                        bool dense = false, bool screen = false) const;
  // The wide-beam geometry, shared by the wide-beam walk (walk_plan) and the wide construction form (build_cfg): a
  // beam of ef over a shared-memory key list of smem_list keys, no visited table in shared memory (each warp has
  // beam_vtab_size(ef) entries in HBM) and, with tombstones, a side queue that grows with the beam.
  ehb::WalkCfg beam_cfg(uint32_t ef, uint32_t smem_list, uint64_t jobs, bool bf16 = false) const;
  uint32_t beam_vtab_size(uint32_t ef) const { return ehb::align_up(2u * M0 * ef + 64u, 32); }  // walk_cfg's "roomy"
  uint32_t wpb_for(const ehb::WalkCfg& c, uint32_t extra, bool bf16 = false) const;
  // every choice of the graph-walk kernel for a search of nq queries with beam ef_eff (the shadow exists if bf16)
  ehb::WalkPlan walk_plan(uint64_t nq, uint32_t ef_eff, bool bf16) const;
  int ensure_capacity(uint64_t want);
  int ensure_upper(uint64_t want_rows);
  int draw_level();
  bool find_id(uint64_t label, uint32_t* id) const;
  int add_rows(uint64_t cnt, const float* src, bool src_is_device, const uint64_t* lab);
  int remove_labels(uint64_t cnt, const uint64_t* lab);
  int ensure_build_scratch(uint64_t edges, uint32_t batch, bool updates);
  ehb::BuildBuffers build_buffers(uint64_t edges);
  ehb::BuildGraph build_graph() const;
  // the search configuration of a build launch of `jobs` warps: walk_cfg's register form for efc <= kMaxRegEfc, else
  // the wide form's (launch_build_batch)
  ehb::WalkCfg build_cfg(uint64_t jobs) const;
  // Grows b_vtab for the wide form's persistent grid and describes it in *bm (all zero for efc <= kMaxRegEfc).  Called
  // before the graph is touched, so that running out of memory (EHB_ERR_OOM) leaves the index as it was.
  int reserve_build_beam(ehb::BuildBeam* bm);
  int build();
  int compact();
  bool needs_build() const { return n_linked != n || !pending_updates.empty(); }
  // (re-)take the writer side until the graph is built and, with bf16, the shadow exists
  // screen: the fp32 walk of this batch wants the int8 screen copy (walk_screens); it is created if it fits
  int ensure_built(std::shared_lock<ehb::RwLock>& lk, bool bf16 = false, bool screen = false);
  // whether an fp32 one-warp walk of nq queries screens on the int8 copy (given that the copy exists)
  bool walk_screens(uint64_t nq) const;
  int try_screen_copy();
  int ensure_shadow(std::shared_lock<ehb::RwLock>& lk);
  int create_shadow();
  int derive_rows(uint64_t first, uint64_t cnt);  // re-derive rows [first, first + cnt) of every copy that exists
  void drop_derived();
  // what a search of nq queries needs before it runs: the graph built (walk) and the copies it reads (ensure_built,
  // ensure_shadow)
  int prepare(std::shared_lock<ehb::RwLock>& lk, bool brute, int precision, uint64_t nq);
  // Caller holds the reader lock and has checked the request (ehb::check_request); `sl` is leased on s.  ef is the
  // beam the check resolved and passed (never 0).
  // sink (optional): extra destinations + slice flags for the sharded exchange; *pushed tells whether the
  // launched kernel honoured it (the one-warp walk does, the team walk does not)
  // precision EHB_BF16 walks the bf16 shadow (caller made sure it exists) and re-ranks the retained set in fp32
  int search_dev(ehb::SearchSlot* sl, uint64_t nq, const float* dq, uint32_t k, uint32_t ef_in, uint64_t* dl, float* dd,
                 uint32_t* dc, cudaStream_t s, const ehb::ResultSink* sink = nullptr, bool* pushed = nullptr,
                 int precision = EHB_FP32);
  // The wide-beam scratch a search_dev of nq queries at beam ef_eff (= max(ef, k)) needs, grown now on s, so that the
  // search's own grow does nothing: the exchange steps call it before their epoch advances, so that an allocation
  // failure (EHB_ERR_OOM) leaves the rank in phase.  Nothing happens when the plan is not the wide-beam walk.  A grow
  // synchronises s and frees the old buffer (which waits for the device).  Caller holds the reader lock, so the plan
  // cannot change before the search.
  int reserve_beam(uint64_t nq, uint32_t ef_eff, int precision, cudaStream_t s);
  // caller holds beam_mu: waits for the previous wide-beam search on s, then grows the scratch for `plan`
  int grow_beam(const ehb::WalkPlan& plan, uint64_t nq, uint32_t ef_eff, cudaStream_t s, uint32_t* warps);
  int bruteforce_dev(uint64_t nq, const float* dq, uint32_t k, int precision, uint64_t* dl, float* dd, uint32_t* dc,
                     cudaStream_t s);
  void reset_content();
};

namespace ehb {
// The only way to use a search slot: one for the length of a call.  take() acquires a slot from ix's pool and orders
// `s` (nullptr: the slot's own stream) after the slot's previous user; the destructor records the slot's `busy` event
// on `s` and returns the slot, so the next user waits for this call's work without a host synchronisation.
class SlotLease {
 public:
  explicit SlotLease(ehb_index* ix) : ix_(ix) {}
  SlotLease(const SlotLease&) = delete;
  SlotLease& operator=(const SlotLease&) = delete;
  ~SlotLease();
  int take(cudaStream_t stream = nullptr);
  SearchSlot* sl = nullptr;
  cudaStream_t s = nullptr;

 private:
  ehb_index* ix_;
};
}  // namespace ehb
