// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product path.
//
// CPU restatement of the hnswlib subset that embeddinghub's ANNIndex calls
// (reference: embeddinghub/embeddingstore/index.cc:10-52, index.h:19-33).  The
// arithmetic itself lives in the third-party header-only library
//   github.com/nmslib/hnswlib @ 21b54fe9544cfbb757b2ea8f3def5542ba2435c7
//   (embeddinghub/WORKSPACE:80-85; Python side hnswlib==0.5.2,
//    embeddinghub/sdk/python/requirements.txt:1)
// which is NOT vendored in the reference tree, so this
// file restates its published algorithm (Malkov & Yashunin, "Efficient and
// robust approximate nearest neighbor search using HNSW graphs", and the
// upstream hnswalg.h / space_l2.h / space_ip.h / bruteforce.h behaviour as
// called from the reference's call sites):
//   HierarchicalNSW ctor defaults  <- index.cc:14-15  (M=16, efC=200, seed=100, ef=10)
//   addPoint (insert + update)     <- index.cc:36
//   resizeIndex                    <- index.cc:31
//   searchKnn                      <- index.cc:41
//   L2Space                        <- index.cc:12-13
//   InnerProductSpace / cosine     <- named by BASELINE.json north_star; cosine is
//                                     hnswlib's Python convention (normalise + IP)
//   BruteforceSearch               <- semantic oracle for the exact path
//   markDelete / has_deletions     <- docs/reading_and_writing_embeddings.md:49-66 promises delete;
//                                     upstream: tombstones are traversed but never returned, a re-added
//                                     label is un-deleted and updated in place (addPoint)
//
// PINNING: checked against the reference's own known-answer tests
// (embeddingstore/test/index_test.cc:17-60, sdk/python/test/offlinehub_test.py:63-86,
// provider/vectorstore_test.go:121-166 fixture) in tests/test_oracle_golden.py.
// Beyond those toy cases the reference holds no vectors for this path; larger
// sizes are pinned by exact fp32 brute force (orc_bruteforce below), whose
// arithmetic order is the canonical one shared with the CUDA exact kernel.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
// reference legs may load this library.

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <mutex>
#include <queue>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace {

enum Metric : int { kL2 = 0, kIP = 1, kCosine = 2 };

// ---------------------------------------------------------------------------
// Distance functors (hnswlib space_l2.h / space_ip.h semantics: squared L2, and
// 1 - dot).  The graph code uses a 16-accumulator form that gcc vectorises to
// the same shape as hnswlib's SIMD16 kernels (fair CPU baseline).  The exact
// path uses the canonical sequential-FMA chain (see canon_* below).
// ---------------------------------------------------------------------------
static inline float l2_fast(const float* a, const float* b, size_t d) {
  float acc[16] = {0};
  size_t i = 0;
  for (; i + 16 <= d; i += 16)
    for (int j = 0; j < 16; ++j) {
      float t = a[i + j] - b[i + j];
      acc[j] += t * t;
    }
  float s = 0.f;
  for (int j = 0; j < 16; ++j) s += acc[j];
  for (; i < d; ++i) {
    float t = a[i] - b[i];
    s += t * t;
  }
  return s;
}
static inline float dot_fast(const float* a, const float* b, size_t d) {
  float acc[16] = {0};
  size_t i = 0;
  for (; i + 16 <= d; i += 16)
    for (int j = 0; j < 16; ++j) acc[j] += a[i + j] * b[i + j];
  float s = 0.f;
  for (int j = 0; j < 16; ++j) s += acc[j];
  for (; i < d; ++i) s += a[i] * b[i];
  return s;
}

// Canonical exact arithmetic: one fp32 accumulator, k ascending, fused
// multiply-add.  The CUDA exact kernel (bf_exact) follows the same chain so
// that brute-force ids can be compared bit-exactly.
static inline float canon_l2(const float* a, const float* b, size_t d) {
  float acc = 0.f;
  for (size_t i = 0; i < d; ++i) {
    float t = a[i] - b[i];
    acc = fmaf(t, t, acc);
  }
  return acc;
}
static inline float canon_dot(const float* a, const float* b, size_t d) {
  float acc = 0.f;
  for (size_t i = 0; i < d; ++i) acc = fmaf(a[i], b[i], acc);
  return acc;
}
// hnswlib Python binding normalize_vector(): norm = 1/(sqrt(sum x^2)+1e-30).
static inline void canon_normalize(const float* in, float* out, size_t d) {
  float acc = 0.f;
  for (size_t i = 0; i < d; ++i) acc = fmaf(in[i], in[i], acc);
  float inv = 1.0f / (sqrtf(acc) + 1e-30f);
  for (size_t i = 0; i < d; ++i) out[i] = in[i] * inv;
}

typedef uint32_t idx_t;
typedef std::pair<float, idx_t> DI;
struct DICmp {
  bool operator()(const DI& a, const DI& b) const { return a.first < b.first; }
};
typedef std::priority_queue<DI, std::vector<DI>, DICmp> MaxHeap;

struct Visited {
  std::vector<uint16_t> tag;
  uint16_t cur = 0;
  void reset(size_t n) {
    if (tag.size() < n) tag.assign(n, 0), cur = 0;
    if (++cur == 0) {
      std::fill(tag.begin(), tag.end(), 0);
      cur = 1;
    }
  }
};

struct Oracle {
  size_t dim;
  int metric;
  size_t cap;
  size_t M, maxM, maxM0, efC, ef;
  double mult;
  std::minstd_rand0 level_rng;   // std::default_random_engine in libstdc++
  std::minstd_rand0 update_rng;
  size_t count = 0;
  int maxlevel = -1;
  idx_t enterpoint = 0;
  bool has_ep = false;

  std::vector<float> vecs;                 // [cap][dim]
  std::vector<uint64_t> labels;            // [cap]
  std::vector<int> levels;                 // [cap]
  std::vector<uint8_t> deleted;            // [cap] hnswlib DELETE_MARK
  size_t num_deleted = 0;
  std::vector<uint32_t> links0;            // [cap][1+maxM0]  (count, ids...)
  std::vector<std::vector<uint32_t>> linksup;  // [cap] -> level*(1+maxM)
  std::unordered_map<uint64_t, idx_t> lookup;
  std::vector<std::mutex> node_locks;
  std::mutex global_lock, lookup_lock, level_lock;
  std::atomic<uint64_t> metric_hops{0}, metric_evals{0}, metric_hops_upper{0};

  std::mutex pool_lock;
  std::vector<std::unique_ptr<Visited>> pool;

  Oracle(size_t d, int met, size_t max_elements, size_t M_, size_t efc, uint64_t seed)
      : dim(d), metric(met), cap(max_elements), M(M_), maxM(M_), maxM0(2 * M_),
        efC(std::max(efc, M_)), ef(10), mult(1.0 / std::log(1.0 * M_)),
        level_rng(seed), update_rng(seed + 1), node_locks(max_elements) {
    vecs.resize(cap * dim);
    labels.resize(cap);
    levels.assign(cap, 0);
    deleted.assign(cap, 0);
    links0.assign(cap * (1 + maxM0), 0);
    linksup.resize(cap);
  }

  inline float dist(const float* a, const float* b) const {
    return metric == kL2 ? l2_fast(a, b, dim) : 1.0f - dot_fast(a, b, dim);
  }
  inline const float* vec(idx_t i) const { return &vecs[(size_t)i * dim]; }
  inline uint32_t* ll(idx_t i, int level) {
    return level == 0 ? &links0[(size_t)i * (1 + maxM0)]
                      : &linksup[i][(size_t)(level - 1) * (1 + maxM)];
  }

  std::unique_ptr<Visited> get_visited() {
    std::unique_ptr<Visited> v;
    {
      std::lock_guard<std::mutex> g(pool_lock);
      if (!pool.empty()) {
        v = std::move(pool.back());
        pool.pop_back();
      }
    }
    if (!v) v.reset(new Visited());
    v->reset(cap);
    return v;
  }
  void put_visited(std::unique_ptr<Visited> v) {
    std::lock_guard<std::mutex> g(pool_lock);
    pool.push_back(std::move(v));
  }

  void resize(size_t new_cap) {
    if (new_cap < count) throw std::runtime_error("Cannot resize, max element is less than the current number of elements");
    vecs.resize(new_cap * dim);
    labels.resize(new_cap);
    levels.resize(new_cap, 0);
    deleted.resize(new_cap, 0);
    links0.resize(new_cap * (1 + maxM0), 0);
    linksup.resize(new_cap);
    std::vector<std::mutex>(new_cap).swap(node_locks);
    cap = new_cap;
    pool.clear();
  }

  int random_level() {
    std::uniform_real_distribution<double> u(0.0, 1.0);
    double r = -std::log(u(level_rng)) * mult;
    return (int)r;
  }

  // Beam search used while building (hnswlib searchBaseLayer).
  MaxHeap search_layer_build(idx_t ep, const float* q, int layer) {
    auto vl = get_visited();
    uint16_t* tags = vl->tag.data();
    uint16_t t = vl->cur;
    MaxHeap top, cand;
    float lower;
    if (!deleted[ep]) {
      lower = dist(q, vec(ep));
      top.emplace(lower, ep);
      cand.emplace(-lower, ep);
    } else {
      lower = std::numeric_limits<float>::max();
      cand.emplace(-lower, ep);
    }
    tags[ep] = t;
    while (!cand.empty()) {
      DI cur = cand.top();
      if (-cur.first > lower && top.size() == efC) break;
      cand.pop();
      idx_t c = cur.second;
      std::unique_lock<std::mutex> lk(node_locks[c]);
      uint32_t* l = ll(c, layer);
      uint32_t sz = l[0];
      for (uint32_t j = 1; j <= sz; ++j) {
        idx_t nb = l[j];
        if (tags[nb] == t) continue;
        tags[nb] = t;
        float dd = dist(q, vec(nb));
        if (top.size() < efC || lower > dd) {
          cand.emplace(-dd, nb);
          if (!deleted[nb]) top.emplace(dd, nb);
          if (top.size() > efC) top.pop();
          if (!top.empty()) lower = top.top().first;
        }
      }
    }
    put_visited(std::move(vl));
    return top;
  }

  // hnswlib getNeighborsByHeuristic2.
  void heuristic(MaxHeap& top, size_t Msel) {
    if (top.size() < Msel) return;
    std::vector<DI> asc;
    asc.reserve(top.size());
    while (!top.empty()) {
      asc.push_back(top.top());
      top.pop();
    }
    std::reverse(asc.begin(), asc.end());  // ascending distance to the query
    std::vector<DI> keep;
    for (const DI& c : asc) {
      if (keep.size() >= Msel) break;
      bool good = true;
      for (const DI& s : keep) {
        if (dist(vec(s.second), vec(c.second)) < c.first) {
          good = false;
          break;
        }
      }
      if (good) keep.push_back(c);
    }
    for (const DI& k : keep) top.push(k);
  }

  idx_t connect(const float* q, idx_t cur, MaxHeap& top, int level, bool is_update) {
    size_t Mmax = level ? maxM : maxM0;
    heuristic(top, M);
    if (top.size() > M) throw std::runtime_error("Should be not be more than M_ candidates returned by the heuristic");
    std::vector<idx_t> sel;
    sel.reserve(M);
    while (!top.empty()) {
      sel.push_back(top.top().second);
      top.pop();
    }
    idx_t next_ep = sel.back();
    {
      // A fresh insert already holds node_locks[cur] for its whole duration (as
      // upstream's lock_el does); only the update path locks here.
      std::unique_lock<std::mutex> lk(node_locks[cur], std::defer_lock);
      if (is_update) lk.lock();
      uint32_t* l = ll(cur, level);
      if (l[0] && !is_update) throw std::runtime_error("The newly inserted element should have blank link list");
      l[0] = (uint32_t)sel.size();
      for (size_t i = 0; i < sel.size(); ++i) l[1 + i] = sel[i];
    }
    for (idx_t s : sel) {
      std::unique_lock<std::mutex> lk(node_locks[s]);
      uint32_t* l = ll(s, level);
      uint32_t sz = l[0];
      bool present = false;
      if (is_update)
        for (uint32_t j = 1; j <= sz; ++j)
          if (l[j] == cur) {
            present = true;
            break;
          }
      if (present) continue;
      if (sz < Mmax) {
        l[1 + sz] = cur;
        l[0] = sz + 1;
      } else {
        MaxHeap c;
        c.emplace(dist(vec(cur), vec(s)), cur);
        for (uint32_t j = 1; j <= sz; ++j) c.emplace(dist(vec(l[j]), vec(s)), l[j]);
        heuristic(c, Mmax);
        uint32_t k = 0;
        while (!c.empty()) {
          l[1 + k++] = c.top().second;
          c.pop();
        }
        l[0] = k;
      }
    }
    return next_ep;
  }

  // collect=true is the query path (no locking, metrics on); false is the build path.
  idx_t greedy(const float* q, idx_t cur, int from_level, int to_level_excl, bool collect) {
    float cd = dist(q, vec(cur));
    for (int level = from_level; level > to_level_excl; --level) {
      bool changed = true;
      while (changed) {
        changed = false;
        std::unique_lock<std::mutex> lk(node_locks[cur], std::defer_lock);
        if (!collect) lk.lock();
        uint32_t* l = ll(cur, level);
        uint32_t sz = l[0];
        if (collect) {
          metric_hops_upper++;
          metric_evals += sz;
        }
        for (uint32_t j = 1; j <= sz; ++j) {
          idx_t nb = l[j];
          float dd = dist(q, vec(nb));
          if (dd < cd) {
            cd = dd;
            cur = nb;
            changed = true;
          }
        }
      }
    }
    return cur;
  }

  std::vector<idx_t> connections(idx_t i, int level) {
    std::unique_lock<std::mutex> lk(node_locks[i]);
    uint32_t* l = ll(i, level);
    return std::vector<idx_t>(l + 1, l + 1 + l[0]);
  }

  void update_point(const float* data, idx_t id) {
    std::memcpy(&vecs[(size_t)id * dim], data, dim * sizeof(float));
    int max_copy = maxlevel;
    idx_t ep_copy = enterpoint;
    if (ep_copy == id && count == 1) return;
    int el_level = levels[id];
    for (int layer = 0; layer <= el_level; ++layer) {
      std::unordered_set<idx_t> sCand, sNeigh;
      std::vector<idx_t> one = connections(id, layer);
      if (one.empty()) continue;
      sCand.insert(id);
      for (idx_t e1 : one) {
        sCand.insert(e1);
        sNeigh.insert(e1);  // updateNeighborProbability = 1.0
        for (idx_t e2 : connections(e1, layer)) sCand.insert(e2);
      }
      for (idx_t nb : sNeigh) {
        MaxHeap c;
        size_t size = sCand.count(nb) ? sCand.size() - 1 : sCand.size();
        size_t keep = std::min(efC, size);
        for (idx_t cd : sCand) {
          if (cd == nb) continue;
          float dd = dist(vec(nb), vec(cd));
          if (c.size() < keep)
            c.emplace(dd, cd);
          else if (dd < c.top().first) {
            c.pop();
            c.emplace(dd, cd);
          }
        }
        heuristic(c, layer == 0 ? maxM0 : maxM);
        std::unique_lock<std::mutex> lk(node_locks[nb]);
        uint32_t* l = ll(nb, layer);
        uint32_t k = 0;
        while (!c.empty()) {
          l[1 + k++] = c.top().second;
          c.pop();
        }
        l[0] = k;
      }
    }
    // repairConnectionsForUpdate
    idx_t cur = ep_copy;
    if (el_level < max_copy) cur = greedy(data, cur, max_copy, el_level, false);
    for (int level = el_level; level >= 0; --level) {
      MaxHeap top = search_layer_build(cur, data, level);
      MaxHeap filt;
      while (!top.empty()) {
        if (top.top().second != id) filt.push(top.top());
        top.pop();
      }
      if (!filt.empty()) cur = connect(data, id, filt, level, true);
    }
  }

  void add(const float* data_in, uint64_t label) {
    std::vector<float> tmp;
    const float* data = data_in;
    if (metric == kCosine) {
      tmp.resize(dim);
      canon_normalize(data_in, tmp.data(), dim);
      data = tmp.data();
    }
    idx_t cur;
    {
      std::unique_lock<std::mutex> lk(lookup_lock);
      auto it = lookup.find(label);
      if (it != lookup.end()) {
        idx_t existing = it->second;
        lk.unlock();
        if (deleted[existing]) {  // upstream addPoint: unmarkDeletedInternal, then updatePoint
          deleted[existing] = 0;
          num_deleted--;
        }
        update_point(data, existing);
        return;
      }
      if (count >= cap) throw std::runtime_error("The number of elements exceeds the specified limit");
      cur = (idx_t)count++;
      lookup[label] = cur;
    }
    std::unique_lock<std::mutex> el_lock(node_locks[cur]);
    int curlevel;
    {
      // level draw is serialised like upstream's single generator
      std::unique_lock<std::mutex> g(level_lock);
      curlevel = random_level();
    }
    levels[cur] = curlevel;
    std::unique_lock<std::mutex> templock(global_lock);
    int max_copy = maxlevel;
    if (curlevel <= max_copy) templock.unlock();
    idx_t cur_obj = enterpoint;
    bool had_ep = has_ep;
    std::memset(ll(cur, 0), 0, (1 + maxM0) * sizeof(uint32_t));
    labels[cur] = label;
    std::memcpy(&vecs[(size_t)cur * dim], data, dim * sizeof(float));
    if (curlevel) linksup[cur].assign((size_t)curlevel * (1 + maxM), 0);
    if (had_ep) {
      if (curlevel < max_copy) cur_obj = greedy(data, cur_obj, max_copy, curlevel, false);
      for (int level = std::min(curlevel, max_copy); level >= 0; --level) {
        MaxHeap top = search_layer_build(cur_obj, data, level);
        cur_obj = connect(data, cur, top, level, false);
      }
    } else {
      enterpoint = cur;
      maxlevel = curlevel;
      has_ep = true;
    }
    if (curlevel > max_copy) {
      enterpoint = cur;
      maxlevel = curlevel;
    }
  }

  // hnswlib searchBaseLayerST (no deletions) + searchKnn.
  size_t search(const float* q_in, size_t k, size_t ef_use, uint64_t* out_l, float* out_d) {
    if (count == 0 || k == 0) return 0;
    std::vector<float> tmp;
    const float* q = q_in;
    if (metric == kCosine) {
      tmp.resize(dim);
      canon_normalize(q_in, tmp.data(), dim);
      q = tmp.data();
    }
    metric_evals++;  // entry point
    idx_t cur = greedy(q, enterpoint, maxlevel, 0, true);
    size_t efs = std::max(ef_use, k);
    auto vl = get_visited();
    uint16_t* tags = vl->tag.data();
    uint16_t t = vl->cur;
    MaxHeap top, cand;
    const bool has_del = num_deleted != 0;  // searchBaseLayerST<has_deletions>
    float lower;
    if (!has_del || !deleted[cur]) {
      lower = dist(q, vec(cur));
      top.emplace(lower, cur);
      cand.emplace(-lower, cur);
    } else {
      lower = std::numeric_limits<float>::max();
      cand.emplace(-lower, cur);
    }
    tags[cur] = t;
    uint64_t hops = 0, evals = 0;
    while (!cand.empty()) {
      DI c = cand.top();
      if (-c.first > lower && (top.size() == efs || !has_del)) break;
      cand.pop();
      uint32_t* l = ll(c.second, 0);
      uint32_t sz = l[0];
      hops++;
      for (uint32_t j = 1; j <= sz; ++j) {
        idx_t nb = l[j];
        if (tags[nb] == t) continue;
        tags[nb] = t;
        evals++;
        float dd = dist(q, vec(nb));
        if (top.size() < efs || lower > dd) {
          cand.emplace(-dd, nb);
          if (!has_del || !deleted[nb]) top.emplace(dd, nb);
          if (top.size() > efs) top.pop();
          if (!top.empty()) lower = top.top().first;
        }
      }
    }
    put_visited(std::move(vl));
    metric_hops += hops;
    metric_evals += evals;
    while (top.size() > k) top.pop();
    size_t n = top.size();
    for (size_t i = n; i-- > 0;) {
      out_l[i] = labels[top.top().second];
      out_d[i] = top.top().first;
      top.pop();
    }
    return n;
  }
};

thread_local std::string g_err;

// Timing hygiene for the CPU baseline (bench.py): with pinning on, worker t runs on the t-th CPU of the
// process affinity mask, so a pass is not at the mercy of the scheduler migrating 128 threads.
std::atomic<int> g_pin_threads{0};

template <class F>
void parallel_for(size_t n, int threads, F f) {
  if (threads <= 1 || n < 2) {
    for (size_t i = 0; i < n; ++i) f(i);
    return;
  }
  std::atomic<size_t> next{0};
  std::vector<std::thread> ts;
  std::mutex em;
  std::string err;
  std::vector<int> cpus;
  if (g_pin_threads.load()) {
    cpu_set_t mask;
    if (sched_getaffinity(0, sizeof(mask), &mask) == 0)
      for (int c = 0; c < CPU_SETSIZE; ++c)
        if (CPU_ISSET(c, &mask)) cpus.push_back(c);
  }
  for (int t = 0; t < threads; ++t)
    ts.emplace_back([&, t] {
      if (!cpus.empty()) {
        cpu_set_t one;
        CPU_ZERO(&one);
        CPU_SET(cpus[(size_t)t % cpus.size()], &one);
        pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
      }
      try {
        for (;;) {
          size_t i = next.fetch_add(1);
          if (i >= n) break;
          f(i);
        }
      } catch (const std::exception& e) {
        std::lock_guard<std::mutex> g(em);
        err = e.what();
        next = n;
      }
    });
  for (auto& t : ts) t.join();
  if (!err.empty()) throw std::runtime_error(err);
}

}  // namespace

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }
void orc_set_thread_pinning(int on) { g_pin_threads = on; }

void* orc_create(uint64_t dim, int metric, uint64_t max_elements, uint64_t M, uint64_t efc, uint64_t seed) {
  try {
    return new Oracle(dim, metric, max_elements, M, efc, seed);
  } catch (const std::exception& e) {
    g_err = e.what();
    return nullptr;
  }
}
void orc_destroy(void* h) { delete (Oracle*)h; }
void orc_set_ef(void* h, uint64_t ef) { ((Oracle*)h)->ef = ef; }
uint64_t orc_count(void* h) { return ((Oracle*)h)->count; }
uint64_t orc_capacity(void* h) { return ((Oracle*)h)->cap; }
int orc_max_level(void* h) { return ((Oracle*)h)->maxlevel; }
uint32_t orc_entry_point(void* h) { return ((Oracle*)h)->enterpoint; }

int orc_resize(void* h, uint64_t new_cap) {
  try {
    ((Oracle*)h)->resize(new_cap);
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// Insert-or-update n rows.  threads<=1 is the reference's behaviour (one
// addPoint at a time under the service mutex, version.cc:69-72).
int orc_add(void* h, uint64_t n, const float* rows, const uint64_t* labels, int threads) {
  Oracle* o = (Oracle*)h;
  try {
    size_t start = 0;
    if (o->count == 0 && n > 0) {  // first element alone, as upstream's add_items does
      o->add(rows, labels[0]);
      start = 1;
    }
    parallel_for(n - start, threads, [&](size_t i) {
      o->add(rows + (start + i) * o->dim, labels[start + i]);
    });
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// k-NN for nq queries; ef=0 -> index ef (default 10, like the reference which
// never calls setEf).  Rows are nearest-first, padded with UINT64_MAX / +inf.
int orc_search(void* h, uint64_t nq, const float* q, uint64_t k, uint64_t ef, uint64_t* out_labels,
               float* out_dists, uint32_t* out_counts, int threads) {
  Oracle* o = (Oracle*)h;
  try {
    size_t efs = ef ? ef : o->ef;
    parallel_for(nq, threads, [&](size_t i) {
      uint64_t* ol = out_labels + i * k;
      float* od = out_dists + i * k;
      size_t n = o->search(q + i * o->dim, k, efs, ol, od);
      for (size_t j = n; j < k; ++j) {
        ol[j] = UINT64_MAX;
        od[j] = INFINITY;
      }
      if (out_counts) out_counts[i] = (uint32_t)n;
    });
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

void orc_metrics(void* h, uint64_t* hops_upper, uint64_t* hops0, uint64_t* evals, int reset) {
  Oracle* o = (Oracle*)h;
  *hops_upper = o->metric_hops_upper;
  *hops0 = o->metric_hops;
  *evals = o->metric_evals;
  if (reset) o->metric_hops_upper = 0, o->metric_hops = 0, o->metric_evals = 0;
}

// hnswlib markDelete(label): unknown label and double delete both throw.
int orc_mark_delete(void* h, uint64_t label) {
  Oracle* o = (Oracle*)h;
  auto it = o->lookup.find(label);
  if (it == o->lookup.end()) {
    g_err = "Label not found";
    return 1;
  }
  if (o->deleted[it->second]) {
    g_err = "The requested to delete element is already deleted";
    return 2;
  }
  o->deleted[it->second] = 1;
  o->num_deleted++;
  return 0;
}
uint64_t orc_deleted_count(void* h) { return ((Oracle*)h)->num_deleted; }

int orc_get_vector(void* h, uint64_t label, float* out) {
  Oracle* o = (Oracle*)h;
  auto it = o->lookup.find(label);
  if (it == o->lookup.end() || o->deleted[it->second]) return 1;  // getDataByLabel: "Label not found"
  std::memcpy(out, o->vec(it->second), o->dim * sizeof(float));
  return 0;
}

// Graph export (for feeding the identical graph to the CUDA walk in tests):
// levels[count], links0[count][maxM0] padded with UINT32_MAX, and for every
// node with level>0 its upper rows [level][maxM] appended to links_up in node
// order; up_off[i] = first row of node i (or UINT32_MAX).
uint64_t orc_upper_rows(void* h) {
  Oracle* o = (Oracle*)h;
  uint64_t r = 0;
  for (size_t i = 0; i < o->count; ++i) r += o->levels[i];
  return r;
}
void orc_export_graph(void* h, uint8_t* levels, uint32_t* links0, uint32_t* up_off, uint32_t* links_up,
                      uint64_t* labels) {
  Oracle* o = (Oracle*)h;
  uint64_t row = 0;
  for (size_t i = 0; i < o->count; ++i) {
    levels[i] = (uint8_t)o->levels[i];
    labels[i] = o->labels[i];
    uint32_t* l = o->ll(i, 0);
    for (size_t j = 0; j < o->maxM0; ++j) links0[i * o->maxM0 + j] = j < l[0] ? l[1 + j] : UINT32_MAX;
    up_off[i] = o->levels[i] ? (uint32_t)row : UINT32_MAX;
    for (int lv = 1; lv <= o->levels[i]; ++lv, ++row) {
      uint32_t* u = o->ll(i, lv);
      for (size_t j = 0; j < o->maxM; ++j) links_up[row * o->maxM + j] = j < u[0] ? u[1 + j] : UINT32_MAX;
    }
  }
}
const float* orc_vectors(void* h) { return ((Oracle*)h)->vecs.data(); }

// Graph import: lets the CPU search (the reference algorithm) run over a graph
// built elsewhere (same layout as orc_export_graph).  Vectors are taken as
// given (already normalised for cosine).
int orc_import_graph(void* h, uint64_t n, const float* vecs, const uint64_t* labels, const uint8_t* levels,
                     const uint32_t* links0, const uint32_t* up_off, const uint32_t* links_up,
                     uint32_t entry, int maxlevel) {
  Oracle* o = (Oracle*)h;
  try {
    if (n > o->cap) o->resize(n);
    std::memcpy(o->vecs.data(), vecs, n * o->dim * sizeof(float));
    o->lookup.clear();
    for (size_t i = 0; i < n; ++i) {
      o->labels[i] = labels[i];
      o->lookup[labels[i]] = (idx_t)i;
      o->levels[i] = levels[i];
      uint32_t* l = o->ll(i, 0);
      uint32_t c = 0;
      for (size_t j = 0; j < o->maxM0; ++j) {
        uint32_t v = links0[i * o->maxM0 + j];
        if (v != UINT32_MAX) l[1 + c++] = v;
      }
      l[0] = c;
      if (levels[i]) {
        o->linksup[i].assign((size_t)levels[i] * (1 + o->maxM), 0);
        for (int lv = 1; lv <= levels[i]; ++lv) {
          uint32_t* u = o->ll(i, lv);
          uint32_t cu = 0;
          const uint32_t* src = links_up + ((size_t)up_off[i] + lv - 1) * o->maxM;
          for (size_t j = 0; j < o->maxM; ++j)
            if (src[j] != UINT32_MAX) u[1 + cu++] = src[j];
          u[0] = cu;
        }
      }
    }
    o->count = n;
    o->enterpoint = entry;
    o->maxlevel = maxlevel;
    o->has_ep = n > 0;
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// Exact k-NN (hnswlib BruteforceSearch semantics) with the canonical
// sequential-FMA arithmetic; total order (distance asc, row index asc).
// base rows are used as given for L2/IP and normalised first for cosine.
int orc_bruteforce(int metric, uint64_t n, uint64_t d, const float* base, uint64_t nq, const float* q, uint64_t k,
                   uint64_t* out_idx, float* out_dists, int threads) {
  try {
    std::vector<float> nbase;
    const float* b = base;
    if (metric == kCosine) {
      nbase.resize(n * d);
      parallel_for(n, threads, [&](size_t i) { canon_normalize(base + i * d, &nbase[i * d], d); });
      b = nbase.data();
    }
    parallel_for(nq, threads, [&](size_t qi) {
      std::vector<float> qn(d);
      const float* qq = q + qi * d;
      if (metric == kCosine) {
        canon_normalize(qq, qn.data(), d);
        qq = qn.data();
      }
      typedef std::pair<float, uint64_t> DL;
      std::priority_queue<DL> heap;  // max-heap on (dist, idx)
      for (uint64_t i = 0; i < n; ++i) {
        float dd = metric == kL2 ? canon_l2(qq, b + i * d, d) : 1.0f - canon_dot(qq, b + i * d, d);
        if (heap.size() < k)
          heap.emplace(dd, i);
        else if (DL(dd, i) < heap.top()) {
          heap.pop();
          heap.emplace(dd, i);
        }
      }
      size_t m = heap.size();
      for (size_t j = m; j < k; ++j) out_idx[qi * k + j] = UINT64_MAX, out_dists[qi * k + j] = INFINITY;
      for (size_t j = m; j-- > 0;) {
        out_idx[qi * k + j] = heap.top().second;
        out_dists[qi * k + j] = heap.top().first;
        heap.pop();
      }
    });
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

void orc_normalize(uint64_t n, uint64_t d, const float* in, float* out) {
  for (uint64_t i = 0; i < n; ++i) canon_normalize(in + i * d, out + i * d, d);
}

}  // extern "C"
