// Range-sharded search behind the C ABI (SURVEY.md §8b B4 "device_ids[], n_dev", §8e).
//
// The index is partitioned by label range; every GPU owns an independent graph; every GPU searches all
// queries; the per-shard top-k lists meet in ONE exchange step and are merged.  Two deployment shapes:
//
//  * ehb_sharded  — one process drives n_dev GPUs (what a C++ ANNIndex or the cgo provider links against).
//    Peer access is enabled between the devices and every shard's search kernels write their top-k
//    STRAIGHT INTO DEVICE 0's gather buffer (stores over NVLink from inside the walk kernel); device 0's
//    merge kernel is ordered after them with events.  No collective, no staging copy.
//
//  * ehb_exchange — one process per GPU (torchrun / MPI style).  Each rank owns a receive buffer
//    [2 parities][world][block] + flags, exported with CUDA IPC and mapped by every peer.  A step is ONE
//    kernel per rank (exchange_merge_kernel): phase 1 pushes this rank's block, slice by slice, into every
//    peer's buffer with coalesced stores over NVLink and raises a per-(rank, slice) flag with a
//    system-scope release; phase 2 waits (acquire) for the flags of each slice and merges the G lists of
//    its queries.  This replaces ncclAllGather + merge kernel: no collective launch, the merge of early
//    slices overlaps the transfer of late ones, and flags are epoch-numbered with parity double
//    buffering so consecutive steps need no barrier.
#include <thread>

#include "exchange_layout.cuh"
#include "index_impl.h"
#include "merge.cuh"

using ehb::fail;

namespace ehb {

// Every rank's exported allocation as mapped HERE, and its layout (exchange_layout.cuh).
struct PeerView {
  unsigned char* base[kMaxWorld];
  uint32_t rank;
  ExchangeLayout L;
};

// The end of slice s's push: every thread's stores are ordered before the slice's flag on every peer.
__device__ __forceinline__ void publish_slice(const PeerView& v, uint32_t parity, uint32_t epoch, uint32_t s) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < v.L.world && threadIdx.x != v.rank)
    st_release_sys(v.L.flags(v.base[threadIdx.x], parity, v.rank) + s, epoch);
  __syncthreads();
}

// Waits until every peer has raised slice s's flag.  Bounded (~20 s): a peer that never arrives must not wedge the
// GPU, so the wait gives up, sets the timeout word the host reads, and returns true (in the threads that gave up).
__device__ __forceinline__ bool await_slice(const PeerView& v, uint32_t parity, uint32_t epoch, uint32_t s,
                                            uint32_t* timeout_word) {
  bool gave_up = false;
  if (threadIdx.x < v.L.world && threadIdx.x != v.rank) {
    const uint32_t* f = v.L.flags(v.base[v.rank], parity, threadIdx.x) + s;
    uint32_t spins = 0;
    while (ld_acquire_sys(f) != epoch) {
      __nanosleep(64);
      if (++spins > (1u << 28)) {
        atomicExch(timeout_word, 1u);
        gave_up = true;
        break;
      }
    }
  }
  __syncthreads();
  return gave_up;
}

// One persistent launch per rank and step; grid <= resident capacity so no CTA waits on an unscheduled one.
// 1024 threads per CTA: the push is a plain copy and the merge is one latency-bound warp per query, so both
// want as many warps per SM as one resident CTA can hold.
constexpr uint32_t kExchangeThreads = 1024;
__global__ void __launch_bounds__(kExchangeThreads) exchange_merge_kernel(PeerView v, uint32_t parity, uint32_t epoch,
                                                             uint64_t nq, uint32_t k, uint32_t qs, uint32_t nslices,
                                                             float* __restrict__ out_dists,
                                                             uint64_t* __restrict__ out_labels,
                                                             uint32_t* __restrict__ out_counts,
                                                             uint32_t* __restrict__ timeout_flag, uint32_t skip_push) {
  const uint32_t W = v.L.world, me = v.rank;
  const unsigned char* mine = v.L.recv(v.base[me], parity, me);  // written by my search kernels
  const uint64_t lab_bytes = nq * k * 8ull;
  // ---- phase 1: push my slices to every peer, then raise their flags ------------------------------------
  // (skipped when the producer was the one-warp walk: its epilogue already stored every query's results into
  //  the peers' buffers and raised the slice flags — search_impl.cuh)
  for (uint32_t s = blockIdx.x; s < nslices && !skip_push; s += gridDim.x) {
    const uint64_t q0 = (uint64_t)s * qs, q1 = min(nq, q0 + qs);
    const uint64_t e0 = q0 * k, e1 = q1 * k;  // element range of the slice
    const uint64_t* src_l = (const uint64_t*)mine;
    const float* src_d = (const float*)(mine + lab_bytes);
    for (uint32_t g = 0; g < W; ++g) {
      if (g == me) continue;
      unsigned char* dst = v.L.recv(v.base[g], parity, me);
      uint64_t* dst_l = (uint64_t*)dst;
      float* dst_d = (float*)(dst + lab_bytes);
      for (uint64_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) dst_l[i] = src_l[i];
      for (uint64_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) dst_d[i] = src_d[i];
    }
    publish_slice(v, parity, epoch, s);
  }
  // ---- phase 2: wait for each slice from every peer, merge its queries -------------------------------------
  const unsigned char* base = v.L.recv(v.base[me], parity, 0);
  const uint32_t warps = blockDim.x >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t s = blockIdx.x; s < nslices; s += gridDim.x) {
    await_slice(v, parity, epoch, s, timeout_flag);
    const uint64_t q0 = (uint64_t)s * qs, q1 = min(nq, q0 + qs);
    for (uint64_t q = q0 + w; q < q1; q += warps)
      merge_one_query(W, q, lane, k, (const float*)(base + lab_bytes), (const uint64_t*)base, v.L.stride, v.L.stride,
                      out_dists, out_labels, out_counts);
  }
}

// Bits of the verdict word of a row step.  Every rank reads the same digests, so kRowsDigest is set on every rank or on
// none; when it is clear every rank was given the same list and reads the same marks, so the whole word is equal.
constexpr uint32_t kRowsMissing = 1;   // a query that no rank holds
constexpr uint32_t kRowsShared = 2;    // a query that more than one rank holds
constexpr uint32_t kRowsDigest = 4;    // a peer's label list differs from this rank's
constexpr uint32_t kRowsTimeout = 8;   // a peer never raised its flags (the timeout word is set too)

// The row step of a by-label search (ehb_exchange_search_by_label_ex_dev); one persistent launch per rank (grid sized
// like exchange_merge_kernel).  Phase 1: every query this rank holds (ids[q] != kInvalid) has its stored row copied
// from vecs (dpad stride) into row q of every rank's row region, this rank's own included: one warp per row, each
// 16-byte chunk read once and stored to every destination.  The whole mark vector and (with slice 0) the digest go to
// every rank too; then the slice flags, released at system scope.  Phase 2: wait for every peer's slice flags, count
// each query's holders over the ranks, compare the digests, and OR the outcome into the local verdict word (zeroed
// before the launch).
__global__ void __launch_bounds__(kExchangeThreads) exchange_rows_kernel(PeerView v, uint32_t parity, uint32_t epoch,
                                                             uint64_t nq, uint32_t qs, uint32_t nslices,
                                                             const uint32_t* __restrict__ ids,
                                                             const float* __restrict__ vecs, uint32_t dpad,
                                                             uint32_t dim, uint64_t digest,
                                                             uint32_t* __restrict__ verdict,
                                                             uint32_t* __restrict__ timeout_flag) {
  const uint32_t W = v.L.world, me = v.rank;
  const uint32_t warps = blockDim.x >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // each parity's part of the row region is 256-byte aligned (exchange_layout.cuh), so a row q * dim floats in is
  // 16-byte aligned when dim is; dpad is a multiple of 4
  const bool vec4 = (dim & 3) == 0;
  // ---- phase 1: rows, marks and digest to every rank, then the flags ------------------------------------------
  for (uint32_t s = blockIdx.x; s < nslices; s += gridDim.x) {
    const uint64_t q0 = min(nq, (uint64_t)s * qs), q1 = min(nq, q0 + qs);
    for (uint64_t q = q0 + w; q < q1; q += warps) {
      const uint32_t id = ids[q];
      if (id == kInvalid) continue;
      const float* src = vecs + (uint64_t)id * dpad;
      const uint64_t at = q * dim;
      if (vec4) {
        for (uint32_t c = lane; c < dim / 4; c += 32) {
          const float4 x = reinterpret_cast<const float4*>(src)[c];
          for (uint32_t g = 0; g < W; ++g) *reinterpret_cast<float4*>(v.L.rows(v.base[g], parity, at + 4 * c)) = x;
        }
      } else {
        for (uint32_t c = lane; c < dim; c += 32) {
          const float x = src[c];
          for (uint32_t g = 0; g < W; ++g) *v.L.rows(v.base[g], parity, at + c) = x;
        }
      }
    }
    for (uint64_t q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
      const unsigned char held = ids[q] != kInvalid;
      for (uint32_t g = 0; g < W; ++g) v.L.marks(v.base[g], parity, me)[q] = held;
    }
    if (s == 0 && threadIdx.x < W) *v.L.digest(v.base[threadIdx.x], parity, me) = digest;
    publish_slice(v, parity, epoch, s);
  }
  // ---- phase 2: wait for each slice from every peer, count the holders ---------------------------------------
  for (uint32_t s = blockIdx.x; s < nslices; s += gridDim.x) {
    uint32_t bits = await_slice(v, parity, epoch, s, timeout_flag) ? kRowsTimeout : 0u;
    const uint64_t q0 = min(nq, (uint64_t)s * qs), q1 = min(nq, q0 + qs);
    for (uint64_t q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
      uint32_t holders = 0;
      for (uint32_t g = 0; g < W; ++g) holders += v.L.marks(v.base[me], parity, g)[q];
      bits |= holders == 0 ? kRowsMissing : holders > 1 ? kRowsShared : 0u;
    }
    if (s == 0 && threadIdx.x < W && *v.L.digest(v.base[me], parity, threadIdx.x) != digest) bits |= kRowsDigest;
    if (bits) atomicOr(verdict, bits);
  }
}

}  // namespace ehb

// =====================================================================================================
// ehb_exchange: one process per GPU
// =====================================================================================================
struct ehb_exchange {
  int device = 0;
  uint32_t world = 1, rank = 0;
  ehb::ExchangeLayout L{};  // of the exported allocation, the same on every rank
  uint64_t max_elems = 0;
  uint32_t max_dim = 0;
  ehb::DevBuf<unsigned char> local;  // the exported allocation: ONE, because an IPC handle covers one allocation
  unsigned char* mapped[ehb::kMaxWorld] = {nullptr};  // base of every rank's allocation as mapped here
  bool opened[ehb::kMaxWorld] = {false};
  bool attached = false;
  ehb::DevBuf<uint32_t> slice_count;  // [kMaxSlices], zero between steps (raised by the walk's epilogue)
  uint32_t same_device_ranks = 1;  // ranks (this one included) whose exchange kernels share this GPU (tests)
  uint32_t epoch = 0;
  uint64_t slot_nq = 0;
  uint32_t slot_k = 0;
  int sms = 132;
  std::mutex mu;
  // by-label steps (max_dim > 0).  Local scratch: the resolved ids, the query labels, the merged k + 1 lists, the
  // verdict word; pinned staging of the labels, ids and verdict; `bl_done` ends the last by-label step's use of them.
  ehb::DevBuf<uint32_t> bl_ids, bl_counts, bl_verdict;
  ehb::DevBuf<uint64_t> bl_self, bl_labels;
  ehb::DevBuf<float> bl_dists;
  ehb::PinBuf h_self, h_ids, h_verdict;
  cudaEvent_t bl_done = nullptr;

  // Waits for this rank's work and closes the peers' mappings before the buffers free themselves.
  ~ehb_exchange() {
    cudaSetDevice(device);
    cudaDeviceSynchronize();
    for (uint32_t g = 0; g < world; ++g)
      if (opened[g]) cudaIpcCloseMemHandle(mapped[g]);
    if (bl_done) cudaEventDestroy(bl_done);
  }
};

extern "C" {

// Everything a step uses is allocated here: a cudaFree inside a step waits for the whole device, which with two ranks
// on one GPU means a peer's spinning kernel.
int ehb_exchange_create_ex(int32_t device, uint32_t world, uint32_t rank, uint64_t max_nq, uint32_t max_k,
                           uint32_t max_dim, ehb_exchange** out) {
  if (!out) return fail(EHB_ERR_INVALID, "null argument");
  if (world == 0 || world > ehb::kMaxWorld || rank >= world) return fail(EHB_ERR_INVALID, "bad world / rank");
  if (max_nq == 0 || max_k == 0) return fail(EHB_ERR_INVALID, "max_nq and max_k must be positive");
  if (max_dim > ehb::kMaxDim) return fail(EHB_ERR_INVALID, "max_dim must be <= 4096");
  CU(cudaSetDevice(device));
  ehb_exchange* ex = new (std::nothrow) ehb_exchange();
  if (!ex) return fail(EHB_ERR_OOM, "host allocation failed");
  ex->device = device;
  ex->world = world;
  ex->rank = rank;
  ex->L = ehb::ExchangeLayout::make(world, max_nq, max_k, max_dim);
  ex->max_elems = max_nq * max_k;
  ex->max_dim = max_dim;
  cudaDeviceGetAttribute(&ex->sms, cudaDevAttrMultiProcessorCount, device);
  cudaError_t e = cudaSuccess;
  auto dev = [&](auto& buf, size_t n, int fill) {
    if (e == cudaSuccess) e = buf.grow(n, 0, fill, nullptr);
  };
  auto pin = [&](ehb::PinBuf& buf, size_t bytes) {
    if (e == cudaSuccess) e = buf.reserve(bytes);
  };
  dev(ex->local, ex->L.total_bytes, -1);
  if (e == cudaSuccess) e = cudaMemset(ex->local.p, 0, ex->L.flag_bytes);
  dev(ex->slice_count, ehb::kMaxSlices, 0);
  if (max_dim) {
    dev(ex->bl_ids, max_nq, -1);
    dev(ex->bl_self, max_nq, -1);
    dev(ex->bl_labels, ex->max_elems, -1);
    dev(ex->bl_dists, ex->max_elems, -1);
    dev(ex->bl_counts, max_nq, -1);
    dev(ex->bl_verdict, 1, -1);
    pin(ex->h_self, max_nq * 8);
    pin(ex->h_ids, max_nq * 4);
    pin(ex->h_verdict, 4);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ex->bl_done, cudaEventDisableTiming);
    // load the step's own kernels now: under lazy module loading a first launch may wait for every kernel running in
    // the context, and with two ranks in one process one of those is a peer's exchange kernel waiting for this rank
    cudaFuncAttributes a;
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, ehb::exchange_rows_kernel);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, ehb::exchange_merge_kernel);
    if (e == cudaSuccess) e = ehb::load_drop_self();
  }
  if (e != cudaSuccess) {
    delete ex;
    return fail(e == cudaErrorMemoryAllocation ? EHB_ERR_OOM : EHB_ERR_CUDA, cudaGetErrorString(e));
  }
  ex->mapped[rank] = ex->local.p;
  ex->attached = world == 1;
  *out = ex;
  return EHB_OK;
}

int ehb_exchange_create(int32_t device, uint32_t world, uint32_t rank, uint64_t max_nq, uint32_t max_k,
                        ehb_exchange** out) {
  return ehb_exchange_create_ex(device, world, rank, max_nq, max_k, 0, out);
}

int ehb_exchange_destroy(ehb_exchange* ex) {
  delete ex;
  return EHB_OK;
}

// 64 bytes (cudaIpcMemHandle_t) other ranks pass to ehb_exchange_open.
int ehb_exchange_ipc_handle(ehb_exchange* ex, void* out_handle) {
  if (!ex || !out_handle) return fail(EHB_ERR_INVALID, "null argument");
  CU(cudaSetDevice(ex->device));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, ex->local.p));
  static_assert(sizeof(cudaIpcMemHandle_t) == EHB_IPC_HANDLE_BYTES, "handle size");
  std::memcpy(out_handle, &h, sizeof(h));
  return EHB_OK;
}

// handles: [world][64] in rank order (this rank's own entry is ignored).
int ehb_exchange_open(ehb_exchange* ex, const void* handles) {
  if (!ex || !handles) return fail(EHB_ERR_INVALID, "null argument");
  CU(cudaSetDevice(ex->device));
  for (uint32_t g = 0; g < ex->world; ++g) {
    if (g == ex->rank || ex->opened[g]) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, (const unsigned char*)handles + (size_t)g * EHB_IPC_HANDLE_BYTES, sizeof(h));
    void* p = nullptr;
    CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ex->mapped[g] = (unsigned char*)p;
    ex->opened[g] = true;
  }
  ex->attached = true;
  return EHB_OK;
}

// Same process, different device: attach a peer exchange directly (peer access must be possible).
int ehb_exchange_attach_local(ehb_exchange* ex, uint32_t peer_rank, ehb_exchange* peer) {
  if (!ex || !peer || peer_rank >= ex->world || peer_rank == ex->rank) return fail(EHB_ERR_INVALID, "bad argument");
  if (peer->max_dim != ex->max_dim) return fail(EHB_ERR_INVALID, "the peers' max_dim differ (their row regions would)");
  CU(cudaSetDevice(ex->device));
  if (peer->device != ex->device) {
    int can = 0;
    CU(cudaDeviceCanAccessPeer(&can, ex->device, peer->device));
    if (!can) return fail(EHB_ERR_CUDA, "devices cannot access each other's memory");
    cudaError_t e = cudaDeviceEnablePeerAccess(peer->device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU(e);
    cudaGetLastError();
  }
  if (!ex->mapped[peer_rank] && peer->device == ex->device) ex->same_device_ranks++;
  ex->mapped[peer_rank] = peer->local.p;
  bool all = true;
  for (uint32_t g = 0; g < ex->world; ++g) all = all && ex->mapped[g] != nullptr;
  ex->attached = all;
  return EHB_OK;
}

// Starts a step: returns where THIS rank's search must write its [nq][k] labels and distances.
int ehb_exchange_begin(ehb_exchange* ex, uint64_t nq, uint32_t k, uint64_t** labels_dev, float** dists_dev) {
  if (!ex || !labels_dev || !dists_dev) return fail(EHB_ERR_INVALID, "null argument");
  if (nq == 0 || k == 0 || nq * k > ex->max_elems) return fail(EHB_ERR_INVALID, "nq * k exceeds the exchange capacity");
  if (!ex->attached) return fail(EHB_ERR_STATE, "peers are not attached yet");
  std::lock_guard<std::mutex> g(ex->mu);
  ex->epoch++;
  ex->slot_nq = nq;
  ex->slot_k = k;
  const uint32_t parity = ex->epoch & 1u;
  unsigned char* blk = ex->L.recv(ex->local.p, parity, ex->rank);
  *labels_dev = (uint64_t*)blk;
  *dists_dev = (float*)(blk + nq * k * 8ull);
  return EHB_OK;
}

}  // extern "C"

namespace {

// slices of whole queries, a multiple of 4 queries so every slice boundary is 16 B aligned
void slice_plan(const ehb_exchange* ex, uint64_t nq, uint32_t* qs, uint32_t* nslices) {
  uint32_t target = std::min<uint32_t>(ehb::kMaxSlices, (uint32_t)ex->sms);
  uint32_t per = (uint32_t)((nq + target - 1) / target);
  per = (per + 3) / 4 * 4;
  *qs = per;
  *nslices = (uint32_t)((nq + per - 1) / per);
}

// Every rank's mapping of the exported allocation, as the exchange kernels and step_sink read it.
ehb::PeerView peer_view(const ehb_exchange* ex) {
  ehb::PeerView v{};
  std::copy(ex->mapped, ex->mapped + ex->world, v.base);
  v.rank = ex->rank;
  v.L = ex->L;
  return v;
}

// Every CTA of an exchange kernel must be resident (a waiting CTA may depend on a peer's CTA): one CTA per SM, and
// when several ranks share this GPU (single-GPU tests) they split the SMs.
uint32_t resident_grid(const ehb_exchange* ex, uint32_t nslices) {
  return std::min<uint32_t>(nslices, std::max<uint32_t>(1, (uint32_t)ex->sms / ex->same_device_ranks));
}

int launch_exchange_merge(ehb_exchange* ex, uint64_t nq, uint32_t k, float* out_dists_dev, uint64_t* out_labels_dev,
                          uint32_t* out_counts_dev, cudaStream_t stream, bool skip_push) {
  uint32_t qs, nslices;
  slice_plan(ex, nq, &qs, &nslices);
  ehb::exchange_merge_kernel<<<resident_grid(ex, nslices), ehb::kExchangeThreads, 0, stream>>>(
      peer_view(ex), ex->epoch & 1u, ex->epoch, nq, k, qs, nslices, out_dists_dev, out_labels_dev, out_counts_dev,
      ex->L.timeout(ex->local.p), skip_push ? 1u : 0u);
  CU(cudaGetLastError());
  return EHB_OK;
}

static_assert(ehb::kMaxSinks >= ehb::kMaxWorld, "step_sink gives every rank a destination");

// The destinations of this rank's [nq][k] results at the current epoch: its own block of its own buffer first, then
// its block of every peer's buffer, with the slice flags the search's last kernel raises.
ehb::ResultSink step_sink(ehb_exchange* ex, uint64_t nq, uint32_t k) {
  const ehb::PeerView v = peer_view(ex);
  const uint32_t parity = ex->epoch & 1u, me = ex->rank;
  uint32_t qs, nslices;
  slice_plan(ex, nq, &qs, &nslices);
  ehb::ResultSink sink;
  std::memset(&sink, 0, sizeof(sink));
  uint32_t t = 0;
  auto add = [&](uint32_t r) {
    unsigned char* blk = v.L.recv(v.base[r], parity, me);
    sink.labels[t] = (uint64_t*)blk;
    sink.dists[t] = (float*)(blk + nq * k * 8ull);
    sink.flags[t] = v.L.flags(v.base[r], parity, me);
    ++t;
  };
  add(me);  // destination 0 = my own block of my own buffer
  for (uint32_t r = 0; r < ex->world; ++r)
    if (r != me) add(r);
  sink.n = t;
  sink.qs = qs;
  sink.epoch = ex->epoch;
  sink.slice_count = ex->slice_count.p;
  return sink;
}

// The row step of a by-label search at the current epoch.  Its slice count does not depend on nq (every rank raises
// the same flags whatever list it was given); the verdict word must be zero on `stream`.
int launch_exchange_rows(ehb_exchange* ex, const ehb_index* ix, uint64_t nq, uint64_t digest, cudaStream_t stream) {
  const uint32_t nslices = std::min<uint32_t>(ehb::kMaxSlices, (uint32_t)ex->sms);
  const uint32_t qs = (uint32_t)((nq + nslices - 1) / nslices);
  ehb::exchange_rows_kernel<<<resident_grid(ex, nslices), ehb::kExchangeThreads, 0, stream>>>(
      peer_view(ex), ex->epoch & 1u, ex->epoch, nq, qs, nslices, ex->bl_ids.p, ix->vecs.p, ix->dpad, ix->dim, digest,
      ex->bl_verdict.p, ex->L.timeout(ex->local.p));
  CU(cudaGetLastError());
  return EHB_OK;
}

// 64-bit digest of a label list (its length included): splitmix64's finaliser over a running sum
uint64_t label_digest(uint64_t nq, const uint64_t* labels) {
  auto mix = [](uint64_t z) {
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
  };
  uint64_t h = mix(nq + 0x9e3779b97f4a7c15ull);
  for (uint64_t i = 0; i < nq; ++i) h = mix(h + 0x9e3779b97f4a7c15ull + labels[i]);
  return h;
}

}  // namespace

extern "C" {

// Finishes the step on `stream` (the stream the search was queued on): push + flags + wait + merge.
int ehb_exchange_merge_dev(ehb_exchange* ex, float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev,
                           void* stream) {
  if (!ex || !out_labels_dev) return fail(EHB_ERR_INVALID, "null argument");
  CU(cudaSetDevice(ex->device));
  std::lock_guard<std::mutex> g(ex->mu);
  if (!ex->slot_nq) return fail(EHB_ERR_STATE, "ehb_exchange_begin was not called");
  const uint64_t nq = ex->slot_nq;
  const uint32_t k = ex->slot_k;
  ex->slot_nq = 0;
  return launch_exchange_merge(ex, nq, k, out_dists_dev, out_labels_dev, out_counts_dev, (cudaStream_t)stream, false);
}

// One sharded graph search step, fused: this rank's search stores every query's top-k straight into every peer's
// receive buffer from its last kernel (the fp32 walk's epilogue, the wide-beam walk's, or the re-rank after a bf16
// walk: coalesced stores over NVLink while the other queries are still running) and raises per-slice flags; then one
// kernel waits for the peers' flags and merges.  Falls back to push-after-walk when the batch is small enough for the
// team walk (fp32 only).  Call in lock step on every rank.  Everything that can be rejected is checked before the
// epoch advances, and the wide-beam scratch is grown before it too: a rank that failed after it would be one step out
// of phase with its peers, whose merges would then wait for it until they time out.  Locks in the order of the
// by-label step: ex->mu, then the reader side of ix->rw, held from the check through the search launch so that the
// walk plan the scratch was reserved for is the one that runs.  max_beam: 512 (_ex) or kMaxBeam (_beam).
static int exchange_fused_step(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                               uint32_t ef, int precision, float* out_dists_dev, uint64_t* out_labels_dev,
                               uint32_t* out_counts_dev, uint32_t* shard_counts_dev, void* stream, uint32_t max_beam) {
  if (!ex || !ix) return fail(EHB_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(ex->mu);
  std::shared_lock<ehb::RwLock> lk(ix->rw);
  bool none;
  RET(ehb::check_request(ix, false, precision, !queries_dev || !out_labels_dev, nq, k, k, &ef, &none, max_beam));
  if (none || nq * k > ex->max_elems) return fail(EHB_ERR_INVALID, "nq * k exceeds the exchange capacity");
  if (!ex->attached) return fail(EHB_ERR_STATE, "peers are not attached yet");
  CU(cudaSetDevice(ex->device));
  const cudaStream_t s = (cudaStream_t)stream;
  RET(ix->prepare(lk, false, precision, nq));
  RET(ix->reserve_beam(nq, std::max(ef, k), precision, s));
  ex->epoch++;
  const ehb::ResultSink sink = step_sink(ex, nq, k);
  bool pushed = false;
  RET(ehb_index_search_dev_sink_held(ix, lk, nq, queries_dev, k, ef, precision, &sink, shard_counts_dev, s, &pushed,
                                     max_beam));
  CU(cudaSetDevice(ex->device));
  return launch_exchange_merge(ex, nq, k, out_dists_dev, out_labels_dev, out_counts_dev, s, pushed);
}

int ehb_exchange_search_ex_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                               uint32_t ef, int precision, float* out_dists_dev, uint64_t* out_labels_dev,
                               uint32_t* out_counts_dev, uint32_t* shard_counts_dev, void* stream) {
  return exchange_fused_step(ex, ix, nq, queries_dev, k, ef, precision, out_dists_dev, out_labels_dev, out_counts_dev,
                             shard_counts_dev, stream, ehb::kMaxEf);
}
int ehb_exchange_search_beam_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                                 uint32_t ef, int precision, float* out_dists_dev, uint64_t* out_labels_dev,
                                 uint32_t* out_counts_dev, uint32_t* shard_counts_dev, void* stream) {
  return exchange_fused_step(ex, ix, nq, queries_dev, k, ef, precision, out_dists_dev, out_labels_dev, out_counts_dev,
                             shard_counts_dev, stream, ehb::kMaxBeam);
}

// Key mode over the exchange: a row step at epoch e (every holder pushes its stored rows to every rank, and every
// rank agrees that each label has exactly one holder and that all ranks were given the same list), then the fused
// k + 1 step at e + 1 over the pushed rows, the merge, and the self-removal.  The reader side of ix->rw is held from
// prepare through the search launch, so the resolved ids cannot move under a compaction.  Locks in the order of
// ehb_exchange_search_ex_dev: ex->mu first, then ix->rw (a writer-preferring lock taken in the other order by a
// second thread on the same exchange could deadlock).  The wide-beam scratch of the k + 1 search is grown before the
// first epoch, like every check.  max_beam: 512 (_ex) or kMaxBeam (_beam).
static int exchange_by_label_step(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const uint64_t* labels_host,
                                  uint32_t k, uint32_t ef, int precision, float* out_dists_dev,
                                  uint64_t* out_labels_dev, uint32_t* out_counts_dev, void* stream,
                                  uint32_t max_beam) {
  if (!ex || !ix) return fail(EHB_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(ex->mu);
  std::shared_lock<ehb::RwLock> lk(ix->rw);
  bool none;
  RET(ehb::check_request(ix, false, precision, !labels_host || !out_labels_dev || !out_dists_dev || !out_counts_dev,
                         nq, k, k + 1ull, &ef, &none, max_beam));
  if (none) return EHB_OK;
  const uint32_t k1 = k + 1;
  if (nq > ex->L.max_nq || nq * k1 > ex->max_elems)
    return fail(EHB_ERR_INVALID, "nq or nq * (k + 1) exceeds the exchange capacity");
  if (ix->dim > ex->max_dim) return fail(EHB_ERR_INVALID, "the exchange has no room for rows of this dim (max_dim)");
  if (!ex->attached) return fail(EHB_ERR_STATE, "peers are not attached yet");
  CU(cudaSetDevice(ex->device));
  const cudaStream_t s = (cudaStream_t)stream;
  RET(ix->prepare(lk, false, precision, nq));
  RET(ix->reserve_beam(nq, std::max(ef, k1), precision, s));
  uint64_t* h_self = (uint64_t*)ex->h_self.p;
  uint32_t* h_ids = (uint32_t*)ex->h_ids.p;
  uint32_t* h_verdict = (uint32_t*)ex->h_verdict.p;
  // hnswlib getDataByLabel, as ehb_index_get_batch: a tombstoned label is not held
  for (uint64_t q = 0; q < nq; ++q)
    if (!ix->find_id(labels_host[q], &h_ids[q]) || ix->h_deleted[h_ids[q]]) h_ids[q] = ehb::kInvalid;
  std::memcpy(h_self, labels_host, nq * 8);
  CU(cudaStreamWaitEvent(s, ex->bl_done, 0));  // the previous by-label step is done with the scratch
  ex->epoch++;
  const uint32_t parity = ex->epoch & 1u;
  CU(cudaMemsetAsync(ex->bl_verdict.p, 0, 4, s));
  CU(cudaMemcpyAsync(ex->bl_ids.p, h_ids, nq * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(ex->bl_self.p, h_self, nq * 8, cudaMemcpyHostToDevice, s));
  RET(launch_exchange_rows(ex, ix, nq, label_digest(nq, labels_host), s));
  CU(cudaMemcpyAsync(h_verdict, ex->bl_verdict.p, 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));  // the step's only host synchronisation
  // every rank reads the same verdict and returns the same status; each has consumed epoch e, so they stay in phase.
  // The digests decide first: they are fresh whatever lists the ranks were given, and a digest mismatch is seen by
  // every rank.  Only when the lists agree (so nq agrees) are the marks all of this step, and the holder counts used.
  const uint32_t v = *h_verdict;
  if (v & ehb::kRowsTimeout) return fail(EHB_ERR_CUDA, "a peer did not arrive within ~20 s (ehb_exchange_timed_out)");
  if (v & ehb::kRowsDigest) return fail(EHB_ERR_INVALID, "the ranks were given different label lists");
  if (v & ehb::kRowsMissing) return fail(EHB_ERR_NOT_FOUND, "label not found on any rank");
  if (v & ehb::kRowsShared) return fail(EHB_ERR_STATE, "a label is stored on more than one rank");
  ex->epoch++;
  const float* rows = ex->L.rows(ex->local.p, parity);
  const ehb::ResultSink sink = step_sink(ex, nq, k1);
  bool pushed = false;
  RET(ehb_index_search_dev_sink_held(ix, lk, nq, rows, k1, ef, precision, &sink, nullptr, s, &pushed, max_beam));
  CU(cudaSetDevice(ex->device));
  RET(launch_exchange_merge(ex, nq, k1, ex->bl_dists.p, ex->bl_labels.p, ex->bl_counts.p, s, pushed));
  CU(ehb::launch_drop_self(ex->bl_self.p, ex->bl_labels.p, ex->bl_dists.p, ex->bl_counts.p, nq, k, out_labels_dev,
                           out_dists_dev, out_counts_dev, s));
  CU(cudaEventRecord(ex->bl_done, s));
  return EHB_OK;
}

int ehb_exchange_search_by_label_ex_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const uint64_t* labels_host,
                                        uint32_t k, uint32_t ef, int precision, float* out_dists_dev,
                                        uint64_t* out_labels_dev, uint32_t* out_counts_dev, void* stream) {
  return exchange_by_label_step(ex, ix, nq, labels_host, k, ef, precision, out_dists_dev, out_labels_dev,
                                out_counts_dev, stream, ehb::kMaxEf);
}
int ehb_exchange_search_by_label_beam_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const uint64_t* labels_host,
                                          uint32_t k, uint32_t ef, int precision, float* out_dists_dev,
                                          uint64_t* out_labels_dev, uint32_t* out_counts_dev, void* stream) {
  return exchange_by_label_step(ex, ix, nq, labels_host, k, ef, precision, out_dists_dev, out_labels_dev,
                                out_counts_dev, stream, ehb::kMaxBeam);
}

int ehb_exchange_search_dev(ehb_exchange* ex, ehb_index* ix, uint64_t nq, const float* queries_dev, uint32_t k,
                            uint32_t ef, float* out_dists_dev, uint64_t* out_labels_dev, uint32_t* out_counts_dev,
                            uint32_t* shard_counts_dev, void* stream) {
  return ehb_exchange_search_ex_dev(ex, ix, nq, queries_dev, k, ef, EHB_FP32, out_dists_dev, out_labels_dev,
                                    out_counts_dev, shard_counts_dev, stream);
}

// 1 when some exchange kernel of this rank gave up waiting for a peer (its results are then invalid).
int ehb_exchange_timed_out(ehb_exchange* ex, uint32_t* out) {
  if (!ex || !out) return fail(EHB_ERR_INVALID, "null argument");
  CU(cudaSetDevice(ex->device));
  CU(cudaMemcpy(out, ex->L.timeout(ex->local.p), 4, cudaMemcpyDeviceToHost));
  return EHB_OK;
}

}  // extern "C"

// =====================================================================================================
// ehb_sharded: one process, n_dev GPUs
// =====================================================================================================
namespace ehb {
// One shard of an ehb_sharded: its index, its device, and the stream, event and buffers it searches with.
struct Shard {
  ehb_index* ix;
  int dev;
  cudaStream_t st = nullptr;
  cudaEvent_t done = nullptr;
  DevBuf<float> q_dev;              // the queries
  DevBuf<unsigned char> local_out;  // [labels | dists] when this device cannot store into device 0
  DevBuf<uint32_t> cnt_dev;
  // by-label searches: the gathered rows in owner order and each row's query position
  DevBuf<float> q_stage;
  DevBuf<uint32_t> q_pos;

  Shard(ehb_index* ix, int dev) : ix(ix), dev(dev) {}
  // Waits for the device before anything is freed; the buffers free themselves after, still on this device.
  ~Shard() {
    cudaSetDevice(dev);
    cudaDeviceSynchronize();
    if (st) cudaStreamDestroy(st);
    if (done) cudaEventDestroy(done);
    ehb_index_destroy(ix);
  }
};
}  // namespace ehb

struct ehb_sharded {
  std::vector<std::unique_ptr<ehb::Shard>> shards;
  uint64_t span = 0;  // labels per shard range (0: label % n_dev)
  ehb_params prm;
  bool peer_direct = true;  // every device can store into device 0
  // device-0 gather + result buffers
  ehb::DevBuf<unsigned char> gather;       // [n_dev][labels | dists]
  ehb::DevBuf<float> m_dists;
  ehb::DevBuf<uint64_t> m_labels;
  ehb::DevBuf<uint32_t> m_counts;
  // by-label searches, on device 0: the query labels and the results after self-removal
  ehb::DevBuf<uint64_t> s_self, s_labels;
  ehb::DevBuf<float> s_dists;
  ehb::DevBuf<uint32_t> s_counts;
  cudaEvent_t q_ready = nullptr;
  std::mutex mu;
  uint64_t next_label = 0;

  // The shards go first; the device-0 buffers free themselves after, on device 0.
  ~ehb_sharded() {
    if (shards.empty()) return;
    const int dev0 = shards[0]->dev;
    shards.clear();
    cudaSetDevice(dev0);
    if (q_ready) cudaEventDestroy(q_ready);
  }

  uint32_t owner(uint64_t label) const {
    const uint64_t G = shards.size();
    return (uint32_t)(span ? (label / span) % G : label % G);
  }
};

extern "C" {

int ehb_sharded_destroy(ehb_sharded* sh) {
  delete sh;
  return EHB_OK;
}

// ehb_index_create over device_ids[0..n_dev): p->device is ignored, p->capacity is per shard.
// shard_span: labels [i*span, (i+1)*span) live on shard i % n_dev (0 = label % n_dev).
int ehb_sharded_create(const ehb_params* p, const int32_t* device_ids, uint32_t n_dev, uint64_t shard_span,
                       ehb_sharded** out) {
  if (!p || !device_ids || !out) return fail(EHB_ERR_INVALID, "null argument");
  if (n_dev == 0 || n_dev > ehb::kMaxWorld) return fail(EHB_ERR_INVALID, "n_dev must be in 1..16");
  // (a device may be listed more than once: several shards then share it — useful on one GPU)
  ehb_sharded* sh = new (std::nothrow) ehb_sharded();
  if (!sh) return fail(EHB_ERR_OOM, "host allocation failed");
  sh->prm = *p;
  sh->span = shard_span;
  auto body = [&]() -> int {
    for (uint32_t g = 0; g < n_dev; ++g) {
      ehb_params pg = *p;
      pg.device = device_ids[g];
      ehb_index* ix = nullptr;
      RET(ehb_index_create(&pg, &ix));
      sh->shards.push_back(std::make_unique<ehb::Shard>(ix, device_ids[g]));
      ehb::Shard& s = *sh->shards.back();
      CU(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
      CU(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
      if (g > 0 && device_ids[g] != device_ids[0]) {  // device g must be able to store into device 0
        int can = 0;
        CU(cudaDeviceCanAccessPeer(&can, device_ids[g], device_ids[0]));
        if (can) {
          cudaError_t pe = cudaDeviceEnablePeerAccess(device_ids[0], 0);
          if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CU(pe);
          cudaGetLastError();
        } else {
          sh->peer_direct = false;
        }
      }
    }
    CU(cudaSetDevice(device_ids[0]));
    CU(cudaEventCreateWithFlags(&sh->q_ready, cudaEventDisableTiming));
    return EHB_OK;
  };
  int rc = body();
  if (rc != EHB_OK) {
    const std::string msg = ehb::last_error_text();
    delete sh;
    return fail(rc, msg);
  }
  *out = sh;
  return EHB_OK;
}

int ehb_sharded_n_shards(ehb_sharded* sh, uint32_t* out) {
  if (!sh || !out) return fail(EHB_ERR_INVALID, "null argument");
  *out = (uint32_t)sh->shards.size();
  return EHB_OK;
}

// Borrow shard i (stats, tuning); owned by the sharded index.
int ehb_sharded_shard(ehb_sharded* sh, uint32_t i, ehb_index** out) {
  if (!sh || !out || i >= sh->shards.size()) return fail(EHB_ERR_INVALID, "bad argument");
  *out = sh->shards[i]->ix;
  return EHB_OK;
}

// Insert-or-update, routed by label range; no communication between shards (SURVEY.md §8e).
int ehb_sharded_add(ehb_sharded* sh, uint64_t n, const float* vecs, const uint64_t* labels) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  if (n && !vecs) return fail(EHB_ERR_INVALID, "null vectors");
  std::lock_guard<std::mutex> g(sh->mu);
  const size_t G = sh->shards.size(), dim = sh->prm.dim;
  std::vector<std::vector<float>> rows(G);
  std::vector<std::vector<uint64_t>> labs(G);
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t l = labels ? labels[i] : sh->next_label + i;
    const uint32_t o = sh->owner(l);
    rows[o].insert(rows[o].end(), vecs + i * dim, vecs + (i + 1) * dim);
    labs[o].push_back(l);
  }
  for (size_t o = 0; o < G; ++o)
    if (!labs[o].empty()) RET(ehb_index_add(sh->shards[o]->ix, labs[o].size(), rows[o].data(), labs[o].data()));
  if (!labels) sh->next_label += n;
  return EHB_OK;
}

int ehb_sharded_remove(ehb_sharded* sh, uint64_t n, const uint64_t* labels) {
  if (!sh || (n && !labels)) return fail(EHB_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(sh->mu);
  for (uint64_t i = 0; i < n; ++i) RET(ehb_index_remove(sh->shards[sh->owner(labels[i])]->ix, 1, labels + i));
  return EHB_OK;
}

int ehb_sharded_get(ehb_sharded* sh, uint64_t label, float* out) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  return ehb_index_get(sh->shards[sh->owner(label)]->ix, label, out);
}

int ehb_sharded_size(ehb_sharded* sh, uint64_t* out) {
  if (!sh || !out) return fail(EHB_ERR_INVALID, "null argument");
  uint64_t tot = 0, v = 0;
  for (const auto& s : sh->shards) {
    RET(ehb_index_size(s->ix, &v));
    tot += v;
  }
  *out = tot;
  return EHB_OK;
}

// Runs fn on every shard concurrently (one host thread per device) and reports the first shard's error.
static int on_every_shard(ehb_sharded* sh, int (*fn)(ehb_index*)) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  std::lock_guard<std::mutex> g(sh->mu);
  const size_t G = sh->shards.size();
  std::vector<int> rc(G, EHB_OK);
  std::vector<std::string> msg(G);
  std::vector<std::thread> th;
  for (size_t i = 0; i < G; ++i)
    th.emplace_back([&, i]() {
      rc[i] = fn(sh->shards[i]->ix);
      if (rc[i] != EHB_OK) msg[i] = ehb::last_error_text();
    });
  for (auto& t : th) t.join();
  for (size_t i = 0; i < G; ++i)
    if (rc[i] != EHB_OK) return fail(rc[i], msg[i]);
  return EHB_OK;
}

// Links every shard; the shards build concurrently.
int ehb_sharded_build(ehb_sharded* sh) { return on_every_shard(sh, ehb_index_build); }

// Compacts every shard; the shards compact concurrently.
int ehb_sharded_compact(ehb_sharded* sh) { return on_every_shard(sh, ehb_index_compact); }

int ehb_sharded_set_ef(ehb_sharded* sh, uint32_t ef) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  for (const auto& s : sh->shards) RET(ehb_index_set_ef(s->ix, ef));
  return EHB_OK;
}

// Every shard searches, device 0 merges into m_labels / m_dists / m_counts (queued on st[0]).  Caller holds mu.
// q: host queries, or nullptr when every q_dev already holds them (queued on the shards' streams).
// brute: the exact / bf16 brute force instead of the graph walk (a bf16 walk re-ranks straight into device 0's gather
// block, like the fp32 walk).  beam: ehb_index_search_beam_dev on every shard instead of ehb_index_search_ex_dev.
static int sharded_merge(ehb_sharded* sh, bool brute, uint64_t nq, const float* q, uint32_t k, uint32_t ef,
                         int precision, bool beam = false) {
  const uint32_t G = (uint32_t)sh->shards.size();
  const uint32_t dim = sh->prm.dim;
  const uint64_t blk = (nq * k * 12ull + 255) / 256 * 256;
  const int dev0 = sh->shards[0]->dev;
  CU(cudaSetDevice(dev0));
  cudaStream_t s0 = sh->shards[0]->st;
  CU(sh->gather.grow(blk * G, 0, -1, s0));
  CU(sh->m_labels.grow(nq * k, 0, -1, s0));
  CU(sh->m_dists.grow(nq * k, 0, -1, s0));
  CU(sh->m_counts.grow(nq, 0, -1, s0));
  CU(cudaEventRecord(sh->q_ready, s0));  // orders the peers' stores after earlier merges on device 0
  for (uint32_t i = 0; i < G; ++i) {
    ehb::Shard& sd = *sh->shards[i];
    CU(cudaSetDevice(sd.dev));
    cudaStream_t s = sd.st;
    CU(sd.q_dev.grow(nq * dim, 0, -1, s));
    CU(sd.cnt_dev.grow(nq, 0, -1, s));
    if (q) CU(cudaMemcpyAsync(sd.q_dev.p, q, nq * dim * 4, cudaMemcpyHostToDevice, s));
    unsigned char* dst;
    if (i == 0 || sh->peer_direct || sd.dev == dev0) {
      dst = sh->gather.p + blk * i;  // device i's kernels store straight into device 0's gather block
      if (i) CU(cudaStreamWaitEvent(s, sh->q_ready, 0));
    } else {
      CU(sd.local_out.grow(blk, 0, -1, s));
      dst = sd.local_out.p;
    }
    uint64_t* dl = (uint64_t*)dst;
    float* dd = (float*)(dst + nq * k * 8ull);
    if (brute)
      RET(ehb_index_search_bruteforce_dev(sd.ix, nq, sd.q_dev.p, k, precision, dl, dd, sd.cnt_dev.p, s));
    else
      RET((beam ? ehb_index_search_beam_dev : ehb_index_search_ex_dev)(sd.ix, nq, sd.q_dev.p, k, ef, precision, dl, dd,
                                                                       sd.cnt_dev.p, s));
    CU(cudaSetDevice(sd.dev));
    if (i && !sh->peer_direct && sd.dev != dev0)
      CU(cudaMemcpyPeerAsync(sh->gather.p + blk * i, dev0, dst, sd.dev, nq * k * 12ull, s));
    CU(cudaEventRecord(sd.done, s));
  }
  CU(cudaSetDevice(dev0));
  for (uint32_t i = 1; i < G; ++i) CU(cudaStreamWaitEvent(s0, sh->shards[i]->done, 0));
  CU(ehb::launch_merge_topk(G, nq, k, (const float*)(sh->gather.p + nq * k * 8ull), (const uint64_t*)sh->gather.p, blk,
                            blk, sh->m_dists.p, sh->m_labels.p, sh->m_counts.p, s0));
  return EHB_OK;
}

// ehb::check_request on every shard, each under its reader lock (ef == 0 reads the shard's default; each shard's search
// resolves and checks it again under its own lock).  max_beam: the graph walk's width limit (512, or kMaxBeam).
static int check_shards(ehb_sharded* sh, bool brute, int precision, bool null_buf, uint64_t nq, uint32_t k,
                        uint64_t k_walk, uint32_t ef, bool* none, uint32_t max_beam = ehb::kMaxEf) {
  for (const auto& s : sh->shards) {
    ehb_index* ix = s->ix;
    std::shared_lock<ehb::RwLock> lk(ix->rw);
    uint32_t ef_shard = ef;
    RET(ehb::check_request(ix, brute, precision, null_buf, nq, k, k_walk, brute ? nullptr : &ef_shard, none,
                           max_beam));
  }
  return EHB_OK;
}

// Host queries in, merged host results out.
static int sharded_search(ehb_sharded* sh, bool brute, uint64_t nq, const float* q, uint32_t k, uint32_t ef,
                          int precision, uint64_t* ol, float* od, uint32_t* oc, bool beam = false) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  bool none;
  RET(check_shards(sh, brute, precision, nq && (!q || !ol), nq, k, k, ef, &none, beam ? ehb::kMaxBeam : ehb::kMaxEf));
  if (none) return EHB_OK;
  std::lock_guard<std::mutex> g(sh->mu);
  RET(sharded_merge(sh, brute, nq, q, k, ef, precision, beam));
  RET(ehb::copy_results(nq, k, sh->m_labels.p, sh->m_dists.p, sh->m_counts.p, ol, od, oc, sh->shards[0]->st));
  CU(cudaStreamSynchronize(sh->shards[0]->st));
  return EHB_OK;
}

int ehb_sharded_search(ehb_sharded* sh, uint64_t nq, const float* q, uint32_t k, uint32_t ef, uint64_t* ol, float* od,
                       uint32_t* oc) {
  return sharded_search(sh, false, nq, q, k, ef, EHB_FP32, ol, od, oc);
}
int ehb_sharded_search_ex(ehb_sharded* sh, uint64_t nq, const float* q, uint32_t k, uint32_t ef, int precision,
                          uint64_t* ol, float* od, uint32_t* oc) {
  return sharded_search(sh, false, nq, q, k, ef, precision, ol, od, oc);
}
int ehb_sharded_search_bruteforce(ehb_sharded* sh, uint64_t nq, const float* q, uint32_t k, int precision, uint64_t* ol,
                                  float* od, uint32_t* oc) {
  return sharded_search(sh, true, nq, q, k, 0, precision, ol, od, oc);
}
int ehb_sharded_search_beam(ehb_sharded* sh, uint64_t nq, const float* q, uint32_t k, uint32_t ef, int precision,
                            uint64_t* ol, float* od, uint32_t* oc) {
  return sharded_search(sh, false, nq, q, k, ef, precision, ol, od, oc, true);
}

int ehb_sharded_get_batch(ehb_sharded* sh, uint64_t n, const uint64_t* labels, float* out) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  if (n && (!labels || !out)) return fail(EHB_ERR_INVALID, "null buffer");
  const size_t G = sh->shards.size(), dim = sh->prm.dim;
  std::vector<std::vector<uint64_t>> labs(G), pos(G);
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t o = sh->owner(labels[i]);
    labs[o].push_back(labels[i]);
    pos[o].push_back(i);
  }
  std::vector<std::vector<float>> rows(G);  // every shard answers before anything is written
  for (size_t o = 0; o < G; ++o) {
    if (labs[o].empty()) continue;
    rows[o].resize(labs[o].size() * dim);
    RET(ehb_index_get_batch(sh->shards[o]->ix, labs[o].size(), labs[o].data(), rows[o].data()));
  }
  for (size_t o = 0; o < G; ++o)
    for (size_t j = 0; j < pos[o].size(); ++j)
      std::copy(rows[o].begin() + j * dim, rows[o].begin() + (j + 1) * dim, out + pos[o][j] * dim);
  return EHB_OK;
}

// The rows are laid out in owner order: shard o gathers its labels' rows into its own staging rows
// [first[o], first[o] + m_o) and copies them into every other shard's staging buffer; each shard then scatters the
// staging rows to their query positions in q_dev, and the k + 1 search + merge of ehb_sharded_search_ex (beam:
// ehb_sharded_search_beam) runs on them.
static int sharded_by_label(ehb_sharded* sh, uint64_t nq, const uint64_t* labels, uint32_t k, uint32_t ef,
                            int precision, uint64_t* ol, float* od, uint32_t* oc, bool beam) {
  if (!sh) return fail(EHB_ERR_INVALID, "null handle");
  bool none;
  RET(check_shards(sh, false, precision, nq && (!labels || !ol), nq, k, k + 1ull, ef, &none,
                   beam ? ehb::kMaxBeam : ehb::kMaxEf));
  if (none) return EHB_OK;
  const uint32_t k1 = k + 1;
  std::lock_guard<std::mutex> g(sh->mu);
  const uint32_t G = (uint32_t)sh->shards.size();
  const uint32_t dim = sh->prm.dim;
  std::vector<std::vector<uint64_t>> labs(G);
  std::vector<uint32_t> order;  // query position of each staging row
  std::vector<uint64_t> first(G);
  order.reserve(nq);
  {
    std::vector<std::vector<uint32_t>> pos(G);
    for (uint64_t i = 0; i < nq; ++i) {
      const uint32_t o = sh->owner(labels[i]);
      labs[o].push_back(labels[i]);
      pos[o].push_back((uint32_t)i);
    }
    for (uint32_t o = 0; o < G; ++o) {
      first[o] = order.size();
      order.insert(order.end(), pos[o].begin(), pos[o].end());
    }
  }
  for (const auto& sd : sh->shards) {
    CU(cudaSetDevice(sd->dev));
    CU(sd->q_stage.grow(nq * dim, 0, -1, sd->st));
    CU(sd->q_pos.grow(nq, 0, -1, sd->st));
    CU(sd->q_dev.grow(nq * dim, 0, -1, sd->st));
  }
  for (uint32_t o = 0; o < G; ++o) {
    if (labs[o].empty()) continue;
    const ehb::Shard& so = *sh->shards[o];
    const uint64_t m = labs[o].size();
    float* rows = so.q_stage.p + first[o] * dim;
    RET(ehb_index_gather_dev(so.ix, m, labs[o].data(), rows, so.st));
    CU(cudaSetDevice(so.dev));
    for (uint32_t i = 0; i < G; ++i)
      if (i != o)
        CU(cudaMemcpyPeerAsync(sh->shards[i]->q_stage.p + first[o] * dim, sh->shards[i]->dev, rows, so.dev,
                               m * dim * 4ull, so.st));
    CU(cudaEventRecord(so.done, so.st));
  }
  for (uint32_t i = 0; i < G; ++i) {
    const ehb::Shard& sd = *sh->shards[i];
    CU(cudaSetDevice(sd.dev));
    for (uint32_t o = 0; o < G; ++o)
      if (o != i && !labs[o].empty()) CU(cudaStreamWaitEvent(sd.st, sh->shards[o]->done, 0));
    CU(cudaMemcpyAsync(sd.q_pos.p, order.data(), nq * 4, cudaMemcpyHostToDevice, sd.st));
    CU(ehb::launch_gather_rows(sd.q_stage.p, dim, nullptr, sd.q_dev.p, dim, sd.q_pos.p, nq, dim, sd.st));
  }
  RET(sharded_merge(sh, false, nq, nullptr, k1, ef, precision, beam));
  CU(cudaSetDevice(sh->shards[0]->dev));
  cudaStream_t s0 = sh->shards[0]->st;
  CU(sh->s_self.grow(nq, 0, -1, s0));
  CU(sh->s_labels.grow(nq * k, 0, -1, s0));
  CU(sh->s_dists.grow(nq * k, 0, -1, s0));
  CU(sh->s_counts.grow(nq, 0, -1, s0));
  CU(cudaMemcpyAsync(sh->s_self.p, labels, nq * 8, cudaMemcpyHostToDevice, s0));
  CU(ehb::launch_drop_self(sh->s_self.p, sh->m_labels.p, sh->m_dists.p, sh->m_counts.p, nq, k, sh->s_labels.p,
                           sh->s_dists.p, sh->s_counts.p, s0));
  RET(ehb::copy_results(nq, k, sh->s_labels.p, sh->s_dists.p, sh->s_counts.p, ol, od, oc, s0));
  CU(cudaStreamSynchronize(s0));
  return EHB_OK;
}

int ehb_sharded_search_by_label_ex(ehb_sharded* sh, uint64_t nq, const uint64_t* labels, uint32_t k, uint32_t ef,
                                   int precision, uint64_t* ol, float* od, uint32_t* oc) {
  return sharded_by_label(sh, nq, labels, k, ef, precision, ol, od, oc, false);
}
int ehb_sharded_search_by_label_beam(ehb_sharded* sh, uint64_t nq, const uint64_t* labels, uint32_t k, uint32_t ef,
                                     int precision, uint64_t* ol, float* od, uint32_t* oc) {
  return sharded_by_label(sh, nq, labels, k, ef, precision, ol, od, oc, true);
}

}  // extern "C"
