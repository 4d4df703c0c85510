// Graph exchange and persistence of an ehb_index (SURVEY.md §8f-3).
//
// The reference persists only key -> vector rows in RocksDB (embeddinghub/embeddingstore/storage.cc:28-36)
// and rebuilds the hnswlib graph with one addPoint per row on every cold start
// (embeddinghub/embeddingstore/version.cc:64-74).  Here the vectors AND the graph go to one flat file whose
// sections are the device arrays themselves; save and load stream them through two page-locked buffers
// straight from / into their final device arrays (no full-size host copies, no second staging pass), so a
// cold start costs file-read + PCIe time instead of a rebuild.
#include <sys/stat.h>

#include "index_impl.h"

using ehb::fail;

namespace {

constexpr size_t kIoChunk = 64ull << 20;  // bytes per pinned buffer

__global__ void validate_links_kernel(const uint32_t* __restrict__ links, uint64_t count, uint32_t n,
                                      unsigned int* __restrict__ bad) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) {
    uint32_t v = links[i];
    if (v != ehb::kInvalid && v >= n) atomicAdd(bad, 1u);
  }
}

// Double-buffered pinned pipe between a FILE and device memory.
struct Pipe {
  ehb::PinBuf buf[2];
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool pending[2] = {false, false};
  cudaStream_t s;
  int cur = 0;
  explicit Pipe(cudaStream_t st) : s(st) {}
  ~Pipe() {
    for (int i = 0; i < 2; ++i)
      if (ev[i]) cudaEventDestroy(ev[i]);
  }
  int init() {
    for (int i = 0; i < 2; ++i) {
      CU(buf[i].reserve(kIoChunk));
      CU(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    }
    return EHB_OK;
  }
  // file -> device: rows of `row_bytes` land at dst + r * dst_pitch
  int read_rows(FILE* f, unsigned char* dst, size_t dst_pitch, size_t row_bytes, uint64_t rows) {
    if (rows == 0 || row_bytes == 0) return EHB_OK;
    const uint64_t per = std::max<uint64_t>(1, kIoChunk / row_bytes);
    for (uint64_t r0 = 0; r0 < rows; r0 += per) {
      const uint64_t m = std::min(per, rows - r0);
      if (pending[cur]) CU(cudaEventSynchronize(ev[cur]));
      if (std::fread(buf[cur].p, row_bytes, m, f) != m) return fail(EHB_ERR_IO, "short read");
      CU(cudaMemcpy2DAsync(dst + r0 * dst_pitch, dst_pitch, buf[cur].p, row_bytes, row_bytes, m,
                           cudaMemcpyHostToDevice, s));
      CU(cudaEventRecord(ev[cur], s));
      pending[cur] = true;
      cur ^= 1;
    }
    return EHB_OK;
  }
  // like read_rows, but also keeps a host copy of what was read
  int read_rows_keep(FILE* f, unsigned char* dst, size_t row_bytes, uint64_t rows, unsigned char* host_copy) {
    if (rows == 0) return EHB_OK;
    const uint64_t per = std::max<uint64_t>(1, kIoChunk / row_bytes);
    for (uint64_t r0 = 0; r0 < rows; r0 += per) {
      const uint64_t m = std::min(per, rows - r0);
      if (pending[cur]) CU(cudaEventSynchronize(ev[cur]));
      if (std::fread(buf[cur].p, row_bytes, m, f) != m) return fail(EHB_ERR_IO, "short read");
      std::memcpy(host_copy + r0 * row_bytes, buf[cur].p, m * row_bytes);
      CU(cudaMemcpyAsync(dst + r0 * row_bytes, buf[cur].p, m * row_bytes, cudaMemcpyHostToDevice, s));
      CU(cudaEventRecord(ev[cur], s));
      pending[cur] = true;
      cur ^= 1;
    }
    return EHB_OK;
  }
  // device -> file
  int write_rows(FILE* f, const unsigned char* src, size_t src_pitch, size_t row_bytes, uint64_t rows) {
    if (rows == 0 || row_bytes == 0) return EHB_OK;
    const uint64_t per = std::max<uint64_t>(1, kIoChunk / row_bytes);
    uint64_t prev_m = 0;
    int prev = -1;
    for (uint64_t r0 = 0; r0 < rows; r0 += per) {
      const uint64_t m = std::min(per, rows - r0);
      CU(cudaMemcpy2DAsync(buf[cur].p, row_bytes, src + r0 * src_pitch, src_pitch, row_bytes, m,
                           cudaMemcpyDeviceToHost, s));
      CU(cudaEventRecord(ev[cur], s));
      if (prev >= 0) {  // the previous chunk goes to the file while this one crosses PCIe
        CU(cudaEventSynchronize(ev[prev]));
        if (std::fwrite(buf[prev].p, row_bytes, prev_m, f) != prev_m) return fail(EHB_ERR_IO, "short write");
      }
      prev = cur;
      prev_m = m;
      cur ^= 1;
    }
    CU(cudaEventSynchronize(ev[prev]));
    if (std::fwrite(buf[prev].p, row_bytes, prev_m, f) != prev_m) return fail(EHB_ERR_IO, "short write");
    pending[0] = pending[1] = false;
    return EHB_OK;
  }
  int drain() {
    CU(cudaStreamSynchronize(s));
    pending[0] = pending[1] = false;
    return EHB_OK;
  }
};

int check_links(ehb_index* ix, const uint32_t* links, uint64_t count, uint64_t n) {
  if (!count) return EHB_OK;
  cudaStream_t s = ix->stream;
  CU(ix->b_counters.grow(8, 0, 0, s));
  CU(cudaMemsetAsync(ix->b_counters.p + 4, 0, 4, s));
  validate_links_kernel<<<(unsigned)((count + 255) / 256), 256, 0, s>>>(links, count, (uint32_t)n, ix->b_counters.p + 4);
  CU(cudaGetLastError());
  uint32_t bad = 0;
  CU(cudaMemcpyAsync(&bad, ix->b_counters.p + 4, 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (bad) return fail(EHB_ERR_IO, "corrupt graph: adjacency ids out of range");
  return EHB_OK;
}

// host-side tables that follow from (labels, levels, up_off, deleted)
int adopt_host_tables(ehb_index* ix, uint64_t n, uint64_t upper_rows, std::vector<uint64_t>&& labels,
                      std::vector<uint8_t>&& levels, std::vector<uint8_t>&& deleted, const uint32_t* up_off,
                      uint32_t entry, int32_t max_level) {
  cudaStream_t s = ix->stream;
  if (upper_rows) {
    std::vector<uint32_t> owners(upper_rows, 0);
    uint64_t expect = 0;
    for (uint64_t i = 0; i < n; ++i) {
      if (levels[i] == 0) continue;
      if (up_off[i] != expect || expect + levels[i] > upper_rows) return fail(EHB_ERR_IO, "corrupt graph: upper rows");
      for (int l = 0; l < levels[i]; ++l) owners[expect + l] = (uint32_t)i;
      expect += levels[i];
    }
    if (expect != upper_rows) return fail(EHB_ERR_IO, "corrupt graph: upper row count");
    CU(cudaMemcpyAsync(ix->up_owner.p, owners.data(), upper_rows * 4, cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));
  }
  if (n && (entry >= n || max_level < 0 || max_level > 31 || levels[entry] != max_level))
    return fail(EHB_ERR_IO, "corrupt graph: entry point");
  ix->identity_labels = true;
  for (uint64_t i = 0; i < n && ix->identity_labels; ++i)
    if (labels[i] != i) ix->identity_labels = false;
  ix->lookup.clear();
  if (!ix->identity_labels) {
    ix->lookup.reserve(n * 2);
    for (uint64_t i = 0; i < n; ++i) ix->lookup[labels[i]] = (uint32_t)i;
    if (ix->lookup.size() != n) return fail(EHB_ERR_IO, "corrupt graph: duplicate labels");
  }
  uint64_t nd = 0;
  for (uint64_t i = 0; i < n; ++i) nd += deleted[i] ? 1 : 0;
  ix->h_labels = std::move(labels);
  ix->h_levels = std::move(levels);
  ix->h_deleted = std::move(deleted);
  ix->n_deleted = nd;
  ix->n = ix->n_linked = n;
  ix->up_rows = upper_rows;
  ix->entry = entry;
  ix->max_level = n ? max_level : -1;
  ix->drop_derived();
  ix->pending_updates.clear();
  return EHB_OK;
}

// rows past the loaded range must read as empty for later inserts
int clear_tails(ehb_index* ix, uint64_t n, uint64_t upper_rows) {
  cudaStream_t s = ix->stream;
  if (ix->cap > n) {
    CU(cudaMemsetAsync(ix->links0.p + n * ix->M0, 0xFF, (ix->cap - n) * ix->M0 * 4, s));
    CU(cudaMemsetAsync(ix->up_off.p + n, 0xFF, (ix->cap - n) * 4, s));
    CU(cudaMemsetAsync(ix->deleted.p + n, 0, ix->cap - n, s));
  }
  if (ix->links_up.n > upper_rows * ix->M)
    CU(cudaMemsetAsync(ix->links_up.p + upper_rows * ix->M, 0xFF, (ix->links_up.n - upper_rows * ix->M) * 4, s));
  return EHB_OK;
}

}  // namespace

extern "C" {

int ehb_index_export_graph(ehb_index* ix, float* vectors, uint64_t* labels, uint8_t* levels, uint32_t* links0,
                           uint32_t* up_off, uint32_t* links_up, uint32_t* entry, int32_t* max_level) {
  if (!ix) return fail(EHB_ERR_INVALID, "null index handle");
  std::unique_lock<ehb::RwLock> g(ix->rw);
  CU(cudaSetDevice(ix->device));
  RET(ix->build());
  cudaStream_t s = ix->stream;
  uint64_t n = ix->n;
  if (vectors && n)
    CU(cudaMemcpy2DAsync(vectors, ix->dim * 4, ix->vecs.p, ix->dpad * 4, ix->dim * 4, n, cudaMemcpyDeviceToHost, s));
  if (labels && n) CU(cudaMemcpyAsync(labels, ix->labels.p, n * 8, cudaMemcpyDeviceToHost, s));
  if (levels && n) CU(cudaMemcpyAsync(levels, ix->levels.p, n, cudaMemcpyDeviceToHost, s));
  if (links0 && n) CU(cudaMemcpyAsync(links0, ix->links0.p, n * ix->M0 * 4, cudaMemcpyDeviceToHost, s));
  if (up_off && n) CU(cudaMemcpyAsync(up_off, ix->up_off.p, n * 4, cudaMemcpyDeviceToHost, s));
  if (links_up && ix->up_rows)
    CU(cudaMemcpyAsync(links_up, ix->links_up.p, ix->up_rows * ix->M * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  if (entry) *entry = ix->entry;
  if (max_level) *max_level = ix->max_level;
  return EHB_OK;
}

int ehb_index_import_graph(ehb_index* ix, uint64_t n, const float* vectors, const uint64_t* labels,
                           const uint8_t* levels, const uint32_t* links0, const uint32_t* up_off, uint64_t upper_rows,
                           const uint32_t* links_up, uint32_t entry, int32_t max_level) {
  if (!ix) return fail(EHB_ERR_INVALID, "null index handle");
  std::unique_lock<ehb::RwLock> g(ix->rw);
  CU(cudaSetDevice(ix->device));
  if (n && (!vectors || !labels || !levels || !links0 || !up_off)) return fail(EHB_ERR_INVALID, "null buffer");
  if (upper_rows && !links_up) return fail(EHB_ERR_INVALID, "null links_up");
  if (n >= 0x7FFFFFFFull) return fail(EHB_ERR_INVALID, "too many vectors");
  cudaStream_t s = ix->stream;
  ix->reset_content();
  RET(ix->ensure_capacity(std::max<uint64_t>(n, 1)));
  RET(ix->ensure_upper(std::max<uint64_t>(upper_rows, 1)));
  if (n) {
    if (ix->dim != ix->dpad) CU(cudaMemsetAsync(ix->vecs.p, 0, n * ix->dpad * 4, s));
    CU(cudaMemcpy2DAsync(ix->vecs.p, ix->dpad * 4, vectors, ix->dim * 4, ix->dim * 4, n, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ix->labels.p, labels, n * 8, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ix->levels.p, levels, n, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(ix->deleted.p, 0, n, s));
    CU(cudaMemcpyAsync(ix->links0.p, links0, n * ix->M0 * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ix->up_off.p, up_off, n * 4, cudaMemcpyHostToDevice, s));
    if (upper_rows) CU(cudaMemcpyAsync(ix->links_up.p, links_up, upper_rows * ix->M * 4, cudaMemcpyHostToDevice, s));
    CU(cudaStreamSynchronize(s));
  }
  RET(clear_tails(ix, n, upper_rows));
  CU(cudaStreamSynchronize(s));
  int rc = check_links(ix, ix->links0.p, n * ix->M0, n);
  if (rc == EHB_OK) rc = check_links(ix, ix->links_up.p, upper_rows * ix->M, n);
  if (rc == EHB_OK) {
    ix->level_rng.seed((unsigned)ix->prm.seed);  // later inserts continue the level sequence after n draws
    for (uint64_t i = 0; i < n; ++i) (void)ix->draw_level();
  }
  if (rc == EHB_OK)
    rc = adopt_host_tables(ix, n, upper_rows, std::vector<uint64_t>(labels, labels + n),
                           std::vector<uint8_t>(levels, levels + n), std::vector<uint8_t>(n, 0), up_off, entry,
                           max_level);
  if (rc != EHB_OK) ix->reset_content();
  return rc;
}

// File format (little endian): "EHB200\0\2", ehb_params, u64 hdr[6] = {n, upper_rows, entry, max_level,
// tombstones, points removed by ehb_index_compact (0 in files written before it existed)}, then the sections in device-array order: vectors [n][dim] f32 (unpadded), labels [n] u64,
// levels [n] u8, deleted [n] u8, links0 [n][2M] u32, up_off [n] u32, links_up [upper_rows][M] u32.
static uint64_t file_bytes(const ehb_params& p, uint64_t n, uint64_t rows) {
  return 8 + sizeof(ehb_params) + 48 + n * p.dim * 4ull + n * 8 + n + n + n * 2ull * p.M * 4 + n * 4 + rows * p.M * 4ull;
}

int ehb_index_save(ehb_index* ix, const char* path) {
  if (!ix || !path) return fail(EHB_ERR_INVALID, "null argument");
  std::unique_lock<ehb::RwLock> g(ix->rw);  // one consistent snapshot: no add can slip in between
  CU(cudaSetDevice(ix->device));
  RET(ix->build());
  FILE* f = std::fopen(path, "wb");
  if (!f) return fail(EHB_ERR_IO, std::string("cannot open ") + path);
  std::setvbuf(f, nullptr, _IOFBF, 8 << 20);
  auto body = [&]() -> int {
    Pipe pipe(ix->stream);
    RET(pipe.init());
    const char magic[8] = {'E', 'H', 'B', '2', '0', '0', 0, 2};
    const uint64_t n = ix->n, rows = ix->up_rows;
    uint64_t hdr[6] = {n, rows, ix->entry, (uint64_t)(int64_t)ix->max_level, ix->n_deleted, ix->n_removed};
    if (std::fwrite(magic, 1, 8, f) != 8 || std::fwrite(&ix->prm, sizeof(ehb_params), 1, f) != 1 ||
        std::fwrite(hdr, 8, 6, f) != 6)
      return fail(EHB_ERR_IO, "short write");
    RET(pipe.write_rows(f, (const unsigned char*)ix->vecs.p, ix->dpad * 4ull, ix->dim * 4ull, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->labels.p, 8, 8, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->levels.p, 1, 1, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->deleted.p, 1, 1, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->links0.p, ix->M0 * 4ull, ix->M0 * 4ull, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->up_off.p, 4, 4, n));
    RET(pipe.write_rows(f, (const unsigned char*)ix->links_up.p, ix->M * 4ull, ix->M * 4ull, rows));
    return EHB_OK;
  };
  int rc = body();
  if (std::fclose(f) != 0 && rc == EHB_OK) rc = fail(EHB_ERR_IO, "close failed");
  return rc;
}

int ehb_index_load(const char* path, int32_t device, ehb_index** out) {
  if (!path || !out) return fail(EHB_ERR_INVALID, "null argument");
  FILE* f = std::fopen(path, "rb");
  if (!f) return fail(EHB_ERR_IO, std::string("cannot open ") + path);
  std::setvbuf(f, nullptr, _IOFBF, 8 << 20);
  ehb_index* ix = nullptr;
  auto body = [&]() -> int {
    char magic[8];
    ehb_params p;
    uint64_t hdr[6];
    if (std::fread(magic, 1, 8, f) != 8 || std::memcmp(magic, "EHB200", 6) != 0 || magic[6] != 0)
      return fail(EHB_ERR_IO, "not an ehb200 index file");
    if (magic[7] != 2) return fail(EHB_ERR_IO, "unsupported ehb200 file version");
    if (std::fread(&p, sizeof(p), 1, f) != 1 || std::fread(hdr, 8, 6, f) != 6) return fail(EHB_ERR_IO, "bad header");
    const uint64_t n = hdr[0], rows = hdr[1];
    if (p.dim == 0 || p.dim > ehb::kMaxDim || p.M < 2 || p.M > 16 || p.metric < 0 || p.metric > 2 ||
        p.ef_construction > ehb::kMaxBeam || n >= 0x7FFFFFFFull || rows > n * 31ull || hdr[5] >= (1ull << 40))
      return fail(EHB_ERR_IO, "corrupt header");
    struct stat st;
    if (fstat(fileno(f), &st) != 0 || (uint64_t)st.st_size != file_bytes(p, n, rows))
      return fail(EHB_ERR_IO, "file size does not match its header");
    p.device = device;
    p.capacity = std::max<uint64_t>(n, 1);
    RET(ehb_index_create(&p, &ix));
    std::unique_lock<ehb::RwLock> g(ix->rw);
    cudaStream_t s = ix->stream;
    RET(ix->ensure_upper(std::max<uint64_t>(rows, 1)));
    Pipe pipe(s);
    RET(pipe.init());
    std::vector<uint64_t> labels;
    std::vector<uint8_t> levels, deleted;
    std::vector<uint32_t> up_off;
    try {
      labels.resize(n);
      levels.resize(n);
      deleted.resize(n);
      up_off.resize(n);
    } catch (const std::bad_alloc&) {
      return fail(EHB_ERR_OOM, "host allocation failed");
    }
    if (ix->dim != ix->dpad && n) CU(cudaMemsetAsync(ix->vecs.p, 0, n * ix->dpad * 4, s));
    RET(pipe.read_rows(f, (unsigned char*)ix->vecs.p, ix->dpad * 4ull, ix->dim * 4ull, n));
    RET(pipe.read_rows_keep(f, (unsigned char*)ix->labels.p, 8, n, (unsigned char*)labels.data()));
    RET(pipe.read_rows_keep(f, (unsigned char*)ix->levels.p, 1, n, levels.data()));
    RET(pipe.read_rows_keep(f, (unsigned char*)ix->deleted.p, 1, n, deleted.data()));
    RET(pipe.read_rows(f, (unsigned char*)ix->links0.p, ix->M0 * 4ull, ix->M0 * 4ull, n));
    RET(pipe.read_rows_keep(f, (unsigned char*)ix->up_off.p, 4, n, (unsigned char*)up_off.data()));
    RET(pipe.read_rows(f, (unsigned char*)ix->links_up.p, ix->M * 4ull, ix->M * 4ull, rows));
    RET(pipe.drain());
    RET(clear_tails(ix, n, rows));
    CU(cudaStreamSynchronize(s));
    RET(check_links(ix, ix->links0.p, n * ix->M0, n));
    RET(check_links(ix, ix->links_up.p, rows * ix->M, n));
    // the level generator continues after the loaded points and the compacted-away ones: replay its draws
    for (uint64_t i = 0; i < n + hdr[5]; ++i) (void)ix->draw_level();
    RET(adopt_host_tables(ix, n, rows, std::move(labels), std::move(levels), std::move(deleted), up_off.data(),
                          (uint32_t)hdr[2], (int32_t)(int64_t)hdr[3]));
    ix->n_removed = hdr[5];
    return EHB_OK;
  };
  int rc = body();
  std::fclose(f);
  if (rc != EHB_OK) {
    const std::string msg = ehb::last_error_text();
    if (ix) ehb_index_destroy(ix);
    return fail(rc, msg);
  }
  *out = ix;
  return EHB_OK;
}

}  // extern "C"
