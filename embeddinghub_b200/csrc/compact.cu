// K6 — compaction of tombstoned points (ehb_index_compact).  The repair kernel itself lives with the
// updatePoint kernel in build_impl.cuh; here are the passes around it: find the rows that name deleted ids
// (and count level-0 in-links), copy the repaired rows back, renumber the adjacency, find the orphans and
// move the vectors down in place.
#include "kernels.h"

namespace ehb {

static __global__ void compact_mark_kernel(const uint32_t* __restrict__ links0, const uint32_t* __restrict__ links_up,
                                           const uint32_t* __restrict__ up_owner, const uint8_t* __restrict__ deleted,
                                           uint64_t n, uint64_t up_rows, uint32_t M0, uint32_t M, uint32_t cap,
                                           uint32_t* rows, uint32_t* nrows, uint32_t* indeg) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n + up_rows) return;
  const bool upper = r >= n;
  const uint32_t owner = upper ? up_owner[r - n] : (uint32_t)r;
  const uint32_t width = upper ? M : M0;
  const uint32_t* row = upper ? links_up + (r - n) * M : links0 + r * M0;
  bool names_dead = false;
  for (uint32_t j = 0; j < width; ++j) {
    const uint32_t v = row[j];
    if (v == kInvalid) break;
    names_dead |= deleted[v] != 0;
    if (!upper) atomicAdd(&indeg[v], 1u);  // in-links from every node, tombstones included
  }
  if (names_dead && !deleted[owner]) rows[atomicAdd(nrows, 1u)] = upper ? cap + (uint32_t)(r - n) : (uint32_t)r;
}

static __global__ void compact_apply_kernel(const uint32_t* __restrict__ rows, uint32_t nrows,
                                            const uint32_t* __restrict__ repair_out, uint32_t* links0,
                                            uint32_t* links_up, uint32_t M0, uint32_t M, uint32_t cap) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t i = t / M0;
  const uint32_t j = (uint32_t)(t % M0);
  if (i >= nrows) return;
  const uint32_t r = rows[i];
  if (r < cap)
    links0[(uint64_t)r * M0 + j] = repair_out[i * M0 + j];
  else if (j < M)
    links_up[(uint64_t)(r - cap) * M + j] = repair_out[i * M0 + j];
}

static __global__ void compact_remap_rows_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ src_row,
                                                 uint64_t rows, uint32_t width, const uint32_t* __restrict__ remap,
                                                 uint32_t* __restrict__ dst) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= rows * width) return;
  const uint64_t i = t / width;
  const uint32_t v = src[(uint64_t)src_row[i] * width + (t % width)];
  dst[t] = v == kInvalid ? kInvalid : remap[v];
}

static __global__ void compact_indeg_kernel(const uint32_t* __restrict__ links0, uint64_t n, uint32_t M0,
                                            uint32_t* indeg) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * M0) return;
  const uint32_t v = links0[t];
  if (v != kInvalid) atomicAdd(&indeg[v], 1u);
}

static __global__ void compact_orphans_kernel(const uint32_t* __restrict__ links0, uint64_t n, uint32_t M0,
                                              const uint32_t* __restrict__ inv, const uint32_t* __restrict__ indeg_old,
                                              const uint32_t* __restrict__ indeg_new, uint8_t* flag) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool empty = links0[i * M0] == kInvalid;
  flag[i] = empty || (indeg_old[inv[i]] > 0 && indeg_new[i] == 0) ? 1 : 0;
}

// one warp per row, float4 copies (rows are 16 B aligned, dpad a multiple of 32)
static __global__ void compact_gather_rows_kernel(const float* __restrict__ vecs, uint32_t dpad,
                                                  const uint32_t* __restrict__ inv, uint64_t lo, uint64_t cnt,
                                                  float* __restrict__ stage) {
  const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (i >= cnt) return;
  const float4* s = reinterpret_cast<const float4*>(vecs + (uint64_t)inv[lo + i] * dpad);
  float4* d = reinterpret_cast<float4*>(stage + i * dpad);
  for (uint32_t c = lane; c < dpad / 4; c += 32) d[c] = s[c];
}

static unsigned blocks_for(uint64_t threads) { return (unsigned)((threads + 255) / 256); }

cudaError_t launch_compact_mark(const uint32_t* links0, const uint32_t* links_up, const uint32_t* up_owner,
                                const uint8_t* deleted, uint64_t n, uint64_t up_rows, uint32_t M0, uint32_t M,
                                uint32_t cap, uint32_t* rows, uint32_t* nrows, uint32_t* indeg, cudaStream_t s) {
  if (n + up_rows == 0) return cudaSuccess;
  compact_mark_kernel<<<blocks_for(n + up_rows), 256, 0, s>>>(links0, links_up, up_owner, deleted, n, up_rows, M0, M,
                                                               cap, rows, nrows, indeg);
  return cudaGetLastError();
}

cudaError_t launch_compact_apply(const uint32_t* rows, uint32_t nrows, const uint32_t* repair_out, uint32_t* links0,
                                 uint32_t* links_up, uint32_t M0, uint32_t M, uint32_t cap, cudaStream_t s) {
  if (!nrows) return cudaSuccess;
  compact_apply_kernel<<<blocks_for((uint64_t)nrows * M0), 256, 0, s>>>(rows, nrows, repair_out, links0, links_up, M0,
                                                                        M, cap);
  return cudaGetLastError();
}

cudaError_t launch_compact_remap_rows(const uint32_t* src, const uint32_t* src_row, uint64_t rows, uint32_t width,
                                      const uint32_t* remap, uint32_t* dst, cudaStream_t s) {
  if (!rows) return cudaSuccess;
  compact_remap_rows_kernel<<<blocks_for(rows * width), 256, 0, s>>>(src, src_row, rows, width, remap, dst);
  return cudaGetLastError();
}

cudaError_t launch_compact_orphans(const uint32_t* links0, uint64_t n, uint32_t M0, const uint32_t* inv,
                                   const uint32_t* indeg_old, uint32_t* indeg_new, uint8_t* flag, cudaStream_t s) {
  if (!n) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(indeg_new, 0, n * 4, s);
  if (e != cudaSuccess) return e;
  compact_indeg_kernel<<<blocks_for(n * M0), 256, 0, s>>>(links0, n, M0, indeg_new);
  compact_orphans_kernel<<<blocks_for(n), 256, 0, s>>>(links0, n, M0, inv, indeg_old, indeg_new, flag);
  return cudaGetLastError();
}

cudaError_t launch_compact_move_rows(float* vecs, uint32_t dpad, const uint32_t* inv, uint64_t lo, uint64_t n,
                                     float* stage, uint64_t stage_rows, cudaStream_t s) {
  for (uint64_t a = lo; a < n; a += stage_rows) {
    const uint64_t cnt = n - a < stage_rows ? n - a : stage_rows;
    compact_gather_rows_kernel<<<blocks_for(cnt * 32), 256, 0, s>>>(vecs, dpad, inv, a, cnt, stage);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(vecs + a * dpad, stage, cnt * dpad * 4, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace ehb
