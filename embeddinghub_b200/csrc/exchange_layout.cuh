// The buffer every rank of an ehb_exchange exports (exchange.cu): ONE cudaMalloc per rank, because a CUDA IPC handle
// covers one allocation, mapped by every peer.  Offsets in bytes from the start of the allocation; W = world.
//
//   flag page   [0, flag_bytes)             u32 flags[2 parities][W senders][kMaxSlices]; the last u32 of the page is
//                                           the timeout word.  flag_bytes = 2·W·kMaxSlices·4 + 4, rounded up to 4096.
//   receive     [flag_bytes, + 2·W·stride)  block (parity, rank): [max_nq·max_k] u64 labels, then as many f32
//                                           distances (a step of nq·k uses the first nq·k of each);
//                                           stride = 12·max_nq·max_k rounded up to 256.
//   key mode only (max_dim > 0), each part rounded up to 256 bytes:
//   rows        at rows_off                 f32 [2 parities][row_stride]; row_stride = max_nq·max_dim rounded up to
//                                           64 floats, so each parity's part starts 256-byte aligned.
//   marks       at marks_off                u8 [2][W][max_nq]: 1 when rank g holds query q's label.
//   digests     at digests_off              u64 [2][W]: each rank's digest of its label list.
//
// With max_dim = 0 the allocation ends after the receive blocks and rows_off = marks_off = digests_off = row_stride = 0.
// Every rank builds the same layout from the same (world, max_nq, max_k, max_dim), so an offset computed here is valid
// in any rank's mapping.  tests/cpp/exchange_layout.cu holds these formulas fixed.
#pragma once
#include <cstdint>

namespace ehb {

constexpr uint32_t kMaxWorld = 16;
constexpr uint32_t kMaxSlices = 256;

struct ExchangeLayout {
  uint32_t world;
  uint64_t max_nq;
  uint64_t stride;      // bytes per receive block
  uint64_t flag_bytes;  // bytes of the flag page (the receive blocks start here)
  uint64_t row_stride;  // floats per parity of the row region
  uint64_t rows_off, marks_off, digests_off;
  uint64_t total_bytes;

  static ExchangeLayout make(uint32_t world, uint64_t max_nq, uint32_t max_k, uint32_t max_dim) {
    auto round_up = [](uint64_t b, uint64_t a) { return (b + a - 1) / a * a; };
    ExchangeLayout L{};
    L.world = world;
    L.max_nq = max_nq;
    L.stride = round_up(max_nq * max_k * 12ull, 256);
    L.flag_bytes = round_up(2ull * world * kMaxSlices * 4 + 4, 4096);
    L.total_bytes = L.flag_bytes + 2ull * world * L.stride;
    if (max_dim) {
      L.row_stride = round_up(max_nq * max_dim, 64);
      L.rows_off = L.total_bytes;
      L.marks_off = L.rows_off + round_up(2ull * L.row_stride * 4, 256);
      L.digests_off = L.marks_off + round_up(2ull * world * max_nq, 256);
      L.total_bytes = L.digests_off + round_up(2ull * world * 8, 256);
    }
    return L;
  }

  // `base` is one rank's allocation as mapped by the caller.
  // Receive block (parity, rank): [nq][k] labels, then [nq][k] distances.
  __host__ __device__ unsigned char* recv(unsigned char* base, uint32_t parity, uint32_t rank) const {
    return base + flag_bytes + ((uint64_t)parity * world + rank) * stride;
  }
  // Flags that rank `from` raises in this allocation at `parity`: one per slice.
  __host__ __device__ uint32_t* flags(unsigned char* base, uint32_t parity, uint32_t from) const {
    return (uint32_t*)base + ((uint64_t)parity * world + from) * kMaxSlices;
  }
  // Set to 1 by an exchange kernel of the owning rank that gave up waiting for a peer.
  __host__ __device__ uint32_t* timeout(unsigned char* base) const { return (uint32_t*)(base + flag_bytes - 4); }
  // Float i of the row part of `parity` (the offset is summed first, so a loop over ranks adds it to each base once).
  __host__ __device__ float* rows(unsigned char* base, uint32_t parity, uint64_t i = 0) const {
    return (float*)(base + (rows_off + (parity * row_stride + i) * 4));
  }
  // [max_nq] marks written by `rank`.
  __host__ __device__ unsigned char* marks(unsigned char* base, uint32_t parity, uint32_t rank) const {
    return base + marks_off + ((uint64_t)parity * world + rank) * max_nq;
  }
  __host__ __device__ uint64_t* digest(unsigned char* base, uint32_t parity, uint32_t rank) const {
    return (uint64_t*)(base + digests_off) + (uint64_t)parity * world + rank;
  }
};

}  // namespace ehb
