// Host-callable launchers of the ehb200 kernels (internal header).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "walk.cuh"

namespace ehb {

constexpr uint32_t kMaxDim = 2048;  // pad_dim() supports rows up to 2048 floats
constexpr uint32_t kMaxEf = 512;    // register-resident list: 16 keys per lane
constexpr uint32_t kUpdCandCap = 1088;  // update path: sCand capacity per moved point, >= 1 + 32 + 32*32

// K2 — batched k-NN graph walk (hnswlib searchKnn).  ef >= k, cfg.lcap >= ef.
// stats: [nq][4] u32 = hops_upper, hops_base, evals, overflow.
cudaError_t launch_search(const GraphView& g, const WalkCfg& cfg, const float* queries, uint32_t nq, uint32_t k,
                          uint32_t ef, const ResultSink& sink, uint32_t* out_counts, uint32_t* stats,
                          uint32_t warps_per_block, cudaStream_t s);

// K2t — team walk (T warps per query, T in {2,3,4}); rows <= 1 KB and ef <= 256 only.
cudaError_t launch_search_team(uint32_t T, const GraphView& g, uint32_t hash_size, const float* queries, uint32_t nq,
                               uint32_t k, uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                               uint32_t* stats, cudaStream_t s);
// the U (4-vector load steps in flight) that launch_search_team instantiates for this shape
uint32_t team_eval_steps(uint32_t T, uint32_t dpad, uint32_t nq);

// row-wise L2 normalisation (hnswlib cosine convention), canonical arithmetic.
cudaError_t launch_normalize(const float* in, uint32_t in_stride, float* out, uint32_t out_stride, uint64_t n,
                             uint32_t dim, cudaStream_t s);
// copy [n][dim] -> [n][dpad] with zero padding (and optional normalisation)
cudaError_t launch_pad_rows(const float* in, float* out, uint64_t n, uint32_t dim, uint32_t dpad, bool normalize,
                            cudaStream_t s);
cudaError_t launch_sum_stats(const uint32_t* stats, uint32_t nq, unsigned long long* out4, cudaStream_t s);

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
};
struct BuildGraph {
  GraphView g;          // links are written through these pointers (const-cast inside)
  const uint8_t* levels;
  const uint32_t* up_owner;  // [upper rows] owning node of each upper row
  uint32_t cap;         // row id space split: rows >= cap are upper rows
  uint32_t efc;
};
// Links points ids[0..b) (or first..first+b when ids == nullptr) into the graph.
cudaError_t launch_build_batch(const BuildGraph& bg, const WalkCfg& cfg, const uint32_t* ids, uint32_t first,
                               uint32_t b, bool is_update, BuildBuffers& bb, uint32_t warps_per_block,
                               cudaStream_t s);

}  // namespace ehb
