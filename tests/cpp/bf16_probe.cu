// Test-only entry points into the bf16 tensor-core brute-force launchers of libehb200.so (K3,
// bf16gemm.cu), so tests/test_gpu_bf16_gemm.py can check the shipped kernels one launch at a time.
// Not part of the product ABI (include/ehb200.h): the signatures follow the internal launchers.
// Pointers are raw device pointers, the stream is the legacy default stream, and every wrapper
// returns the launcher's cudaError_t as an int.
#include "kernels.h"

extern "C" {

int probe_to_bf16(const float* in, uint32_t in_stride, void* out_bf16, float* norms, uint64_t n, uint32_t dpad) {
  return (int)ehb::launch_to_bf16(in, in_stride, out_bf16, norms, n, dpad, 0);
}

int probe_bf16_dist_tile(const void* q_bf16, uint64_t q_rows, const void* x_bf16, uint64_t x_rows, uint32_t dpad,
                         int metric, const float* qnorm, const float* xnorm, uint64_t q0, uint64_t qn, uint64_t n0,
                         uint64_t nn, float* dist, uint64_t ldd) {
  return (int)ehb::launch_bf16_dist_tile(q_bf16, q_rows, x_bf16, x_rows, dpad, metric, qnorm, xnorm, q0, qn, n0, nn,
                                         dist, ldd, 0);
}

int probe_bf16_topk_chunk(const void* q_bf16, uint64_t nq, const void* x_bf16, uint64_t x_rows, uint32_t dpad,
                          int metric, const float* qnorm, const float* xnorm, uint64_t n_lo, uint64_t n_hi, float* thr,
                          uint64_t* cbuf, uint32_t* ccount, uint32_t ccap, uint64_t* run_keys, uint32_t kc,
                          uint32_t* overflow, int sms) {
  return (int)ehb::launch_bf16_topk_chunk(q_bf16, nq, x_bf16, x_rows, dpad, metric, qnorm, xnorm, n_lo, n_hi, thr,
                                          cbuf, ccount, ccap, run_keys, kc, overflow, sms, 0);
}

}  // extern "C"
