// Test-only entry point into the int8 screen-copy conversion of libehb200.so (search.cu launch_to_i8), so
// tests/test_gpu_walk_screen_int8.py can check the shipped kernel against its numpy replica.  Not part of the product
// ABI (include/ehb200.h).  Pointers are raw device pointers, the stream is the legacy default stream, and the wrapper
// returns the launcher's cudaError_t as an int.
#include "kernels.h"

extern "C" int probe_to_i8(const float* in, uint32_t dpad, int8_t* codes, float* terms, uint64_t n) {
  return (int)ehb::launch_to_i8(in, dpad, codes, (float4*)terms, n, 0);
}
