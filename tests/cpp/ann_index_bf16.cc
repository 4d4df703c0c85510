// The C++ ANNIndex twin (include/ehb200_ann_index.hpp) with a bf16 graph search.  Inner-product rows
// x_i = (B u_i, 256 floor((i+1) / 256), (i+1) mod 256) and queries (v, 1, 1), u, v in {-1, 0, 1}, B = 1024: every
// coordinate is exact in bf16, every partial sum is an integer below 2^24, and q.x_i = B (u_i.v) + i + 1 differs
// for every i.  The bf16 walk then computes the fp32 walk's distances exactly and nothing ties, so both
// precisions must return the same keys in the same order.  An unknown precision must throw.
// Run on the GPU by tests/test_gpu_bf16_walk.py.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "ehb200_ann_index.hpp"

using featureform::embedding::ANNIndex;

int main() {
  const size_t dims = 24, n = 800, nq = 40;
  const float B = 1024.f;
  ANNIndex idx(dims, 128, EHB_IP);
  uint32_t s = 12345;
  auto tri = [&]() {  // -1, 0 or 1
    s = s * 1664525u + 1013904223u;
    return (float)((int)((s >> 16) % 3u) - 1);
  };
  for (size_t i = 0; i < n; ++i) {
    std::vector<float> v(dims);
    for (size_t j = 0; j + 2 < dims; ++j) v[j] = B * tri();
    v[dims - 2] = 256.f * (float)((i + 1) / 256);
    v[dims - 1] = (float)((i + 1) % 256);
    idx.set("k" + std::to_string(i), v);
  }
  std::vector<std::vector<float>> q(nq, std::vector<float>(dims, 1.f));
  for (auto& r : q)
    for (size_t j = 0; j + 2 < dims; ++j) r[j] = tri();
  int failed = 0;
  auto expect = [&](bool ok, const char* what) {
    std::printf("%s %s\n", ok ? "ok  " : "FAIL", what);
    failed += ok ? 0 : 1;
  };
  const auto f = idx.approx_nearest_batch(q, 10, 64, EHB_FP32);
  const auto b = idx.approx_nearest_batch(q, 10, 64, EHB_BF16);
  bool same = f.size() == nq && b.size() == nq;
  for (size_t i = 0; same && i < nq; ++i) same = b[i].size() == 10 && f[i] == b[i];
  expect(same, "bf16 batch equals fp32 batch on bf16-exact tie-free rows");
  const auto one_f = idx.approx_nearest_batch({q[3]}, 5, 0, EHB_FP32);
  const auto one_b = idx.approx_nearest_batch({q[3]}, 5, 0, EHB_BF16);
  expect(one_b.size() == 1 && one_b[0].size() == 5 && one_b == one_f, "a single query at the default ef agrees");
  bool threw = false;
  try {
    idx.approx_nearest_batch(q, 10, 64, 7);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  expect(threw, "unknown precision throws");
  return failed;
}
