// Host-only check of ehb::ExchangeLayout (csrc/exchange_layout.cuh): the exported buffer of an exchange rank keeps the
// byte layout every peer relies on.  The expected values are written out here independently of the header, so a change
// to the header's formulas (which would make ranks built from different sources disagree, or move a region) fails.
// No GPU needed.
#include <cstdint>
#include <cstdio>

#include "../../embeddinghub_b200/csrc/exchange_layout.cuh"

static int failures = 0;

static void expect(const char* what, uint64_t got, uint64_t want, uint32_t W, uint64_t nq, uint32_t k, uint32_t dim) {
  if (got == want) return;
  std::printf("FAILED %s: %llu, expected %llu (world %u, max_nq %llu, max_k %u, max_dim %u)\n", what,
              (unsigned long long)got, (unsigned long long)want, W, (unsigned long long)nq, k, dim);
  ++failures;
}

static void check(uint32_t W, uint64_t max_nq, uint32_t max_k, uint32_t max_dim) {
  const ehb::ExchangeLayout L = ehb::ExchangeLayout::make(W, max_nq, max_k, max_dim);
  auto up = [](uint64_t b, uint64_t a) { return (b + a - 1) / a * a; };
  const uint64_t stride = (max_nq * max_k * 12 + 255) / 256 * 256;
  const uint64_t flag_bytes = (2ull * W * 256 * 4 + 4 + 4095) / 4096 * 4096;
  uint64_t total = flag_bytes + 2ull * W * stride, rows_off = 0, marks_off = 0, digests_off = 0, row_stride = 0;
  if (max_dim) {
    row_stride = (max_nq * max_dim + 63) / 64 * 64;
    rows_off = total;
    marks_off = rows_off + up(2 * row_stride * 4, 256);
    digests_off = marks_off + up(2ull * W * max_nq, 256);
    total = digests_off + up(2ull * W * 8, 256);
  }
  unsigned char* const base = reinterpret_cast<unsigned char*>(uintptr_t(1) << 40);  // any address; never read
  auto at = [&](const void* p) { return (uint64_t)((uintptr_t)p - (uintptr_t)base); };
  expect("stride", L.stride, stride, W, max_nq, max_k, max_dim);
  expect("flag_bytes", L.flag_bytes, flag_bytes, W, max_nq, max_k, max_dim);
  expect("total_bytes", L.total_bytes, total, W, max_nq, max_k, max_dim);
  expect("row_stride", L.row_stride, row_stride, W, max_nq, max_k, max_dim);
  expect("rows_off", L.rows_off, rows_off, W, max_nq, max_k, max_dim);
  expect("marks_off", L.marks_off, marks_off, W, max_nq, max_k, max_dim);
  expect("digests_off", L.digests_off, digests_off, W, max_nq, max_k, max_dim);
  expect("timeout", at(L.timeout(base)), flag_bytes - 4, W, max_nq, max_k, max_dim);
  for (uint32_t p = 0; p < 2; ++p)
    for (uint32_t r = 0; r < W; ++r) {
      expect("recv", at(L.recv(base, p, r)), flag_bytes + (p * W + r) * stride, W, max_nq, max_k, max_dim);
      expect("flags", at(L.flags(base, p, r)), (p * W + r) * 256 * 4, W, max_nq, max_k, max_dim);
      if (!max_dim) continue;
      expect("marks", at(L.marks(base, p, r)), marks_off + (p * W + r) * max_nq, W, max_nq, max_k, max_dim);
      expect("digest", at(L.digest(base, p, r)), digests_off + (p * W + r) * 8, W, max_nq, max_k, max_dim);
      expect("rows", at(L.rows(base, p)), rows_off + p * row_stride * 4, W, max_nq, max_k, max_dim);
      expect("row float", at(L.rows(base, p, r)), rows_off + (p * row_stride + r) * 4, W, max_nq, max_k, max_dim);
    }
  // the regions neither overlap nor leave the allocation
  expect("flags fit", L.flags(base, 1, W - 1) + 256 <= L.timeout(base), 1, W, max_nq, max_k, max_dim);
  if (max_dim) {
    expect("rows 256-byte aligned", at(L.rows(base, 1)) % 256, 0, W, max_nq, max_k, max_dim);
    expect("rows fit", at(L.rows(base, 1) + max_nq * max_dim) <= marks_off, 1, W, max_nq, max_k, max_dim);
    expect("marks fit", at(L.marks(base, 1, W - 1) + max_nq) <= digests_off, 1, W, max_nq, max_k, max_dim);
    expect("digests fit", at(L.digest(base, 1, W - 1) + 1) <= total, 1, W, max_nq, max_k, max_dim);
  }
}

int main() {
  static_assert(ehb::kMaxSlices == 256, "the flag page above holds 256 slices per (parity, rank)");
  const uint32_t worlds[] = {1, 2, 3, 16};
  const uint64_t nqs[] = {1, 5, 1000, 10000};
  const uint32_t ks[] = {1, 10, 101, 4096};
  const uint32_t dims[] = {0, 1, 3, 64, 127, 768, 4096};
  int cases = 0;
  for (uint32_t W : worlds)
    for (uint64_t nq : nqs)
      for (uint32_t k : ks)
        for (uint32_t dim : dims) {
          check(W, nq, k, dim);
          ++cases;
        }
  std::printf("%d layouts checked, %d mismatches\n", cases, failures);
  std::printf(failures ? "FAILED\n" : "OK\n");
  return failures ? 1 : 0;
}
