// Known-answer cases of the reference's ANNIndex unit test
// (embeddinghub/embeddingstore/test/index_test.cc:17-60: TestSimpleANN, TestMultiANN,
// TestUpdateANN, TestANN0Items), table-driven and without gtest, run against the drop-in
// twin in include/ehb200_ann_index.hpp on the GPU (tests/test_gpu_host.py).
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "ehb200_ann_index.hpp"

using featureform::embedding::ANNIndex;
using Keys = std::vector<std::string>;
using Vec = std::vector<float>;

struct Case {
  const char* name;
  std::vector<std::pair<std::string, Vec>> extra_sets;  // applied after the common a/b/c fixture
  Vec query;
  size_t num;
  Keys expect;
};

int main() {
  const std::vector<std::pair<std::string, Vec>> fixture = {{"a", {0, 1, 0}}, {"b", {1, 1, 0}}, {"c", {1, 0, 0}}};
  const std::vector<Case> cases = {
      {"TestSimpleANN", {}, {0, 1, 0}, 1, {"a"}},
      {"TestMultiANN", {}, {0, 1, 0}, 2, {"a", "b"}},
      {"TestUpdateANN", {{"a", {0, -1, 0}}}, {0, 1, 0}, 1, {"b"}},  // re-set of "a" must update in place
      {"TestANN0Items", {}, {0, 1, 0}, 0, {}},
  };
  int failed = 0;
  for (const Case& c : cases) {
    ANNIndex idx(3);
    for (const auto& kv : fixture) idx.set(kv.first, kv.second);
    for (const auto& kv : c.extra_sets) idx.set(kv.first, kv.second);
    Keys got = idx.approx_nearest(c.query, c.num);
    bool ok = got == c.expect;
    std::printf("%s %s\n", ok ? "ok  " : "FAIL", c.name);
    failed += ok ? 0 : 1;
  }
  return failed;
}
