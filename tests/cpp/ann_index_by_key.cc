// Key mode of the reference's NearestNeighbor (embeddinghub/embeddingstore/server.cc:190-207) through the C++ twin's
// approx_nearest_by_key, on the a/b/c fixture of embeddinghub/embeddingstore/test/index_test.cc:17-60.  Prints one
// line per (case, key, num) for tests/test_gpu_search_by_label.py to compare with the Python layer, and checks the
// answers that have no distance ties.
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "ehb200_ann_index.hpp"

using featureform::embedding::ANNIndex;
using Keys = std::vector<std::string>;
using Vec = std::vector<float>;

int main() {
  const std::vector<std::pair<std::string, Vec>> fixture = {{"a", {0, 1, 0}}, {"b", {1, 1, 0}}, {"c", {1, 0, 0}}};
  struct Case {
    const char* name;
    std::vector<std::pair<std::string, Vec>> extra_sets;
    std::vector<std::pair<std::string, Keys>> expect;  // key -> its 2 nearest other keys (tie-free ones)
  };
  const std::vector<Case> cases = {
      {"fixture", {}, {{"a", {"b", "c"}}, {"c", {"b", "a"}}}},
      {"update", {{"a", {0, -1, 0}}}, {{"a", {"c", "b"}}, {"b", {"c", "a"}}, {"c", {"b", "a"}}}},
  };
  int failed = 0;
  for (const Case& c : cases) {
    ANNIndex idx(3);
    for (const auto& kv : fixture) idx.set(kv.first, kv.second);
    for (const auto& kv : c.extra_sets) idx.set(kv.first, kv.second);
    for (const char* key : {"a", "b", "c"})
      for (size_t num = 0; num <= 3; ++num) {
        Keys got = idx.approx_nearest_by_key(key, num);
        std::printf("%s %s %zu:", c.name, key, num);
        for (const auto& g : got) std::printf(" %s", g.c_str());
        std::printf("\n");
        for (const auto& e : c.expect)
          if (e.first == key && num == 2 && got != e.second) {
            std::printf("FAIL %s %s\n", c.name, key);
            ++failed;
          }
      }
  }
  try {
    ANNIndex idx(3);
    idx.set("a", {0, 1, 0});
    idx.approx_nearest_by_key("zz", 1);
    std::printf("FAIL unknown key accepted\n");
    ++failed;
  } catch (const std::runtime_error&) {
  }
  return failed;
}
