// Drop-in twin of featureform::embedding::ANNIndex
// (embeddinghub/embeddingstore/index.h:19-33, index.cc:10-52) over the ehb200 C ABI.
// Same class name, constructor and member signatures, so version.h:49's
// std::shared_ptr<ANNIndex> and server.cc:202-203 compile unchanged when
// "index.h" is replaced by this header and the target links libehb200.so.
//
// Differences that are deliberate:
//   * errors from the library surface as std::runtime_error (hnswlib throws the
//     same type for capacity errors, which the reference lets propagate);
//   * approx_nearest returns the keys that exist when fewer than `num` points are
//     stored (index.cc:42-50 pops `num` entries regardless — undefined behaviour);
//   * a batched approx_nearest_batch() is added (docs/inference.md:14-22), with an optional ef and precision
//     (EHB_BF16: the graph walk over bf16 rows, re-ranked in fp32; ehb_index_search_ex);
//   * approx_nearest_by_key() / approx_nearest_by_keys() answer the server's key mode (server.cc:190-207) on the
//     device.
#pragma once
#include <algorithm>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "ehb200.h"

namespace featureform {
namespace embedding {

class ANNIndex {
 public:
  ANNIndex(size_t dims, size_t init_cap = 128, int metric = EHB_L2, int device = 0) : dims_(dims), next_label_(0) {
    ehb_params p;
    ehb_params_default(&p, (uint32_t)dims);
    p.capacity = init_cap;
    p.metric = metric;
    p.device = device;
    check(ehb_index_create(&p, &ix_));
  }
  ~ANNIndex() { ehb_index_destroy(ix_); }
  ANNIndex(const ANNIndex&) = delete;
  ANNIndex& operator=(const ANNIndex&) = delete;

  // index.cc:20-37 — new key -> next label; existing key -> same label (update in place).
  void set(std::string key, std::vector<float> value) {
    if (value.size() != dims_) throw std::runtime_error("ANNIndex::set: wrong dimension");
    auto it = key_to_label_.find(key);
    uint64_t label;
    if (it == key_to_label_.end()) {
      label = next_label_++;
      label_to_key_[label] = key;
      key_to_label_[key] = label;
    } else {
      label = it->second;
    }
    check(ehb_index_add(ix_, 1, value.data(), &label));
    deleted_.erase(key);  // hnswlib addPoint un-deletes a re-added label
  }

  // index.cc:39-52 — keys nearest-first.
  std::vector<std::string> approx_nearest(std::vector<float> value, size_t num) const {
    std::vector<std::vector<float>> one{std::move(value)};
    return approx_nearest_batch(one, num)[0];
  }

  std::vector<std::vector<std::string>> approx_nearest_batch(const std::vector<std::vector<float>>& values,
                                                             size_t num, uint32_t ef = 0,
                                                             int precision = EHB_FP32) const {
    std::vector<std::vector<std::string>> out(values.size());
    if (num == 0 || values.empty()) return out;
    std::vector<float> q(values.size() * dims_);
    for (size_t i = 0; i < values.size(); ++i) {
      if (values[i].size() != dims_) throw std::runtime_error("ANNIndex::approx_nearest: wrong dimension");
      std::copy(values[i].begin(), values[i].end(), q.begin() + i * dims_);
    }
    std::vector<uint64_t> labels(values.size() * num);
    std::vector<uint32_t> counts(values.size());
    check(ehb_index_search_ex(ix_, values.size(), q.data(), (uint32_t)num, ef, precision, labels.data(), nullptr,
                              counts.data()));
    for (size_t i = 0; i < values.size(); ++i)
      for (uint32_t j = 0; j < counts[i]; ++j) out[i].push_back(label_to_key_.at(labels[i * num + j]));
    return out;
  }

  // Key mode of NearestNeighbor (server.cc:190-207): the `num` nearest other keys of a stored key.  The key's row
  // is searched at num + 1 on the device and the key removed there, or the last hit dropped when the key is not
  // among them (ehb_index_search_by_label_ex), so a server calls this one member instead of get + approx_nearest
  // with num + 1 + erase.  An unknown or removed key throws.
  std::vector<std::string> approx_nearest_by_key(const std::string& key, size_t num) const {
    return approx_nearest_by_keys(std::vector<std::string>{key}, num)[0];
  }

  std::vector<std::vector<std::string>> approx_nearest_by_keys(const std::vector<std::string>& keys, size_t num,
                                                               uint32_t ef = 0, int precision = EHB_FP32) const {
    std::vector<uint64_t> q(keys.size());
    for (size_t i = 0; i < keys.size(); ++i) {
      auto it = key_to_label_.find(keys[i]);
      if (it == key_to_label_.end() || deleted_.count(keys[i]))
        throw std::runtime_error("ANNIndex::approx_nearest_by_key: unknown key");
      q[i] = it->second;
    }
    std::vector<std::vector<std::string>> out(keys.size());
    if (num == 0 || keys.empty()) return out;
    std::vector<uint64_t> labels(keys.size() * num);
    std::vector<uint32_t> counts(keys.size());
    if (std::max<size_t>(num + 1, ef) > 512)  // beyond the graph walk's beam: the exact scan
      check(ehb_index_search_bruteforce_by_label(ix_, keys.size(), q.data(), (uint32_t)num, precision, labels.data(),
                                                 nullptr, counts.data()));
    else
      check(ehb_index_search_by_label_ex(ix_, keys.size(), q.data(), (uint32_t)num, ef, precision, labels.data(),
                                         nullptr, counts.data()));
    for (size_t i = 0; i < keys.size(); ++i)
      for (uint32_t j = 0; j < counts[i]; ++j) out[i].push_back(label_to_key_.at(labels[i * num + j]));
    return out;
  }

  void set_ef(uint32_t ef) { check(ehb_index_set_ef(ix_, ef)); }

  // docs/reading_and_writing_embeddings.md:49-66 (space.delete): tombstone, never returned again; a later
  // set() of the same key brings it back (hnswlib markDelete / addPoint).
  void remove(const std::string& key) {
    auto it = key_to_label_.find(key);
    if (it == key_to_label_.end()) throw std::runtime_error("ANNIndex::remove: unknown key");
    uint64_t label = it->second;
    check(ehb_index_remove(ix_, 1, &label));
    deleted_.insert(key);
  }

  // Removes the deleted keys for good (ehb_index_compact): the graph is repaired on the GPU and the tombstone-free
  // search paths apply again.  A removed key that is set later gets a fresh label.
  void compact() {
    check(ehb_index_compact(ix_));
    for (const std::string& key : deleted_) {
      auto it = key_to_label_.find(key);
      label_to_key_.erase(it->second);
      key_to_label_.erase(it);
    }
    deleted_.clear();
  }

 private:
  static void check(int rc) {
    if (rc != EHB_OK) throw std::runtime_error(std::string("ehb200: ") + ehb_last_error());
  }
  size_t dims_;
  ehb_index* ix_ = nullptr;
  std::unordered_map<std::string, uint64_t> key_to_label_;
  std::unordered_map<uint64_t, std::string> label_to_key_;
  uint64_t next_label_;
  std::unordered_set<std::string> deleted_;  // removed (and not set again) since the last compact()
};

}  // namespace embedding
}  // namespace featureform
