"""Host-side mirror of featureform::embedding::ANNIndex
(embeddinghub/embeddingstore/index.h:19-33, index.cc:10-52) over the ehb200 C ABI.

Same surface and semantics: string keys, insert-or-update on a duplicate key,
`approx_nearest(value, num)` returning keys nearest-first, `num == 0 -> []`.
The metric is a per-index parameter defaulting to L2 (the reference hard-codes
hnswlib::L2Space, index.cc:12-13).  Capacity doubling (index.cc:29-32) happens
inside the library.  ef stays at hnswlib's default 10 unless set_ef is called,
exactly as the reference (which never calls setEf).
"""
import numpy as np

from ._native import FP32, NativeIndex


class ANNIndex:
    def __init__(self, dims, init_cap=128, metric="l2", device=0, **kw):
        self._nn = NativeIndex(dims, metric=metric, capacity=init_cap, device=device, **kw)
        self._dims = int(dims)
        self._key_to_label = {}
        self._label_to_key = {}
        self._next_label = 0
        self._deleted = set()

    # index.cc:20-37
    def set(self, key, value):
        self.multiset([(key, value)])

    def multiset(self, items):
        """Batched form of `set` (the reference loops set() per row, version.cc:69-72).  Every row is validated
        before any key is registered, and the key maps are committed only after the native add succeeded, so a
        bad row (wrong length) or a failed add leaves the index exactly as it was."""
        items = list(items.items()) if hasattr(items, "items") else list(items)
        if not items:
            return
        vecs = np.empty((len(items), self._dims), np.float32)
        for i, (_, value) in enumerate(items):
            v = np.asarray(value, dtype=np.float32)
            if v.ndim != 1 or v.shape[0] != self._dims:
                raise ValueError(f"embedding has {v.size} values, the index has {self._dims} dimensions")
            vecs[i] = v
        labels = np.empty(len(items), np.uint64)
        fresh, nxt = {}, self._next_label
        for i, (key, _) in enumerate(items):
            label = self._key_to_label.get(key)
            if label is None:
                label = fresh.get(key)
            if label is None:
                label = fresh[key] = nxt
                nxt += 1
            labels[i] = label
        self._nn.add(vecs, labels)
        for key, label in fresh.items():
            self._key_to_label[key] = label
            self._label_to_key[label] = key
        self._next_label = nxt
        self._deleted.difference_update(k for k, _ in items)   # a re-set key is un-deleted (hnswlib addPoint)

    # docs/reading_and_writing_embeddings.md:49-66 (promised by the reference; hnswlib markDelete semantics)
    def delete(self, key):
        self.multidelete([key])

    def multidelete(self, keys):
        keys = list(keys)
        for k in keys:
            if k not in self:
                raise KeyError(k)
        if keys:
            self._nn.remove(np.array([self._key_to_label[k] for k in keys], np.uint64))
            self._deleted.update(keys)

    def compact(self):
        """Removes the deleted keys for good (ehb_index_compact): the graph is repaired on the GPU and the index
        searches at full speed again.  len, keys, `in`, get and approx_nearest answer as before; a deleted key
        that is set again later gets a fresh label."""
        self._nn.compact()
        for k in self._deleted:
            del self._label_to_key[self._key_to_label.pop(k)]
        self._deleted.clear()

    def delete_all(self):
        self.multidelete([k for k in self._key_to_label if k not in self._deleted])

    # index.cc:39-52
    def approx_nearest(self, value, num):
        return self.approx_nearest_batch(np.asarray(value, np.float32)[None, :], num)[0]

    def approx_nearest_batch(self, values, num, ef=0, precision=FP32):
        """Batched k-NN (docs/inference.md:14-22 promises multi_nearest_neighbor;
        the reference never implemented it).  precision=BF16 walks the graph over bf16 rows and re-ranks in fp32
        (ehb_index_search_ex); the exact-scan fallback below runs at the same precision."""
        if num == 0:
            return [[] for _ in range(len(values))]
        values = np.asarray(values, np.float32)
        if values.ndim != 2 or values.shape[1] != self._dims:
            raise ValueError(f"query has {values.shape[-1] if values.ndim else 0} values, the index has {self._dims} dimensions")
        extra = () if precision == FP32 else (precision,)   # the default keeps the plain fp32 call
        if max(num, ef) > 512:
            # beyond the register-resident beam (ef <= 512) the exact scan answers (any num the reference accepts)
            labels, _, counts = self._nn.search_bruteforce(values, num, *extra)
        else:
            labels, _, counts = self._nn.search(values, num, ef, *extra)
        return [[self._label_to_key[int(l)] for l in row[:c]] for row, c in zip(labels, counts)]

    def _labels_of(self, keys):
        for k in keys:
            if k not in self:
                raise KeyError(k)
        return np.array([self._key_to_label[k] for k in keys], np.uint64)

    def approx_nearest_by_keys(self, keys, num, ef=0, precision=FP32):
        """Key mode of NearestNeighbor (server.cc:190-207): for each stored key, the `num` nearest other keys.  The
        key's stored row is searched at num + 1 on the device and the key itself removed there (or, when it is not
        among the hits, the last hit dropped), so this answers what get + approx_nearest_batch(num + 1) + that rule
        answers.  KeyError for an unknown or deleted key; beyond the register-resident beam (max(num + 1, ef) > 512)
        the exact scan answers, like approx_nearest_batch."""
        keys = list(keys)
        labels = self._labels_of(keys)
        if num == 0 or not keys:
            return [[] for _ in keys]
        extra = () if precision == FP32 else (precision,)
        if max(num + 1, ef) > 512:
            out, _, counts = self._nn.search_bruteforce_by_label(labels, num, *extra)
        else:
            out, _, counts = self._nn.search_by_label(labels, num, ef, *extra)
        return [[self._label_to_key[int(l)] for l in row[:c]] for row, c in zip(out, counts)]

    def neighbor_table(self, num, ef=0, precision=FP32):
        """{key: its `num` nearest other keys} for every stored key, in insertion order: approx_nearest_by_keys of
        all keys, computed in batches on the device (ehb_index_neighbor_table; graph walk, so max(num + 1, ef) <= 512).
        Writers wait until it returns."""
        if num == 0:
            return {k: [] for k in self.keys()}
        q, out, _, counts = self._nn.neighbor_table(num, ef, precision)
        key = self._label_to_key
        return {key[int(lq)]: [key[int(l)] for l in row[:c]] for lq, row, c in zip(q, out, counts)}

    def get(self, key):
        if key in self._deleted:
            raise KeyError(key)
        return self._nn.get(self._key_to_label[key])

    def multiget(self, keys):
        """The stored rows of `keys` ([n][dims]) in one device gather (ehb_index_get_batch); KeyError for an unknown
        or deleted key."""
        keys = list(keys)
        if not keys:
            return np.empty((0, self._dims), np.float32)
        return self._nn.get_batch(self._labels_of(keys))

    def set_ef(self, ef):
        self._nn.set_ef(ef)

    def keys(self):
        """Stored keys in insertion order (what Download streams, server.cc:212-233)."""
        return [k for k in self._key_to_label if k not in self._deleted]

    def __len__(self):
        return len(self._key_to_label) - len(self._deleted)

    def __contains__(self, key):
        return key in self._key_to_label and key not in self._deleted
