"""CPU tier of the by-label searches: the new entry points are declared, exported and bound, and the numpy model
of the self-removal rule (server.cc:190-207) that the GPU tests compare against behaves as the reference does."""
import ctypes as C

import numpy as np

from embeddinghub_b200 import _native
from label_rule_model import NO_LABEL, drop_self

NEW = ["ehb_index_get_batch", "ehb_index_search_by_label_ex", "ehb_index_search_bruteforce_by_label",
       "ehb_index_neighbor_table", "ehb_sharded_get_batch", "ehb_sharded_search_by_label_ex"]


def test_new_entry_points_exported_and_bound():
    L = C.CDLL(_native.LIB_PATH)
    for n in NEW:
        assert hasattr(L, n), n
        assert n in _native.SYMBOLS, n
    for m in ("get_batch", "search_by_label", "search_bruteforce_by_label", "neighbor_table"):
        assert callable(getattr(_native.NativeIndex, m))
    for m in ("get_batch", "search_by_label"):
        assert callable(getattr(_native.ShardedIndex, m))


def _one(self_label, labels, k):
    c = len(labels)
    L = np.full((1, k + 1), NO_LABEL, np.uint64)
    D = np.full((1, k + 1), np.inf, np.float32)
    L[0, :c] = labels
    D[0, :c] = np.arange(c, dtype=np.float32)
    ol, od, oc = drop_self(np.array([self_label], np.uint64), L, D, np.array([c], np.uint32), k)
    return list(ol[0][:oc[0]]), od[0], int(oc[0]), ol[0]


def test_rule_self_first():
    got, d, c, _ = _one(7, [7, 1, 2, 3], 3)
    assert got == [1, 2, 3] and c == 3 and list(d) == [1, 2, 3]


def test_rule_self_in_the_middle():
    got, d, c, _ = _one(2, [5, 2, 9, 4], 3)
    assert got == [5, 9, 4] and list(d) == [0, 2, 3]


def test_rule_self_absent_with_k_plus_one_hits_drops_the_last():
    got, d, c, _ = _one(42, [5, 2, 9, 4], 3)
    assert got == [5, 2, 9] and c == 3


def test_rule_self_absent_with_at_most_k_hits_keeps_all():
    got, d, c, row = _one(42, [5, 2], 3)
    assert got == [5, 2] and c == 2 and row[2] == NO_LABEL and np.isinf(d[2])


def test_rule_self_present_among_few_hits_pads():
    got, d, c, row = _one(5, [5, 2], 3)
    assert got == [2] and c == 1 and row[1] == NO_LABEL and row[2] == NO_LABEL


def test_rule_no_hits():
    got, d, c, row = _one(5, [], 3)
    assert got == [] and c == 0 and (row == NO_LABEL).all() and np.isinf(d).all()
