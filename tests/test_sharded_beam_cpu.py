"""The wide-beam shard entry points without a GPU: the four symbols resolve in the built library and are bound with
their _ex counterparts' argument lists, the Python surfaces exist, and the NCCL searcher rejects key mode."""
import ctypes as C
import os
import re

import pytest

import embeddinghub_b200 as ehb
from embeddinghub_b200 import _native
from embeddinghub_b200.sharded import ShardedSearcher

PAIRS = {"ehb_exchange_search_beam_dev": "ehb_exchange_search_ex_dev",
         "ehb_exchange_search_by_label_beam_dev": "ehb_exchange_search_by_label_ex_dev",
         "ehb_sharded_search_beam": "ehb_sharded_search_ex",
         "ehb_sharded_search_by_label_beam": "ehb_sharded_search_by_label_ex"}
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ehb200.h")


def test_sharded_beam_symbols_resolve_and_are_bound_like_ex():
    raw = C.CDLL(_native.LIB_PATH)
    text = open(HEADER).read()
    for name, ex in PAIRS.items():
        getattr(raw, name)                                  # AttributeError when the library lacks it
        assert _native.SYMBOLS[name] == _native.SYMBOLS[ex], name
        assert getattr(ehb.lib(), name).argtypes == _native.SYMBOLS[ex][1]
        assert re.search(rf"\bint {name}\(", text), name
    for m in ("search_beam", "search_by_label_beam"):
        assert callable(getattr(_native.ShardedIndex, m))
    for m in ("search_beam_dev", "search_by_label_beam_dev"):
        assert callable(getattr(ShardedSearcher, m))


def test_nccl_searcher_rejects_key_mode_beam():
    s = ShardedSearcher.__new__(ShardedSearcher)            # no process group or GPU needed to reach the check
    s.exchange, s.world, s._ex = "nccl", 2, None
    with pytest.raises(ValueError):
        s.search_by_label_beam_dev([1, 2], 10, 1000, 0)
