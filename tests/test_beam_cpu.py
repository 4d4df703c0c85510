"""The wide-beam entry points without a GPU: the three symbols resolve in the built library, _native binds them with
the header's argument lists, and the header's limit is 4096."""
import ctypes as C
import os
import re

import embeddinghub_b200 as ehb
from embeddinghub_b200 import _native

NAMES = {"ehb_index_search_beam": 9, "ehb_index_search_beam_dev": 10, "ehb_index_search_by_label_beam": 9}
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ehb200.h")


def test_beam_symbols_resolve_and_are_bound():
    raw = C.CDLL(_native.LIB_PATH)
    for name, nargs in NAMES.items():
        getattr(raw, name)                                  # AttributeError when the library lacks it
        res, args = _native.SYMBOLS[name]
        assert res is C.c_int and len(args) == nargs
        assert getattr(ehb.lib(), name).argtypes == args
    for m in ("search_beam", "search_beam_dev", "search_by_label_beam"):
        assert callable(getattr(_native.NativeIndex, m))


def test_header_declares_the_beam_limit():
    text = open(HEADER).read()
    assert re.search(r"#define EHB_MAX_BEAM 4096\b", text)
    for name in NAMES:
        assert re.search(rf"\bint {name}\(", text), name
