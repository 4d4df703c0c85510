"""CPU-side checks of key mode over the one-process-per-GPU exchange: the binding's shape, the NCCL searcher's
refusal and the probe's vectorised self-removal rule, none of which needs a device."""
import os
import re

import numpy as np
import pytest

from embeddinghub_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _params(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ehb200.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", src)
    return [p for p in m.group(1).split(",") if p.strip()]


@pytest.mark.parametrize("name", ["ehb_exchange_create_ex", "ehb_exchange_search_by_label_ex_dev"])
def test_binding_takes_the_declared_arguments(name):
    assert len(_native.SYMBOLS[name][1]) == len(_params(name))


def test_nccl_searcher_rejects_key_mode_before_touching_a_device():
    from embeddinghub_b200.sharded import ShardedSearcher
    s = ShardedSearcher(None, 2, 0, exchange="nccl")
    with pytest.raises(ValueError, match="peer exchange"):
        s.search_by_label_dev(np.arange(3, dtype=np.uint64), 10, 64, 0)
    assert s._ex is None and not s._buf


def test_probe_rule_equals_the_model():
    """tools/exchange_by_label_probe.py applies the self-removal rule vectorised; it is the model's rule."""
    import importlib.util

    from label_rule_model import NO_LABEL, drop_self

    spec = importlib.util.spec_from_file_location("probe", os.path.join(ROOT, "tools", "exchange_by_label_probe.py"))
    probe = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(probe)
    rng = np.random.default_rng(3)
    for k in (1, 3, 10):
        nq = 400
        labels = rng.integers(0, 30, (nq, k + 1)).astype(np.uint64)
        dists = rng.standard_normal((nq, k + 1)).astype(np.float32)
        counts = rng.integers(0, k + 2, nq).astype(np.uint32)
        for q in range(nq):
            labels[q, counts[q]:], dists[q, counts[q]:] = NO_LABEL, np.inf
        self_labels = rng.integers(0, 30, nq).astype(np.uint64)
        want = drop_self(self_labels, labels, dists, counts, k)
        got = probe.drop_self(self_labels, labels, dists, counts, k)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), k
