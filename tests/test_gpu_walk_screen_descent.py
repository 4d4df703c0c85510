"""The screened fp32 walk also screens its upper-layer descent: each hop's neighbours are scored on the int8 copy
against the current node's distance, and only those whose lower bound is below it are read in fp32.  The descent
must take the same path: screen on vs off must give the same ids, distance bits, counts and hop / evaluation /
overflow counters, and the screened walk must still match hnswlib's walk on the same graph exactly.
"""
import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure
from test_gpu_walk_exact import assert_exact, ip_dist, oracle_run, tiefree
from test_gpu_walk_screen import DIMS, check_same, gaussian, make_index, run


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


@pytest.mark.gpu
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("metric", ["ip", "cosine"])
@pytest.mark.parametrize("deleted", [False, True])
def test_on_off_every_dpad_class(d, metric, deleted):
    x = gaussian(6000, d, 71)
    q = gaussian(200, d, 72)
    ix = make_index(x, metric)
    if deleted:
        ix.remove(np.arange(0, len(x), 6, dtype=np.uint64))
    check_same(ix, q, 10, 128)


@pytest.mark.gpu
def test_on_off_after_compaction():
    x = gaussian(8000, 768, 73)
    q = gaussian(200, 768, 74)
    ix = make_index(x, "ip")
    ix.remove(np.arange(0, len(x), 4, dtype=np.uint64))
    ix.compact()
    check_same(ix, q, 10, 128)


def _screened_walk_equals_oracle(g, o, x, q, k, ef):
    """walk_screen forced on and off over graph g: both equal the oracle's walk over the same graph."""
    d = x.shape[1]
    ix = _ehb().NativeIndex(d, metric="ip", capacity=len(x))
    ix.import_graph(g)
    ref = oracle_run(o, q, k, ef)
    D = ip_dist(x, q)
    for screen in (0, 1):
        res, st, _ = run(ix, q, k, ef, screen)
        assert_exact(res, st, ref, D, k)
    check_same(ix, q, k, ef)
    return st


@pytest.mark.gpu
def test_oracle_built_graph():
    """A graph built by the oracle (hnswlib's insert order and links), imported and walked screened."""
    n, d = 3000, 768
    x, q = tiefree(n, d, 160, seed=75)
    o = orc.OracleHNSW(d, "ip", n)
    o.add(x.astype(np.float32), threads=8)
    g = o.export_graph()
    assert int(g["maxlevel"]) >= 1
    st = _screened_walk_equals_oracle(g, o, x, q, 10, 128)
    assert st["screened_evals"] > 0


@pytest.mark.gpu
def test_descent_alone_is_screened():
    """ef = 512 over a few hundred points: the base layer's result set never fills, so only the upper-layer descent
    screens, and it must still screen (and reject) some of its candidates."""
    n, d = 400, 768
    x, q = tiefree(n, d, 160, seed=77)
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n)
    ix.add(x.astype(np.float32))
    ix.build()
    g = ix.export_graph()
    assert int(g["maxlevel"]) >= 1
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    st = _screened_walk_equals_oracle(g, o, x, q, 10, 512)
    assert st["hops_upper"] > 0
    assert 0 < st["screened_evals"] and st["fp32_row_reads"] < st["dist_evals"], st
