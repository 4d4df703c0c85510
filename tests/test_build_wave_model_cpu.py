"""The wave model of the GPU build (tests/wave_model.py) anchored to hnswlib: with waves of one point it must be
sequential addPoint / updatePoint, so on build-tie-free data its graph equals OracleHNSW's row for row (as sets:
hnswlib stores a selection in reverse order)."""
import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure
from wave_model import INV, WaveModel, ip_matrix, tiefree_ip


def _sets(links):
    return [frozenset(int(v) for v in r if v != INV) for r in links]


def assert_same_graph_sets(mg, og):
    assert np.array_equal(mg["levels"], og["levels"])
    assert (int(mg["entry"]), int(mg["maxlevel"])) == (int(og["entry"]), int(og["maxlevel"]))
    assert np.array_equal(mg["up_off"], og["up_off"])
    a0, b0 = _sets(mg["links0"]), _sets(og["links0"])
    bad = [i for i in range(len(a0)) if a0[i] != b0[i]]
    assert not bad, (len(bad), bad[:5])
    assert _sets(mg["links_up"]) == _sets(og["links_up"])


def _oracle(x, M, n_cap=None):
    o = orc.OracleHNSW(x.shape[1], "ip", n_cap or x.shape[0], M=M)
    o.add(x.astype(np.float32), threads=1)
    return o


@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("M", [4, 16])
def test_model_waves_of_one_equal_oracle(d, M):
    n = 500
    x, _ = tiefree_ip(n, d)
    og = _oracle(x, M).export_graph()
    m = WaveModel(ip_matrix(x), og["levels"], M).build(build_batch=1)
    assert m.trace["waves"] == [1] * n
    assert_same_graph_sets(m.export(), og)


@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("M", [4, 16])
def test_model_single_moves_equal_oracle(d, M):
    """updatePoint one move at a time (each move is a wave of one), some labels moved twice."""
    n = 400
    x, B = tiefree_ip(n, d)
    o = _oracle(x, M)
    m = WaveModel(ip_matrix(x), o.export_graph()["levels"], M).build(build_batch=1)
    rng = np.random.default_rng(M * 7 + d)
    moved = rng.choice(n, 30, replace=False)
    moved = np.concatenate([moved, moved[:6]])
    for lab in moved.tolist():
        x[lab, :d - 1] = B * rng.integers(-1, 2, d - 1)       # the last coordinate keeps the data tie-free
        o.add(x[lab:lab + 1].astype(np.float32), np.array([lab], np.uint64), threads=1)
        m.set_distances(ip_matrix(x))
        m.update([lab])
    og = o.export_graph()
    assert np.array_equal(og["vectors"], x.astype(np.float32))
    assert_same_graph_sets(m.export(), og)


@pytest.mark.parametrize("M", [4, 16])
def test_model_inserts_after_tombstones_equal_oracle(M):
    """Tombstoned points are traversed during construction but never selected."""
    n0, n, d = 400, 500, 32
    x, _ = tiefree_ip(n, d)
    o = orc.OracleHNSW(d, "ip", n, M=M)
    o.add(x[:n0].astype(np.float32), threads=1)
    dead = np.random.default_rng(M).choice(n0, n0 // 10, replace=False)
    for lab in dead.tolist():
        o.mark_delete(lab)
    o.add(x[n0:].astype(np.float32), np.arange(n0, n, dtype=np.uint64), threads=1)
    og = o.export_graph()
    m = WaveModel(ip_matrix(x), og["levels"], M).build(n0, build_batch=1)
    m.mark_deleted(dead)
    m.build(build_batch=1)
    assert_same_graph_sets(m.export(), og)
    # the new points never link to a tombstone
    dset = set(dead.tolist())
    assert not any(v in dset for p in range(n0, n) for v in m.row(p, 0))
