"""The CPU model of ehb_index_compact (tests/compact_model.py) on the oracle: structure, labels, entry point rule,
edge cases and recall.  No GPU needed."""
import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure
from compact_model import INV, compact_oracle, float_dist


def _gauss(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)


def _oracle(x, M=8, metric="l2"):
    o = orc.OracleHNSW(x.shape[1], metric, len(x), M=M)
    o.add(x, threads=1)
    return o


def _recall(o, x_live, lab_live, q, k, ef):
    got, _, _ = o.search(q, k, ef=ef)
    idx, _ = orc.bruteforce(x_live, q, k, "l2")
    truth = lab_live[idx.astype(np.int64)]
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(got, truth)]))


@pytest.mark.parametrize("frac", [0.1, 0.5, 0.9])
def test_structure_labels_entry(frac):
    n, d, M = 1500, 16, 8
    x = _gauss(n, d, 1)
    o = _oracle(x, M)
    g = o.export_graph()
    rng = np.random.default_rng(int(frac * 100))
    dead = np.union1d(rng.choice(n, int(frac * n), replace=False), [int(g["entry"])]).astype(np.uint64)
    for lab in dead:
        o.mark_delete(int(lab))
    c, cg, orphans = compact_oracle(o, dead, float_dist(g["vectors"], "l2"))
    out = c.export_graph()
    nn = n - len(dead)
    assert c.count == nn and len(out["labels"]) == nn
    live = np.setdiff1d(np.arange(n, dtype=np.uint64), dead)
    assert np.array_equal(out["labels"], live)                              # insertion order kept
    for lab in live[:: max(1, nn // 50)]:
        assert np.array_equal(c.get(int(lab)), x[int(lab)])
    for lab in dead[:20]:
        with pytest.raises(KeyError):
            c.get(int(lab))
    l0 = out["links0"]
    assert np.all((l0 == INV) | (l0 < nn))
    assert np.all((out["links_up"] == INV) | (out["links_up"] < nn))
    assert out["links_up"].shape[0] == int(out["levels"].astype(np.int64).sum())
    # rule 3: the entry point was deleted -> the live node of highest level, smallest id on a tie
    lv = out["levels"].astype(np.int64)
    assert int(out["maxlevel"]) == lv.max() and int(out["entry"]) == int(np.argmax(lv))
    # every survivor keeps a non-empty level-0 row (orphans were re-linked), and no row names itself
    assert np.all(l0[:, 0] != INV)
    assert not np.any(l0 == np.arange(nn, dtype=np.uint32)[:, None])
    print(f"deleted {frac:.0%}+entry: {len(orphans)} orphans re-linked")


def test_live_entry_is_kept():
    n, d = 800, 8
    x = _gauss(n, d, 2)
    o = _oracle(x)
    g = o.export_graph()
    e = int(g["entry"])
    dead = np.setdiff1d(np.arange(0, n, 3), [e]).astype(np.uint64)
    for lab in dead:
        o.mark_delete(int(lab))
    c, _, _ = compact_oracle(o, dead, float_dist(g["vectors"], "l2"))
    out = c.export_graph()
    assert int(out["labels"][int(out["entry"])]) == e and int(out["maxlevel"]) == int(g["maxlevel"])


def test_nothing_deleted_changes_nothing():
    x = _gauss(600, 8, 3)
    o = _oracle(x)
    g = o.export_graph()
    c, _, orphans = compact_oracle(o, [], float_dist(g["vectors"], "l2"))
    out = c.export_graph()
    assert len(orphans) == 0
    for f in ("labels", "levels", "links0", "up_off", "links_up", "vectors"):
        assert np.array_equal(out[f], g[f]), f
    assert (out["entry"], out["maxlevel"]) == (g["entry"], g["maxlevel"])


def test_everything_deleted_gives_an_empty_index_that_accepts_adds():
    x = _gauss(300, 8, 4)
    o = _oracle(x)
    g = o.export_graph()
    for lab in range(300):
        o.mark_delete(lab)
    c, cg, _ = compact_oracle(o, np.arange(300, dtype=np.uint64), float_dist(g["vectors"], "l2"))
    assert c.count == 0 and cg["maxlevel"] == -1
    y = _gauss(200, 8, 5)
    c.resize(200)
    c.add(y, np.arange(1000, 1200, dtype=np.uint64), threads=1)
    lab, _, cnt = c.search(y[:5], 1, ef=32)
    assert np.array_equal(lab[:, 0], np.arange(1000, 1005, dtype=np.uint64)) and np.all(cnt == 1)


@pytest.mark.parametrize("frac", [0.1, 0.5, 0.9])
def test_recall_not_below_tombstones(frac):
    """Gaussian data: recall after compaction >= recall of the tombstoned index - 0.005."""
    n, d, k, ef = 3000, 16, 10, 64
    x = _gauss(n, d, 6)
    q = _gauss(200, d, 7)
    o = _oracle(x, M=16)
    dead = np.random.default_rng(8).choice(n, int(frac * n), replace=False).astype(np.uint64)
    for lab in dead:
        o.mark_delete(int(lab))
    live = np.setdiff1d(np.arange(n), dead.astype(np.int64))
    before = _recall(o, x[live], live.astype(np.uint64), q, k, ef)
    c, _, orphans = compact_oracle(o, dead, float_dist(x, "l2"))
    after = _recall(c, x[live], live.astype(np.uint64), q, k, ef)
    print(f"oracle recall@{k} deleted {frac:.0%}: tombstones {before:.4f}, compacted {after:.4f} "
          f"({len(orphans)} orphans)")
    assert after >= before - 0.005, (after, before)
