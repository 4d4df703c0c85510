"""The wide construction form (ef_construction 257 ... 4096) held to hnswlib and to the wave model.

Above efc 256 the build's search keeps its result set in shared memory (SList) and its visited table in HBM, and the
update and compaction re-selections keep their candidates in an SList too.  The algorithm is the same: with waves of
one point the graph is hnswlib's sequential addPoint (the oracle's, as row sets), and on build-tie-free inner-product
data every wave equals tests/wave_model.py at that efc, row for row and in order: every row width, real wave sizes,
tombstones, update waves, compaction, save / load and shards.  At scale two builds are bit-identical and recall does
not drop below the efc 200 build's or the oracle's at the same efc.
"""
import os
import tempfile

import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure
from compact_model import compact_oracle, int_ip_dist
from test_gpu_build_waves import assert_same_ordered, assert_well_formed, levels_of
from test_gpu_walk_exact import _assert_same_graph
from wave_model import WaveModel, ip_matrix, tiefree_ip

pytestmark = pytest.mark.gpu

# one per dpad class 32 ... 4096
DIMS = [29, 64, 128, 250, 383, 512, 768, 1000, 1535, 2048, 3000, 4096]


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def data(n, d, seed=11, nnz=None):
    """Build-tie-free inner-product rows: dense up to d = 64 when they stay exact, else `nnz` (or as many as stay
    exact, at most 48) non-zeros."""
    if nnz is None:
        B2 = (1 << n.bit_length()) ** 2
        exact = ((1 << 24) - (n + 1) ** 2 - 1) // B2
        nnz = None if d <= 64 and d - 1 <= exact else min(48, exact, d - 1)
    return tiefree_ip(n, d, seed, nnz=nnz)[0]


def gpu_build(x, M, efc, build_batch=0, build_frac=0):
    n, d = x.shape
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, ef_construction=efc, build_batch=build_batch)
    if build_frac:
        ix.set_option("build_frac", build_frac)
    ix.add(x.astype(np.float32))
    ix.build()
    return ix


def model(x, M, efc, levels=None, **build):
    n, d = x.shape
    lv = levels_of(n, d, M) if levels is None else levels
    return WaveModel(ip_matrix(x), lv, M, ef_construction=efc).build(**build)


def check(ix, m, n):
    g = ix.export_graph()
    assert_well_formed(g, n)
    assert_same_ordered(g, m.export())
    return g


def _sets(links):
    return [frozenset(int(v) for v in r if v != 0xFFFFFFFF) for r in links]


# ---- waves of one: hnswlib's sequential build ----------------------------------------------------------------------
@pytest.mark.parametrize("efc", [257, 512, 1000])
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_gpu_wave_of_one_equals_oracle_wide_efc(metric, efc):
    n, d, M = efc + 300, 32, 8
    x = np.random.default_rng(efc).standard_normal((n, d), dtype=np.float32)
    ix = _ehb().NativeIndex(d, metric=metric, capacity=n, M=M, ef_construction=efc, build_batch=1)
    ix.add(x)
    g = ix.export_graph()
    o = orc.OracleHNSW(d, metric, n, M=M, ef_construction=efc)
    o.add(x, threads=1)
    og = o.export_graph()
    assert np.array_equal(g["levels"], og["levels"])
    assert (int(g["entry"]), int(g["maxlevel"])) == (int(og["entry"]), int(og["maxlevel"]))
    assert np.array_equal(g["up_off"], og["up_off"])
    same0 = np.mean([a == b for a, b in zip(_sets(g["links0"]), _sets(og["links0"]))])
    sameu = np.mean([a == b for a, b in zip(_sets(g["links_up"]), _sets(og["links_up"]))]) if len(g["links_up"]) else 1.0
    assert same0 >= 0.99 and sameu >= 0.99, (same0, sameu)   # float summation order may flip rare ties


@pytest.mark.parametrize("efc", [257, 512, 1000])
def test_gpu_wave_of_one_equals_model_tiefree(efc):
    n, d, M = efc + 100, 16, 8
    x = data(n, d, seed=efc)
    check(gpu_build(x, M, efc, build_batch=1), model(x, M, efc, build_batch=1), n)


# ---- real waves ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DIMS)
def test_gpu_waves_every_dpad_efc300(d):
    """Waves of up to 1/4 of the linked graph at every row width; n > efc, so the set fills."""
    n, M, efc = 400, 8, 300
    x = data(n, d)
    m = model(x, M, efc, build_frac=4)
    assert max(m.trace["waves"]) >= 60
    check(gpu_build(x, M, efc, build_frac=4), m, n)


@pytest.mark.parametrize("d", DIMS)
def test_gpu_waves_every_dpad_efc4096(d):
    """The widest beam at every row width (the launch fits at least one warp per SM); the set never fills."""
    n, M, efc = 160, 8, 4096
    x = data(n, d, seed=2)
    check(gpu_build(x, M, efc, build_frac=4), model(x, M, efc, build_frac=4), n)


@pytest.mark.parametrize("build_frac", [1, 4, 64])
@pytest.mark.parametrize("build_batch", [0, 7, 64])
def test_gpu_waves_frac_batch_efc512(build_frac, build_batch):
    n, d, M, efc = 600, 48, 8, 512
    x = data(n, d, seed=3)
    m = model(x, M, efc, build_batch=build_batch, build_frac=build_frac)
    assert 1 < max(m.trace["waves"]) <= (build_batch or 16384)
    check(gpu_build(x, M, efc, build_batch, build_frac), m, n)


def test_gpu_waves_efc1024_set_fills():
    n, d, M, efc = 1500, 24, 8, 1024
    x = data(n, d, seed=4)
    m = model(x, M, efc, build_frac=8)
    check(gpu_build(x, M, efc, build_frac=8), m, n)


@pytest.mark.parametrize("efc", [512, 1100])
def test_gpu_waves_after_tombstones_wide_efc(efc):
    """Batched inserts into an index with 10 % of its points tombstoned (the HASDEL form)."""
    n0, n, d, M = 600, 700, 32, 8
    x = data(n, d, seed=13)
    levels = levels_of(n, d, M)
    dead = np.random.default_rng(efc).choice(n0, n0 // 10, replace=False)
    m = WaveModel(ip_matrix(x), levels, M, ef_construction=efc).build(n0, build_frac=4)
    m.mark_deleted(dead)
    m.build(build_frac=4)
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, ef_construction=efc)
    ix.set_option("build_frac", 4)
    ix.add(x[:n0].astype(np.float32))
    ix.build()
    ix.remove(dead.astype(np.uint64))
    ix.add(x[n0:].astype(np.float32))
    ix.build()
    check(ix, m, n)


# ---- update waves --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("efc", [512, 1100])
@pytest.mark.parametrize("mode", ["sequential", "waves", "waves16"])
def test_gpu_update_waves_wide_efc(efc, mode):
    """Moves (some labels moved twice) one point per wave, all in one wave, or 16 per wave (seq_updates = 0)."""
    n, d, M = 600, 32, 8
    x = data(n, d, seed=17)
    g0 = model(x, M, efc, build_frac=4).export()
    g0.update(vectors=x.astype(np.float32), labels=np.arange(n, dtype=np.uint64))
    rng = np.random.default_rng(23)
    first = rng.choice(n, 120 if mode == "sequential" else 220, replace=False)
    again = first[rng.choice(len(first), 30, replace=False)]
    B = 1 << n.bit_length()
    bb = 16 if mode == "waves16" else 0
    x1 = x.copy()
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, ef_construction=efc, build_batch=bb)
    ix.import_graph(g0)
    if mode != "sequential":
        ix.set_option("seq_updates", 0)
    nz = x[:, :d - 1] != 0
    for ids in (first, again):
        # the moved rows keep their number of non-zeros, so the data stays exact
        x1[ids, :d - 1] = np.where(nz[ids], B * rng.choice([-1, 1], (len(ids), d - 1)), 0)
        ix.add(x1[ids].astype(np.float32), ids.astype(np.uint64))
    ix.build()
    m = WaveModel(ip_matrix(x1), g0["levels"], M, ef_construction=efc)
    m.load(g0, n)
    m.update(np.concatenate([first, again]), build_batch=bb, seq_updates=4096 if mode == "sequential" else 0)
    g = check(ix, m, n)
    assert np.array_equal(g["vectors"], x1.astype(np.float32))


# ---- compaction, save / load, shards -------------------------------------------------------------------------------
def test_gpu_compaction_wide_efc():
    """Wave-of-one build at efc 512, 30 % of the points and the entry deleted, compacted on both sides: the repair keeps
    min(efc, |C|) and the orphans are re-linked through the wide search."""
    n, d, M, efc = 700, 16, 8, 512
    x = data(n, d, seed=19)
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, ef_construction=efc, build_batch=1)
    ix.add(x.astype(np.float32))
    o = orc.OracleHNSW(d, "ip", n, M=M, ef_construction=efc)
    o.add(x.astype(np.float32), threads=1)
    g0 = ix.export_graph()
    _assert_same_graph(g0, o.export_graph())
    rng = np.random.default_rng(29)
    dead = np.union1d(rng.choice(n, int(0.3 * n), replace=False), [int(g0["entry"])]).astype(np.uint64)
    ix.remove(dead)
    for lab in dead:
        o.mark_delete(int(lab))
    ix.compact()
    c, _, orphans = compact_oracle(o, dead, int_ip_dist(x), efc=efc)
    g, og = ix.export_graph(), c.export_graph()
    assert ix.size == n - len(dead) and ix.stats()["deleted"] == 0
    assert np.array_equal(g["labels"], og["labels"])
    _assert_same_graph(g, og)


def test_gpu_save_load_then_add_wide_efc():
    n0, n, d, M, efc = 500, 800, 64, 8, 512
    x = np.random.default_rng(31).standard_normal((n, d), dtype=np.float32)
    ehb = _ehb()
    twin = ehb.NativeIndex(d, metric="l2", capacity=n0, M=M, ef_construction=efc)
    ix = ehb.NativeIndex(d, metric="l2", capacity=n0, M=M, ef_construction=efc)
    for t in (twin, ix):
        t.add(x[:n0])
        t.build()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "wide.ehb")
        ix.save(path)
        ld = ehb.NativeIndex.load(path)
    for t in (twin, ld):
        t.add(x[n0:])
        t.build()
    a, b = twin.export_graph(), ld.export_graph()
    for k in ("levels", "up_off", "links0", "links_up", "labels"):
        assert np.array_equal(a[k], b[k]), k
    assert (int(a["entry"]), int(a["maxlevel"])) == (int(b["entry"]), int(b["maxlevel"]))


def test_gpu_sharded_shards_equal_native_wide_efc():
    """Each shard of ShardedIndex(ef_construction=512) is a NativeIndex built from that shard's rows, labels and
    arrival order (devices [0, 0]: a device may repeat)."""
    n, d, M, efc = 1600, 48, 8, 512
    x = np.random.default_rng(37).standard_normal((n, d), dtype=np.float32)
    ehb = _ehb()
    sh = ehb.ShardedIndex(d, [0, 0], metric="ip", capacity=n, M=M, ef_construction=efc)
    sh.add(x)
    sh.build()
    for i in range(2):
        g = sh.shard(i).export_graph()
        assert len(g["labels"]) > efc
        ix = ehb.NativeIndex(d, metric="ip", capacity=len(g["labels"]), M=M, ef_construction=efc)
        ix.add(x[g["labels"].astype(np.int64)], g["labels"])
        ix.build()
        assert_same_ordered(ix.export_graph(), g)


# ---- scale ---------------------------------------------------------------------------------------------------------
def _recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(r.tolist()) & set(t.tolist())) / k for r, t in zip(a, b)]))


def test_gpu_wide_efc_at_scale():
    """Gaussian n = 50k, d = 128, L2: two builds at efc 512 are bit-identical and well formed; recall@10 at ef 32 is
    no lower than the efc 200 build's (- 0.002) and the oracle's at efc 512 (- 0.01)."""
    n, d, nq, k = 50_000, 128, 2000, 10
    rng = np.random.default_rng(41)
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    ehb = _ehb()
    gs, rec = [], {}
    for efc in (512, 512, 200):
        ix = ehb.NativeIndex(d, metric="l2", capacity=n, ef_construction=efc)
        ix.add(x)
        ix.build()
        if efc == 512:
            gs.append(ix.export_graph())
        gt = ix.search_bruteforce(q, k)[0]
        rec[efc] = _recall(ix.search(q, k, ef=32)[0], gt)
    assert_well_formed(gs[0], n)
    for key in ("links0", "links_up", "levels", "up_off"):
        assert np.array_equal(gs[0][key], gs[1][key]), key
    assert (int(gs[0]["entry"]), int(gs[0]["maxlevel"])) == (int(gs[1]["entry"]), int(gs[1]["maxlevel"]))
    r_orc = {}
    for efc in (512, 200):
        o = orc.OracleHNSW(d, "l2", n, ef_construction=efc)
        o.add(x, threads=os.cpu_count() or 1)
        r_orc[efc] = _recall(o.search(q, k, ef=32)[0], gt)
    print(f"recall@10 ef 32: GPU {rec}, oracle {r_orc}")
    assert rec[512] >= r_orc[512] - 0.01, (rec, r_orc)
    assert rec[512] >= rec[200] - 0.002, (rec, r_orc)
