"""The batched GPU build held to the wave model (tests/wave_model.py), row for row and in order.

On build-tie-free inner-product data every distance is exact in fp32 under any summation order and no two
candidates of one selection tie, so the GPU's levels, up_off, entry, max_level and every row (selection order, then
append order) must equal the model's: real wave sizes, every build instantiation (dpad 32 ... 2048), hub rows that
receive more than 128 links in one wave, tombstones, and update waves.  On Gaussian data at scale, where nothing is
exact, two builds must still be bit-identical and every graph must be well formed.
"""
import numpy as np
import pytest

from wave_model import INV, WaveModel, hub_ip, ip_matrix, tiefree_ip

pytestmark = pytest.mark.gpu

DIMS = [29, 64, 128, 250, 383, 512, 768, 1000, 1535, 2048]   # one per dpad class 32 ... 2048


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


# ---- data and helpers ---------------------------------------------------------------------------------------------
def data(n, d, seed=11):
    """Dense tie-free rows up to d = 64, sparse ones (48 non-zeros over all d - 1 coordinates) above."""
    return tiefree_ip(n, d, seed, nnz=None if d <= 64 else 48)[0]


def levels_of(n, d, M):
    """The index's level sequence for n points (it depends on M and the seed only)."""
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M)
    ix.add(np.zeros((n, d), np.float32) + np.arange(1, n + 1, dtype=np.float32)[:, None])
    return ix.export_graph()["levels"]


def gpu_build(x, M, build_batch=0, build_frac=0):
    n, d = x.shape
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, build_batch=build_batch)
    if build_frac:
        ix.set_option("build_frac", build_frac)
    ix.add(x.astype(np.float32))
    ix.build()
    return ix


_MODELS = {}


def model_build(key, x, M, build_batch=0, build_frac=0):
    """The model's graph for one configuration (cached: the model is the slow part)."""
    k = (key, x.shape, M, build_batch, build_frac)
    if k not in _MODELS:
        m = WaveModel(ip_matrix(x), levels_of(x.shape[0], x.shape[1], M), M)
        _MODELS[k] = m.build(build_batch=build_batch, build_frac=build_frac)
    return _MODELS[k]


def assert_same_ordered(g, mg):
    """levels, up_off, entry, max_level and every row, in order (kInvalid padding included)."""
    assert np.array_equal(g["levels"], mg["levels"])
    assert np.array_equal(g["up_off"], mg["up_off"])
    assert (int(g["entry"]), int(g["maxlevel"])) == (int(mg["entry"]), int(mg["maxlevel"]))
    for name in ("links0", "links_up"):
        a, b = np.asarray(g[name]), np.asarray(mg[name])
        assert a.shape == b.shape, (name, a.shape, b.shape)
        bad = np.flatnonzero((a != b).any(1))
        assert bad.size == 0, (name, bad.size, [(int(i), a[i].tolist(), b[i].tolist()) for i in bad[:3]])


def assert_well_formed(g, n):
    """Valid ids first, then INV; no self links, no duplicates, ids < n; upper rows exactly for nodes of level >= 1,
    naming only nodes of at least that level."""
    levels = np.asarray(g["levels"]).astype(np.int64)
    up_off = np.asarray(g["up_off"])
    assert np.array_equal(up_off == INV, levels == 0)
    assert int(levels.sum()) == len(g["links_up"])
    owner = np.repeat(np.arange(n), levels)
    layer = np.concatenate([np.arange(1, lv + 1) for lv in levels]) if len(owner) else np.zeros(0, np.int64)
    assert np.array_equal(up_off[owner].astype(np.int64) + layer - 1, np.arange(len(owner)))
    for rows, own, lay in ((np.asarray(g["links0"]), np.arange(n), np.zeros(n, np.int64)),
                           (np.asarray(g["links_up"]), owner, layer)):
        if not len(rows):
            continue
        valid = rows != INV
        cnt = valid.sum(1)
        assert np.array_equal(valid, np.arange(rows.shape[1])[None, :] < cnt[:, None]), "INV before a valid id"
        r = np.where(valid, rows, 0).astype(np.int64)
        assert (r[valid] < n).all()
        assert not (valid & (r == own[:, None])).any(), "self link"
        s = np.sort(np.where(valid, r, -1 - np.arange(rows.shape[1])[None, :]), 1)
        assert not (s[:, 1:] == s[:, :-1]).any(), "duplicate id in a row"
        assert (levels[r[valid]] >= np.repeat(lay, cnt)).all(), "upper row names a node below its layer"


def check(ix, m, n):
    g = ix.export_graph()
    assert_well_formed(g, n)
    assert_same_ordered(g, m.export())
    return g


# ---- batched inserts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DIMS)
def test_gpu_waves_every_dpad(d):
    """Waves of up to 1/4 of the linked graph at every row width (each BuildShape instantiation)."""
    n, M = 400, 8
    x = data(n, d)
    m = model_build("dpad", x, M, build_frac=4)
    assert max(m.trace["waves"]) >= 60 and m.trace["reselects"] > 100
    check(gpu_build(x, M, build_frac=4), m, n)


@pytest.mark.parametrize("d", [32, 250])
@pytest.mark.parametrize("M", [4, 8, 16])
def test_gpu_waves_M(d, M):
    n = 400
    x = data(n, d, seed=5)
    m = model_build("M", x, M, build_frac=4)
    check(gpu_build(x, M, build_frac=4), m, n)


@pytest.mark.parametrize("build_frac", [1, 4, 64])
@pytest.mark.parametrize("build_batch", [0, 7, 64])
def test_gpu_waves_frac_batch(build_frac, build_batch):
    n, d, M = 500, 48, 8
    x = data(n, d, seed=3)
    m = model_build("fb", x, M, build_batch, build_frac)
    assert 1 < max(m.trace["waves"]) <= (build_batch or 16384)
    check(gpu_build(x, M, build_batch, build_frac), m, n)


def test_gpu_single_wave_isolated():
    """One wave on top of an imported model graph: when a build differs, this names the phase, not the wave."""
    n0, n, d, M = 300, 480, 40, 8
    x = data(n, d, seed=9)
    levels = levels_of(n, d, M)
    base = WaveModel(ip_matrix(x[:n0]), levels[:n0], M).build(build_frac=4)
    g0 = base.export()
    g0.update(vectors=x[:n0].astype(np.float32), labels=np.arange(n0, dtype=np.uint64))
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M)
    ix.import_graph(g0)
    ix.set_option("build_frac", 1)
    ix.add(x[n0:].astype(np.float32), np.arange(n0, n, dtype=np.uint64))
    ix.build()
    m = WaveModel(ip_matrix(x), levels, M)
    m.load(g0, n0)
    m.build(build_frac=1)
    assert m.trace["waves"] == [n - n0]
    check(ix, m, n)


def test_gpu_hub_rows_fold_every_link():
    """x_i = (i + 1) e_{d-1}: every point of a wave selects the same M rows, so from n_linked >= 129 on those rows
    receive more than 128 links in one wave; the fold must consider all of them."""
    n, d, M = 600, 32, 8
    x = hub_ip(n, d)
    m = model_build("hub", x, M, build_frac=1)
    assert m.trace["max_incoming"] > 128 and m.trace["hub_folds"] > 0, m.trace
    check(gpu_build(x, M, build_frac=1), m, n)


@pytest.mark.parametrize("M", [4, 8])
def test_gpu_waves_after_tombstones(M):
    """Batched inserts into an index with 10 % of its points tombstoned (the HASDEL build kernel)."""
    n0, n, d = 400, 500, 32
    x = data(n, d, seed=13)
    levels = levels_of(n, d, M)
    dead = np.random.default_rng(M).choice(n0, n0 // 10, replace=False)
    m = WaveModel(ip_matrix(x), levels, M).build(n0, build_frac=4)
    m.mark_deleted(dead)
    m.build(build_frac=4)
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M)
    ix.set_option("build_frac", 4)
    ix.add(x[:n0].astype(np.float32))
    ix.build()
    ix.remove(dead.astype(np.uint64))
    ix.add(x[n0:].astype(np.float32))
    ix.build()
    check(ix, m, n)


# ---- update waves ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("build_batch", [0, 16])
def test_gpu_update_waves(build_batch):
    """250 moves (30 labels moved twice) applied in waves (seq_updates = 0): all at once, or 16 per wave.  Moved
    points of one wave share neighbours, so re-selections of one row compete and re-links read rows others rewrite."""
    n, d, M = 500, 32, 8
    x = data(n, d, seed=17)
    m0 = model_build("upd", x, M, build_frac=4)
    g0 = m0.export()
    g0.update(vectors=x.astype(np.float32), labels=np.arange(n, dtype=np.uint64))
    rng = np.random.default_rng(23)
    first = rng.choice(n, 220, replace=False)
    again = first[rng.choice(220, 30, replace=False)]
    B = 1 << n.bit_length()
    x1 = x.copy()
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n, M=M, build_batch=build_batch)
    ix.import_graph(g0)
    ix.set_option("seq_updates", 0)
    for ids in (first, again):
        x1[ids, :d - 1] = B * rng.integers(-1, 2, (len(ids), d - 1))
        ix.add(x1[ids].astype(np.float32), ids.astype(np.uint64))
    ix.build()
    m = WaveModel(ip_matrix(x1), g0["levels"], M)
    m.load(g0, n)
    # the first wave's moved points share one-hop rows: the winner rule is exercised
    wave = first[:build_batch or len(first)].tolist()
    hits = {}
    for p in wave:
        for nb in m.row(p, 0):
            hits[nb] = hits.get(nb, 0) + 1
    assert max(hits.values()) >= 2
    m.update(np.concatenate([first, again]), build_batch=build_batch, seq_updates=0)
    g = check(ix, m, n)
    assert np.array_equal(g["vectors"], x1.astype(np.float32))


# ---- determinism at scale -------------------------------------------------------------------------------------------
def gaussian(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)


def _same_graph_bits(a, b):
    for k in ("links0", "links_up", "levels", "up_off"):
        assert np.array_equal(a[k], b[k]), k
    assert (int(a["entry"]), int(a["maxlevel"])) == (int(b["entry"]), int(b["maxlevel"]))


_SCALE = {}


def scale_graph(metric, d):
    key = (metric, d)
    if key not in _SCALE:
        n = 100_000
        x = gaussian(n, d, 31)
        gs = []
        for _ in range(2):
            ix = _ehb().NativeIndex(d, metric=metric, capacity=n)
            ix.add(x)
            ix.build()
            gs.append(ix.export_graph())
        _SCALE[key] = (x, gs)
    return _SCALE[key]


@pytest.mark.parametrize("metric,d", [("l2", 128), ("ip", 96)])
def test_gpu_build_deterministic_at_scale(metric, d):
    x, (a, b) = scale_graph(metric, d)
    assert_well_formed(a, len(x))
    _same_graph_bits(a, b)


def test_gpu_update_waves_deterministic_at_scale():
    """6000 moves exceed the default one-at-a-time limit (4096), so the default wave path runs; two imports of
    the same graph must come out identical."""
    x, (g, _) = scale_graph("l2", 128)
    n, d = x.shape
    rng = np.random.default_rng(41)
    ids = rng.choice(n, 6000, replace=False).astype(np.uint64)
    newx = gaussian(len(ids), d, 43)
    out = []
    for _ in range(2):
        ix = _ehb().NativeIndex(d, metric="l2", capacity=n)
        ix.import_graph(g)
        ix.add(newx, ids)
        ix.build()
        out.append(ix.export_graph())
    assert_well_formed(out[0], n)
    _same_graph_bits(out[0], out[1])
    assert np.array_equal(out[0]["vectors"][ids.astype(np.int64)], newx)
    assert not np.array_equal(out[0]["links0"], g["links0"])
