"""Wide rows, dim 2049 ... 4096 (dpad 3072 and 4096): the wide form of the one-warp walk (the fp32 query in shared
memory, rows read straight into registers in d-slices) and of the build kernels, and every other entry point at
these widths.

  * The walk on the tie-free integer data of test_gpu_walk_exact (exact in any summation order; B (d + 1) <= 2^24
    allows n = 4000 up to d = 3584 and n = 2000 at d = 4096) equals the oracle's hnswlib walk on the identical graph:
    ids, distance bits, hop and evaluation counters, every KPL class, with and without tombstones.  The bf16 walk
    re-ranks in fp32: every distance it returns is the exact path's for that id.
  * A wave of one builds and updates the oracle's graph row for row; batched waves equal tests/wave_model.py;
    compaction equals tests/compact_model.py.
  * GPU build + GPU walk recall at d = 3072 is at least the oracle's (graph and walk) at the same ef.
  * At d = 4096: brute force (fp32 exact, bf16), key mode, get_batch, save / load, export / import, ShardedIndex at
    n_dev = 2 and the one-process-per-GPU exchange at world 2 (both skip without two GPUs where they need them).
  * The hub, the gRPC server, offline.Index and ANNIndex at d = 3072.
"""
import numpy as np
import pytest

from compact_model import compact_oracle, int_ip_dist
from oracle import oracle as orc  # test infrastructure
from test_gpu_bf16_walk import assert_same_walk
from test_gpu_walk_exact import _assert_same_graph, assert_exact, build_tiefree, ip_dist, l2_exact, tiefree
from wave_model import WaveModel, ip_matrix, tiefree_ip

pytestmark = pytest.mark.gpu

DIMS = [2049, 2560, 3072, 3073, 3584, 4096]
NO_LABEL = 0xFFFFFFFFFFFFFFFF


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def _bf16():
    from embeddinghub_b200._native import BF16
    return BF16


def dpad_of(d):
    return 3072 if d <= 3072 else 4096


def kpl_of(ef):
    return 2 if ef <= 64 else (4 if ef <= 128 else (8 if ef <= 256 else 16))


def wide_name(d, ef, deleted=False, bf16=False):
    return (f"hnsw_search_wide_kernel<LPV=32,NQ={dpad_of(d) // 128},KPL={kpl_of(ef)}"
            f"{',HASDEL=1' if deleted else ''}{',ROW=bf16' if bf16 else ''}>")


def n_for(d):
    return 4000 if d <= 4095 else 2000                                  # B * (d + 1) <= 2^24


_CACHE = {}


def graph(d, nq=96):
    """A GPU-built (wide build kernels) graph over tie-free IP data, and the oracle walking the identical graph."""
    if d not in _CACHE:
        ehb = _ehb()
        n = n_for(d)
        x, q = tiefree(n, d, nq)
        ix = ehb.NativeIndex(d, metric="ip", capacity=n)
        ix.add(x.astype(np.float32))
        ix.build()
        g = ix.export_graph()
        assert np.array_equal(g["vectors"], x.astype(np.float32))
        o = orc.OracleHNSW(d, "ip", n)
        o.import_graph(g)
        _CACHE[d] = (x, q, g, o, ix)
    return _CACHE[d]


def oracle_run(o, q, k, ef):
    o.metrics(reset=True)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    return ol, od, oc, o.metrics()


# ---- the walk, exact --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DIMS)
def test_wide_walk_every_kpl_exact(d):
    x, q, g, o, ix = graph(d)
    D = ip_dist(x, q)
    ix.set_search_width(1)
    for ef, k in [(40, 1), (65, 33), (129, 10), (257, 257), (512, 500)]:
        res = ix.search(q.astype(np.float32), k, ef=ef)
        assert ix.last_kernel_name() == wide_name(d, max(ef, k)), ix.last_kernel_name()
        assert_exact(res, ix.stats(), oracle_run(o, q, k, ef), D, k)


@pytest.mark.parametrize("d", [2049, 3072, 4096])
@pytest.mark.parametrize("ef", [64, 256])
def test_wide_walk_tombstones_exact(d, ef):
    """One query per call (the overflow flag is that query's): an unflagged query equals the oracle exactly."""
    ehb = _ehb()
    x, q, g, _, _ = graph(d)
    n, nq, k = x.shape[0], 32, 10
    q = q[:nq]
    D = ip_dist(x, q)
    dead = np.random.default_rng(d + ef).choice(n, n // 10, replace=False)
    dead = np.union1d(dead, [int(g["entry"])]).astype(np.uint64)
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    for lab in dead:
        o.mark_delete(int(lab))
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.import_graph(g)
    ix.set_search_width(1)
    ix.set_option("combine", 0)
    ix.remove(dead)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    flagged = 0
    for i in range(nq):
        l, dd, c = ix.search(q[i:i + 1].astype(np.float32), k, ef=ef)
        assert ix.last_kernel_name() == wide_name(d, ef, deleted=True)
        got = l[0, :c[0]].astype(np.int64)
        assert not np.isin(got, dead.astype(np.int64)).any()
        assert np.array_equal(dd[0, :c[0]].view(np.uint32), D[i, got].view(np.uint32))
        if ix.stats()["visited_overflow"]:
            flagged += 1
            continue
        assert c[0] == oc[i] and np.array_equal(l[0], ol[i]), (i, l[0], ol[i])
        assert np.array_equal(dd[0].view(np.uint32), od[i].view(np.uint32))
    assert flagged < nq // 2


@pytest.mark.parametrize("d", DIMS)
def test_wide_bf16_walk_reranked_exact(d):
    """On rows exact in bf16 (integers in [-8, 8]) the bf16 walk computes the fp32 walk's distances, so it walks the
    same way: distance bits, counts, hop / evaluation counters and (distance, id) pairs equal the fp32 wide walk's,
    every KPL class (the fp32 re-rank orders exact ties its own way).
    On the tie-free rows (not exact in bf16) every distance the re-rank returns is the exact one of its id."""
    ehb, BF16 = _ehb(), _bf16()
    n, nq = 3000, 64
    rng = np.random.default_rng(d + 1)
    x = rng.integers(-8, 9, (n, d)).astype(np.float32)
    q = rng.integers(-8, 9, (nq, d)).astype(np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(x)
    ix.build()
    ix.set_search_width(1)
    for ef, k in [(40, 10), (100, 10), (200, 50), (400, 100)]:
        f = ix.search(q, k, ef=ef)
        fs = ix.stats()
        b = ix.search(q, k, ef=ef, precision=BF16)
        bs = ix.stats()
        assert ix.last_kernel_name() == wide_name(d, ef, bf16=True), ix.last_kernel_name()
        assert_same_walk(f, b, k)                  # (distance, label) pairs; ties cut by the k-th only by distance
        assert (fs["hops_upper"], fs["hops_base"]) == (bs["hops_upper"], bs["hops_base"])
        if fs["visited_overflow"] == 0 and bs["visited_overflow"] == 0:   # a full table only adds re-evaluations
            assert fs["dist_evals"] == bs["dist_evals"]
    tx, tq, _, _, tix = graph(d)
    l, dd, c = tix.search(tq.astype(np.float32), 10, ef=128, precision=BF16)
    assert tix.last_kernel_name() == wide_name(d, 128, bf16=True), tix.last_kernel_name()
    assert np.all(c == 10)
    exact = np.take_along_axis(ip_dist(tx, tq), l.astype(np.int64), 1)
    assert np.array_equal(dd.view(np.uint32), exact.view(np.uint32))


@pytest.mark.parametrize("d", [2049, 3584, 4096])
@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_wide_walk_l2_cosine(d, metric):
    """L2 on integer rows: every distance is the exact squared distance of its id; ids equal the oracle's walk on
    the identical graph (ties aside).  Cosine: ids equal the oracle's walk, distances within 1e-4 |d|."""
    ehb = _ehb()
    n, nq, k, ef = 2000, 64, 10, 64
    r = min(200, int(2048 / np.sqrt(d)) - 1)
    rng = np.random.default_rng(d)
    x = rng.integers(-r, r + 1, (n, d)).astype(np.int64)
    q = rng.integers(-r, r + 1, (nq, d)).astype(np.int64)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(x.astype(np.float32))
    ix.build()
    o = orc.OracleHNSW(d, metric, n)
    o.import_graph(ix.export_graph())
    ix.set_search_width(1)
    l, dd, c = ix.search(q.astype(np.float32), k, ef=ef)
    assert ix.last_kernel_name() == wide_name(d, ef)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    assert np.all(c == k) and np.array_equal(c, oc)
    assert np.mean(l == ol) >= 0.99
    if metric == "l2":
        assert np.array_equal(dd.view(np.uint32), l2_exact(x, q, l).view(np.uint32))
    else:
        m = l == ol
        np.testing.assert_allclose(dd[m], od[m], rtol=1e-4, atol=1e-6)


# ---- the build, exact --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [2049, 3072, 4096])
def test_wide_wave_of_one_build_update_compact_equal_oracle(d):
    """build_tiefree at d <= 4096 allows n < 64 (B = 64): sequential addPoint, updatePoint moves and a compaction
    reproduce the oracle's graphs row for row."""
    ehb = _ehb()
    n, M = 60, 4
    x, B = build_tiefree(n, d)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n, M=M, build_batch=1)
    ix.add(x.astype(np.float32))
    o = orc.OracleHNSW(d, "ip", n, M=M)
    o.add(x.astype(np.float32), threads=1)
    _assert_same_graph(ix.export_graph(), o.export_graph())
    rng = np.random.default_rng(d)
    moved = rng.choice(n, 8, replace=False)
    newx = x[moved].copy()
    newx[:, :d - 1] = B * rng.integers(-1, 2, (len(moved), d - 1))
    for i, lab in enumerate(moved):
        ix.add(newx[i:i + 1].astype(np.float32), np.array([lab], np.uint64))
        ix.build()
        o.add(newx[i:i + 1].astype(np.float32), np.array([lab], np.uint64), threads=1)
    _assert_same_graph(ix.export_graph(), o.export_graph())
    x[moved] = newx
    g0 = ix.export_graph()
    dead = np.union1d(rng.choice(n, n // 4, replace=False), [int(g0["entry"])]).astype(np.uint64)
    ix.remove(dead)
    for lab in dead:
        o.mark_delete(int(lab))
    ix.compact()
    c, _, _ = compact_oracle(o, dead, int_ip_dist(x))
    g, og = ix.export_graph(), c.export_graph()
    assert np.array_equal(g["labels"], og["labels"]) and np.array_equal(g["vectors"], og["vectors"])
    _assert_same_graph(g, og)


@pytest.mark.parametrize("d", [2049, 3073, 4096])
def test_wide_batched_waves_equal_model(d):
    ehb = _ehb()
    n, M = 400, 8
    x = tiefree_ip(n, d, 11, nnz=48)[0]
    lv = ehb.NativeIndex(d, metric="ip", capacity=n, M=M)
    lv.add(np.zeros((n, d), np.float32) + np.arange(1, n + 1, dtype=np.float32)[:, None])
    m = WaveModel(ip_matrix(x), lv.export_graph()["levels"], M).build(build_frac=4)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n, M=M)
    ix.set_option("build_frac", 4)
    ix.add(x.astype(np.float32))
    ix.build()
    g, mg = ix.export_graph(), m.export()
    for name in ("levels", "up_off", "links0", "links_up"):
        assert np.array_equal(np.asarray(g[name]), np.asarray(mg[name])), name
    assert (int(g["entry"]), int(g["maxlevel"])) == (int(mg["entry"]), int(mg["maxlevel"]))


# ---- recall parity -------------------------------------------------------------------------------------------------
def test_wide_recall_parity_gmm_3072():
    ehb = _ehb()
    n, d, nq, k, ef = 50_000, 3072, 500, 10, 64
    rng = np.random.default_rng(3072)
    centers = rng.standard_normal((64, d), dtype=np.float32) * 2
    x = (centers[rng.integers(0, 64, n)] + rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)
    q = (centers[rng.integers(0, 64, nq)] + rng.standard_normal((nq, d), dtype=np.float32)).astype(np.float32)
    ix = ehb.NativeIndex(d, metric="l2", capacity=n)
    ix.add(x)
    ix.build()
    ix.set_search_width(1)
    gl, gd, _ = ix.search(q, k, ef=ef)
    assert ix.last_kernel_name() == wide_name(d, ef)
    el, ed, _ = ix.search_bruteforce(q, k)
    o = orc.OracleHNSW(d, "l2", n)
    o.add(x, threads=32)
    ol, _, _ = o.search(q, k, ef=ef, threads=8)
    rec = lambda a: np.mean([len(set(r.tolist()) & set(t.tolist())) / k for r, t in zip(a, el)])
    assert rec(gl) >= rec(ol) - 0.005, (rec(gl), rec(ol))
    exact = ((x[gl.astype(np.int64)].astype(np.float64) - q[:, None, :]) ** 2).sum(-1)
    assert np.all(np.abs(gd - exact) <= 1e-4 * np.abs(exact) + 1e-3)


# ---- every other entry point at d = 4096 ---------------------------------------------------------------------------
def _gauss_index(ehb, d=4096, n=3000, metric="ip", seed=4096):
    x = np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(x)
    ix.build()
    return ix, x


def test_wide_bruteforce_against_numpy():
    ehb = _ehb()
    ix, x = _gauss_index(ehb, metric="l2")
    q = np.random.default_rng(1).standard_normal((64, 4096), dtype=np.float32)
    k = 10
    ref = ((q[:, None, :].astype(np.float64) - x[None].astype(np.float64)) ** 2).sum(-1)
    truth = np.argsort(ref, 1, kind="stable")[:, :k]
    l, dd, c = ix.search_bruteforce(q, k)
    assert np.all(c == k) and np.mean(l == truth) >= 0.999
    np.testing.assert_allclose(dd, np.take_along_axis(ref, l.astype(np.int64), 1), rtol=1e-4)
    bl, bd, bc = ix.search_bruteforce(q, k, precision=_bf16())
    same = bl == l
    assert same.mean() >= 0.99 and np.array_equal(bd[same].view(np.uint32), dd[same].view(np.uint32))


@pytest.mark.parametrize("precision", [0, 1])
def test_wide_key_mode_get_batch_and_round_trips(precision, tmp_path):
    from label_rule_model import drop_self
    ehb = _ehb()
    ix, x = _gauss_index(ehb)
    labels = np.arange(0, 3000, 37, dtype=np.uint64)
    rows = ix.get_batch(labels)
    assert np.array_equal(rows, x[labels.astype(np.int64)])
    k, ef = 10, 64
    L, D, Cn = ix.search(rows, k + 1, ef, precision)
    want = drop_self(labels, L, D, Cn, k)
    got = ix.search_by_label(labels, k, ef, precision)
    for a, b in zip(got, want):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    _, tl, td, tc = ix.neighbor_table(k, ef, precision)
    tw = drop_self(np.arange(3000, dtype=np.uint64), *ix.search(x, k + 1, ef, precision), k)
    assert np.array_equal(tl, tw[0]) and np.array_equal(td.view(np.uint32), tw[1].view(np.uint32))
    base = ix.search(x[:100], k, ef, precision)
    path = str(tmp_path / "wide.ehb")
    ix.save(path)
    lx = ehb.NativeIndex.load(path)
    ex = ehb.NativeIndex(4096, metric="ip", capacity=3000)
    ex.import_graph(ix.export_graph())
    for other in (lx, ex):
        r = other.search(x[:100], k, ef, precision)
        assert np.array_equal(r[0], base[0]) and np.array_equal(r[1].view(np.uint32), base[1].view(np.uint32))


def _two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")


def test_wide_sharded_two_devices():
    _two_gpus()
    ehb = _ehb()
    d, n, k, ef = 4096, 4000, 10, 64
    x = np.random.default_rng(7).standard_normal((n, d), dtype=np.float32)
    sx = ehb.ShardedIndex(d, [0, 1], metric="ip", capacity=n)
    sx.add(x)
    sx.build()
    q = np.random.default_rng(8).standard_normal((50, d), dtype=np.float32)
    l, dd, c = sx.search(q, k, ef)
    el, ed, _ = sx.search_bruteforce(q, k)
    rec = np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(l, el)])
    assert np.all(c == k) and rec >= 0.9
    labels = np.arange(0, n, 97, dtype=np.uint64)
    bl, bd, bc = sx.search_by_label(labels, k, ef)
    assert np.all(bc == k) and not np.any(bl == labels[:, None])
    assert np.array_equal(sx.get_batch(labels), x[labels.astype(np.int64)])


@pytest.mark.parametrize("precision", [0, 1])
def test_wide_exchange_key_mode_world_two(precision):
    """The one-process-per-GPU exchange with max_dim = 4096: key-mode steps (owners push 16 KB rows, fused
    k + 1 step) equal the rule over the fused step on both ranks."""
    _two_gpus()
    from test_gpu_exchange_by_label import Pair, assert_held, batches, gauss
    d, n, cap, k, ef = 4096, 1500, 64, 10, 64
    x = gauss(2 * n, d, 4096)
    p = Pair([x[:n], x[n:]], d, "ip", cap, ef, max_dim=4096)
    try:
        bs = batches(n, cap, 4097)
        p.warm(bs[0], k, ef, precision)
        for labels in bs[:3]:
            assert_held(p.by_label(labels, k, ef, precision), p.reference(labels, k, ef, precision), len(labels))
    finally:
        p.close()


# ---- surfaces ------------------------------------------------------------------------------------------------------
def test_wide_hub_grpc_offline_ann_index():
    import grpc

    from embeddinghub_b200 import grpc_server as gs
    from embeddinghub_b200.ann_index import ANNIndex
    from embeddinghub_b200.offline import Index

    d = 3072
    rng = np.random.default_rng(3)
    emb = {f"k{i}": rng.standard_normal(d).astype(np.float32).tolist() for i in range(40)}
    server, port = gs.make_server("127.0.0.1:0", max_workers=4)
    server.start()
    try:
        with grpc.insecure_channel(f"127.0.0.1:{port}") as ch:
            stub = gs.Stub(ch)
            stub.CreateSpace(gs.M["CreateSpaceRequest"](name="s", dims=d))
            for key, v in emb.items():
                stub.Set(gs.M["SetRequest"](space="s", key=key, embedding=gs.M["Embedding"](values=v)))
            got = stub.Get(gs.M["GetRequest"](space="s", key="k3"))
            assert np.array_equal(np.float32(got.embedding.values), np.float32(emb["k3"]))
            nn = stub.NearestNeighbor(gs.M["NearestNeighborRequest"](space="s", key="k3", num=5))
            assert len(nn.keys) == 5 and "k3" not in nn.keys
    finally:
        server.stop(0)
    ix = Index(iter(emb.items()), d)
    assert ix.nearest_neighbor(3, embedding=emb["k5"])[0] == "k5"
    ann = ANNIndex(d)
    for key, v in emb.items():
        ann.set(key, v)
    assert ann.approx_nearest(emb["k7"], 1)[0] == "k7"
