"""The wide-beam walk (ehb_index_search_beam and friends, max(ef, k) 513 .. 4096) held exactly against hnswlib.

On the tie-free inner-product data of test_gpu_walk_exact the walk must return the oracle's ids, distance bits,
counts and hop / evaluation counters with its result set in shared memory and its visited table in device memory,
for every row shape; up to 512 every beam entry point is exactly its _ex counterpart.
"""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import embeddinghub_b200 as ehb  # noqa: E402
from embeddinghub_b200._native import BF16, FP32, _p, lib  # noqa: E402
from label_rule_model import drop_self  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from test_gpu_bf16_walk import split_tiefree  # noqa: E402
from test_gpu_walk_exact import assert_exact, ip_dist, l2_exact, tiefree  # noqa: E402
from test_gpu_wide_rows import graph as wide_graph  # noqa: E402

EHB_ERR_INVALID = 1
DIMS = [29, 64, 128, 250, 383, 512, 768, 1000, 1535, 2048]   # one per dpad class 32 ... 2048
EFS = [513, 1057, 2049, 4096]
NQ = 24


def n_for(d):
    """The largest n <= 20000 whose tie-free data keeps B (d + 1) <= 2^24 (B: the power of two tiefree picks)."""
    b = 1 << ((1 << 24) // (d + 1)).bit_length() - 1
    return min(20000, b - 2)


def dpad_of(d):
    return next(s for s in (32, 64, 128, 256, 384, 512, 768, 1024, 1536, 2048, 3072, 4096) if d <= s)


def beam_name(d, deleted=False, bf16=False):
    row = dpad_of(d) * (2 if bf16 else 4)
    lpv = 32 if row > 1024 else 8
    return (f"hnsw_search_beam_kernel<LPV={lpv},NQ={dpad_of(d) // (4 * lpv)}"
            f"{',HASDEL=1' if deleted else ''}{',ROW=bf16' if bf16 else ''}>")


_CACHE = {}


def graph(d):
    """A GPU-built graph over tie-free IP data (n_for(d) rows), a walker on it, and the oracle on the same graph."""
    if d not in _CACHE:
        n = n_for(d)
        x, q = tiefree(n, d, NQ)
        ix = ehb.NativeIndex(d, metric="ip", capacity=n)
        ix.add(x.astype(np.float32))
        ix.build()
        g = ix.export_graph()
        assert np.array_equal(g["vectors"], x.astype(np.float32))
        o = orc.OracleHNSW(d, "ip", n)
        o.import_graph(g)
        ix.set_option("combine", 0)
        _CACHE[d] = (x, q, g, o, ix)
    return _CACHE[d]


def oracle_run(o, q, k, ef):
    o.metrics(reset=True)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    return ol, od, oc, o.metrics()


def same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def check_exact(res, st, ref, D, k):
    """assert_exact; when k exceeds the n points every query returns, the padding tail is compared on its own."""
    n = D.shape[1]
    if k > n:
        assert np.all(res[0][:, n:] == ehb.NO_LABEL) and np.all(np.isinf(res[1][:, n:]))
        res = (res[0][:, :n], res[1][:, :n], res[2])
        ref = (ref[0][:, :n], ref[1][:, :n], ref[2], ref[3])
    assert_exact(res, st, ref, D, min(k, n))


# ---- the walk, exact ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DIMS)
def test_beam_walk_every_row_shape_exact(d):
    x, q, g, o, ix = graph(d)
    D = ip_dist(x, q)
    for ef in EFS:
        for k in sorted({1, 600, ef}):
            res = ix.search_beam(q.astype(np.float32), k, ef=ef)
            st = ix.stats()
            assert ix.last_kernel_name() == beam_name(d), ix.last_kernel_name()
            assert st["visited_overflow"] == 0
            check_exact(res, st, oracle_run(o, q, k, ef), D, k)


@pytest.mark.parametrize("d", [3072, 4096])
def test_beam_walk_wide_rows_exact(d):
    x, q, g, o, ix = wide_graph(d)
    D = ip_dist(x, q)
    q = q[:NQ]
    D = D[:NQ]
    for ef, k in [(513, 1), (1057, 600), (4096, 600), (4096, 4096)]:
        res = ix.search_beam(q.astype(np.float32), k, ef=ef)
        st = ix.stats()
        assert ix.last_kernel_name() == beam_name(d), ix.last_kernel_name()
        assert st["visited_overflow"] == 0
        check_exact(res, st, oracle_run(o, q, k, ef), D, k)


@pytest.mark.parametrize("frac", [0.1, 0.5])
@pytest.mark.parametrize("d", [64, 768])
def test_beam_walk_tombstones_exact(d, frac):
    """Deleted points (and the entry point) are traversed, never returned: one query per call, so the overflow flag
    is that query's.  Every query returns sorted, unique, live ids with exact distances; a query with a clear flag
    equals the oracle after mark_delete exactly, and at 10 % deleted every query must have a clear flag."""
    x, q, g, _, _ = graph(d)
    n = x.shape[0]
    D = ip_dist(x, q)
    rng = np.random.default_rng(int(frac * 100) + d)
    dead = np.union1d(rng.choice(n, int(frac * n), replace=False), [int(g["entry"])]).astype(np.uint64)
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    for lab in dead:
        o.mark_delete(int(lab))
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.import_graph(g)
    ix.set_option("combine", 0)
    ix.remove(dead)
    live = np.ones(n, bool)
    live[dead.astype(np.int64)] = False
    for ef, k in [(1057, 600), (4096, 100)]:
        ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
        flagged = 0
        for i in range(8):
            l, dd, c = ix.search_beam(q[i:i + 1].astype(np.float32), k, ef=ef)
            assert ix.last_kernel_name() == beam_name(d, deleted=True)
            got = l[0, :c[0]].astype(np.int64)
            assert np.all(live[got]) and len(set(got.tolist())) == c[0]
            assert np.all(l[0, c[0]:] == ehb.NO_LABEL)
            assert np.array_equal(dd[0, :c[0]].view(np.uint32), D[i, got].view(np.uint32))
            assert np.all(np.diff(dd[0, :c[0]]) > 0)
            if ix.stats()["visited_overflow"]:
                flagged += 1
                continue
            assert c[0] == oc[i] and np.array_equal(l[0], ol[i]), i
            assert np.array_equal(dd[0].view(np.uint32), od[i].view(np.uint32))
        print(f"beam tombstones d={d} ef={ef} deleted={frac:.0%}+entry: {flagged}/8 queries flagged")
        if frac <= 0.1:
            assert flagged == 0


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_beam_walk_l2_cosine(metric):
    """The integer data of test_l2_integer_distances_exact: L2 distances are the exact squared distances of their
    ids, ids equal the oracle's walk on the identical graph (ties aside); cosine ids equal the oracle's."""
    d, n, nq, k, ef = 64, 3000, 32, 600, 1057
    r = min(200, int(2048 / np.sqrt(d)) - 1)
    rng = np.random.default_rng(d)
    x = rng.integers(-r, r + 1, (n, d)).astype(np.int64)
    q = rng.integers(-r, r + 1, (nq, d)).astype(np.int64)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(x.astype(np.float32))
    ix.build()
    o = orc.OracleHNSW(d, metric, n)
    o.import_graph(ix.export_graph())
    l, dd, c = ix.search_beam(q.astype(np.float32), k, ef=ef)
    assert ix.last_kernel_name() == beam_name(d)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    assert np.all(c == k) and np.array_equal(c, oc)
    assert np.mean(l == ol) >= 0.995
    assert np.all(np.diff(dd, axis=1) >= 0)
    if metric == "l2":
        assert np.array_equal(dd.view(np.uint32), l2_exact(x, q, l).view(np.uint32))
    else:
        m = l == ol
        np.testing.assert_allclose(dd[m], od[m], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("d", [64, 768])
def test_beam_bf16_equals_oracle(d):
    """bf16-exact tie-free rows: the bf16 walk plus the fp32 re-rank of all max(ef, k) retained keys returns the
    oracle's ids and distance bits, and every distance is the canonical fp32 distance of its id."""
    n = 6000
    x, q = split_tiefree(n, d, NQ)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(x.astype(np.float32))
    ix.build()
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(ix.export_graph())
    D = (1 - q @ x.T).astype(np.float32)
    for ef, k in [(513, 10), (2049, 600), (4096, 4096)]:
        o.metrics(reset=True)
        ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
        om = o.metrics()
        l, dd, c = ix.search_beam(q.astype(np.float32), k, ef=ef, precision=BF16)
        st = ix.stats()
        assert ix.last_kernel_name() == beam_name(d, bf16=True)
        assert np.array_equal(c, oc) and np.array_equal(l, ol)
        assert np.array_equal(dd.view(np.uint32), od.view(np.uint32))
        ok = l != ehb.NO_LABEL
        exact = np.take_along_axis(D, np.where(ok, l, 0).astype(np.int64), 1)
        assert np.array_equal(dd[ok].view(np.uint32), exact[ok].view(np.uint32))
        assert st["hops_upper"] == om["hops_upper"] and st["hops_base"] == om["hops0"]
        assert st["visited_overflow"] == 0 and st["dist_evals"] == om["evals"]


@pytest.mark.parametrize("precision", [FP32, BF16])
def test_beam_by_label_is_the_host_composition(precision):
    x, q, g, o, ix = graph(128)
    labels = np.array([5, 17, 1234, 9999, 17], np.uint64)
    for ef, k in [(600, 10), (1057, 1056), (4096, 4095)]:
        got = ix.search_by_label_beam(labels, k, ef=ef, precision=precision)
        assert ix.last_kernel_name() == beam_name(128, bf16=precision == BF16)
        rows = ix.get_batch(labels)
        l1, d1, c1 = ix.search_beam(rows, k + 1, ef=ef, precision=precision)
        same(got, drop_self(labels, l1, d1, c1, k))


# ---- up to 512: the _ex entry points ---------------------------------------------------------------------------
def test_beam_up_to_512_is_the_ex_path():
    """Gaussian rows: stored rows of the tie-free data, used as by-label queries, have distances far beyond 2^24 and
    so exact fp32 ties, whose order is not part of any contract."""
    import torch
    rng = np.random.default_rng(64)
    ix = ehb.NativeIndex(64, metric="ip", capacity=6000)
    ix.add(rng.standard_normal((6000, 64), dtype=np.float32))
    ix.build()
    qf = rng.standard_normal((NQ, 64), dtype=np.float32)
    labels = np.array([3, 99, 4000], np.uint64)
    for precision in (FP32, BF16):
        for ef, k in [(0, 10), (40, 10), (256, 100), (512, 512), (100, 512)]:
            a = ix.search(qf, k, ef=ef, precision=precision)
            na = ix.last_kernel_name()
            b = ix.search_beam(qf, k, ef=ef, precision=precision)
            assert ix.last_kernel_name() == na and "beam" not in na
            same(a, b)
            if k < 512:
                a = ix.search_by_label(labels, k, ef=ef, precision=precision)
                na = ix.last_kernel_name()
                b = ix.search_by_label_beam(labels, k, ef=ef, precision=precision)
                assert ix.last_kernel_name() == na
                same(a, b)
            dq = torch.from_numpy(qf).cuda()
            outs = []
            for fn in (ix.search_dev, ix.search_beam_dev):
                lab = torch.empty((len(qf), k), dtype=torch.int64, device="cuda")
                dst = torch.empty((len(qf), k), dtype=torch.float32, device="cuda")
                cnt = torch.empty(len(qf), dtype=torch.int32, device="cuda")
                fn(dq.data_ptr(), len(qf), k, ef, lab.data_ptr(), dst.data_ptr(), cnt.data_ptr(), precision=precision)
                torch.cuda.synchronize()
                outs.append((lab.cpu().numpy().view(np.uint64), dst.cpu().numpy(), cnt.cpu().numpy().view(np.uint32),
                             ix.last_kernel_name()))
            same(outs[0][:3], outs[1][:3])
            assert outs[0][3] == outs[1][3]


def test_beam_dev_matches_host():
    import torch
    x, q, g, o, ix = graph(512)
    qf = np.ascontiguousarray(q.astype(np.float32))
    for precision in (FP32, BF16):
        ref = ix.search_beam(qf, 700, ef=2049, precision=precision)
        dq = torch.from_numpy(qf).cuda()
        lab = torch.empty((len(qf), 700), dtype=torch.int64, device="cuda")
        dst = torch.empty((len(qf), 700), dtype=torch.float32, device="cuda")
        cnt = torch.empty(len(qf), dtype=torch.int32, device="cuda")
        ix.search_beam_dev(dq.data_ptr(), len(qf), 700, 2049, lab.data_ptr(), dst.data_ptr(), cnt.data_ptr(),
                           precision=precision)
        torch.cuda.synchronize()
        same(ref, (lab.cpu().numpy().view(np.uint64), dst.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)))


# ---- argument checks --------------------------------------------------------------------------------------------
CASES = ["ef4097", "k4097", "by_label_k4096", "precision", "null_query", "null_out", "nq0", "k0"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("entry", ["host", "dev", "by_label"])
def test_beam_rejects_and_leaves_buffers(entry, case):
    import torch
    x, q, g, o, ix = graph(64)
    if case == "by_label_k4096" and entry != "by_label":
        pytest.skip("k + 1 applies to the by-label form")
    nq = 0 if case == "nq0" else 2
    k = {"k4097": 4097, "by_label_k4096": 4096, "k0": 0}.get(case, 5)
    ef = 4097 if case == "ef4097" else 600
    precision = 7 if case == "precision" else FP32
    kk = max(k, 1)
    if entry == "dev":
        dq = torch.from_numpy(np.ascontiguousarray(q[:2].astype(np.float32))).cuda()
        lab = torch.full((2, kk), 7, dtype=torch.int64, device="cuda")
        dst = torch.full((2, kk), 3.0, dtype=torch.float32, device="cuda")
        cnt = torch.full((2,), 9, dtype=torch.int32, device="cuda")
        rc = lib().ehb_index_search_beam_dev(ix._h, nq, None if case == "null_query" else C.c_void_p(dq.data_ptr()), k,
                                             ef, precision, None if case == "null_out" else C.c_void_p(lab.data_ptr()),
                                             C.c_void_p(dst.data_ptr()), C.c_void_p(cnt.data_ptr()), None)
        torch.cuda.synchronize()
        untouched = bool((lab == 7).all() and (dst == 3.0).all() and (cnt == 9).all())
    else:
        lab = np.full((2, kk), 7, np.uint64)
        dst = np.full((2, kk), 3.0, np.float32)
        cnt = np.full(2, 9, np.uint32)
        if entry == "host":
            qf = np.ascontiguousarray(q[:2].astype(np.float32))
            rc = lib().ehb_index_search_beam(ix._h, nq, None if case == "null_query" else _p(qf), k, ef, precision,
                                             None if case == "null_out" else _p(lab), _p(dst), _p(cnt))
        else:
            labels = np.array([1, 123456789], np.uint64)      # the second is not stored: a lookup would fail
            rc = lib().ehb_index_search_by_label_beam(ix._h, nq, None if case == "null_query" else _p(labels), k, ef,
                                                      precision, None if case == "null_out" else _p(lab), _p(dst),
                                                      _p(cnt))
        untouched = bool((lab == 7).all() and (dst == 3.0).all() and (cnt == 9).all())
    assert rc == (0 if case in ("nq0", "k0") else EHB_ERR_INVALID), rc
    assert untouched


def test_beam_default_ef_above_512():
    x, q, g, o, ix = graph(64)
    D = ip_dist(x, q)
    ix.set_ef(600)
    try:
        res = ix.search_beam(q.astype(np.float32), 10)
        assert ix.last_kernel_name() == beam_name(64)
        assert_exact(res, ix.stats(), oracle_run(o, q, 10, 600), D, 10)
        with pytest.raises(ehb.EhbError):
            ix.search(q.astype(np.float32), 10)           # the _ex path keeps its limit
    finally:
        ix.set_ef(10)


# ---- concurrency --------------------------------------------------------------------------------------------------
def test_beam_concurrent_with_ex_and_mutation():
    """Host threads run wide-beam searches (fp32 and bf16) beside _ex searches and an add followed by a build; every
    result equals the same search run alone on the same index state (before or after the add)."""
    d, n = 128, 6000
    rng = np.random.default_rng(5)
    x = rng.standard_normal((n + 500, d), dtype=np.float32)
    q = rng.standard_normal((16, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n + 500)
    ix.add(x[:n])
    ix.build()
    ix.search(q, 10, precision=BF16)                       # the bf16 copy exists before the threads start
    jobs = [("beam", 600, 1057, FP32), ("beam", 100, 2049, BF16), ("ex", 10, 128, FP32), ("beam", 4096, 4096, FP32)]

    def run(job):
        kind, k, ef, prec = job
        return (ix.search_beam if kind == "beam" else ix.search)(q, k, ef=ef, precision=prec)

    before = [run(j) for j in jobs]
    out, errs = {}, []

    def worker(i, j):
        try:
            out[i] = [run(j) for _ in range(3)]
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    def mutate():
        try:
            ix.add(x[n:])
            ix.build()
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=worker, args=(i, j)) for i, j in enumerate(jobs)]
    ts.append(threading.Thread(target=mutate))
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    after = [run(j) for j in jobs]
    for i in range(len(jobs)):
        for r in out[i]:
            assert any(np.array_equal(r[0], ref[0]) and np.array_equal(r[1].view(np.uint32), ref[1].view(np.uint32))
                       and np.array_equal(r[2], ref[2]) for ref in (before[i], after[i])), jobs[i]
