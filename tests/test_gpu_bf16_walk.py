"""The bf16 graph search (ehb_index_search_ex with EHB_BF16): the HNSW walk over the bf16 copy of the rows, then an
fp32 re-rank of the walk's whole result set.

Held exactly:
  * on data bf16 represents exactly (small integers), the bf16 walk computes the fp32 walk's distances in any
    summation order, so it must retain the same set with the same hop and evaluation counters.  The re-rank
    orders equal distances by internal id while the fp32 walk orders them by its result-set slot, so rows are
    compared as (distance, label) pairs in distance order, with the members of a tie group that straddles the
    k-th position compared by distance only;
  * on tie-free integer inner-product data split so that every coordinate is exact in bf16, the bf16 search
    returns the oracle's ids, distance bits, counts and counters on the same graph;
  * every returned distance is the canonical fp32 distance of its id, bit for bit, on any data.
Held within a tolerance: recall@10 against the exact path, at least the fp32 walk's minus 0.01 on iid Gaussian and
1024-centre GMM data.  1000 queries: with 400, sampling noise alone once put one case 0.011 below (iid Gaussian,
d = 128, cosine, ef = 64: 0.341 against 0.352; 0.3348 against 0.3343 with 1000 queries).
"""
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIMS = [29, 64, 128, 250, 383, 512, 768, 1000, 1535, 2048]   # one per dpad class 32 ... 2048
NO_LABEL = np.uint64(0xFFFFFFFFFFFFFFFF)


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def _bf16():
    from embeddinghub_b200._native import BF16
    return BF16


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def dpad_of(d):
    return next(s for s in (32, 64, 128, 256, 384, 512, 768, 1024, 1536, 2048) if d <= s)


def kpl_of(ef):
    return 2 if ef <= 64 else (4 if ef <= 128 else (8 if ef <= 256 else 16))


def name_of(d, ef, bf16, kind="hnsw_search_kernel", deleted=False):
    dpad = dpad_of(d)
    rb = dpad * (2 if bf16 else 4)
    lpv = 32 if rb > 1024 else 8
    return (f"{kind}<LPV={lpv},NQ={dpad // (4 * lpv)},KPL={kpl_of(ef)}{',HASDEL=1' if deleted else ''}"
            f"{',ROW=bf16' if bf16 else ''}>")


def intdata(n, d, nq, seed=5, lo=-8, hi=8):
    rng = np.random.default_rng(seed)
    return (rng.integers(lo, hi + 1, (n, d)).astype(np.float32), rng.integers(lo, hi + 1, (nq, d)).astype(np.float32))


def exact_dist(x, q, labels, metric):
    """int64 reference distances of the returned labels (exact in fp32 for these small integers)."""
    ok = labels != NO_LABEL
    rows = x[np.where(ok, labels, 0).astype(np.int64)].astype(np.int64)
    qi = q.astype(np.int64)[:, None, :]
    if metric == "l2":
        r = ((rows - qi) ** 2).sum(-1)
    else:
        r = 1 - (rows * qi).sum(-1)
    assert np.abs(r).max() < 1 << 24
    return np.where(ok, r.astype(np.float32), np.float32(np.inf))


def walk_stats(ix):
    st = ix.stats()
    return st["hops_upper"], st["hops_base"], st["dist_evals"], st["visited_overflow"]


def assert_same_counters(fs, bs):
    """Equal hops; equal evaluations unless a visited table ran full.  The table's size follows the shared memory
    left beside the TMA staging ring (sized from the row bytes) and the dense form's occupancy target, so the two
    walks may get different tables, and a full table adds re-evaluations (never a different result)."""
    assert fs[:2] == bs[:2], (fs, bs)
    if fs[3] == 0 and bs[3] == 0:
        assert fs[2] == bs[2], (fs, bs)


def assert_same_walk(f, b, k):
    """fp32-walk result f and bf16 result b on bf16-exact data: same counts, same distance bits in order, same
    (distance, label) pairs; inside a tie group cut by the k-th position only the distances must agree."""
    fl, fd, fc = f
    bl, bd, bc = b
    assert np.array_equal(fc, bc)
    assert np.array_equal(fd.view(np.uint32), bd.view(np.uint32))
    for i in range(len(fc)):
        c = int(fc[i])
        if c == 0:
            continue
        cut = fd[i, c - 1]
        full = c < k or not np.isfinite(cut)
        keep = slice(0, c) if full else fd[i, :c] < cut
        pf = sorted(zip(fd[i, :c][keep].tolist(), fl[i, :c][keep].tolist()))
        pb = sorted(zip(bd[i, :c][keep].tolist(), bl[i, :c][keep].tolist()))
        assert pf == pb, (i, pf[:5], pb[:5])
        assert len(set(bl[i, :c].tolist())) == c
    assert np.all(bl[fc[:, None] <= np.arange(k)[None, :]] == NO_LABEL)


def both(ix, q, k, ef):
    """(fp32 result, its counters), (bf16 result, its counters) on one index."""
    BF16 = _bf16()
    f = ix.search(q, k, ef=ef)
    fs = walk_stats(ix)
    b = ix.search(q, k, ef=ef, precision=BF16)
    bs = walk_stats(ix)
    return f, fs, b, bs


_G = {}


def int_index(n, d, metric, seed=5):
    """A GPU-built graph over bf16-exact integer rows (cached), walked at width 1."""
    key = (n, d, metric, seed)
    if key not in _G:
        ehb = _ehb()
        x, q = intdata(n, d, 200, seed)
        ix = ehb.NativeIndex(d, metric=metric, capacity=n)
        ix.add(x)
        ix.build()
        _G[key] = (x, q, ix.export_graph())
    x, q, g = _G[key]
    ix = _ehb().NativeIndex(d, metric=metric, capacity=n)
    ix.import_graph(g)
    ix.set_search_width(1)
    return x, q, ix


# ---- 1. bf16 walk == fp32 walk on bf16-exact data ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("d", DIMS)
def test_bf16_walk_equals_fp32_walk_every_class(d, metric):
    x, q, ix = int_index(3000, d, metric)
    q = q[:100]
    for ef, k in [(40, 1), (40, 40), (65, 33), (129, 10), (129, 129), (257, 33), (512, 500)]:
        f, fs, b, bs = both(ix, q, k, ef)
        assert ix.last_kernel_name() == name_of(d, max(ef, k), True), ix.last_kernel_name()
        assert_same_walk(f, b, k)
        assert_same_counters(fs, bs)
        assert np.array_equal(b[1].view(np.uint32), exact_dist(x, q, b[0], metric).view(np.uint32))
    ix.set_tuning(hash_bits=12)                        # one table size for both walks: every counter equal
    f, fs, b, bs = both(ix, q, 50, 129)
    assert_same_walk(f, b, 50)
    assert fs == bs
    ix.search(q, 10, ef=64)
    assert ix.last_kernel_name() == name_of(d, 64, False)     # the fp32 entry point still runs fp32 rows


@pytest.mark.gpu
@pytest.mark.parametrize("d,ef,k", [(29, 64, 10), (64, 100, 10), (128, 128, 10), (128, 256, 100)])
def test_bf16_dense_form(d, ef, k):
    """nq = 20 x SMs: the dense form where bf16 has one (rows <= 256 B; at d = 128 only up to ef = 128)."""
    x, q, ix = int_index(3000, d, "l2")
    nq = 20 * sms()
    _, q = intdata(1, d, nq, seed=77)
    ix.set_search_width(0)
    f, fs, b, bs = both(ix, q, k, ef)
    dense_bf16 = d <= 64 or ef <= 128
    assert ix.last_kernel_name() == name_of(d, ef, True, kind="hnsw_search_dense_kernel" if dense_bf16
                                            else "hnsw_search_kernel")
    ix.search(q, k, ef=ef)
    assert ix.last_kernel_name() == name_of(d, ef, False, kind="hnsw_search_dense_kernel")
    assert_same_walk(f, b, k)
    assert_same_counters(fs, bs)


@pytest.mark.gpu
@pytest.mark.parametrize("d,ef", [(64, 256), (768, 256), (768, 512)])
def test_bf16_walk_visited_table_full(d, ef):
    x, q, ix = int_index(3000, d, "ip")
    ix.set_tuning(hash_bits=8)
    f, fs, b, bs = both(ix, q[:96], 50, ef)
    assert ix.stats()["visited_overflow"] > 0
    assert_same_walk(f, b, 50)
    assert fs == bs                                    # same table: the same re-evaluations


@pytest.mark.gpu
@pytest.mark.parametrize("frac", [0.1, 0.5])
@pytest.mark.parametrize("d", [64, 383, 768])
def test_bf16_walk_tombstones(d, frac):
    x, q, ix = int_index(3000, d, "l2")
    st = ix.stats()
    rng = np.random.default_rng(int(frac * 100) + d)
    dead = np.union1d(rng.choice(3000, int(frac * 3000), replace=False), [st["entry_point"]]).astype(np.uint64)
    ix.remove(dead)
    for ef, k in [(64, 10), (257, 100)]:
        f, fs, b, bs = both(ix, q[:100], k, ef)
        assert ix.last_kernel_name() == name_of(d, ef, True, deleted=True)
        assert_same_walk(f, b, k)
        assert_same_counters(fs, bs)
        assert not np.isin(b[0], dead).any()


# ---- 2. against the oracle, exactly -----------------------------------------------------------------------------
def split_tiefree(n, d, nq, seed=7):
    """x_i = (B u_i, 256 floor((i+1)/256), (i+1) mod 256), q = (v, 1, 1): q.x_i = B (u_i.v) + i + 1, all distinct,
    every coordinate exact in bf16 and every partial sum an integer below 2^24."""
    B = 1 << (n + 1).bit_length()
    assert B * (d + 1) <= 1 << 24
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.int64)
    x[:, :d - 2] = B * rng.integers(-1, 2, (n, d - 2))
    x[:, d - 2] = 256 * (np.arange(1, n + 1) // 256)
    x[:, d - 1] = np.arange(1, n + 1) % 256
    q = np.ones((nq, d), np.int64)
    q[:, :d - 2] = rng.integers(-1, 2, (nq, d - 2))
    return x, q


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 768])
def test_bf16_search_equals_oracle(d):
    ehb, BF16 = _ehb(), _bf16()
    n = 6000
    x, q = split_tiefree(n, d, 160)
    xf = x.astype(np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(xf)
    ix.build()
    g = ix.export_graph()
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    D = (1 - q @ x.T).astype(np.float32)
    for ef, k in [(64, 10), (128, 10), (257, 100)]:
        o.metrics(reset=True)
        ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
        om = o.metrics()
        l, dd, c = ix.search(q.astype(np.float32), k, ef=ef, precision=BF16)
        st = ix.stats()
        assert ix.last_kernel_name() == name_of(d, ef, True)
        assert np.array_equal(c, oc) and np.array_equal(l, ol)
        assert np.array_equal(dd.view(np.uint32), od.view(np.uint32))
        assert np.array_equal(dd.view(np.uint32), np.take_along_axis(D, l.astype(np.int64), 1).view(np.uint32))
        assert st["hops_upper"] == om["hops_upper"] and st["hops_base"] == om["hops0"]
        if st["visited_overflow"] == 0:
            assert st["dist_evals"] == om["evals"]
        # algorithmic bytes: every query retained ef keys (n >> ef, no tombstones)
        M, M0 = 16, 32
        want = (st["hops_upper"] * 4 * M + st["hops_base"] * 4 * M0 + st["dist_evals"] * 2 * d + len(q) * 4 * d
                + len(q) * max(ef, k) * 4 * d)
        assert st["algorithmic_bytes"] == want
        assert ix.last_kernel_ms() > 0


# ---- 3. Gaussian and clustered data -----------------------------------------------------------------------------
def gmm(n, d, seed):
    centres = np.random.default_rng(99).standard_normal((1024, d), dtype=np.float32)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d), dtype=np.float32) * np.float32(0.3)
    return x + centres[rng.integers(0, 1024, n)]


def recall(a, b, k):
    return float(np.mean([len(set(r[:k].tolist()) & set(s[:k].tolist())) / k for r, s in zip(a, b)]))


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["gaussian", "gmm"])
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("d", [128, 768])
def test_bf16_search_real_data(d, metric, dist):
    ehb, BF16 = _ehb(), _bf16()
    n, nq, k = 50_000, 1000, 10
    if dist == "gmm":
        x, q = gmm(n, d, 1234), gmm(nq, d, 4321)
    else:
        x = np.random.default_rng(1234).standard_normal((n, d), dtype=np.float32)
        q = np.random.default_rng(4321).standard_normal((nq, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(x)
    ix.build()
    dead = np.arange(0, n, 50, dtype=np.uint64)
    ex_l, _, _ = ix.search_bruteforce(q, k)
    base = orc.normalize(x) if metric == "cosine" else x
    qq = orc.normalize(q) if metric == "cosine" else q
    om = "l2" if metric == "l2" else "ip"
    for ef in (64, 128):
        fl, _, _ = ix.search(q, k, ef=ef)
        bl, bd, bc = ix.search(q, k, ef=ef, precision=BF16)
        assert np.all(bc == k)
        for i in range(nq):
            rows = bl[i].astype(np.int64)
            assert len(set(rows.tolist())) == k
            _, od = orc.bruteforce(base[rows], qq[i:i + 1], k, om)
            assert np.array_equal(bd[i].view(np.uint32), od[0].view(np.uint32)), i
        assert np.all(np.diff(bd, axis=1) >= 0)
        rf, rb = recall(fl, ex_l, k), recall(bl, ex_l, k)
        print(f"d={d} {metric} {dist} ef={ef}: recall@10 fp32 walk {rf:.4f}, bf16 walk {rb:.4f}, "
              f"id overlap {recall(bl, fl, k):.4f}")
        assert rb >= rf - 0.01, (rb, rf)
    ix.remove(dead)
    bl, bd, bc = ix.search(q, k, ef=64, precision=BF16)
    assert not np.isin(bl, dead).any() and np.all(np.diff(bd, axis=1) >= 0)


# ---- 4. shadow lifecycle ----------------------------------------------------------------------------------------
def check_equal_paths(ix, x, q, k=10, ef=64, metric="l2"):
    """case 1 on the current index, and bf16 brute force == the exact path (x: rows by label)."""
    BF16 = _bf16()
    f, fs, b, bs = both(ix, q, k, ef)
    assert_same_walk(f, b, k)
    assert_same_counters(fs, bs)
    assert np.array_equal(b[1].view(np.uint32), exact_dist(x, q, b[0], metric).view(np.uint32))
    el, ed, ec = ix.search_bruteforce(q, k)
    bl, bd, bc = ix.search_bruteforce(q, k, precision=BF16)
    assert np.array_equal(el, bl) and np.array_equal(ed.view(np.uint32), bd.view(np.uint32))
    assert np.array_equal(ec, bc)


@pytest.mark.gpu
def test_shadow_follows_every_mutation(tmp_path):
    ehb, BF16 = _ehb(), _bf16()
    d = 64
    xs, q = intdata(6000, d, 80, seed=21)
    rows = xs.copy()                                   # rows[label] = the label's current vector
    ix = ehb.NativeIndex(d, metric="l2", capacity=1000)
    ix.set_search_width(1)
    ix.add(xs[:1000])
    check_equal_paths(ix, rows, q)                     # the first bf16 search creates the shadow
    ix.add(xs[1000:4000])                              # capacity 1000 -> 4096: the shadow grows with the rows
    check_equal_paths(ix, rows, q)
    # in-place update: label 7 becomes the first query, which the bf16 search must see
    rows[7] = q[0]
    ix.add(q[:1], np.array([7], np.uint64))
    l, dd, _ = ix.search(q[:1], 1, ef=64, precision=BF16)
    assert l[0, 0] == 7 and dd[0, 0] == 0
    check_equal_paths(ix, rows, q)
    # remove, then re-add some of the removed labels with new vectors
    dead = np.arange(100, 700, 3, dtype=np.uint64)
    ix.remove(dead)
    l, _, _ = ix.search(q, 10, ef=64, precision=BF16)
    assert not np.isin(l, dead).any()
    back = dead[::2]
    rows[back.astype(np.int64)] = xs[4000:4000 + len(back)]
    ix.add(xs[4000:4000 + len(back)], back)
    still = np.setdiff1d(dead, back)
    l, _, _ = ix.search(q, 10, ef=64, precision=BF16)
    assert not np.isin(l, still).any()
    check_equal_paths(ix, rows, q)
    ix.compact()                                       # survivors move down: the shadow follows
    check_equal_paths(ix, rows, q)
    ix.add(xs[4500:5000], np.arange(4500, 5000, dtype=np.uint64))
    rows[4500:5000] = xs[4500:5000]
    check_equal_paths(ix, rows, q)
    path = str(tmp_path / "ix.ehb")
    ix.save(path)
    lx = ehb.NativeIndex.load(path)
    lx.set_search_width(1)
    check_equal_paths(lx, rows, q)
    g = lx.export_graph()
    ix.import_graph(g)                                 # replaces the content: the old shadow goes
    check_equal_paths(ix, rows, q)


@pytest.mark.gpu
def test_no_shadow_without_a_bf16_search():
    import torch

    ehb, BF16 = _ehb(), _bf16()
    n, d = 200_000, 768
    x = np.random.default_rng(3).standard_normal((n, d), dtype=np.float32)
    q = np.random.default_rng(4).standard_normal((16, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(x)
    ix.build()
    ix.search(q, 10, ef=64)                            # slot scratch of the graph search exists from here on
    ix.search_bruteforce(q, 10)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(3):
        ix.search(q, 10, ef=128)
        ix.search_bruteforce(q, 10)
    free1 = torch.cuda.mem_get_info(0)[0]
    shadow = n * dpad_of(d) * 2
    assert free0 - free1 < shadow // 8, (free0 - free1, shadow)
    ix.search(q, 10, ef=128, precision=BF16)           # now the shadow exists
    free2 = torch.cuda.mem_get_info(0)[0]
    assert free1 - free2 >= shadow, (free1 - free2, shadow)


# ---- 5. concurrency ---------------------------------------------------------------------------------------------
def _run_threads(fns):
    errs = []

    def wrap(fn):
        try:
            fn()
        except BaseException as e:  # noqa: BLE001 - reported below
            errs.append(e)

    ts = [threading.Thread(target=wrap, args=(fn,)) for fn in fns]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]


@pytest.mark.gpu
def test_concurrent_mixed_precision_through_the_combining_queue():
    BF16 = _bf16()
    x, q, ix = int_index(3000, 64, "l2")
    k, ef = 10, 64
    ref = {0: ix.search(q, k, ef=ef), BF16: ix.search(q, k, ef=ef, precision=BF16)}
    before = ix.stats()["combined_batches"]

    def worker(t):
        def run():
            rng = np.random.default_rng(t)
            for it in range(60):
                p = BF16 if (it + t) % 2 else 0
                i = int(rng.integers(0, len(q) - 4))
                m = int(rng.integers(1, 4))
                l, dd, c = ix.search(q[i:i + m], k, ef=ef, precision=p)
                rl, rd, rc = ref[p]
                assert np.array_equal(l, rl[i:i + m]) and np.array_equal(c, rc[i:i + m])
                assert np.array_equal(dd.view(np.uint32), rd[i:i + m].view(np.uint32))
        return run

    _run_threads([worker(t) for t in range(4)])
    assert ix.stats()["combined_batches"] > before


@pytest.mark.gpu
def test_first_bf16_searches_race_to_create_the_shadow():
    ehb, BF16 = _ehb(), _bf16()
    d = 128
    x, q = intdata(5000, d, 100, seed=9)
    for _ in range(3):
        ix = ehb.NativeIndex(d, metric="l2", capacity=5000)
        ix.add(x)
        ix.build()
        ix.set_search_width(1)
        out = {}
        bar = threading.Barrier(2)

        def graph():
            bar.wait()
            out["g"] = ix.search(q, 10, ef=64, precision=BF16)

        def brute():
            bar.wait()
            out["b"] = ix.search_bruteforce(q, 10, precision=BF16)

        _run_threads([graph, brute])
        g2 = ix.search(q, 10, ef=64, precision=BF16)
        b2 = ix.search_bruteforce(q, 10, precision=BF16)
        for a, b in ((out["g"], g2), (out["b"], b2)):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
            assert np.array_equal(a[2], b[2])


@pytest.mark.gpu
def test_searches_in_both_precisions_while_rows_are_added():
    ehb, BF16 = _ehb(), _bf16()
    d = 64
    xs, q = intdata(12000, d, 64, seed=13)
    ix = ehb.NativeIndex(d, metric="l2", capacity=2000)
    ix.set_search_width(1)
    ix.add(xs[:2000])
    ix.search(q, 10, ef=64, precision=BF16)
    stop = threading.Event()

    def adder():
        try:
            for lo in range(2000, 12000, 500):
                ix.add(xs[lo:lo + 500])
        finally:
            stop.set()

    def searcher(t):
        def run():
            it = 0
            while not stop.is_set() or it < 4:
                p = BF16 if (it + t) % 2 else 0
                l, dd, c = ix.search(q[t * 8:t * 8 + 8], 10, ef=64, precision=p)
                for r in range(len(c)):
                    got = l[r, :c[r]]
                    assert len(set(got.tolist())) == c[r] and np.all(np.diff(dd[r, :c[r]]) >= 0)
                if p == BF16:
                    ex = exact_dist(xs, q[t * 8:t * 8 + 8], l, "l2")
                    assert np.array_equal(dd.view(np.uint32), ex.view(np.uint32))
                it += 1
        return run

    _run_threads([adder] + [searcher(t) for t in range(4)])
    assert ix.size == 12000
    check_equal_paths(ix, xs, q)


# ---- 6. surfaces ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sharded_bf16_equals_merge_of_shard_searches():
    ehb, BF16 = _ehb(), _bf16()
    d, n, k, ef = 64, 6000, 10, 64
    x, q = split_tiefree(n, d, 100)
    sh = ehb.ShardedIndex(d, [0, 0], metric="ip", capacity=n)
    sh.add(x.astype(np.float32), np.arange(n, dtype=np.uint64))
    sh.build()
    l, dd, c = sh.search(q.astype(np.float32), k, ef=ef, precision=BF16)
    parts = [sh.shard(i).search(q.astype(np.float32), k, ef=ef, precision=BF16) for i in range(2)]
    assert "ROW=bf16" in sh.shard(0).last_kernel_name()
    ml = np.concatenate([p[0] for p in parts], 1)
    md = np.concatenate([p[1] for p in parts], 1)
    order = np.argsort(md, axis=1, kind="stable")[:, :k]
    assert np.array_equal(l, np.take_along_axis(ml, order, 1))
    assert np.array_equal(dd.view(np.uint32), np.take_along_axis(md, order, 1).view(np.uint32))
    assert np.all(c == k)
    with pytest.raises(ehb.EhbError) as e:
        sh.search(q.astype(np.float32), k, ef=ef, precision=5)
    assert e.value.code == 1


@pytest.mark.gpu
def test_ann_index_and_native_pass_precision():
    import torch

    ehb, BF16 = _ehb(), _bf16()
    d, n = 64, 3000
    x, q = split_tiefree(n, d, 50)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    a = ehb.ANNIndex(d, metric="ip", init_cap=n)
    a.multiset([(f"k{i}", xf[i]) for i in range(n)])
    nat = a._nn
    nat.set_search_width(1)
    l, _, c = nat.search(qf, 10, 64, BF16)
    assert "ROW=bf16" in nat.last_kernel_name()
    got = a.approx_nearest_batch(qf, 10, ef=64, precision=BF16)
    assert got == [[f"k{int(v)}" for v in row[:cc]] for row, cc in zip(l, c)]
    assert "ROW=bf16" in nat.last_kernel_name()
    # beyond ef 512: brute force at the same precision
    bl, _, bc = nat.search_bruteforce(qf, 600, BF16)
    got = a.approx_nearest_batch(qf, 600, precision=BF16)
    assert got == [[f"k{int(v)}" for v in row[:cc]] for row, cc in zip(bl, bc)]
    # the device entry point
    dq = torch.from_numpy(qf).cuda()
    dl = torch.empty((len(qf), 10), dtype=torch.int64, device="cuda")
    dd = torch.empty((len(qf), 10), dtype=torch.float32, device="cuda")
    dc = torch.empty(len(qf), dtype=torch.int32, device="cuda")
    nat.search_dev(dq.data_ptr(), len(qf), 10, 64, dl.data_ptr(), dd.data_ptr(), dc.data_ptr(), precision=BF16)
    torch.cuda.synchronize()
    l2, d2, c2 = nat.search(qf, 10, 64, BF16)
    assert np.array_equal(dl.cpu().numpy().view(np.uint64), l2)
    assert np.array_equal(dd.cpu().numpy().view(np.uint32), d2.view(np.uint32))
    assert np.array_equal(dc.cpu().numpy().astype(np.uint32), c2)
    # invalid precision: EHB_ERR_INVALID on every entry point, before anything runs
    for call in (lambda: nat.search(qf, 10, 64, 2),
                 lambda: nat.search(qf, 0, 64, -1),
                 lambda: nat.search_dev(dq.data_ptr(), len(qf), 10, 64, dl.data_ptr(), 0, 0, precision=9)):
        with pytest.raises(ehb.EhbError) as e:
            call()
        assert e.value.code == 1
    # the plain entry point is the fp32 search
    nat.search(qf, 10, 64)
    assert nat.last_kernel_name() == "hnsw_search_kernel<LPV=8,NQ=2,KPL=2>"


@pytest.mark.gpu
def test_cpp_ann_index_twin_bf16():
    exe = os.path.join(ROOT, "tests", "cpp", "ann_index_bf16")
    assert os.path.exists(exe), "tests/cpp/ann_index_bf16 not built (make)"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("ok  ") == 3, out.stdout
