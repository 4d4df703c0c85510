"""The HNSW walk kernels held exactly: every instantiation against hnswlib's order, on tie-free integer data.

Inner-product rows x_i = (B*u_i, i+1) and queries q = (v, 1), with u_i, v in {-1, 0, 1}^(d-1) and B a power of
two >= n+2, give q.x_i = B*(u_i.v) + i+1.  Every partial sum of that dot product is an integer below
B*(d+1) <= 2^24, so any summation order (the walk's lane / shuffle tree, the oracle's 16 accumulators, int64)
gives the same fp32 value, 1 - dot is exact, and the n distances of one query are all different.  Tie order
never matters, so the one-warp walk must return the oracle's ids, distance bits and hop / evaluation counters
exactly, and the team walk must match a small numpy model of its rounds exactly.

The walk's stats report, per query, whether the visited table ran out of probes (or the side queue of
tombstoned candidates overflowed).  Without tombstones that only adds re-evaluations: a re-evaluated node is
either still in the result set (filtered) or not closer than the current worst result (rejected), so ids, hops
and distances stay exact and only the evaluation count may grow.
"""
import bisect

import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure

INV = 0xFFFFFFFF
DIMS = [29, 64, 128, 250, 383, 512, 768, 1000, 1535, 2048]   # one per dpad class 32 ... 2048


# ---- data ------------------------------------------------------------------------------------------------
def tiefree(n, d, nq, seed=7):
    """Search-tie-free IP data: int64 rows / queries and their fp32 copies."""
    B = 1 << (n + 1).bit_length()                   # power of two >= n + 2
    assert B * (d + 1) <= 1 << 24
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.int64)
    x[:, :d - 1] = B * rng.integers(-1, 2, (n, d - 1))
    x[:, d - 1] = np.arange(1, n + 1)
    q = np.ones((nq, d), np.int64)
    q[:, :d - 1] = rng.integers(-1, 2, (nq, d - 1))
    return x, q


def build_tiefree(n, d, seed=11):
    """Tie-free per inserted point: x_a.x_b = B^2 (u_a.u_b) + (a+1)(b+1) is exact and distinct over b."""
    B = 1 << n.bit_length()                         # power of two > n + 1
    assert B * B * (d - 1) + (n + 1) ** 2 < 1 << 24
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.int64)
    x[:, :d - 1] = B * rng.integers(-1, 2, (n, d - 1))
    x[:, d - 1] = np.arange(1, n + 1)
    return x, B


def ip_dist(x, q):
    """int64 reference: 1 - q.x as float32 ([nq][n]); exact because |1 - q.x| < 2^24."""
    r = 1 - q @ x.T
    assert np.abs(r).max() < 1 << 24
    return r.astype(np.float32)


def l2_exact(x, q, ids):
    """Exact squared L2 of the returned ids (int64, then fp32: all values < 2^24)."""
    diff = x[ids.astype(np.int64)] - q[:, None, :]
    return (diff * diff).sum(-1).astype(np.float32)


# ---- numpy model of the walk -----------------------------------------------------------------------------
def adjacency(g):
    return [r[r != INV].tolist() for r in g["links0"]]


def walk_model(g, adj0, dist, ef, k, T):
    """T warps per query (T = 1: hnswlib's searchKnn).  dist: exact distances of one query to every row.
    Each round pops the T closest unexpanded entries, evaluates the union of their unvisited neighbours once,
    publishes those passing `cnt < ef or d < worst` (state from before the round) and applies them with the
    same test against the running state.  Returns (ids, dists, hops_upper, hops_base, evals)."""
    dl = dist.tolist()
    cur = int(g["entry"])
    cd, evals, hu = dl[cur], 1, 0
    for level in range(int(g["maxlevel"]), 0, -1):           # greedy descent (warp 0 of a team)
        changed = True
        while changed:
            changed = False
            row = g["links_up"][int(g["up_off"][cur]) + level - 1]
            row = row[row != INV].tolist()
            hu += 1
            evals += len(row)
            if row:
                j = min(row, key=dl.__getitem__)
                if dl[j] < cd:
                    cd, cur, changed = dl[j], j, True
    visited = {cur}
    res = [(cd, cur)]                                         # ascending (distance, id), <= ef entries
    expanded = set()
    hb = 0
    while True:
        pops = []
        for e in res:
            if e[1] not in expanded:
                pops.append(e[1])
                if len(pops) == T:
                    break
        if not pops:
            break
        full = len(res) >= ef
        worst = res[-1][0]
        pub = []
        for node in pops:
            expanded.add(node)
            hb += 1
            for nb in adj0[node]:
                if nb in visited:
                    continue
                visited.add(nb)
                evals += 1
                if not full or dl[nb] < worst:
                    pub.append((dl[nb], nb))
        for e in pub:
            if len(res) >= ef and e[0] >= res[-1][0]:
                continue
            bisect.insort(res, e)
            if len(res) > ef:
                res.pop()
    top = res[:k]
    return [i for _, i in top], [d for d, _ in top], hu, hb, evals


def model_batch(g, adj0, D, ef, k, T):
    ids = np.full((D.shape[0], k), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    dd = np.full((D.shape[0], k), np.inf, np.float32)
    cnt = np.zeros(D.shape[0], np.uint32)
    hu = hb = ev = 0
    for i in range(D.shape[0]):
        a, b, u, h, e = walk_model(g, adj0, D[i], ef, k, T)
        ids[i, :len(a)] = np.asarray(a, np.uint64)
        dd[i, :len(b)] = np.asarray(b, np.float32)
        cnt[i] = len(a)
        hu, hb, ev = hu + u, hb + h, ev + e
    return ids, dd, cnt, {"hops_upper": hu, "hops0": hb, "evals": ev}


def test_walk_model_t1_equals_oracle():
    """CPU only: the model with one warp is hnswlib's search (ids, distance bits, hops, evaluations)."""
    n, d, nq, ef, k = 3000, 32, 60, 48, 10
    x, q = tiefree(n, d, nq)
    o = orc.OracleHNSW(d, "ip", n, M=8)
    o.add(x.astype(np.float32), threads=1)
    g = o.export_graph()
    assert np.array_equal(g["vectors"], x.astype(np.float32))     # sequential inserts: row i is label i
    D = ip_dist(x, q)
    o.metrics(reset=True)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef)
    om = o.metrics()
    ml, md, mc, mm = model_batch(g, adjacency(g), D, ef, k, 1)
    assert np.array_equal(ml, ol) and np.array_equal(md.view(np.uint32), od.view(np.uint32))
    assert np.array_equal(mc, oc)
    assert mm == om, (mm, om)
    assert mm["hops0"] > 20 * nq                                # long enough walks: evictions happen
    # the model itself is checked against exact ground truth: every distance is the int64 one
    assert np.array_equal(md, np.take_along_axis(D, ml.astype(np.int64), 1))


# ---- GPU -------------------------------------------------------------------------------------------------
def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_CACHE = {}


def graph(n, d, nq):
    """A GPU-built graph over tie-free data (cached per shape), and the oracle walking the identical graph."""
    key = (n, d, nq)
    if key not in _CACHE:
        ehb = _ehb()
        x, q = tiefree(n, d, nq)
        ix = ehb.NativeIndex(d, metric="ip", capacity=n)
        ix.add(x.astype(np.float32))
        ix.build()
        g = ix.export_graph()
        assert np.array_equal(g["vectors"], x.astype(np.float32))
        o = orc.OracleHNSW(d, "ip", n)
        o.import_graph(g)
        _CACHE[key] = (x, q, g, o)
    return _CACHE[key]


def walker(g, d, width=1, **tuning):
    ehb = _ehb()
    ix = ehb.NativeIndex(d, metric="ip", capacity=g["vectors"].shape[0])
    ix.import_graph(g)
    ix.set_search_width(width)
    if tuning:
        ix.set_tuning(**tuning)
    return ix


def oracle_run(o, q, k, ef):
    o.metrics(reset=True)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    return ol, od, oc, o.metrics()


def assert_exact(res, st, ref, D, k):
    """GPU result == reference exactly; counters exact unless a visited-table overflow was reported."""
    l, dd, c = res
    rl, rd, rc, rm = ref
    assert np.array_equal(c, rc)
    assert np.array_equal(l, rl), np.argwhere(l != rl)[:5]
    assert np.array_equal(dd.view(np.uint32), rd.view(np.uint32))
    ok = l != np.uint64(0xFFFFFFFFFFFFFFFF)
    exact = np.take_along_axis(D, np.where(ok, l, 0).astype(np.int64), 1)
    assert np.array_equal(dd[ok].view(np.uint32), exact[ok].view(np.uint32))     # 1 - int64 dot, bit for bit
    assert np.all(np.diff(dd, axis=1) >= 0)
    assert st["hops_upper"] == rm["hops_upper"] and st["hops_base"] == rm["hops0"]
    assert st["dist_evals"] >= rm["evals"]
    if st["visited_overflow"] == 0:
        assert st["dist_evals"] == rm["evals"], (st["dist_evals"], rm["evals"])


def dpad_of(d):
    return next(s for s in (32, 64, 128, 256, 384, 512, 768, 1024, 1536, 2048) if d <= s)


def name_of(d, ef, lpv=None, kind="hnsw_search_kernel", deleted=False):
    dpad = dpad_of(d)
    lpv = lpv or (32 if dpad > 256 else 8)
    kpl = 2 if ef <= 64 else (4 if ef <= 128 else (8 if ef <= 256 else 16))
    return f"{kind}<LPV={lpv},NQ={dpad // (4 * lpv)},KPL={kpl}{',HASDEL=1' if deleted else ''}>"


def _n_for(d):
    return 6000 if d <= 1024 else 4000                     # B * (d + 1) <= 2^24


# ---- 2. every plain-walk instantiation --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d", DIMS)
def test_plain_walk_every_instantiation_exact(d):
    x, q, g, o = graph(_n_for(d), d, 160)
    D = ip_dist(x, q)
    ix = walker(g, d)
    # every KPL class, ef just above each boundary and not a multiple of 32, k in {1, 33, ef}, k = 500 at ef = 512
    for ef, k in [(40, 1), (40, 40), (65, 33), (129, 129), (257, 33), (257, 257), (512, 500)]:
        res = ix.search(q, k, ef=ef)
        assert ix.last_kernel_name() == name_of(d, max(ef, k)), ix.last_kernel_name()
        assert_exact(res, ix.stats(), oracle_run(o, q, k, ef), D, k)


@pytest.mark.gpu
def test_bench_instance_exact():
    """bench.py's walk: d = 768, ef = 128, k = 10 -> hnsw_search_kernel<LPV=32,NQ=6,KPL=4>."""
    x, q, g, o = graph(6000, 768, 160)
    ix = walker(g, 768)
    res = ix.search(q, 10, ef=128)
    assert ix.last_kernel_name() == "hnsw_search_kernel<LPV=32,NQ=6,KPL=4>"
    st = ix.stats()
    assert_exact(res, st, oracle_run(o, q, 10, 128), ip_dist(x, q), 10)
    assert st["hops_base"] > 100 * len(q)


# ---- 3. dense form ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d,ef,k", [(29, 64, 10), (64, 100, 10), (128, 256, 100)])
def test_dense_walk_exact(d, ef, k):
    """nq >= 20 SMs, rows <= 512 B, no tombstones: the automatic width picks the low-register dense walk
    (d = 128, ef = 256, k = 100 is the C5 shape)."""
    nq = 20 * sms()
    x, q, g, o = graph(6000, d, nq)
    ix = walker(g, d, width=0)
    res = ix.search(q, k, ef=ef)
    assert ix.last_kernel_name() == name_of(d, ef, kind="hnsw_search_dense_kernel")
    assert_exact(res, ix.stats(), oracle_run(o, q, k, ef), ip_dist(x, q), k)


# ---- 4. tuning knobs do not change results ----------------------------------------------------------------
def _same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    assert np.array_equal(a[2], b[2])


@pytest.mark.gpu
@pytest.mark.parametrize("d", [128, 768])
def test_prefetch_and_warps_per_block_invariant(d):
    x, q, g, o = graph(6000, d, 160)
    D = ip_dist(x, q)
    ef, k = 100, 20
    ref = oracle_run(o, q, k, ef)
    ix = walker(g, d)
    base = ix.search(q, k, ef=ef)
    assert_exact(base, ix.stats(), ref, D, k)
    for pf in (0, 1):
        ix.set_option("walk_prefetch", pf)
        r = ix.search(q, k, ef=ef)
        _same(r, base)
        assert_exact(r, ix.stats(), ref, D, k)
    ix.set_option("walk_prefetch", 1)
    for wpb in (1, 2, 4):
        ix.set_tuning(warps_per_block=wpb)
        r = ix.search(q, k, ef=ef)
        assert ix.last_kernel_name() == name_of(d, ef)
        _same(r, base)
        assert_exact(r, ix.stats(), ref, D, k)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [768, 2048])
def test_staging_ring_shapes_invariant(d):
    """(vectors per group G, groups NG) of the TMA ring, G not a multiple of the 4-vector math step included;
    only rings whose staging fits one warp's shared memory."""
    x, q, g, o = graph(_n_for(d), d, 160)
    D = ip_dist(x, q)
    ef, k = 129, 10
    ref = oracle_run(o, q, k, ef)
    ix = walker(g, d)
    base = ix.search(q, k, ef=ef)
    assert_exact(base, ix.stats(), ref, D, k)
    shapes = [(G, NG) for G, NG in [(1, 1), (3, 2), (7, 3), (4, 8), (2, 8), (32, 1)] if G * NG * d * 4 <= 180 * 1024]
    assert len(shapes) >= 4
    for G, NG in shapes:
        for wpb in (1, 2):
            ix.set_tuning(stage_slots=G, stage_groups=NG, warps_per_block=wpb)
            r = ix.search(q, k, ef=ef)
            assert ix.last_kernel_name() == name_of(d, ef, lpv=32)
            _same(r, base)
            assert_exact(r, ix.stats(), ref, D, k)


# ---- 5. forced visited-table overflow ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d,ef,width", [(64, 256, 1), (64, 512, 1), (768, 256, 1), (768, 512, 1),
                                        (64, 256, 2), (128, 200, 4)])
def test_visited_overflow_stays_exact(d, ef, width):
    """hash_bits = 8: a 256-entry table for walks that visit thousands of nodes."""
    nq, k = 96, 50
    x, q, g, o = graph(6000, d, 160)
    q = q[:nq]
    D = ip_dist(x, q)
    ix = walker(g, d, width=width, hash_bits=8)
    res = ix.search(q, k, ef=ef)
    st = ix.stats()
    if width == 1:
        assert ix.last_kernel_name() == name_of(d, ef)
        ref = oracle_run(o, q, k, ef)
    else:
        assert ix.last_kernel_name().startswith(f"hnsw_search_team_kernel<NQ={d // 32},")
        ref = model_batch(g, adjacency(g), D, ef, k, width)
    assert st["visited_overflow"] > 0
    assert_exact(res, st, ref, D, k)
    assert st["dist_evals"] > ref[3]["evals"]                   # the re-evaluations happened
    assert all(len(set(r.tolist())) == k for r in res[0])


# ---- 6. tombstones ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("frac", [0.1, 0.5, 0.9])
@pytest.mark.parametrize("d,ef", [(64, 64), (64, 256), (768, 64), (768, 256)])
def test_tombstones_exact(d, ef, frac):
    """Deleted points (and the entry point) are traversed, never returned.  One query per call, so the overflow
    flag belongs to that query: a query with a clear flag must equal the oracle exactly; every query returns
    sorted, unique, live ids with exact distances."""
    ehb = _ehb()
    n, nq, k = 6000, 64, 10
    x, q, g, _ = graph(n, d, 160)
    q = q[:nq]
    D = ip_dist(x, q)
    rng = np.random.default_rng(int(frac * 100) + d)
    dead = rng.choice(n, int(frac * n), replace=False)
    dead = np.union1d(dead, [int(g["entry"])]).astype(np.uint64)
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    for lab in dead:
        o.mark_delete(int(lab))
    ix = walker(g, d)
    ix.set_option("combine", 0)
    ix.remove(dead)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    live = np.ones(n, bool)
    live[dead.astype(np.int64)] = False
    flagged = 0
    for i in range(nq):
        l, dd, c = ix.search(q[i:i + 1], k, ef=ef)
        if i == 0:
            assert ix.last_kernel_name() == name_of(d, ef, deleted=True)
        flag = ix.stats()["visited_overflow"]
        got = l[0, :c[0]].astype(np.int64)
        assert np.all(live[got]) and len(set(got.tolist())) == c[0]
        assert np.all(l[0, c[0]:] == ehb.NO_LABEL)
        assert np.array_equal(dd[0, :c[0]].view(np.uint32), D[i, got].view(np.uint32))
        assert np.all(np.diff(dd[0, :c[0]]) > 0)
        if flag:
            flagged += 1
            continue
        assert c[0] == oc[i] and np.array_equal(l[0], ol[i]), (i, l[0], ol[i])
        assert np.array_equal(dd[0].view(np.uint32), od[i].view(np.uint32))
    print(f"tombstones d={d} ef={ef} deleted={frac:.0%}+entry: {flagged}/{nq} queries flagged")
    if frac <= 0.1:
        assert flagged < nq // 2                                # the exact comparison ran


@pytest.mark.gpu
def test_side_queue_overflow_in_last_hop_is_reported():
    """90 % deleted, ef = 64: the side queue of tombstoned candidates (64 entries) fills.  A query whose result
    differs from the oracle must carry the overflow flag, including when the queue overflowed while the last
    hop's candidates were admitted (that flag used to be dropped)."""
    d, n, nq, k, ef = 64, 6000, 160, 10, 64
    x, q, g, _ = graph(n, d, 160)
    dead = np.random.default_rng(5).choice(n, int(0.9 * n), replace=False)
    dead = np.union1d(dead, [int(g["entry"])]).astype(np.uint64)
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    for lab in dead:
        o.mark_delete(int(lab))
    ix = walker(g, d)
    ix.set_option("combine", 0)
    ix.remove(dead)
    ol, _, _ = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    flagged = differ = 0
    for i in range(nq):
        l, _, _ = ix.search(q[i:i + 1], k, ef=ef)
        f = ix.stats()["visited_overflow"]
        flagged += f
        if not np.array_equal(l[0], ol[i]):
            differ += 1
            assert f == 1, i
    print(f"side queue: {flagged}/{nq} flagged, {differ} differ from the oracle")
    assert flagged > 0


# ---- 7. team walk -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", [2, 3, 4])
@pytest.mark.parametrize("d", [30, 64, 128, 200])
def test_team_walk_matches_model(d, T):
    nq = 48
    x, q, g, _ = graph(6000, d, 160)
    q = q[:nq]
    D = ip_dist(x, q)
    adj0 = adjacency(g)
    ix = walker(g, d, width=T)
    roomy = walker(g, d, width=T, hash_bits=14)
    nqr = dpad_of(d) // 32
    wide, narrow = (8, 4) if nqr <= 2 else ((4, 2) if nqr <= 4 else (2, 1))    # U: 4-vector load steps in flight
    U = narrow if T == 3 else wide                                               # (T = 4 at <= 396 queries: wide)
    for ef, k in [(50, 10), (100, 33), (200, 200)]:
        res = ix.search(q, k, ef=ef)
        kpl = 2 if ef <= 64 else (4 if ef <= 128 else 8)
        assert ix.last_kernel_name() == f"hnsw_search_team_kernel<NQ={nqr},KPL={kpl},T={T},U={U}>"
        ref = model_batch(g, adj0, D, ef, k, T)
        assert_exact(res, ix.stats(), ref, D, k)
        again = ix.search(q, k, ef=ef)
        _same(again, res)
        r2 = roomy.search(q, k, ef=ef)
        st = roomy.stats()
        assert st["visited_overflow"] == 0 and st["dist_evals"] == ref[3]["evals"]
        _same(r2, res)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 128])
def test_team4_u2_and_u4_forms_agree(d):
    """T = 4 keeps 16-vector batches (U2) for batches of <= 396 queries and 8 (U4) above: the same queries give
    identical results and counters in both forms, and match the model."""
    x, q, g, _ = graph(6000, d, 400)
    D = ip_dist(x, q)
    ef, k = 120, 10
    ix = walker(g, d, width=4, hash_bits=14)
    wide = 8 if d == 64 else 4
    r4 = ix.search(q, k, ef=ef)
    assert ix.last_kernel_name().endswith(f",T=4,U={wide // 2}>")
    st4 = ix.stats()
    ra = ix.search(q[:396], k, ef=ef)
    assert ix.last_kernel_name().endswith(f",T=4,U={wide}>")
    sta = ix.stats()
    rb = ix.search(q[396:], k, ef=ef)
    stb = ix.stats()
    for i in range(3):
        assert np.array_equal(np.concatenate([ra[i], rb[i]]).view(np.uint32), r4[i].view(np.uint32))
    for f in ("hops_upper", "hops_base", "dist_evals"):
        assert st4[f] == sta[f] + stb[f]
    assert st4["visited_overflow"] == 0
    sub = slice(0, 40)
    ml, md, mc, _ = model_batch(g, adjacency(g), D[sub], ef, k, 4)
    assert np.array_equal(r4[0][sub], ml) and np.array_equal(r4[1][sub].view(np.uint32), md.view(np.uint32))


# ---- 8. build -------------------------------------------------------------------------------------------------------
def _rows(links):
    return [frozenset(int(v) for v in r if v != INV) for r in links]


def _assert_same_graph(g, og):
    assert np.array_equal(g["levels"], og["levels"])
    assert (int(g["entry"]), int(g["maxlevel"])) == (int(og["entry"]), int(og["maxlevel"]))
    assert np.array_equal(g["up_off"], og["up_off"])
    a0, b0 = _rows(g["links0"]), _rows(og["links0"])
    bad = [i for i in range(len(a0)) if a0[i] != b0[i]]
    assert not bad, (len(bad), bad[:5])
    au, bu = _rows(g["links_up"]), _rows(og["links_up"])
    assert au == bu


@pytest.mark.gpu
@pytest.mark.parametrize("d", [16, 32, 64])
@pytest.mark.parametrize("M", [4, 8, 16])
def test_wave_of_one_build_and_update_equal_oracle_graph(d, M):
    """One point per wave is sequential addPoint; on build-tie-free data the graph equals the oracle's row for
    row (100 %).  Then a sequence of updatePoint moves (the same tie-free form, new u) keeps it equal."""
    ehb = _ehb()
    n = 500
    x, B = build_tiefree(n, d)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n, M=M, build_batch=1)
    ix.add(x.astype(np.float32))
    o = orc.OracleHNSW(d, "ip", n, M=M)
    o.add(x.astype(np.float32), threads=1)
    _assert_same_graph(ix.export_graph(), o.export_graph())
    rng = np.random.default_rng(M * 100 + d)
    moved = rng.choice(n, 24, replace=False)
    newx = x[moved].copy()
    newx[:, :d - 1] = B * rng.integers(-1, 2, (len(moved), d - 1))
    for i, lab in enumerate(moved):     # one move at a time on both sides, as updatePoint runs
        ix.add(newx[i:i + 1].astype(np.float32), np.array([lab], np.uint64))
        ix.build()
        o.add(newx[i:i + 1].astype(np.float32), np.array([lab], np.uint64), threads=1)
    g = ix.export_graph()
    _assert_same_graph(g, o.export_graph())
    assert np.array_equal(g["vectors"][moved], newx.astype(np.float32))


# ---- 9. L2 on integer data ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d", DIMS)
def test_l2_integer_distances_exact(d):
    """L2 cannot be made tie-free in fp32 at useful n, so ids are held to the usual bound; every returned distance
    must still be the exact squared distance of its id, bit for bit.  Integers in [-r, r] with 4 r^2 d < 2^24 keep
    every partial sum exact; the widest such range keeps exact ties rare."""
    ehb = _ehb()
    n, nq, k, ef = 3000, 80, 10, 64
    r = min(200, int(2048 / np.sqrt(d)) - 1)
    assert 4 * r * r * d < 1 << 24
    rng = np.random.default_rng(d)
    x = rng.integers(-r, r + 1, (n, d)).astype(np.int64)
    q = rng.integers(-r, r + 1, (nq, d)).astype(np.int64)
    ix = ehb.NativeIndex(d, metric="l2", capacity=n)
    ix.add(x.astype(np.float32))
    ix.build()
    o = orc.OracleHNSW(d, "l2", n)
    o.import_graph(ix.export_graph())
    ix.set_search_width(1)
    l, dd, c = ix.search(q.astype(np.float32), k, ef=ef)
    assert ix.last_kernel_name() == name_of(d, ef)
    ol, od, oc = o.search(q.astype(np.float32), k, ef=ef, threads=8)
    assert np.all(c == k) and np.array_equal(c, oc)
    assert np.array_equal(dd.view(np.uint32), l2_exact(x, q, l).view(np.uint32))
    assert np.mean(l == ol) >= 0.995
    assert np.all(np.diff(dd, axis=1) >= 0)
