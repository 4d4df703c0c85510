"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle.

bit-exact for the exact path; for the graph walk: same ids as the oracle when it
walks the identical graph, recall >= the oracle's at matched ef on its own graph,
distances within 1e-4 relative (the tolerance BASELINE.json's north_star states).
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (test infrastructure)
import embeddinghub_b200 as ehb  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")
RTOL = 1e-4


def data(n, d, nq, seed=1234, qseed=4321):
    base = np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)
    q = np.random.default_rng(qseed).standard_normal((nq, d)).astype(np.float32)
    return base, q


def recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


# ---- exact path: bit-exact ids and distances -----------------------------------
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("n,d,nq,k", [(10000, 128, 100, 10), (777, 3, 9, 5), (3000, 50, 33, 100), (500, 130, 7, 1)])
def test_bruteforce_bit_exact(metric, n, d, nq, k):
    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    labels, dists, counts = ix.search_bruteforce(q, k)
    ex, exd = orc.bruteforce(base, q, k, metric)
    assert np.array_equal(labels, ex)
    assert np.array_equal(dists.view(np.uint32), exd.view(np.uint32))
    assert np.all(counts == min(k, n))


def test_bruteforce_k_larger_than_n_and_empty():
    base, q = data(5, 16, 3)
    ix = ehb.NativeIndex(16, capacity=8)
    labels, dists, counts = ix.search_bruteforce(q, 4)
    assert np.all(labels == ehb.NO_LABEL) and np.all(np.isinf(dists)) and np.all(counts == 0)
    ix.add(base)
    labels, dists, counts = ix.search_bruteforce(q, 8)
    ex, _ = orc.bruteforce(base, q, 8, "l2")
    assert np.array_equal(labels, ex) and np.all(counts == 5)
    assert np.all(labels[:, 5:] == ehb.NO_LABEL) and np.all(np.isinf(dists[:, 5:]))


def test_bruteforce_tie_order_is_insertion_index():
    base = np.ones((300, 8), np.float32)
    ix = ehb.NativeIndex(8, capacity=300)
    ix.add(base)
    labels, dists, _ = ix.search_bruteforce(base[:2], 20)
    assert np.array_equal(labels[0], np.arange(20, dtype=np.uint64)) and np.all(dists == 0)


# ---- graph walk on the identical graph -------------------------------------------
@pytest.mark.parametrize("metric,d", [("l2", 128), ("ip", 128), ("cosine", 64), ("l2", 768), ("l2", 20), ("ip", 300)])
def test_walk_matches_oracle_on_same_graph(metric, d):
    n, nq, k, ef = 6000, 200, 10, 64
    base, q = data(n, d, nq)
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=4)
    g = o.export_graph()
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.set_search_width(1)          # one warp per query = hnswlib's exact expansion order
    ix.import_graph(g)
    o.metrics(reset=True)
    ol, od, oc = o.search(q, k, ef=ef)
    om = o.metrics()
    labels, dists, counts = ix.search(q, k, ef=ef)
    st = ix.stats()
    assert np.all(counts == k)
    same = np.mean(labels == ol)
    assert same >= 0.995, same          # float summation order may flip rare near-ties
    m = labels == ol
    np.testing.assert_allclose(dists[m], od[m], rtol=RTOL, atol=1e-6)
    assert np.all(np.diff(dists, axis=1) >= 0)
    # hnswlib metric_hops / metric_distance_computations semantics
    assert abs(st["hops_base"] - om["hops0"]) <= 0.01 * om["hops0"]
    assert abs(st["dist_evals"] - om["evals"]) <= 0.01 * om["evals"]
    # (the visited table may run full — that only costs re-evaluations, bounded by the 1 % above)


def test_walk_reference_default_ef_and_k_gt_ef():
    n, d = 3000, 32
    base, q = data(n, d, 64)
    o = orc.OracleHNSW(d, "l2", n)
    o.add(base)
    ix = ehb.NativeIndex(d, capacity=n)
    ix.set_search_width(1)
    ix.import_graph(o.export_graph())
    for k in (1, 10, 25):                       # ef defaults to 10 -> walk uses max(10, k)
        ol, od, _ = o.search(q, k)
        labels, dists, _ = ix.search(q, k)
        assert np.mean(labels == ol) >= 0.99


@pytest.mark.parametrize("metric,d,width", [("l2", 128, 2), ("ip", 64, 4), ("cosine", 32, 3), ("l2", 256, 2)])
def test_team_walk_recall_not_below_sequential(metric, d, width):
    """T warps per query expand T candidates per round: a superset-style exploration.  Same graph,
    same ef: recall must not drop below the one-warp (hnswlib-order) walk, results stay sorted,
    unique, and distances stay exact."""
    n, nq, k = 20000, 500, 10
    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    ix.build()
    gt, gtd, _ = ix.search_bruteforce(q, k)
    for ef in (10, 64, 200):
        ix.set_search_width(1)
        l1, d1, _ = ix.search(q, k, ef=ef)
        ev1 = ix.stats()["dist_evals"]
        ix.set_search_width(width)
        lt, dt, ct = ix.search(q, k, ef=ef)
        evt = ix.stats()["dist_evals"]
        assert np.all(ct == k) and np.all(np.diff(dt, axis=1) >= 0)
        assert all(len(set(r.tolist())) == k for r in lt)
        assert recall(lt, gt) >= recall(l1, gt) - 0.003, (ef, recall(lt, gt), recall(l1, gt))
        assert evt <= 1.6 * ev1
        hit = lt == gt
        np.testing.assert_allclose(dt[hit], gtd[hit], rtol=RTOL, atol=1e-6)


# ---- GPU construction ----------------------------------------------------------------
@pytest.mark.parametrize("metric,d", [("l2", 16), ("ip", 24), ("cosine", 64)])
def test_gpu_build_wave_of_one_reproduces_sequential_hnswlib_graph(metric, d):
    """With one point per wave the GPU builder is sequential addPoint: same level
    generator, same searches, same heuristic -> the graph must equal the oracle's
    row for row (ids are sets: row order is not part of the contract)."""
    n = 1500
    base, _ = data(n, d, 1)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n, build_batch=1)
    ix.add(base)
    g = ix.export_graph()
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=1)
    og = o.export_graph()
    assert np.array_equal(g["levels"], og["levels"])
    assert (g["entry"], g["maxlevel"]) == (og["entry"], og["maxlevel"])
    assert np.array_equal(g["up_off"], og["up_off"])
    rows = lambda l: [frozenset(int(x) for x in r if x != 0xFFFFFFFF) for r in l]
    same0 = np.mean([a == b for a, b in zip(rows(g["links0"]), rows(og["links0"]))])
    sameu = np.mean([a == b for a, b in zip(rows(g["links_up"]), rows(og["links_up"]))]) if len(g["links_up"]) else 1.0
    assert same0 >= 0.99 and sameu >= 0.99, (same0, sameu)   # float summation order may flip rare ties


# ---- GPU-built graph (default waves): recall vs the oracle's at matched ef ----------------
# Waves of up to 1/64 of the graph cannot see their own members; the measured
# recall difference to the sequential build is within the seed-to-seed noise of
# the oracle itself (+-0.005 at these sizes), hence the 0.01 allowance.
@pytest.mark.parametrize("metric,d,n", [("l2", 128, 20000), ("ip", 96, 12000), ("cosine", 128, 12000)])
def test_gpu_build_recall_vs_oracle(metric, d, n):
    nq, k = 300, 10
    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    ix.build()
    gt, gtd, _ = ix.search_bruteforce(q, k)
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=8)
    for ef in (16, 64, 128):
        labels, dists, _ = ix.search(q, k, ef=ef)
        ol, _, _ = o.search(q, k, ef=ef)
        r_gpu, r_orc = recall(labels, gt), recall(ol, gt)
        assert r_gpu >= r_orc - 0.01, (ef, r_gpu, r_orc)
        # returned distances are the true distances of the returned ids
        ex = {}
        for row_l, row_d, gl, gd in zip(labels, dists, gt, gtd):
            for l, dd in zip(gl, gd):
                ex[int(l)] = dd
            for l, dd in zip(row_l, row_d):
                if int(l) in ex:
                    assert abs(dd - ex[int(l)]) <= RTOL * max(abs(ex[int(l)]), 1e-3)
            ex.clear()


def test_incremental_add_and_update_in_place():
    d = 24
    base, q = data(4000, d, 50)
    ix = ehb.NativeIndex(d, capacity=16)      # grows by doubling like index.cc:29-32
    for i in range(0, 4000, 500):
        ix.add(base[i:i + 500])
        ix.build()
    assert ix.size == 4000
    gt, _, _ = ix.search_bruteforce(q, 10)
    labels, _, _ = ix.search(q, 10, ef=100)
    assert recall(labels, gt) >= 0.9
    # move 200 points far away and onto the queries: they must be found / vanish
    moved = np.arange(0, 2000, 10, dtype=np.uint64)
    newv = (np.tile(q[:20], (10, 1)) + 0.05 * np.random.default_rng(7).standard_normal((200, d))).astype(np.float32)
    ix.add(newv, moved)
    assert ix.size == 4000
    np.testing.assert_array_equal(ix.get(int(moved[3])), newv[3])
    gt2, _, _ = ix.search_bruteforce(q[:20], 5)
    labels2, _, _ = ix.search(q[:20], 5, ef=100)
    assert recall(labels2, gt2) >= 0.9
    assert all(int(gt2[i, 0]) in set(moved.tolist()) for i in range(20))


def test_arbitrary_labels_and_get():
    d = 8
    base, q = data(100, d, 4)
    labels = (np.arange(100, dtype=np.uint64) * 7919 + 12345678901)
    ix = ehb.NativeIndex(d, capacity=128)
    ix.add(base, labels)
    l, dd, c = ix.search(q, 3, ef=50)
    ex, _ = orc.bruteforce(base, q, 3, "l2")
    assert np.array_equal(l, labels[ex.astype(np.int64)])
    np.testing.assert_array_equal(ix.get(int(labels[17])), base[17])
    with pytest.raises(KeyError):
        ix.get(5)


def test_save_load_roundtrip(tmp_path):
    base, q = data(3000, 40, 20)
    ix = ehb.NativeIndex(40, metric="ip", capacity=3000)
    ix.add(base)
    a = ix.search(q, 10, ef=64)
    path = str(tmp_path / "ix.ehb")
    ix.save(path)
    ix2 = ehb.NativeIndex.load(path)
    b = ix2.search(q, 10, ef=64)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---- the reference's own known-answer tests through the product path ----------------
def _abc():
    idx = ehb.ANNIndex(3)
    idx.set("a", [0, 1, 0])
    idx.set("b", [1, 1, 0])
    idx.set("c", [1, 0, 0])
    return idx


def test_index_test_cc_cases():
    # embeddinghub/embeddingstore/test/index_test.cc:17-60
    assert _abc().approx_nearest([0, 1, 0], 1) == ["a"]
    assert _abc().approx_nearest([0, 1, 0], 2) == ["a", "b"]
    idx = _abc()
    idx.set("a", [0, -1, 0])
    assert idx.approx_nearest([0, 1, 0], 1) == ["b"]
    assert _abc().approx_nearest([0, 1, 0], 0) == []


def test_vectorstore_fixture():
    # provider/vectorstore_test.go:121-166 (asserts len == 2) + exact ids from the oracle
    fx = np.load(os.path.join(GOLD, "vectorstore_fixture.npz"))
    for metric in ("l2", "ip", "cosine"):
        ix = ehb.NativeIndex(768, metric=metric, capacity=8)
        ix.add(fx["vectors"])
        l, d, c = ix.search(fx["query"][None, :], 2)
        ex, exd = orc.bruteforce(fx["vectors"], fx["query"][None, :], 2, metric)
        assert c[0] == 2 and l[0].tolist() == ex[0].tolist()
        np.testing.assert_allclose(d[0], exd[0], rtol=RTOL, atol=1e-6)


def test_merge_topk_dev():
    import torch

    G, nq, k = 4, 37, 10
    rng = np.random.default_rng(0)
    d = np.sort(rng.standard_normal((G, nq, k)).astype(np.float32), axis=2)
    lab = rng.permutation(G * nq * k).astype(np.uint64).reshape(G, nq, k)
    d[1, :, 7:] = np.inf
    lab[1, :, 7:] = ehb.NO_LABEL
    td = torch.from_numpy(d).cuda()
    tl = torch.from_numpy(lab.view(np.int64)).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    ol = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    oc = torch.empty(nq, dtype=torch.int32, device="cuda")
    from embeddinghub_b200._native import check, lib
    import ctypes as C
    check(lib().ehb_merge_topk_dev(G, nq, k, C.c_void_p(td.data_ptr()), C.c_void_p(tl.data_ptr()),
                                   C.c_void_p(od.data_ptr()), C.c_void_p(ol.data_ptr()), C.c_void_p(oc.data_ptr()),
                                   0, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    flat_d = np.transpose(d, (1, 0, 2)).reshape(nq, -1)
    flat_l = np.transpose(lab, (1, 0, 2)).reshape(nq, -1)
    order = np.argsort(flat_d, axis=1, kind="stable")[:, :k]
    assert np.array_equal(od.cpu().numpy(), np.take_along_axis(flat_d, order, 1))
    assert np.array_equal(ol.cpu().numpy().view(np.uint64), np.take_along_axis(flat_l, order, 1))
    assert np.all(oc.cpu().numpy() == k)


# ---- bf16 tensor-core brute force (wgmma GEMM + fp32 re-rank) -----------------------------------------
@pytest.mark.parametrize("metric,d,n,nq,k", [("ip", 128, 20000, 300, 10), ("l2", 64, 5000, 130, 20),
                                             ("cosine", 768, 3000, 70, 5), ("ip", 100, 777, 5, 100),
                                             ("l2", 256, 140000, 257, 10)])
def test_bf16_bruteforce_matches_exact(metric, d, n, nq, k):
    """The bf16 GEMM only nominates 4k (>= k+64) candidates; the fp32 re-rank uses the canonical arithmetic,
    so every returned distance is bit-identical to the exact path's and the ids agree except where bf16
    rounding pushed a true neighbour out of the candidate set (random Gaussian data: essentially never)."""
    from embeddinghub_b200._native import BF16

    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    el, ed, ec = ix.search_bruteforce(q, k)
    bl, bd, bc = ix.search_bruteforce(q, k, precision=BF16)
    assert np.array_equal(ec, bc)
    assert recall(bl, el) >= 0.995
    same = bl == el
    assert same.mean() >= 0.99
    assert np.array_equal(bd[same].view(np.uint32), ed[same].view(np.uint32))
    assert np.all(np.diff(bd, axis=1) >= 0)
    # mutation invalidates the bf16 shadow copy
    ix.add(q[:3] * 1.0, np.arange(3, dtype=np.uint64))
    el2, _, _ = ix.search_bruteforce(q[:3], 1)
    bl2, _, _ = ix.search_bruteforce(q[:3], 1, precision=BF16)
    assert np.array_equal(el2, bl2) and el2[:, 0].tolist() == [0, 1, 2]


def test_merge_topk_packed_dev():
    """One packed gather buffer [G][nq*k u64 labels | nq*k f32 dists] merged in place == separate-array merge."""
    import ctypes as C

    import torch

    from embeddinghub_b200._native import check, lib

    G, nq, k = 3, 50, 8
    rng = np.random.default_rng(1)
    d = np.sort(rng.standard_normal((G, nq, k)).astype(np.float32), axis=2)
    lab = rng.permutation(G * nq * k).astype(np.uint64).reshape(G, nq, k)
    nl, nd = nq * k * 8, nq * k * 4
    packed = np.zeros((G, nl + nd), np.uint8)
    for g in range(G):
        packed[g, :nl] = lab[g].reshape(-1).view(np.uint8)
        packed[g, nl:] = d[g].reshape(-1).view(np.uint8)
    tp = torch.from_numpy(packed).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    ol = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    oc = torch.empty(nq, dtype=torch.int32, device="cuda")
    check(lib().ehb_merge_topk_packed_dev(G, nq, k, C.c_void_p(tp.data_ptr()), nl + nd, C.c_void_p(od.data_ptr()),
                                          C.c_void_p(ol.data_ptr()), C.c_void_p(oc.data_ptr()), 0,
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    flat_d = np.transpose(d, (1, 0, 2)).reshape(nq, -1)
    flat_l = np.transpose(lab, (1, 0, 2)).reshape(nq, -1)
    order = np.argsort(flat_d, axis=1, kind="stable")[:, :k]
    assert np.array_equal(od.cpu().numpy(), np.take_along_axis(flat_d, order, 1))
    assert np.array_equal(ol.cpu().numpy().view(np.uint64), np.take_along_axis(flat_l, order, 1))


# ---- BASELINE.json configs[1] at full size: size-independent properties ---------------------------------
def test_c2_full_size_properties():
    """N=1M d=128 Q=1000 k=10 ef=64 L2 (the bench workload): the oracle cannot BUILD this in test time, so the
    walk is checked through properties — sortedness, uniqueness, full counts, idempotence, returned distances
    equal to the exact distances of the returned ids, recall against the exact kernel — and, for the
    hnswlib-order walk (one warp per query), id equality with the CPU oracle walking the SAME exported graph."""
    from bench import gen, BASE_SEED, QUERY_SEED

    n, d, nq, k, ef = 1_000_000, 128, 1000, 10, 64
    base, q = gen(n, d, BASE_SEED), gen(nq, d, QUERY_SEED)
    ix = ehb.NativeIndex(d, capacity=n)
    ix.add(base)
    ix.build()
    gt, gtd, _ = ix.search_bruteforce(q, k)
    for width in (1, 0):                                   # exact order, then the automatic (team) mode
        ix.set_search_width(width)
        l, dd, c = ix.search(q, k, ef=ef)
        l2, dd2, _ = ix.search(q, k, ef=ef)
        assert np.array_equal(l, l2) and np.array_equal(dd, dd2)          # idempotent / deterministic
        assert np.all(c == k) and np.all(np.diff(dd, axis=1) >= 0)
        assert all(len(set(r.tolist())) == k for r in l)
        ex = ((base[l.astype(np.int64)] - q[:, None, :]) ** 2).sum(-1)    # exact distances of the returned ids
        np.testing.assert_allclose(dd, ex, rtol=RTOL, atol=1e-5)
        rec = recall(l, gt)
        assert rec >= 0.20, rec                                           # iid Gaussian d=128: hard for any graph
        if width == 1:
            l_seq, rec_seq = l, rec
        else:
            assert rec >= rec_seq - 0.003
    o = orc.OracleHNSW(d, "l2", n)
    o.import_graph(ix.export_graph())
    ol, od, _ = o.search(q[:200], k, ef=ef, threads=8)
    assert np.mean(ol == l_seq[:200]) >= 0.995
    st = ix.stats()
    assert st["size"] == n and st["max_level"] >= 3


def test_walk_edge_cases_empty_tiny_and_ragged():
    """Empty index, fewer points than k, a single point, k == 1, and a batch whose size is not a multiple of
    anything — the shapes the reference's unit tests and its `num > count` bug (index.cc:42-50) touch."""
    d = 6
    ix = ehb.NativeIndex(d, capacity=4)
    q = np.random.default_rng(0).standard_normal((7, d), dtype=np.float32)
    for width in (1, 2, 4):
        ix.set_search_width(width)
        l, dd, c = ix.search(q, 5, ef=10)
        assert np.all(l == ehb.NO_LABEL) and np.all(np.isinf(dd)) and np.all(c == 0)
    base = np.random.default_rng(1).standard_normal((3, d), dtype=np.float32)
    ix.add(base[:1])
    for width in (1, 2, 4):
        ix.set_search_width(width)
        l, dd, c = ix.search(q, 5, ef=10)
        assert np.all(c == 1) and np.all(l[:, 0] == 0) and np.all(l[:, 1:] == ehb.NO_LABEL)
    ix.add(base[1:])
    ex, exd = orc.bruteforce(base, q, 3, "l2")
    for width in (1, 2, 4):
        ix.set_search_width(width)
        l, dd, c = ix.search(q, 5, ef=10)          # k > n: 3 results, then padding
        assert np.all(c == 3) and np.array_equal(l[:, :3], ex) and np.all(l[:, 3:] == ehb.NO_LABEL)
        np.testing.assert_allclose(dd[:, :3], exd, rtol=RTOL, atol=1e-6)
        assert np.all(np.isinf(dd[:, 3:]))
        l1, _, c1 = ix.search(q[:1], 1)            # ef defaults to 10 -> max(10, k)
        assert c1[0] == 1 and l1[0, 0] == ex[0, 0]


@pytest.mark.parametrize("M", [4, 8])
def test_smaller_M_graphs(M):
    """M below the reference default: level-0 rows are 2M wide; wave-of-one construction must still reproduce
    the sequential oracle graph and the walk must match the oracle on it."""
    n, d, nq = 1200, 24, 60
    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, capacity=n, M=M, build_batch=1)
    ix.add(base)
    g = ix.export_graph()
    o = orc.OracleHNSW(d, "l2", n, M=M)
    o.add(base, threads=1)
    og = o.export_graph()
    assert np.array_equal(g["levels"], og["levels"])
    rows = lambda l: [frozenset(int(x) for x in r if x != 0xFFFFFFFF) for r in l]
    assert np.mean([a == b for a, b in zip(rows(g["links0"]), rows(og["links0"]))]) >= 0.99
    ix.set_search_width(1)
    l, dd, _ = ix.search(q, 5, ef=40)
    ol, od, _ = o.search(q, 5, ef=40)
    assert np.mean(l == ol) >= 0.99


def test_large_ef_and_large_k():
    """ef = 400 (16 entries per lane, one warp per query) with k = 300, and exact brute force at k = 1000."""
    n, d, nq = 8000, 32, 40
    base, q = data(n, d, nq)
    ix = ehb.NativeIndex(d, capacity=n)
    ix.add(base)
    ix.build()
    gt, gtd, _ = ix.search_bruteforce(q, 300)
    l, dd, c = ix.search(q, 300, ef=400)
    assert np.all(c == 300) and np.all(np.diff(dd, axis=1) >= 0)
    assert all(len(set(r.tolist())) == 300 for r in l)
    assert recall(l, gt) >= 0.9
    ex, exd = orc.bruteforce(base, q[:8], 1000, "l2")
    bl, bd, _ = ix.search_bruteforce(q[:8], 1000)
    assert np.array_equal(bl, ex) and np.array_equal(bd.view(np.uint32), exd.view(np.uint32))
    with pytest.raises(ehb.EhbError):
        ix.search(q, 10, ef=513)                      # documented limit
