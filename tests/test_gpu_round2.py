"""GPU parity tests of the round-2 surface: north-star shapes at scale, tombstones, faithful
updatePoint, re-entrant / combined host searches, streaming persistence, the sharded index and the
peer-memory shard exchange.  Everything calls through the C ABI; the oracle is the checker."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

import embeddinghub_b200 as ehb
from embeddinghub_b200._native import check, lib
from oracle import oracle as orc  # test infrastructure

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-4


def gen(n, d, seed):
    """SURVEY.md §8d: PCG64 standard_normal in chunks of 1M rows."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, d), np.float32)
    for i in range(0, n, 1 << 20):
        m = min(1 << 20, n - i)
        out[i:i + m] = rng.standard_normal((m, d), dtype=np.float32)
    return out


def recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


# ---- north-star shapes at N >= 100k on the prescribed data (VERDICT r1 #1) -------------------------------
@pytest.mark.parametrize("name,d,k,ef,metric,n", [("c3", 768, 10, 128, "ip", 100_000),
                                                  ("c5", 128, 100, 256, "cosine", 200_000)])
def test_north_star_shapes_recall_and_distances_vs_oracle(name, d, k, ef, metric, n):
    """Parity gate of SURVEY.md §8d at scale: recall@k(GPU-built, GPU walk) >= recall@k(oracle-built, oracle
    walk) - 0.01 at the same ef on the prescribed iid-Gaussian data, the GPU walk reproduces the oracle's ids
    on the oracle's own graph, and every returned distance is the true fp32 distance within 1e-4."""
    nq = 2000       # enough queries that the recall gate is not decided by sampling noise
    base, q = gen(n, d, 1234), gen(nq, d, 4321)
    cores = len(os.sched_getaffinity(0))
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    ix.build()
    gt, gtd, _ = ix.search_bruteforce(q, k)
    labels, dists, counts = ix.search(q, k, ef=ef)
    assert np.all(counts == k)
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=cores)
    ol, od, _ = o.search(q, k, ef=ef, threads=cores)
    r_gpu, r_orc = recall(labels, gt), recall(ol, gt)
    # per-query paired difference: the gate allows 0.01 or three standard errors of the sample, whichever is larger
    # (the oracle's multi-threaded build is not deterministic: its own recall moves by a few 1e-3 between runs)
    per_q = np.array([(len(set(a.tolist()) & set(t.tolist())) - len(set(b.tolist()) & set(t.tolist()))) / k
                      for a, b, t in zip(labels, ol, gt)])
    assert per_q.mean() >= -max(0.01, 3.0 * per_q.std() / np.sqrt(nq)), (name, r_gpu, r_orc, per_q.std())
    # same graph -> same walk
    gi = ehb.NativeIndex(d, metric=metric, capacity=n)
    gi.import_graph(o.export_graph())
    gi.set_search_width(1)
    l1, d1, _ = gi.search(q, k, ef=ef)
    same = l1 == ol
    assert same.mean() >= 0.995, same.mean()
    assert np.max(np.abs(d1[same] - od[same]) / np.maximum(np.abs(od[same]), 1e-6)) <= RTOL
    # returned distances are true distances: recompute the returned ids exactly on the host (float64)
    xb = base.astype(np.float64)
    if metric == "cosine":
        xb /= np.linalg.norm(xb, axis=1, keepdims=True)
    for i in range(0, nq, 200):
        qq = q[i].astype(np.float64)
        if metric == "cosine":
            qq /= np.linalg.norm(qq)
        ref = 1.0 - xb[labels[i].astype(np.int64)] @ qq
        assert np.max(np.abs(ref - dists[i]) / np.maximum(np.abs(ref), 1e-3)) <= RTOL


# ---- tombstones (hnswlib markDelete) ------------------------------------------------------------------------
@pytest.mark.parametrize("metric,d", [("l2", 32), ("ip", 48), ("cosine", 128)])
def test_remove_matches_oracle_mark_delete(metric, d):
    n, nq, k, ef = 6000, 200, 10, 64
    base, q = gen(n, d, 11), gen(nq, d, 12)
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=1)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.import_graph(o.export_graph())
    ix.set_search_width(1)
    rng = np.random.default_rng(5)
    dead = rng.choice(n, n // 10, replace=False).astype(np.uint64)
    for l in dead:
        o.mark_delete(int(l))
    ix.remove(dead)
    assert ix.stats()["deleted"] == len(dead) and ix.size == n       # size counts tombstones, like hnswlib
    gl, gd, gc = ix.search(q, k, ef=ef)
    ol, od, _ = o.search(q, k, ef=ef)
    assert not np.isin(gl, dead).any()
    same = gl == ol
    assert same.mean() >= 0.995, same.mean()
    np.testing.assert_allclose(gd[same], od[same], rtol=RTOL, atol=1e-6)
    # exact path filters tombstones too
    ex, _, _ = ix.search_bruteforce(q, k)
    alive = np.setdiff1d(np.arange(n, dtype=np.uint64), dead)
    ref, _ = orc.bruteforce(base[alive.astype(np.int64)], q, k, metric)
    assert np.array_equal(ex, alive[ref.astype(np.int64)])
    # error behaviour: unknown -> KeyError (hnswlib "Label not found"), double delete -> state error, get -> KeyError
    with pytest.raises(KeyError):
        ix.remove([n + 5])
    with pytest.raises(ehb.EhbError) as e:
        ix.remove([int(dead[0])])
    assert e.value.code == 4
    with pytest.raises(KeyError):
        ix.get(int(dead[0]))
    # re-adding a deleted label un-deletes it and updates it in place (hnswlib addPoint)
    back = dead[:50]
    newv = gen(50, d, 13)
    ix.add(newv, back)
    o.add(newv, back, threads=1)
    assert ix.stats()["deleted"] == len(dead) - 50
    gl2, _, _ = ix.search(q, k, ef=ef)
    ol2, _, _ = o.search(q, k, ef=ef)
    assert not np.isin(gl2, dead[50:]).any()
    cur = base.copy()
    cur[back.astype(np.int64)] = newv
    alive2 = np.setdiff1d(np.arange(n, dtype=np.uint64), dead[50:])
    ref2, _ = orc.bruteforce(cur[alive2.astype(np.int64)], q, k, metric)
    ref2 = alive2[ref2.astype(np.int64)]
    assert recall(gl2, ref2) >= recall(ol2, ref2) - 0.02      # (the batch moved 50 points at once; hnswlib one by one)
    hit, _, _ = ix.search(newv[:10], 1, ef=ef)
    assert np.array_equal(hit[:, 0], back[:10])                # the resurrected points are found at their new place


def test_remove_entry_point_and_everything_but_one():
    d, n = 16, 300
    base, q = gen(n, d, 21), gen(5, d, 22)
    ix = ehb.NativeIndex(d, capacity=n)
    ix.add(base)
    ix.build()
    ep = ix.stats()["entry_point"]
    ix.remove([ep])
    l, _, c = ix.search(q, 5, ef=50)
    assert np.all(c == 5) and not (l == ep).any()
    rest = np.setdiff1d(np.arange(n, dtype=np.uint64), [ep, 7])
    ix.remove(rest)
    l, dd, c = ix.search(q, 5, ef=50)
    assert np.all(c == 1) and np.all(l[:, 0] == 7) and np.all(l[:, 1:] == ehb.NO_LABEL) and np.all(np.isinf(dd[:, 1:]))


# ---- updatePoint: neighbour re-selection + repair, row for row -------------------------------------------------
@pytest.mark.parametrize("metric,d", [("l2", 16), ("ip", 24)])
def test_update_point_reproduces_oracle_graph(metric, d):
    """index_test.cc:39-49 (TestUpdateANN) at scale: after in-place updates the GPU graph must equal the graph
    hnswlib's updatePoint produces — the moved points' one-hop neighbours re-selected from the two-hop set, then
    repairConnectionsForUpdate — row for row (a wave of one = sequential semantics)."""
    n = 1200
    base = gen(n, d, 31)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n, build_batch=1)
    ix.add(base)
    ix.build()
    o = orc.OracleHNSW(d, metric, n)
    o.add(base, threads=1)
    moved = np.array([3, 500, 77, 1100, 640, 9], dtype=np.uint64)
    newv = gen(len(moved), d, 32)
    for i, l in enumerate(moved):      # one at a time on both sides
        ix.add(newv[i:i + 1], moved[i:i + 1])
        ix.build()
        o.add(newv[i:i + 1], moved[i:i + 1], threads=1)
    g, og = ix.export_graph(), o.export_graph()
    assert np.array_equal(g["levels"], og["levels"]) and (g["entry"], g["maxlevel"]) == (og["entry"], og["maxlevel"])
    rows = lambda l: [frozenset(int(x) for x in r if x != 0xFFFFFFFF) for r in l]
    same0 = np.mean([a == b for a, b in zip(rows(g["links0"]), rows(og["links0"]))])
    sameu = np.mean([a == b for a, b in zip(rows(g["links_up"]), rows(og["links_up"]))]) if len(g["links_up"]) else 1.0
    assert same0 >= 0.99 and sameu >= 0.99, (same0, sameu)
    np.testing.assert_array_equal(g["vectors"][moved.astype(np.int64)], og["vectors"][moved.astype(np.int64)])


def test_index_test_cc_update_case_with_neighbour_repair():
    """index_test.cc:39-49 verbatim: a={0,1,0} b={1,1,0} c={1,0,0}; set(a,{0,-1,0}); NN({0,1,0},1) == [b]."""
    ix = ehb.ANNIndex(3)
    ix.set("a", [0, 1, 0])
    ix.set("b", [1, 1, 0])
    ix.set("c", [1, 0, 0])
    ix.set("a", [0, -1, 0])
    assert ix.approx_nearest([0, 1, 0], 1) == ["b"]


# ---- re-entrancy and the combining queue ----------------------------------------------------------------------
def test_concurrent_single_query_callers_are_combined_and_correct():
    d, n, k, ef = 64, 20000, 10, 64
    base = gen(n, d, 41)
    ix = ehb.NativeIndex(d, capacity=n)
    ix.add(base)
    ix.build()
    ix.set_search_width(1)           # identical kernel shape for every batch size -> identical results
    T, per = 32, 40
    qs = gen(T * per, d, 42)
    want = ix.search(qs, k, ef=ef)
    before = ix.stats()
    got_l = np.empty((T * per, k), np.uint64)
    got_d = np.empty((T * per, k), np.float32)
    errs = []

    def worker(t):
        try:
            for j in range(per):
                i = t * per + j
                l, dd, c = ix.search(qs[i:i + 1], k, ef=ef)    # ctypes releases the GIL: truly concurrent calls
                got_l[i], got_d[i] = l[0], dd[0]
        except Exception as e:  # pragma: no cover
            errs.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    assert np.array_equal(got_l, want[0]) and np.array_equal(got_d, want[1])
    st = ix.stats()
    batches = st["combined_batches"] - before["combined_batches"]
    queries = st["combined_queries"] - before["combined_queries"]
    assert queries == T * per and batches < queries, (batches, queries)


def test_concurrent_search_and_add_do_not_interfere():
    d, n, k = 32, 8000, 5
    base = gen(n + 2000, d, 43)
    ix = ehb.NativeIndex(d, capacity=16)
    ix.add(base[:n])
    ix.build()
    q = gen(64, d, 44)
    stop, errs = threading.Event(), []

    def searcher():
        try:
            while not stop.is_set():
                l, dd, c = ix.search(q, k, ef=40)
                assert np.all(c == k) and np.all(np.diff(dd, axis=1) >= 0)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    th = [threading.Thread(target=searcher) for _ in range(4)]
    [t.start() for t in th]
    for i in range(n, n + 2000, 250):
        ix.add(base[i:i + 250])       # capacity doubling + lazy linking while searches are in flight
    stop.set()
    [t.join() for t in th]
    assert not errs, errs
    assert ix.size == n + 2000
    gt, _, _ = ix.search_bruteforce(q, k)
    l, _, _ = ix.search(q, k, ef=100)
    assert recall(l, gt) >= 0.9


def test_pthread_callers_c_program():
    """tests/cpp/concurrent_search.c: 64 pthreads issuing Q=1 ehb_index_search calls — the stand-in for the cgo
    provider's goroutine-per-request pattern (serving/serving.go:744-771).  It checks every answer against a
    batched search and prints the throughput with and without the combining queue."""
    exe = os.path.join(ROOT, "tests", "cpp", "concurrent_search")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/concurrent_search not built (make)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "OK" in out.stdout, out.stdout
    line = [l for l in out.stdout.splitlines() if l.startswith("speedup")][0]
    assert float(line.split()[1]) >= 4.0, out.stdout


# ---- persistence ------------------------------------------------------------------------------------------------
def test_save_load_streams_tombstones_and_rejects_corrupt_files(tmp_path):
    d, n = 100, 30000        # dim != padded dim: the 2D copies pad / unpad
    base, q = gen(n, d, 51), gen(50, d, 52)
    ix = ehb.NativeIndex(d, metric="cosine", capacity=n)
    ix.add(base, np.arange(n, dtype=np.uint64) * 3 + 1)
    ix.build()
    ix.remove([1, 4, 31])
    a = ix.search(q, 10, ef=64)
    path = str(tmp_path / "ix.ehb")
    ix.save(path)
    ix2 = ehb.NativeIndex.load(path)
    assert ix2.metric == "cosine" and ix2.size == n and ix2.stats()["deleted"] == 3
    b = ix2.search(q, 10, ef=64)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    np.testing.assert_array_equal(ix.get(7), ix2.get(7))
    with pytest.raises(KeyError):
        ix2.get(4)
    # inserts continue identically after a load (same level sequence)
    extra = gen(500, d, 53)
    lab = np.arange(n, n + 500, dtype=np.uint64) * 3 + 1
    ix.add(extra, lab)
    ix2.add(extra, lab)
    ga, gb = ix.export_graph(), ix2.export_graph()
    assert np.array_equal(ga["levels"], gb["levels"]) and np.array_equal(ga["links0"], gb["links0"])
    # corrupt files are refused, not trusted
    raw = open(path, "rb").read()
    bad = str(tmp_path / "bad.ehb")
    open(bad, "wb").write(raw[:-8])
    with pytest.raises(ehb.EhbError):
        ehb.NativeIndex.load(bad)
    broken = bytearray(raw)
    broken[7] = 9
    open(bad, "wb").write(bytes(broken))
    with pytest.raises(ehb.EhbError):
        ehb.NativeIndex.load(bad)
    off = len(raw) - 64      # inside links_up or up_off: an out-of-range adjacency id / offset
    broken = bytearray(raw)
    broken[off:off + 4] = (0x7FFFFFF0).to_bytes(4, "little")
    open(bad, "wb").write(bytes(broken))
    with pytest.raises(ehb.EhbError):
        ehb.NativeIndex.load(bad)


# ---- sharded index behind the C ABI -------------------------------------------------------------------------------
def _devices(n):
    import torch

    have = torch.cuda.device_count()
    return [i % have for i in range(n)]


@pytest.mark.parametrize("shards", [2, 3])
def test_sharded_index_matches_single_index(shards):
    d, n, nq, k = 48, 30000, 200, 10
    base, q = gen(n, d, 61), gen(nq, d, 62)
    sh = ehb.ShardedIndex(d, _devices(shards), metric="ip", capacity=1024, shard_span=n // shards + 1)
    sh.add(base)                       # labels = insertion order, routed by range
    sh.build()
    assert sh.size == n
    one = ehb.NativeIndex(d, metric="ip", capacity=n)
    one.add(base)
    ex1 = one.search_bruteforce(q, k)
    exs = sh.search_bruteforce(q, k)
    assert np.array_equal(ex1[0], exs[0]) and np.array_equal(ex1[1].view(np.uint32), exs[1].view(np.uint32))
    l1, _, _ = one.search(q, k, ef=64)
    ls, ds, cs = sh.search(q, k, ef=64)
    assert np.all(cs == k) and np.all(np.diff(ds, axis=1) >= 0)
    assert recall(ls, ex1[0]) >= recall(l1, ex1[0]) - 0.01    # G graphs at the same ef do at least the work of one
    np.testing.assert_array_equal(sh.get(12345), base[12345])
    sh.remove([int(ex1[0][0, 0])])
    ls2, _, _ = sh.search(q[:1], k, ef=64)
    assert int(ex1[0][0, 0]) not in ls2[0].tolist()


def test_sharded_two_devices_c_program():
    """tests/cpp/sharded_two_dev.c: n_dev = 2 through include/ehb200.h from plain C (both shards on GPU 0 when the
    box has one GPU; two GPUs exercise the peer stores into device 0's gather buffer)."""
    exe = os.path.join(ROOT, "tests", "cpp", "sharded_two_dev")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/sharded_two_dev not built (make)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "OK" in out.stdout, out.stdout + out.stderr


def test_exchange_two_ranks_in_one_process():
    """ehb_exchange with both 'ranks' in this process (attach_local instead of CUDA IPC): each rank's search
    writes into its block, one exchange_merge_kernel per rank pushes / flags / waits / merges; both ranks must
    end up with the exact global top-k."""
    import torch

    d, n, nq, k = 32, 20000, 333, 12
    base, q = gen(n, d, 71), gen(nq, d, 72)
    devs = _devices(2)
    half = n // 2
    L = lib()
    ixs, exs = [], []
    for r in range(2):
        ix = ehb.NativeIndex(d, capacity=half, device=devs[r])
        ix.add(base[r * half:(r + 1) * half], np.arange(r * half, (r + 1) * half, dtype=np.uint64))
        ixs.append(ix)
        h = C.c_void_p()
        check(L.ehb_exchange_create(devs[r], 2, r, nq, k, C.byref(h)))
        exs.append(h)
    check(L.ehb_exchange_attach_local(exs[0], 1, exs[1]))
    check(L.ehb_exchange_attach_local(exs[1], 0, exs[0]))
    ref, refd = orc.bruteforce(base, q, k, "l2")
    for step in range(3):              # parity double buffering + epochs across steps
        outs = []
        streams = []
        for r in range(2):
            torch.cuda.set_device(devs[r])
            s = torch.cuda.Stream(device=devs[r])
            streams.append(s)
            dq = torch.from_numpy(q).to(f"cuda:{devs[r]}")
            lp, dp = C.c_void_p(), C.c_void_p()
            check(L.ehb_exchange_begin(exs[r], nq, k, C.byref(lp), C.byref(dp)))
            cnt = torch.empty(nq, dtype=torch.int32, device=f"cuda:{devs[r]}")
            ixs[r].search_bruteforce_dev(dq.data_ptr(), nq, k, 0, lp.value, dp.value, cnt.data_ptr(), s.cuda_stream)
            ml = torch.empty((nq, k), dtype=torch.int64, device=f"cuda:{devs[r]}")
            md = torch.empty((nq, k), dtype=torch.float32, device=f"cuda:{devs[r]}")
            mc = torch.empty(nq, dtype=torch.int32, device=f"cuda:{devs[r]}")
            outs.append((ml, md, mc, dq, cnt))
        for r in range(2):             # both merges are queued before anyone synchronises
            torch.cuda.set_device(devs[r])
            ml, md, mc, _, _ = outs[r]
            check(L.ehb_exchange_merge_dev(exs[r], C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                           C.c_void_p(mc.data_ptr()), C.c_void_p(streams[r].cuda_stream)))
        for r in range(2):
            streams[r].synchronize()
            ml, md, mc, _, _ = outs[r]
            assert np.array_equal(ml.cpu().numpy().view(np.uint64), ref), (step, r)
            assert np.array_equal(md.cpu().numpy().view(np.uint32), refd.view(np.uint32))
            assert np.all(mc.cpu().numpy() == k)
            t = C.c_uint32()
            check(L.ehb_exchange_timed_out(exs[r], C.byref(t)))
            assert t.value == 0
    # graph search: the fused step (walk epilogue stores into the peers' buffers + slice flags, merge waits) must
    # give exactly what push-after-walk gives
    def run(fused):
        res, streams = [], []
        for r in range(2):
            torch.cuda.set_device(devs[r])
            s = torch.cuda.Stream(device=devs[r])
            streams.append(s)
            dev = f"cuda:{devs[r]}"
            dq = torch.from_numpy(q).to(dev)
            ml = torch.empty((nq, k), dtype=torch.int64, device=dev)
            md = torch.empty((nq, k), dtype=torch.float32, device=dev)
            mc = torch.empty(nq, dtype=torch.int32, device=dev)
            cnt = torch.empty(nq, dtype=torch.int32, device=dev)
            res.append((ml, md, mc, dq, cnt))
            if not fused:
                lp, dp = C.c_void_p(), C.c_void_p()
                check(L.ehb_exchange_begin(exs[r], nq, k, C.byref(lp), C.byref(dp)))
                ixs[r].search_dev(dq.data_ptr(), nq, k, 64, lp.value, dp.value, cnt.data_ptr(), s.cuda_stream)
        for r in range(2):
            torch.cuda.set_device(devs[r])
            ml, md, mc, dq, cnt = res[r]
            if fused:
                check(L.ehb_exchange_search_dev(exs[r], ixs[r]._h, nq, C.c_void_p(dq.data_ptr()), k, 64,
                                                C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                                C.c_void_p(mc.data_ptr()), C.c_void_p(cnt.data_ptr()),
                                                C.c_void_p(streams[r].cuda_stream)))
            else:
                check(L.ehb_exchange_merge_dev(exs[r], C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                               C.c_void_p(mc.data_ptr()), C.c_void_p(streams[r].cuda_stream)))
        out = []
        for r in range(2):
            streams[r].synchronize()
            out.append((res[r][0].cpu().numpy().copy(), res[r][1].cpu().numpy().copy(), res[r][2].cpu().numpy().copy()))
        return out

    for ix in ixs:
        ix.build()
        ix.set_search_width(1)      # the one-warp walk is the kernel that pushes from its epilogue
    plain = run(False)
    for step in range(3):
        fused = run(True)
        for r in range(2):
            for a, b in zip(plain[r], fused[r]):
                assert np.array_equal(a, b), (step, r)
    assert np.array_equal(plain[0][0], plain[1][0])             # both ranks hold the same global top-k
    assert recall(plain[0][0].view(np.uint64), ref) >= 0.9
    for r in range(2):
        t = C.c_uint32()
        check(L.ehb_exchange_timed_out(exs[r], C.byref(t)))
        assert t.value == 0
    for h in exs:
        L.ehb_exchange_destroy(h)
