"""Key-mode searches on the GPU (ehb_index_search_by_label_ex and friends): stored points as queries, named by
label, with the reference's self-removal (server.cc:190-207).  Every result is compared with the host composition
the contract names -- get each label -> search_ex(rows, k + 1) -> the rule (tests/label_rule_model.py) -- bit for bit,
and on tie-free data with the CPU reference walk."""
import ctypes as C
import os
import subprocess
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import embeddinghub_b200 as ehb  # noqa: E402
from embeddinghub_b200._native import BF16, FP32, _p, lib  # noqa: E402
from label_rule_model import drop_self  # noqa: E402
from oracle import oracle as orc  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def host_composition(ix, labels, k, ef=0, precision=FP32):
    rows = np.stack([ix.get(int(l)) for l in labels])
    L, D, Cn = ix.search(rows, k + 1, ef, precision)
    return drop_self(np.asarray(labels, np.uint64), L, D, Cn, k), ix.last_kernel_name()


def assert_same(a, b):
    (al, ad, ac), (bl, bd, bc) = a, b
    assert np.array_equal(ac, bc)
    assert np.array_equal(al, bl)
    assert np.array_equal(ad.view(np.uint32), bd.view(np.uint32))


def check_identity(ix, labels, k, ef=0, precision=FP32):
    ref, ref_kernel = host_composition(ix, labels, k, ef, precision)
    got = ix.search_by_label(labels, k, ef, precision)
    assert ix.last_kernel_name() == ref_kernel
    assert_same(got, ref)
    return ref_kernel


_CACHE = {}


def index(metric, d, n=4000):
    key = (metric, d, n)
    if key not in _CACHE:
        x = np.random.default_rng(d + n).standard_normal((n, d), dtype=np.float32)
        ix = ehb.NativeIndex(d, metric=metric, capacity=n)
        ix.add(x)
        ix.build()
        _CACHE[key] = ix
    return _CACHE[key]


# ---- 1. bit-identity with the host composition, every walk form ---------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("d", [29, 128, 768])
def test_identity_with_host_composition(metric, d):
    ix = index(metric, d)
    rng = np.random.default_rng(5)
    small = rng.choice(4000, 64, replace=False).astype(np.uint64)
    for precision in (FP32, BF16):
        for k in (1, 10, 100):
            name = check_identity(ix, small, k, 0, precision)
            if precision == FP32 and d <= 128:
                assert "team" in name, name
            if precision == BF16:
                assert "ROW=bf16" in name, name
    if d == 128:   # the dense one-warp form needs 20 queries per SM
        big = rng.choice(4000, 20 * sms(), replace=False).astype(np.uint64)
        assert "dense" in check_identity(ix, big, 10), "dense form not exercised"
    if d == 768 and metric == "ip":  # the int8-screened fp32 walk: 4 queries per SM and up
        big = rng.choice(4000, 4 * sms(), replace=False).astype(np.uint64)
        check_identity(ix, big, 10)
        assert ix.stats()["screened_evals"] > 0, "screened walk not exercised"


@pytest.mark.parametrize("case", ["tomb10", "tomb50", "compact", "update", "saveload"])
def test_identity_after_mutations(case, tmp_path):
    n, d = 3000, 64
    rng = np.random.default_rng(17)
    x = rng.standard_normal((n, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(x)
    ix.build()
    live = np.arange(n, dtype=np.uint64)
    if case in ("tomb10", "tomb50", "compact"):
        frac = {"tomb10": 0.1, "tomb50": 0.5, "compact": 0.3}[case]
        entry = np.uint64(ix.stats()["entry_point"])
        dead = np.union1d(rng.choice(n, int(frac * n), replace=False).astype(np.uint64), [entry])
        ix.remove(dead)
        live = np.setdiff1d(live, dead)
        if case == "compact":
            ix.compact()
        with pytest.raises(KeyError):
            ix.search_by_label(dead[:3], 5)
    elif case == "update":
        upd = rng.choice(n, 100, replace=False).astype(np.uint64)
        ix.add(rng.standard_normal((100, d), dtype=np.float32), upd)
    else:
        ix.save(str(tmp_path / "ix.ehb"))
        ix = ehb.NativeIndex.load(str(tmp_path / "ix.ehb"))
    q = rng.choice(live, 200, replace=False).astype(np.uint64)
    for precision in (FP32, BF16):
        for k in (1, 10):
            name = check_identity(ix, q, k, 32, precision)
            if case.startswith("tomb"):
                assert "HASDEL=1" in name


# ---- 2. exact against the CPU reference walk on tie-free data ------------------------------------------------------
@pytest.mark.parametrize("d", [8, 16, 64])
def test_exact_against_reference_walk(d):
    n, B = 400, 512
    assert B * B * (d - 1) + (n + 1) ** 2 < 1 << 24
    rng = np.random.default_rng(11)
    x = np.empty((n, d), np.int64)
    x[:, :d - 1] = B * rng.integers(-1, 2, (n, d - 1))
    x[:, d - 1] = np.arange(1, n + 1)
    xf = x.astype(np.float32)
    ix = ehb.NativeIndex(d, metric="ip", capacity=n)
    ix.add(xf)
    ix.build()
    g = ix.export_graph()
    o = orc.OracleHNSW(d, "ip", n)
    o.import_graph(g)
    ix.set_search_width(1)
    labels = np.arange(n, dtype=np.uint64)
    for k in (1, 10):
        ol, od, oc = o.search(xf, k + 1, ef=16, threads=8)
        ref = drop_self(labels, ol.astype(np.uint64), od.astype(np.float32), oc, k)
        got = ix.search_by_label(labels, k, 16)
        assert_same(got, ref)
        present = np.array([l in row[:c] for l, row, c in zip(labels, ol, oc)])
        assert present.any()
        if d == 8:   # under IP a point is often not its own nearest neighbour: both branches of the rule run
            assert (~present).any()


# ---- 3. edge cases -------------------------------------------------------------------------------------------------
def test_twin_rows_never_return_self():
    n, d = 500, 32
    x = np.random.default_rng(3).standard_normal((n, d), dtype=np.float32)
    ix = ehb.NativeIndex(d, metric="l2", capacity=n + 1)
    ix.add(np.vstack([x, x[:1]]))          # label n is a bitwise twin of label 0
    l, dd, c = ix.search_by_label(np.array([0, n], np.uint64), 5, 64)
    assert l[0][0] == n and l[1][0] == 0 and dd[0][0] == 0 and dd[1][0] == 0
    assert 0 not in l[0][:c[0]] and n not in l[1][:c[1]]


def test_fewer_points_than_k():
    x = np.random.default_rng(4).standard_normal((5, 16), dtype=np.float32)
    ix = ehb.NativeIndex(16, metric="ip", capacity=8)
    ix.add(x)
    got = ix.search_by_label(np.arange(5, dtype=np.uint64), 10)
    assert np.all(got[2] == 4)
    ref, _ = host_composition(ix, np.arange(5, dtype=np.uint64), 10)
    assert_same(got, ref)


def _raw(ix, labels, k, ef=0, brute=False):
    lab = np.ascontiguousarray(labels, np.uint64)
    nq = lab.shape[0]
    ol = np.full((max(nq, 1), max(k, 1)), 77, np.uint64)
    od = np.full((max(nq, 1), max(k, 1)), 7.5, np.float32)
    oc = np.full(max(nq, 1), 9, np.uint32)
    if brute:
        rc = lib().ehb_index_search_bruteforce_by_label(ix._h, nq, _p(lab), k, FP32, _p(ol), _p(od), _p(oc))
    else:
        rc = lib().ehb_index_search_by_label_ex(ix._h, nq, _p(lab), k, ef, FP32, _p(ol), _p(od), _p(oc))
    untouched = (ol == 77).all() and (od == 7.5).all() and (oc == 9).all()
    return rc, untouched


def test_errors_leave_buffers_untouched():
    ix = index("l2", 29)
    ix2 = ehb.NativeIndex(29, capacity=64)
    ix2.add(np.ones((10, 29), np.float32))
    ix2.remove([3])
    assert _raw(ix2, [1, 3], 2) == (5, True)          # tombstoned
    assert _raw(ix2, [1, 99], 2) == (5, True)         # unknown
    assert _raw(ix, [1, 2], 512) == (1, True)         # k + 1 > 512
    assert _raw(ix, [1, 2], 10, ef=513) == (1, True)  # ef > 512
    assert _raw(ix, [1, 2], 2048, brute=True) == (1, True)
    assert _raw(ix, [], 10) == (0, True)              # nq == 0
    assert _raw(ix, [1, 2], 0) == (0, True)           # k == 0
    rc = lib().ehb_index_search_by_label_ex(ix._h, 2, None, 3, 0, FP32, None, None, None)
    assert rc == 1


@pytest.mark.parametrize("precision", [FP32, BF16])
def test_bruteforce_by_label(precision):
    ix = index("ip", 128)
    labels = np.random.default_rng(8).choice(4000, 40, replace=False).astype(np.uint64)
    rows = ix.get_batch(labels)
    for k in (1, 10, 2047):
        L, D, Cn = ix.search_bruteforce(rows, k + 1, precision)
        ref = drop_self(labels, L, D, Cn, k)
        assert_same(ix.search_bruteforce_by_label(labels, k, precision), ref)


# ---- 4. batched get --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric,d", [("cosine", 29), ("l2", 64), ("ip", 768)])
def test_get_batch_equals_get(metric, d):
    ix = index(metric, d) if d != 64 else index(metric, d, 2000)
    labels = np.random.default_rng(9).choice(ix.size, 300).astype(np.uint64)  # repeats allowed
    rows = ix.get_batch(labels)
    ref = np.stack([ix.get(int(l)) for l in labels])
    assert np.array_equal(rows.view(np.uint32), ref.view(np.uint32))
    ix2 = ehb.NativeIndex(d, metric=metric, capacity=16)
    ix2.add(np.ones((4, d), np.float32))
    ix2.remove([2])
    with pytest.raises(KeyError):
        ix2.get_batch([1, 2])
    out = np.zeros((2, d), np.float32)
    assert lib().ehb_index_get_batch(ix2._h, 2, _p(np.array([1, 2], np.uint64)), _p(out)) == 5


# ---- 5. neighbour table ----------------------------------------------------------------------------------------------
def test_neighbor_table_chunks_and_order():
    n, d, k = 6000, 32, 10
    rng = np.random.default_rng(12)
    ix = ehb.NativeIndex(d, metric="l2", capacity=n)
    ix.add(rng.standard_normal((n, d), dtype=np.float32), np.arange(100, 100 + n, dtype=np.uint64))
    # one chunk holds everything: the table is search_by_label of every label
    q, L, D, Cn = ix.neighbor_table(k, 32)
    assert np.array_equal(q, np.arange(100, 100 + n, dtype=np.uint64))
    assert_same((L, D, Cn), ix.search_by_label(q, k, 32))
    dead = rng.choice(np.arange(100, 100 + n), 600, replace=False).astype(np.uint64)
    ix.remove(dead)
    ix.set_option("table_chunk", 1000)
    q, L, D, Cn = ix.neighbor_table(k, 32)
    live = np.setdiff1d(np.arange(100, 100 + n, dtype=np.uint64), dead)
    assert np.array_equal(q, live)          # live internal-id order (= insertion order here)
    for off in range(0, len(q), 1000):      # 5 full chunks and a short last one
        sl = slice(off, off + 1000)
        assert_same((L[sl], D[sl], Cn[sl]), ix.search_by_label(q[sl], k, 32))
    # a buffer too small for the table is refused, nothing else written
    ql, ll = np.zeros(10, np.uint64), np.zeros((10, k), np.uint64)
    rows = C.c_uint64(10)
    rc = lib().ehb_index_neighbor_table(ix._h, k, 32, FP32, _p(ql), _p(ll), None, None, C.byref(rows))
    assert rc == 1 and rows.value == len(live) and (ql == 0).all()


def test_neighbor_table_is_a_snapshot_under_concurrency():
    n, d, k = 6000, 32, 10
    rng = np.random.default_rng(13)
    ix = ehb.NativeIndex(d, metric="l2", capacity=2 * n)
    ix.add(rng.standard_normal((n, d), dtype=np.float32))
    ix.build()
    ix.set_option("table_chunk", 200)
    ix.set_option("combine", 0)   # each search is its own launch, so its answer is the serial one
    ix.set_search_width(1)        # the multi-warp team walk's speculative expansions depend on warp timing
    qs = [rng.standard_normal((16, d), dtype=np.float32) for _ in range(4)]
    serial = [ix.search(q, k, 32) for q in qs]
    ref_table = ix.neighbor_table(k, 32)

    def run(workers):
        started, out = threading.Event(), {}

        def table():
            started.set()
            out["table"] = ix.neighbor_table(k, 32)
            out["t_table"] = time.monotonic()

        th = [threading.Thread(target=table)] + [threading.Thread(target=w, args=(started, out)) for w in workers]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert_same(out["table"][1:], ref_table[1:])
        return out

    # 1. four threads search while the table runs: their answers are the serial ones
    errors = []

    def searcher(i):
        def w(started, out):
            started.wait()
            for _ in range(20):
                r = ix.search(qs[i], k, 32)
                if not all(np.array_equal(a, b) for a, b in zip(r, serial[i])):
                    errors.append(i)
        return w

    run([searcher(i) for i in range(4)])
    assert not errors

    # 2. an add issued during the call completes after it, and the table does not see it
    def adder(started, out):
        started.wait()
        time.sleep(0.002)
        out["t_add_start"] = time.monotonic()
        ix.add(rng.standard_normal((1, d), dtype=np.float32))
        out["t_add"] = time.monotonic()

    out = run([adder])
    assert len(out["table"][0]) == n
    if out["t_add_start"] < out["t_table"]:
        assert out["t_add"] >= out["t_table"]
    assert ix.size == n + 1


# ---- 6. sharded ------------------------------------------------------------------------------------------------------
def _devices(n):
    import torch
    return [i % torch.cuda.device_count() for i in range(n)]


@pytest.mark.parametrize("precision", [FP32, BF16])
def test_sharded_by_label(precision):
    n, d, k = 3000, 64, 10
    rng = np.random.default_rng(21)
    x = rng.standard_normal((n, d), dtype=np.float32)
    sh = ehb.ShardedIndex(d, _devices(2), metric="ip", capacity=n, shard_span=n // 2 + 1)
    sh.add(x)
    sh.build()
    labels = rng.choice(n, 300, replace=False).astype(np.uint64)   # both shards, interleaved
    rows = np.stack([sh.get(int(l)) for l in labels])
    assert np.array_equal(sh.get_batch(labels).view(np.uint32), rows.view(np.uint32))
    L, D, Cn = sh.search(rows, k + 1, 0, precision)
    ref = drop_self(labels, L, D, Cn, k)
    assert_same(sh.search_by_label(labels, k, 0, precision), ref)
    sh.remove(labels[:2])
    with pytest.raises(KeyError):
        sh.search_by_label(labels[:5], k)


# ---- 7. Python and C++ layers ----------------------------------------------------------------------------------------
def test_ann_index_by_keys_equals_hub_key_mode():
    from embeddinghub_b200.hub import EmbeddingHub

    n, d = 3000, 32
    rng = np.random.default_rng(31)
    x = rng.standard_normal((n, d), dtype=np.float32)
    hub = EmbeddingHub()
    hub.create_space("s", d)
    keys = [f"k{i}" for i in range(n)]
    hub.multiset("s", list(zip(keys, x)))
    idx = hub._spaces["s"].index
    idx.multidelete(keys[:50])
    ask = [keys[i] for i in rng.choice(np.arange(50, n), 20, replace=False)]
    for num in (0, 1, 10, 511, 512, 600):
        assert idx.approx_nearest_by_keys(ask, num) == hub.multi_nearest_neighbor("s", num, keys=ask), num
    with pytest.raises(KeyError):
        idx.approx_nearest_by_keys([keys[0]], 3)
    assert np.array_equal(idx.multiget(ask), np.stack([idx.get(k) for k in ask]))
    table = idx.neighbor_table(5)
    assert list(table) == idx.keys()
    sub = idx.keys()[:40]
    assert [table[k] for k in sub] == idx.approx_nearest_by_keys(sub, 5)


def test_cpp_twin_key_mode_matches_python():
    exe = os.path.join(ROOT, "tests", "cpp", "ann_index_by_key")
    assert os.path.exists(exe), "run make"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    got = {}
    for line in out.stdout.splitlines():
        head, _, tail = line.partition(":")
        case, key, num = head.split()
        got[(case, key, int(num))] = tail.split()
    fixture = [("a", [0, 1, 0]), ("b", [1, 1, 0]), ("c", [1, 0, 0])]
    for case, extra in (("fixture", []), ("update", [("a", [0, -1, 0])])):
        idx = ehb.ANNIndex(3)
        for kk, v in fixture + extra:
            idx.set(kk, v)
        for num in range(4):
            py = idx.approx_nearest_by_keys(["a", "b", "c"], num)
            for key, r in zip("abc", py):
                assert got[(case, key, num)] == r, (case, key, num)
