"""The bf16 tensor-core brute force (K3, bf16gemm.cu) checked exactly, kernel by kernel and end to end.

Integer-valued data makes the bf16 path exact.  Entries are integers in [-8, 8] and d <= 2048, so every
|dot|, squared norm and squared distance stays below 2^20: every entry is a bf16 value, every product is
exact in fp32 and every partial sum is an exactly representable integer whatever the accumulation order.
The distance tiles must then equal the integer reference bit for bit, and the whole bf16 pipeline must
return exactly what the fp32 exact path and a float64 numpy reference return (ids, distance bits, counts).
A single misplaced element in the TMA / swizzle / descriptor / accumulator chain changes an integer.
This relies on the H100's wgmma fp32 accumulation being exact for integer partial sums below 2^20.  On an
H100 80GB HBM3 (700 W power limit) it is: every integer case here passes with no tolerance.

Gaussian data and cosine are not exact; they are held to an error bound (tiles) or to agreement between
the fused and the unfused selection (end to end).

The kernel-level tests go through tests/cpp/libbf16_probe.so, thin extern "C" wrappers around the launchers
of the shipped libehb200.so (built by `make`).
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import embeddinghub_b200 as ehb  # noqa: E402
from embeddinghub_b200._native import BF16  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tests", "cpp", "libbf16_probe.so")
MAX_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
U32 = np.uint64(0xFFFFFFFF)

_probe = None


def probe():
    global _probe
    if _probe is None:
        if not os.path.exists(PROBE):
            pytest.fail(f"{PROBE} is missing: run make")
        ehb.lib()  # the probe binds to the same libehb200.so the package loaded
        L = C.CDLL(PROBE)
        vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32
        L.probe_to_bf16.argtypes = [vp, u32, vp, vp, u64, u32]
        L.probe_bf16_dist_tile.argtypes = [vp, u64, vp, u64, u32, i32, vp, vp, u64, u64, u64, u64, vp, u64]
        L.probe_bf16_topk_chunk.argtypes = [vp, u64, vp, u64, u32, i32, vp, vp, u64, u64, vp, vp, vp, u32, vp, u32,
                                            vp, i32]
        for f in (L.probe_to_bf16, L.probe_bf16_dist_tile, L.probe_bf16_topk_chunk):
            f.restype = C.c_int
        _probe = L
    return _probe


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _call(fn, *args):
    import torch

    rc = fn(*args)
    assert rc == 0, f"cudaError {rc}"
    torch.cuda.synchronize()


def ints(rng, rows, dim, width=None):
    """[rows, width] float32 integers in [-8, 8], zero beyond column dim."""
    a = np.zeros((rows, width or dim), np.float32)
    a[:, :dim] = rng.integers(-8, 9, size=(rows, dim), dtype=np.int8)
    return a


def to_dev_bf16(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda().to(torch.bfloat16)


def bf16_round(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.bfloat16).to(torch.float32).numpy()


# ---- ordered keys (common.cuh: f2ord / make_key) restated in numpy -----------------------------------------------
def f2ord(d32):
    b = np.asarray(d32, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(b >> np.uint64(31) == 1, b ^ U32, b ^ np.uint64(0x80000000))


def key_dist(keys):
    o = (np.asarray(keys, np.uint64) >> np.uint64(32)).astype(np.uint64)
    b = np.where(o >> np.uint64(31) == 1, o ^ np.uint64(0x80000000), o ^ U32)
    return b.astype(np.uint32).view(np.float32)


def make_keys(d32, ids):
    return (f2ord(d32) << np.uint64(32)) | np.asarray(ids, np.uint64)


def exact_dist(q, x, metric):
    """float32 distances of integer data, computed exactly in float64 (metric 0: L2, 1: 1 - dot)."""
    qd, xd = q.astype(np.float64), x.astype(np.float64)
    dot = qd @ xd.T
    if metric == 0:
        d = (qd * qd).sum(1)[:, None] + (xd * xd).sum(1)[None, :] - 2.0 * dot
    else:
        d = 1.0 - dot
    return d.astype(np.float32)


# ---- fp32 -> bf16 rows ---------------------------------------------------------------------------------------------
def _near_ties(rng, n):
    """Floats at, just below and just above the midpoint between two adjacent bf16 values (both signs)."""
    hi = rng.integers(0x3000, 0x5000, size=n, dtype=np.uint32)        # |x| in [2^-31, 2^33): squares stay normal
    hi |= rng.integers(0, 2, size=n, dtype=np.uint32) << 15             # sign
    low = rng.choice(np.array([0x7FFF, 0x8000, 0x8001, 0x0001, 0xFFFF, 0x0000], np.uint32), size=n)
    return ((hi << 16) | low).view(np.float32)


@pytest.mark.parametrize("kind,n,dim,dpad,extra", [("gauss", 1000, 128, 128, 0), ("ties", 777, 768, 768, 0),
                                                    ("gauss", 300, 100, 128, 7), ("ties", 33, 2048, 2048, 64)])
def test_to_bf16_rounds_to_nearest_even(kind, n, dim, dpad, extra):
    """Rows are bit-equal to torch's round-to-nearest-even; columns [dim, dpad) of a zero-padded source stay
    zero; source columns beyond dpad (in_stride > dpad) are never read; the norms are those of the rounded
    values within the fp32 error of a 32-lane strided sum."""
    import torch

    rng = np.random.default_rng(n + dim)
    stride = dpad + extra
    src = np.full((n, stride), np.nan, np.float32)
    src[:, dim:dpad] = 0.0
    if kind == "gauss":
        src[:, :dim] = rng.standard_normal((n, dim)).astype(np.float32) * 3.0
    else:
        src[:, :dim] = _near_ties(rng, n * dim).reshape(n, dim)
    s = torch.from_numpy(src).cuda()
    out = torch.full((n, dpad), float("nan"), dtype=torch.bfloat16, device="cuda")
    norms = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    _call(probe().probe_to_bf16, _ptr(s), stride, _ptr(out), _ptr(norms), n, dpad)
    got = out.cpu().view(torch.int16).numpy()
    want = torch.from_numpy(np.ascontiguousarray(src[:, :dpad])).to(torch.bfloat16).view(torch.int16).numpy()
    assert np.array_equal(got, want)
    assert np.all(got[:, dim:] == 0)
    r = torch.from_numpy(got.copy()).view(torch.bfloat16).to(torch.float32).numpy().astype(np.float64)
    ref = (r * r).sum(1)
    tol = (dpad // 32 + 6) * 2.0 ** -24 * ref
    err = np.abs(norms.cpu().numpy().astype(np.float64) - ref)
    assert np.all(err <= tol), float((err / np.maximum(tol, 1e-300)).max())


# ---- unfused distance tiles ----------------------------------------------------------------------------------------
# dpad, q_rows, q0, qn, x_rows, n0, nn, ldd: every k-block count 1..32; windows off the origin; qn and nn on both
# sides of the 128 x 256 tile; operands smaller than one TMA box; odd ldd (scalar stores) and ldd > nn
TILES = [
    (64, 1, 0, 1, 1, 0, 1, 1),
    (128, 200, 5, 63, 600, 3, 255, 255),
    (256, 64, 0, 64, 256, 0, 256, 260),
    (384, 400, 100, 65, 2000, 700, 257, 257),
    (512, 127, 0, 127, 1000, 0, 1000, 1000),
    (768, 300, 0, 300, 1300, 300, 1000, 1001),
    (1024, 130, 2, 128, 257, 1, 256, 258),
    (1536, 129, 0, 129, 300, 43, 257, 264),
    (2048, 63, 0, 63, 255, 0, 255, 256),
]
_GUARD = 64  # NaN floats before and after the output rows


def run_tile(q, x, qnorm, xnorm, metric, case):
    """Launches one distance tile over a NaN-filled buffer; asserts that exactly the window was written."""
    import torch

    dpad, q_rows, q0, qn, x_rows, n0, nn, ldd = case
    qb, xb = to_dev_bf16(q), to_dev_bf16(x)
    qnt = torch.from_numpy(qnorm.astype(np.float32)).cuda()
    xnt = torch.from_numpy(xnorm.astype(np.float32)).cuda()
    buf = torch.full((2 * _GUARD + qn * ldd,), float("nan"), dtype=torch.float32, device="cuda")
    _call(probe().probe_bf16_dist_tile, _ptr(qb), q_rows, _ptr(xb), x_rows, dpad, metric, _ptr(qnt), _ptr(xnt), q0, qn,
          n0, nn, C.c_void_p(buf.data_ptr() + 4 * _GUARD), ldd)
    h = buf.cpu().numpy()
    body = h[_GUARD:_GUARD + qn * ldd].reshape(qn, ldd)
    assert np.isnan(h[:_GUARD]).all() and np.isnan(h[_GUARD + qn * ldd:]).all(), "store outside the buffer rows"
    assert np.isnan(body[:, nn:]).all(), "store beyond column nn"
    win = body[:, :nn]
    assert not np.isnan(win).any(), "window element not written"
    return win


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("case", TILES, ids=[f"dpad{c[0]}" for c in TILES])
def test_dist_tile_integer_exact(case, metric):
    dpad, q_rows, q0, qn, x_rows, n0, nn, ldd = case
    rng = np.random.default_rng(dpad + metric)
    q, x = ints(rng, q_rows, dpad), ints(rng, x_rows, dpad)
    qnorm = (q.astype(np.float64) ** 2).sum(1)
    xnorm = (x.astype(np.float64) ** 2).sum(1)
    win = run_tile(q, x, qnorm, xnorm, metric, case)
    ref = exact_dist(q[q0:q0 + qn], x[n0:n0 + nn], metric)
    bad = win.view(np.uint32) != ref.view(np.uint32)
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} differ; first at {np.argwhere(bad)[0].tolist()}: "
                           f"{win[bad][0]} vs {ref[bad][0]}; max |diff| {float(np.abs(win - ref).max())}")


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("case", TILES, ids=[f"dpad{c[0]}" for c in TILES])
def test_dist_tile_gaussian_error_bound(case, metric):
    """Against float64 on the bf16-rounded inputs: |err| <= 2^-14 sum|q_i x_i| (+ 2^-14 (|q|^2 + |x|^2) for L2).
    A structural error (a wrong k-slice, row or column) is ~1e-2 relative, far outside the bound."""
    dpad, q_rows, q0, qn, x_rows, n0, nn, ldd = case
    rng = np.random.default_rng(100 + dpad + metric)
    q = bf16_round(rng.standard_normal((q_rows, dpad)).astype(np.float32))
    x = bf16_round(rng.standard_normal((x_rows, dpad)).astype(np.float32))
    qd, xd = q.astype(np.float64), x.astype(np.float64)
    qnorm, xnorm = (qd * qd).sum(1), (xd * xd).sum(1)
    win = run_tile(q, x, qnorm, xnorm, metric, case).astype(np.float64)
    qw, xw = qd[q0:q0 + qn], xd[n0:n0 + nn]
    dot = qw @ xw.T
    bound = 2.0 ** -14 * (np.abs(qw) @ np.abs(xw).T)
    if metric == 0:
        ref = qnorm[q0:q0 + qn, None] + xnorm[None, n0:n0 + nn] - 2.0 * dot
        bound += 2.0 ** -14 * (qnorm[q0:q0 + qn, None] + xnorm[None, n0:n0 + nn])
    else:
        ref = 1.0 - dot
    ratio = float((np.abs(win - ref) / bound).max())
    print(f"dpad {dpad} metric {metric}: largest |err| / bound = {ratio:.3e}")
    assert ratio <= 1.0


# ---- fused top-k chunk (bf16_topk_gemm_kernel + compact_candidates_kernel) -------------------------------------------
# metric, dpad, nq, kc, sms: one CTA walking every tile (sms 1) carries the ring phase across tiles; kc spans the
# compaction sizes P = 128 .. 8192 (one warp per block at 8192)
CHUNKS = [
    (0, 384, 129, 64, 1),
    (1, 64, 1, 1, 3),
    (0, 768, 300, 400, 132),
    (1, 2048, 127, 2048, 132),
    (0, 2048, 129, 1, 3),
    (1, 768, 127, 64, 1),
    (0, 64, 300, 2048, 132),
    (1, 384, 1, 400, 3),
]


@pytest.mark.parametrize("metric,dpad,nq,kc,sms", CHUNKS)
def test_topk_chunk_matches_driver_model(metric, dpad, nq, kc, sms):
    """Drives launch_bf16_topk_chunk like launch_bruteforce does and checks every chunk against a numpy model:
    run_keys = the first kc (distance, index) keys of the rows seen so far, thr = the kc-th distance, and the
    overflow flag raised exactly when a query admitted more than ccap rows with d < thr.  The last chunk is
    built to overflow (more than ccap rows beat query 0's threshold); its survivors depend on atomic order,
    so for the overflowing queries only the invariants are checked."""
    import torch

    rng = np.random.default_rng(7 * dpad + kc + nq)
    ccap = 2 * kc + 64
    # thr = +inf admits every row of the first chunk: exactly ccap rows fill the buffer without overflowing;
    # the later chunks double (a chunk as large as everything seen admits about kc rows) and end off the
    # 256-row tile grid
    bounds = [0, ccap]
    while bounds[-1] < max(3 * ccap, 2500):
        bounds.append(2 * bounds[-1] - 13)
    n_norm = bounds[-1]
    q = ints(rng, nq, dpad)
    if metric == 0:
        near = np.repeat(q[:1], ccap + 5, axis=0)                          # distance 0 to query 0
    else:
        near = np.repeat(np.where(q[:1] >= 0, 8.0, -8.0).astype(np.float32), ccap + 5, axis=0)  # largest dot
    x = np.concatenate([ints(rng, n_norm, dpad), near])
    bounds.append(x.shape[0])
    D = exact_dist(q, x, metric)
    ids = np.arange(x.shape[0], dtype=np.uint64)

    qb, xb = to_dev_bf16(q), to_dev_bf16(x)
    qnt = torch.from_numpy((q.astype(np.float64) ** 2).sum(1).astype(np.float32)).cuda()
    xnt = torch.from_numpy((x.astype(np.float64) ** 2).sum(1).astype(np.float32)).cuda()
    thr = torch.full((nq,), float("nan"), dtype=torch.float32, device="cuda")
    cbuf = torch.zeros(nq * ccap, dtype=torch.int64, device="cuda")
    ccount = torch.zeros(nq, dtype=torch.int32, device="cuda")
    overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
    run = torch.full((nq, kc), -1, dtype=torch.int64, device="cuda")      # kMaxKey

    def chunk(lo, hi):
        overflow.zero_()
        _call(probe().probe_bf16_topk_chunk, _ptr(qb), nq, _ptr(xb), x.shape[0], dpad, metric, _ptr(qnt), _ptr(xnt),
              lo, hi, _ptr(thr), _ptr(cbuf), _ptr(ccount), ccap, _ptr(run), kc, _ptr(overflow), sms)
        assert np.all(ccount.cpu().numpy() == 0), "counters not reset"
        return run.cpu().numpy().view(np.uint64), thr.cpu().numpy(), int(overflow.item())

    r, t, ovf = chunk(0, 0)                                                # publishes thr from the empty lists
    assert np.all(r == MAX_KEY) and np.all(np.isposinf(t)) and ovf == 0
    model = np.full((nq, kc), MAX_KEY, np.uint64)
    mthr = np.full(nq, np.inf, np.float32)
    for ci, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
        admitted = (D[:, lo:hi] < mthr[:, None]).sum(1)
        merged = np.sort(np.concatenate([model, make_keys(D[:, lo:hi], ids[lo:hi])], axis=1), axis=1)[:, :kc]
        model = merged
        mthr = np.where(model[:, -1] != MAX_KEY, key_dist(model[:, -1]), np.float32(np.inf)).astype(np.float32)
        r, t, ovf = chunk(lo, hi)
        over = admitted > ccap
        assert ovf == int(over.any()), (ci, lo, hi, int(admitted.max()), ccap)
        assert hi == x.shape[0] or not over.any(), "test data: only the last chunk may overflow"
        ok = ~over
        assert np.array_equal(r[ok], model[ok]), f"chunk {ci} [{lo}, {hi}): run_keys differ from the model"
        assert np.array_equal(t[ok].view(np.uint32), mthr[ok].view(np.uint32)), f"chunk {ci}: thr differs"
        for qi in np.flatnonzero(over):
            rk = r[qi]
            valid = rk[rk != MAX_KEY]
            assert valid.size == min(kc, hi), "run list lost entries"
            assert np.all(valid[1:] > valid[:-1]), "run_keys not sorted and unique"
            rid = (valid & U32).astype(np.int64)
            assert np.all(rid < hi), "key names a row not seen yet"
            assert np.array_equal(key_dist(valid).view(np.uint32), D[qi, rid].view(np.uint32)), "key distance"
            assert t[qi] == key_dist(valid[-1:])[0]
    assert over[0] and ovf == 1, "the last chunk must overflow"


# ---- end to end: NativeIndex.search_bruteforce(..., precision=BF16) ------------------------------------------------
def ref_topk(base, q, k, metric, alive=None):
    """numpy reference: (distance, insertion index) order over the live rows; exact on integer data."""
    n = base.shape[0]
    nq = q.shape[0]
    live = n if alive is None else int(alive.sum())
    kk = min(k, live)
    labels = np.full((nq, k), ehb.NO_LABEL, np.uint64)
    dists = np.full((nq, k), np.inf, np.float32)
    m = 0 if metric == "l2" else 1
    ids = np.arange(n, dtype=np.uint64)
    for b in range(0, nq, 256):
        keys = make_keys(exact_dist(q[b:b + 256], base, m), ids)
        if alive is not None:
            keys[:, ~alive] = MAX_KEY
        if kk:
            top = np.sort(np.partition(keys, kk - 1, axis=1)[:, :kk], axis=1)
            labels[b:b + 256, :kk] = top & U32
            dists[b:b + 256, :kk] = key_dist(top)
    return labels, dists, np.full(nq, kk, np.uint32)


def assert_same(got, want, what):
    gl, gd, gc = got
    wl, wd, wc = want
    bad = np.flatnonzero((gl != wl).any(1))
    assert bad.size == 0, f"{what}: labels differ in {bad.size} queries, first {bad[0]}: {gl[bad[0]][:8]} vs {wl[bad[0]][:8]}"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"{what}: distance bits differ"
    assert np.array_equal(gc, wc), f"{what}: counts differ"


# d < dpad and every dpad class; n = 8192 (unfused only), 8193 (a one-row fused chunk), ~20k and ~70k (several
# fused chunks); nq > 2048 (q-blocked bootstrap); k up to 2048 (kc = 2048, compaction P = 8192)
E2E = [
    ("ip", 33, 8192, 129, 10),
    ("l2", 100, 8193, 129, 100),
    ("ip", 200, 20011, 1, 1),
    ("l2", 300, 20011, 129, 2048),
    ("l2", 384, 70000, 129, 10),
    ("ip", 512, 20011, 2049, 10),
    ("l2", 700, 8193, 2049, 100),
    ("ip", 768, 70000, 129, 100),
    ("ip", 1024, 20011, 129, 2048),
    ("l2", 1100, 8193, 1, 1),
    ("l2", 2048, 20011, 129, 100),
]


@pytest.mark.parametrize("metric,d,n,nq,k", E2E)
def test_bf16_bruteforce_integer_bitwise(metric, d, n, nq, k):
    """Integer data: the bf16 keys are exact, so the candidate sets hold the true top-kc and the fp32 re-rank
    returns exactly the exact path's result.  Integer data has many exact ties, so this also pins the strict
    d < thr admission and the tie order by insertion index."""
    rng = np.random.default_rng(d * 7 + n + nq)
    base, q = ints(rng, n, d), ints(rng, nq, d)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    want = ref_topk(base, q, k, metric)
    assert_same(ix.search_bruteforce(q, k), want, "exact path vs numpy")
    assert_same(ix.search_bruteforce(q, k, precision=BF16), want, "bf16 path vs numpy")


def test_bf16_overflow_fallback_bitwise():
    """Rows 0..8191 lie far from the queries, every later row near them: every row of the first fused chunk
    [8192, 16384) beats the bootstrap threshold, 8192 > ccap survivors per query overflow the candidate
    buffer, and the driver re-runs that chunk unfused over the partly merged running lists."""
    d, n, nq, k = 128, 20011, 129, 10
    rng = np.random.default_rng(5)
    base, q = ints(rng, n, d), ints(rng, nq, d)
    base[:8192] += 40.0                          # squared distances >= 128 * 24^2 > every near row's 128 * 16^2
    ix = ehb.NativeIndex(d, metric="l2", capacity=n)
    ix.add(base)
    want = ref_topk(base, q, k, "l2")
    assert_same(ix.search_bruteforce(q, k), want, "exact path vs numpy")
    assert_same(ix.search_bruteforce(q, k, precision=BF16), want, "bf16 path (overflow fallback) vs numpy")


@pytest.mark.parametrize("metric", ["ip", "l2", "cosine"])
def test_bf16_fused_equals_unfused(metric):
    """Both selections keep the exact top-kc by the same bf16 keys, computed at the same tile positions (chunk
    starts are multiples of 256, query blocks multiples of 128), so their outputs are identical."""
    d, n, nq, k = 768, 20011, 129, 10
    rng = np.random.default_rng(11)
    base = rng.standard_normal((n, d)).astype(np.float32)
    q = rng.standard_normal((nq, d)).astype(np.float32)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    fused = ix.search_bruteforce(q, k, precision=BF16)
    ix.set_option("bf16_unfused", 1)
    unfused = ix.search_bruteforce(q, k, precision=BF16)
    ix.set_option("bf16_unfused", 0)
    assert_same(fused, unfused, "fused vs unfused")
    assert_same(ix.search_bruteforce(q, k, precision=BF16), fused, "fused, repeated")


@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_bf16_tombstones(metric):
    """Tombstones force the unfused selection (they are filtered where keys are formed): no removed label is
    returned, the result is the exact one over the survivors, and a re-added label is found again."""
    d, n, nq, k = 128, 20011, 129, 10
    rng = np.random.default_rng(13)
    base, q = ints(rng, n, d), ints(rng, nq, d)
    ix = ehb.NativeIndex(d, metric=metric, capacity=n)
    ix.add(base)
    top0 = int(ref_topk(base, q[:1], 1, metric)[0][0, 0])
    dead = np.union1d(rng.choice(n, n // 10, replace=False), [top0]).astype(np.uint64)
    ix.remove(dead)
    alive = np.ones(n, bool)
    alive[dead.astype(np.int64)] = False
    got = ix.search_bruteforce(q, k, precision=BF16)
    assert not np.isin(got[0], dead).any()
    want = ref_topk(base, q, k, metric, alive)
    assert_same(ix.search_bruteforce(q, k), want, "exact path with tombstones vs numpy")
    assert_same(got, want, "bf16 path with tombstones vs numpy")
    ix.add(base[top0:top0 + 1], np.array([top0], np.uint64))
    alive[top0] = True
    got = ix.search_bruteforce(q, k, precision=BF16)
    assert int(got[0][0, 0]) == top0
    assert_same(got, ref_topk(base, q, k, metric, alive), "bf16 path after re-adding a label")


def test_bf16_edges():
    q = ints(np.random.default_rng(3), 7, 100)
    empty = ehb.NativeIndex(100, metric="l2", capacity=16)
    l, dd, c = empty.search_bruteforce(q, 4, precision=BF16)
    assert np.all(l == ehb.NO_LABEL) and np.all(np.isposinf(dd)) and np.all(c == 0)
    for n, k in [(1, 1), (1, 8), (5, 8), (5, 3)]:
        for metric in ("l2", "ip"):
            base = ints(np.random.default_rng(n), n, 100)
            ix = ehb.NativeIndex(100, metric=metric, capacity=16)
            ix.add(base)
            want = ref_topk(base, q, k, metric)       # kc is clamped to n: counts == n, NO_LABEL / inf padding
            assert_same(ix.search_bruteforce(q, k, precision=BF16), want, f"bf16 n={n} k={k} {metric}")
            assert_same(ix.search_bruteforce(q, k), want, f"exact n={n} k={k} {metric}")
    for d in (32, 5):                                  # one 32-wide row has no 64-wide k-block
        ix = ehb.NativeIndex(d, capacity=16)
        ix.add(ints(np.random.default_rng(d), 10, d))
        with pytest.raises(ehb.EhbError):
            ix.search_bruteforce(ints(np.random.default_rng(1), 2, d), 1, precision=BF16)


def _devices(n):
    import torch

    have = torch.cuda.device_count()
    return [i % have for i in range(n)]


@pytest.mark.parametrize("shards", [2, 3])
def test_sharded_bf16_bitwise(shards):
    """Each shard runs the bf16 path over its label range (fused at ~10k rows, unfused at ~6.7k); the merged
    result equals the single index's exact result."""
    d, n, nq, k = 128, 20011, 129, 10
    rng = np.random.default_rng(17)
    base, q = ints(rng, n, d), ints(rng, nq, d)
    sh = ehb.ShardedIndex(d, _devices(shards), metric="ip", capacity=1024, shard_span=n // shards + 1)
    sh.add(base)
    one = ehb.NativeIndex(d, metric="ip", capacity=n)
    one.add(base)
    want = one.search_bruteforce(q, k)
    assert_same(want, ref_topk(base, q, k, "ip"), "exact path vs numpy")
    assert_same(sh.search_bruteforce(q, k, precision=BF16), want, f"sharded bf16 ({shards} shards)")
