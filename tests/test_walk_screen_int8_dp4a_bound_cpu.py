"""The integer form of the fp32 walk's int8 screen (walk.cuh screen_regs, DESIGN.md §9), checked on the CPU.

The query is quantised once per query (beam_search): sq = RN_fp32(max |q| / 8191) (0 when that is not a normal fp32
value), k = RN(q / sq) clamped to +-8191, split into signed byte planes k = 128 h + l with h = floor((k + 64) / 128),
and e = q - sq k in double, |e|_2 rounded up.  Per candidate, K = sum k_i c_i over the int8 codes, exactly (int32: the
lane sums 128 dp4a(c, h) + dp4a(c, l) and a warp add-reduction, every partial sum bounded by sum |k_i| |c_i|), and
  L = RD(RD(1 - RU(RU(s RU(K)) sq)) - M'),  M' = RU(g |q|_2 |x|_2 + min(|q|_1 max|r|, |q|_2 |r|_2) + en (|x|_2 + |r|_2) + A)
must never exceed the walk's distance RN(1 - P^) of the fp32 chain.  M' replaces the float screen's M
(tests/test_walk_screen_int8_bound_cpu.py) and must stay within 3 % of it on Gaussian rows at d = 768.
"""
import numpy as np
import pytest

from test_walk_screen_int8_bound_cpu import F32, adversarial, chain, f32_down, f32_up, lower_bound, to_i8

KQ = 8191
UP = 1.0 + 2.0 ** -30   # the double sums below are rounded up by far more than their rounding error


def quantise(q):
    """(sq, k, en, kh, kl) as the kernel's prologue computes them"""
    q = np.asarray(q, F32)
    mx = F32(np.abs(np.where(np.isnan(q), 0, q)).max())     # fmaxf ignores NaN
    with np.errstate(over="ignore", invalid="ignore"):
        sq = F32(mx / F32(KQ))
    if not (sq >= F32(2.0 ** -126) and np.isfinite(sq)):
        sq = F32(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.zeros(q.shape, np.int64) if sq == 0 else np.clip(np.nan_to_num(np.rint(q / sq)), -KQ, KQ).astype(np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        e = q.astype(np.float64) - float(sq) * k.astype(np.float64)
        en = f32_up(np.sqrt((e * e).sum() * UP) * UP)
    kh = (k + 64) >> 7
    kl = k - 128 * kh
    return sq, k, en, kh, kl


def int_dot(kh, kl, codes):
    """K in the kernel's order: per lane (chunks lane + 32 t, four codes each) 128 dp4a(c, h) + dp4a(c, l), then the
    warp sum; every intermediate is checked against the int32 range"""
    dpad = codes.shape[-1]
    c = codes.astype(np.int64).reshape(-1, dpad // 128, 32, 4)
    h = kh.reshape(dpad // 128, 32, 4)
    l = kl.reshape(dpad // 128, 32, 4)
    lane = 128 * (c * h).sum((1, 3)) + (c * l).sum((1, 3))
    assert np.abs(lane).max(initial=0) < 2 ** 31
    K = lane.sum(1)
    assert np.abs(K).max(initial=0) < 2 ** 31
    return K


def int_lower_bound(q, codes, terms):
    """the kernel's L and M' from the codes and the row terms, every step rounded in the kernel's direction"""
    dpad = q.shape[-1]
    qd = q.astype(np.float64)
    sq, k, en, kh, kl = quantise(q)
    assert np.all((-64 <= kh) & (kh <= 64) & (-64 <= kl) & (kl <= 63))
    assert np.array_equal(128 * kh + kl, k)
    K = int_dot(kh, kl, codes)
    with np.errstate(invalid="ignore", over="ignore"):
        l1, l2 = f32_up(np.abs(qd).sum()), f32_up(np.sqrt((qd * qd).sum()))
        mxq = np.abs(np.where(np.isnan(qd), 0, qd)).max()
        a = f32_up(dpad * f32_up(mxq * 2.0 ** -125 + 2.0 ** -124).astype(np.float64))
        e = dpad * 2.0 ** -24
        gam = f32_up(e / (1 - e))
        t = terms.astype(np.float64)
        s, rinf, r2, nx = t[:, 0], t[:, 1], t[:, 2], t[:, 3]
        se = f32_up(f32_up(s * f32_up(K.astype(np.float64)).astype(np.float64)).astype(np.float64) * float(sq))
        mg = f32_up(f32_up(float(gam) * float(l2)).astype(np.float64) * nx)
        mg = f32_up(mg + np.minimum(f32_up(float(l1) * rinf), f32_up(float(l2) * r2)))
        mg = f32_up(mg + f32_up(float(en) * f32_up(nx + r2).astype(np.float64) + float(a)))
        L = f32_down(f32_down(1.0 - se.astype(np.float64)).astype(np.float64) - mg.astype(np.float64))
    return L, mg


def check(q, x, codes, terms):
    L, mg = int_lower_bound(q, codes, terms)
    D = (F32(1.0) - chain(q, x)).astype(F32)
    fin = np.isfinite(L)
    assert np.all(L[fin] <= D[fin]), (L - D)[fin].max()
    return L, mg


@pytest.mark.parametrize("dpad", [384, 512, 768, 1024, 1536])
def test_bound_holds_on_adversarial_rows(dpad):
    q, x, codes, terms = adversarial(dpad, 64, dpad)
    L, _ = check(q, x, codes, terms)
    assert np.all(np.isfinite(L))


@pytest.mark.parametrize("dpad", [384, 768, 1536])
@pytest.mark.parametrize("kind", ["dominant", "subnormal", "zeros", "limit", "overflow"])
def test_bound_holds_on_extreme_queries(dpad, kind):
    rng = np.random.default_rng(dpad + len(kind))
    x = rng.standard_normal((64, dpad)).astype(F32)
    q = rng.standard_normal(dpad).astype(F32)
    if kind == "dominant":            # one element carries the scale: the others quantise coarsely
        q[5] = F32(3e4)
    elif kind == "subnormal":         # subnormal elements next to normal ones, and an all-subnormal query
        q[::3] = F32(1e-41)
        check(np.full(dpad, 3e-42, F32), x, *to_i8(x))
    elif kind == "zeros":             # an all-zero query (sq = 0) and one with zero runs
        check(np.zeros(dpad, F32), x, *to_i8(x))
        q[: dpad // 2] = 0
    elif kind == "limit":             # elements exactly at +-sq * 8191 and at half-way points
        sq = F32(2.0 ** -10)
        q = (sq * rng.integers(-KQ, KQ + 1, dpad)).astype(F32)
        q[0] = sq * KQ
        q[1::7] = (sq * (rng.integers(-KQ, KQ, q[1::7].size) + 0.5)).astype(F32)
    elif kind == "overflow":          # |k| = 8191 everywhere against codes +-127 of the same sign: the int32 edge
        q = np.where(rng.standard_normal(dpad) > 0, 1.0, -1.0).astype(F32)
        x = (np.sign(q) * 127 * 2.0 ** -7 * np.ones((4, dpad))).astype(F32)
    codes, terms = to_i8(x)
    if kind == "overflow":
        _, k, _, _, _ = quantise(q)
        assert np.abs(k).min() == KQ and np.abs(codes).min() == 127
        assert KQ * 127 * dpad < 2 ** 31
    L, _ = check(q, x, codes, terms)
    assert np.all(np.isfinite(L))


def test_non_finite_query_keeps_every_candidate():
    x = np.random.default_rng(5).standard_normal((16, 384)).astype(F32)
    codes, terms = to_i8(x)
    for bad in (np.inf, -np.inf, np.nan):
        q = np.random.default_rng(6).standard_normal(384).astype(F32)
        q[17] = bad
        L, _ = int_lower_bound(q, codes, terms)
        assert not np.any(np.isfinite(L))


@pytest.mark.parametrize("dpad", [384, 768, 1536])
def test_integer_margin_stays_within_three_percent_of_the_float_one(dpad):
    rng = np.random.default_rng(11 + dpad)
    x = rng.standard_normal((256, dpad)).astype(F32)
    q = rng.standard_normal(dpad).astype(F32)
    codes, terms = to_i8(x)
    _, mg_int = check(q, x, codes, terms)
    _, mg = lower_bound(q, chain(q, codes.astype(F32)), terms)
    ratio = mg_int.astype(np.float64) / mg.astype(np.float64)
    assert ratio.max() <= 1.03, ratio.max()
