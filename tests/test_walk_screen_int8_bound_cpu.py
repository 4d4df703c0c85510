"""The bound behind the fp32 walk's int8 screen (walk.cuh screen_staged, DESIGN.md §9), checked on the CPU.

`to_i8` is a numpy replica of the conversion kernel (search.cu to_i8_rows_kernel): s = RN_fp32(max |x_i| / 127),
codes c = RN(x / s) clamped to [-127, 127], and the per-row terms (s, max |r_i|, |r|_2, |x|_2) rounded up, r = x - s c
in double.  tests/test_gpu_walk_screen_int8.py checks it against the device.  Both fp32 chains are emulated in the
kernel's lane order: lane l holds the chunks l + 32 t (t < dpad / 128), accumulates component j with fp32 FMAs over t,
adds (a0 + a1) + (a2 + a3), and the warp sums the lanes with a butterfly of xor-shuffles 16, 8, 4, 2, 1.  The walk's
chain runs over the fp32 row x (P^), the screen's over the codes (E^).  The screen's lower bound
  L = RD(RD(1 - RU(s E^)) - M),  M = RU(g |q|_2 (2 |x|_2 + |r|_2) + min(|q|_1 max|r|, |q|_2 |r|_2) + A + s A_s)
must never exceed the walk's distance RN(1 - P^).  On adversarial rows (every residual just inside +-s/2, its sign
that of the query's element) the actual gap |P^ - s E^| must also fill most of M, so the bound is not vacuous.
"""
import numpy as np
import pytest

F32 = np.float32


def to_i8(x):
    """codes [n][d] int8 and terms [n][4] fp32, as the conversion kernel computes them"""
    x = np.asarray(x, F32)
    xd = x.astype(np.float64)
    finite = np.isfinite(x).all(1)
    mx = np.where(finite, np.abs(np.where(np.isfinite(x), x, 0)).max(1), 0).astype(F32)
    s = (mx.astype(np.float64) / 127.0).astype(F32)
    bad = ~finite | ((s != 0) & (s < F32(2.0 ** -126)))
    sd = s.astype(np.float64)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.where(bad[:, None] | (sd == 0), 0.0, np.clip(np.rint(xd / np.where(sd == 0, 1, sd)), -127, 127))
    r = xd - sd * c
    up = 1.0 + 2.0 ** -30
    terms = np.stack([s, f32_up(np.abs(r).max(1)), f32_up(np.sqrt((r * r).sum(1)) * up),
                      f32_up(np.sqrt((xd * xd).sum(1)) * up)], 1).astype(F32)
    terms[bad] = np.nan
    return c.astype(np.int8), terms


def f32_up(v):
    v = np.asarray(v, np.float64)
    f = v.astype(F32)
    return np.where(f.astype(np.float64) < v, np.nextafter(f, F32(np.inf)), f).astype(F32)


def f32_down(v):
    v = np.asarray(v, np.float64)
    f = v.astype(F32)
    return np.where(f.astype(np.float64) > v, np.nextafter(f, F32(-np.inf)), f).astype(F32)


def fma(a, b, c):
    # a * b is exact in float64 for float32 inputs; the sum is rounded once to float64 and once to float32 (the
    # double rounding can differ from a true FMA in the last bit, far inside the bound's slack)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def chain(q, x):
    """fp32 dot product of q and the rows of x in the kernel's lane order"""
    nq = q.shape[-1] // 128
    qq = q.reshape(nq, 32, 4)            # [t][lane][j] = element 4 (lane + 32 t) + j
    xx = x.astype(F32).reshape(-1, nq, 32, 4)
    acc = np.zeros((x.shape[0], 32, 4), F32)
    for t in range(nq):
        acc = fma(np.broadcast_to(qq[t], acc.shape), xx[:, t], acc)
    lane = (acc[..., 0] + acc[..., 1]) + (acc[..., 2] + acc[..., 3])
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[:, np.arange(32) ^ o]
    return lane[:, 0]


def lower_bound(q, e_hat, terms):
    """the kernel's L from E^ and the row terms, every step rounded in the kernel's direction"""
    dpad = q.shape[-1]
    qd = q.astype(np.float64)
    l1, l2 = f32_up(np.abs(qd).sum()), f32_up(np.sqrt((qd * qd).sum()))
    a = f32_up(dpad * f32_up(np.abs(qd).max() * 2.0 ** -125 + 2.0 ** -124).astype(np.float64))
    e = dpad * 2.0 ** -24
    gam, a_s = f32_up(e / (1 - e)), f32_up(dpad * 2.0 ** -118)
    t = terms.astype(np.float64)
    s, rinf, r2, nx = t[:, 0], t[:, 1], t[:, 2], t[:, 3]
    se = f32_up(s * e_hat.astype(np.float64))
    mg = f32_up(f32_up(float(gam) * float(l2)).astype(np.float64) * f32_up(2 * nx + r2))
    mg = f32_up(mg + np.minimum(f32_up(float(l1) * rinf), f32_up(float(l2) * r2)))
    mg = f32_up(mg + f32_up(s * float(a_s) + float(a)))
    return f32_down(f32_down(1.0 - se.astype(np.float64)).astype(np.float64) - mg.astype(np.float64)), mg


def adversarial(dpad, rows, seed):
    """rows whose residuals sit just inside +-s/2, signed like the query's elements, with an exact scale"""
    rng = np.random.default_rng(seed)
    sign = np.where(rng.standard_normal(dpad) > 0, 1.0, -1.0)
    q = (np.abs(rng.standard_normal(dpad)) * sign).astype(F32)
    s = (2.0 ** rng.integers(-8, 2, rows) * (1 + rng.integers(0, 64, rows) / 64)).astype(F32)[:, None]
    c = rng.integers(-126, 127, (rows, dpad)).astype(np.float64)
    x = (s * c + s * sign * (0.5 - 2.0 ** -10)).astype(F32)
    x[:, 0] = (127 * s[:, 0]).astype(F32)       # the largest element fixes s exactly
    codes, terms = to_i8(x)
    assert np.array_equal(terms[:, 0], s[:, 0])
    assert np.array_equal(codes[:, 1:], c[:, 1:].astype(np.int8))
    return q, x, codes, terms


@pytest.mark.parametrize("dpad", [384, 512, 768, 1024, 1536, 2048])
def test_bound_holds_and_is_reached_on_adversarial_rows(dpad):
    q, x, codes, terms = adversarial(dpad, 64, dpad)
    p_hat = chain(q, x)
    e_hat = chain(q, codes.astype(F32))
    L, mg = lower_bound(q, e_hat, terms)
    D = (F32(1.0) - p_hat).astype(F32)
    assert np.all(np.isfinite(L))
    assert np.all(L <= D), (L - D).max()
    gap = np.abs(p_hat.astype(np.float64) - terms[:, 0].astype(np.float64) * e_hat.astype(np.float64))
    assert (gap / mg).max() > 0.9, (gap / mg).max()


@pytest.mark.parametrize("dpad", [384, 768, 1536])
def test_bound_holds_on_gaussian_rows(dpad):
    rng = np.random.default_rng(7 + dpad)
    x = rng.standard_normal((256, dpad)).astype(F32)
    q = rng.standard_normal(dpad).astype(F32)
    codes, terms = to_i8(x)
    p_hat = chain(q, x)
    L, mg = lower_bound(q, chain(q, codes.astype(F32)), terms)
    assert np.all(L <= (F32(1.0) - p_hat).astype(F32))
    # the screen decides on a band of a few tenths of a standard deviation of the inner products
    assert np.median(mg) < 0.4 * np.std(p_hat)


def test_degenerate_rows():
    dpad = 384
    x = np.zeros((5, dpad), F32)
    x[1, :3] = [1e-40, -2e-41, 3e-42]          # subnormal scale: never rejected
    x[2, 5] = np.inf                            # non-finite: never rejected
    x[3, 7] = np.nan
    x[4, :] = 1e-39                             # subnormal elements with ...
    x[4, 0] = 1.0                               # ... a normal scale: a finite bound
    codes, terms = to_i8(x)
    assert np.array_equal(terms[0], np.zeros(4, F32)) and not codes[0].any()   # all zero: s = 0, no residual
    assert np.all(np.isnan(terms[1:4]))
    assert np.all(np.isfinite(terms[4])) and terms[4, 0] == F32(1.0 / 127)
    q = np.random.default_rng(3).standard_normal(dpad).astype(F32)
    L, _ = lower_bound(q, chain(q, codes.astype(F32)), terms)
    assert np.all(np.isnan(L[1:4]))             # a non-finite L keeps the candidate
    p_hat = chain(q, x[[0, 4]])
    assert np.all(L[[0, 4]] <= (F32(1.0) - p_hat).astype(F32))
