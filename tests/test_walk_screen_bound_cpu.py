"""The bound behind the fp32 walk's bf16 screen (walk.cuh screen_constant, DESIGN.md §9), checked on the CPU.

Both fp32 chains are emulated in the kernel's order: lane l holds the float4 chunks l + 32 t (t < dpad / 128),
accumulates component j with fp32 FMAs over t, adds (a0 + a1) + (a2 + a3), and the warp sums the lanes with a
butterfly of xor-shuffles 16, 8, 4, 2, 1.  The walk's chain runs over the fp32 row x, the screen's over
b = RN_bf16(x) (as to_bf16_rows_kernel rounds), together with S = sum |q| |b|.  On adversarial vectors (x just
below the bf16 rounding midpoints, every error aligned with the query's sign) the test checks
|P^ - E^| <= c S^ + A with the kernel's constant and absolute term, and that the screen's lower bound
L = RD(RD(1 - E^) - B) never exceeds the walk's distance RN(1 - P^).
"""
import numpy as np
import pytest

F32 = np.float32


def screen_constant(n):
    u, e = 1.0 / 256.0, n * 2.0 ** -24
    g = e / (1.0 - e)
    return (u + (2.0 + u) * g) / (1.0 - g) * (1.0 + 2.0 ** -20)


def f32_up(v):
    f = F32(v)
    return f if float(f) >= v else np.nextafter(f, F32(np.inf))


def fma(a, b, c):
    # a * b is exact in float64 for float32 inputs; the sum is rounded once to float64 and once to float32 (the
    # double rounding can differ from a true FMA in the last bit, far inside the bound's slack)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def chain(q, x):
    """fp32 dot product of q and x over the rows of x in the kernel's lane order."""
    nq = q.shape[-1] // 128
    qq = q.reshape(nq, 32, 4)            # [t][lane][j] = element 4 (lane + 32 t) + j
    xx = x.reshape(-1, nq, 32, 4)
    acc = np.zeros((x.shape[0], 32, 4), F32)
    for t in range(nq):
        acc = fma(np.broadcast_to(qq[t], acc.shape), xx[:, t], acc)
    lane = (acc[..., 0] + acc[..., 1]) + (acc[..., 2] + acc[..., 3])
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[:, np.arange(32) ^ o]
    return lane[:, 0]


def to_bf16(x):
    u = x.view(np.uint32).astype(np.uint64)
    r = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return r.astype(np.uint32).view(F32)


def rd_sub(a, b):
    """a - b rounded down to float32."""
    r = (a.astype(np.float64) - b.astype(np.float64))
    f = r.astype(F32)
    return np.where(f.astype(np.float64) > r, np.nextafter(f, F32(-np.inf)), f)


def adversarial(dpad, rows, seed):
    rng = np.random.default_rng(seed)
    b = to_bf16(rng.standard_normal((rows, dpad)).astype(F32))
    sign = np.where(rng.standard_normal(dpad) > 0, 1.0, -1.0).astype(F32)
    q = (np.abs(rng.standard_normal(dpad)) * sign).astype(F32)
    # just below the midpoint towards q's sign: rounds back to b, with nearly the largest error bf16 keeps
    x = (b * (1 + F32(2.0 ** -9 * (1 - 2.0 ** -10)) * np.sign(b) * sign)).astype(F32)
    assert np.array_equal(to_bf16(x), b)
    return q, x, b


@pytest.mark.parametrize("dpad", [384, 512, 768, 1024, 1536])
def test_bound_holds_in_the_kernels_lane_order(dpad):
    q, x, b = adversarial(dpad, 64, dpad)
    p_hat = chain(q, x)
    e_hat = chain(q, b)
    s_hat = chain(np.abs(q), np.abs(b))
    c = f32_up(screen_constant(dpad))
    babs = dpad * (float(np.abs(q).max()) * 2.0 ** -125 + 2.0 ** -124)
    bound = float(c) * s_hat.astype(np.float64) + babs
    gap = np.abs(p_hat.astype(np.float64) - e_hat.astype(np.float64))
    assert np.all(gap <= bound), (gap / bound).max()
    # adversarial: the errors add up coherently.  A value's rounding error is at most 2^-8 of it only at the bottom
    # of its binade (about 2^-9 of it on average), so coherent errors fill a bit less than half the band.
    assert (gap / bound).max() > 0.4
    # the screen's lower bound never exceeds the walk's distance
    B = np.array([f32_up(v) for v in bound], F32)
    L = rd_sub(rd_sub(np.full_like(e_hat, 1.0), e_hat), B)
    D = (F32(1.0) - p_hat).astype(F32)
    assert np.all(L <= D)


def test_constant_is_monotone_and_small():
    prev = 0.0
    for n in (384, 512, 768, 1024, 1536):
        c = screen_constant(n)
        assert c > prev and 2.0 ** -8 < c < 2.0 ** -8 * 1.1
        prev = c
