"""The fp32 walk's int8 screen on data that stresses its bound, its copy of the rows, and what it reports.

Every walk case compares walk_screen = 1 with walk_screen = 0 on the same index and queries (check_same: ids,
distance bits, counts and the hop / evaluation / overflow counters).  The conversion kernel is checked against its
numpy replica (tests/test_walk_screen_int8_bound_cpu.py) through tests/cpp/libi8_probe.so.
"""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_walk_screen import check_same, gaussian, make_index, run
from test_walk_screen_int8_bound_cpu import to_i8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tests", "cpp", "libi8_probe.so")


def survivors(s):
    return s["fp32_row_reads"] - (s["dist_evals"] - s["screened_evals"])


@pytest.mark.gpu
def test_conversion_matches_the_numpy_replica():
    import torch

    lib = C.CDLL(PROBE)
    lib.probe_to_i8.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64]
    dpad = 768
    rng = np.random.default_rng(5)
    x = rng.standard_normal((64, dpad)).astype(np.float32)
    x[1] = 0
    x[2, :] = 0
    x[2, :3] = [1e-40, -2e-41, 3e-42]                    # subnormal scale
    x[3, 9] = np.inf
    x[4, 9] = np.nan
    x[5, :] = 1e-39
    x[5, 0] = 1.0                                         # subnormal elements, normal scale
    x[6, 17] = 1e4                                        # one dominant element
    x[7] = (np.round(x[7] * 50) / 50 + 0.5 / 50 * (1 - 2.0 ** -10)).astype(np.float32)
    dx = torch.from_numpy(x).cuda()
    codes = torch.empty((64, dpad), dtype=torch.int8, device="cuda")
    terms = torch.empty((64, 4), dtype=torch.float32, device="cuda")
    assert lib.probe_to_i8(dx.data_ptr(), dpad, codes.data_ptr(), terms.data_ptr(), 64) == 0
    torch.cuda.synchronize()
    c_ref, t_ref = to_i8(x)
    c_dev, t_dev = codes.cpu().numpy(), terms.cpu().numpy()
    assert np.array_equal(c_dev, c_ref)
    nan = np.isnan(t_ref)
    assert np.array_equal(np.isnan(t_dev), nan)
    assert np.array_equal(t_dev[:, :2][~nan[:, :2]], t_ref[:, :2][~nan[:, :2]])    # s and max |r| exactly
    # the norms are double sums in a different order: equal up to their last fp32 bit, and still upper bounds
    np.testing.assert_allclose(t_dev[:, 2:][~nan[:, 2:]], t_ref[:, 2:][~nan[:, 2:]], rtol=2.0 ** -22)


@pytest.mark.gpu
def test_int8_adversarial_band():
    """Near-duplicate rows whose residuals sit at the rounding extremes, signed like the queries' elements: many
    candidates land inside the bound's band, so both rejections and band survivors occur."""
    d, n = 768, 12_000
    rng = np.random.default_rng(71)
    sign = np.where(rng.standard_normal(d) > 0, 1.0, -1.0)
    s = 2.0 ** -5
    base = rng.integers(-126, 127, (n // 40, d)).astype(np.float64)
    x = (s * base + s * sign * (0.5 - 2.0 ** -10)).astype(np.float32)
    x[:, 0] = 127 * s                                      # the largest element fixes every row's scale at s
    x = np.repeat(x, 40, axis=0)
    x[:, 1:] += (rng.standard_normal((n, d - 1)) * 1e-4).astype(np.float32)
    q = (np.abs(rng.standard_normal((200, d))) * sign).astype(np.float32)
    ix = make_index(x.astype(np.float32), "ip")
    st = check_same(ix, q, 10, 128)
    assert 0 < survivors(st) < st["screened_evals"], st


@pytest.mark.gpu
def test_dominant_element_rows_all_survive():
    """One large element, the same in every row, makes s large (about 1.6 against unit-variance elements): the
    bound is far wider than the spread of the inner products, and every screened candidate survives."""
    d, n = 1024, 8000
    rng = np.random.default_rng(72)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[:, 0] = 200
    q = rng.standard_normal((200, d)).astype(np.float32)
    ix = make_index(x, "ip")
    st = check_same(ix, q, 10, 128, expect_screen=False)
    assert st["screened_evals"] > 0 and survivors(st) == st["screened_evals"], st


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_zero_and_subnormal_rows(metric):
    d, n = 512, 10_000
    rng = np.random.default_rng(73)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[::50] = 0                                            # all-zero rows
    x[1::50] = (rng.standard_normal((len(x[1::50]), d)) * 1e-40).astype(np.float32)   # subnormal rows
    x[2::50, 3:] = np.float32(1e-39)                       # subnormal elements next to normal ones
    q = rng.standard_normal((200, d)).astype(np.float32)
    ix = make_index(x, metric)
    check_same(ix, q, 10, 128)


@pytest.mark.gpu
def test_screen_copy_memory():
    """A screened fp32 search allocates the int8 copy (dpad + 16 bytes per row of capacity) and no bf16 shadow; a
    later bf16 search adds the bf16 shadow (2 dpad + 4 bytes per row)."""
    from embeddinghub_b200._native import BF16

    d, n = 768, 20_000
    x = gaussian(n, d, 74)
    q = gaussian(300, d, 75)
    ix = make_index(x, "ip")
    ix.search(q[:8], 10, ef=64)                            # unscreened: no copy
    b0 = ix.stats()["device_bytes"]
    cap = ix.stats()["capacity"]
    _, st, _ = run(ix, q, 10, 128, 1)
    assert st["screened_evals"] > 0
    assert st["device_bytes"] - b0 == cap * (d + 16)
    ix.search(q, 10, ef=128, precision=BF16)
    assert ix.stats()["device_bytes"] - b0 == cap * (d + 16) + cap * (2 * d + 4)
    check_same(ix, q, 10, 128)                             # both copies exist: the screen still runs on int8


@pytest.mark.gpu
def test_algorithmic_bytes_formula():
    d, n = 1024, 20_000
    ix = make_index(gaussian(n, d, 76), "ip")
    q = gaussian(300, d, 77)
    for screen in (1, 0):
        _, st, _ = run(ix, q, 10, 128, screen)
        M = st["M"]
        want = (st["hops_upper"] * 4 * M + st["hops_base"] * 8 * M + st["fp32_row_reads"] * 4 * d
                + st["screened_evals"] * (d + 16) + st["queries"] * 4 * d)
        assert st["algorithmic_bytes"] == want, (screen, st)
    ix.set_option("walk_screen", -1)
