"""The fp32 walk's bf16 screen (option "walk_screen"): once the result set is full, a hop's candidates are evaluated
on the bf16 copy of their rows with a rigorous error bound first, and only those that could still be admitted are
read in fp32.  The screen must not change anything the walk returns or counts: every test compares walk_screen = 1
with walk_screen = 0 on the same index and queries, for ids, distance bits, counts and the hop / evaluation /
overflow counters, and checks the screen's own counters (screened evaluations, fp32 row reads).
"""
import numpy as np
import pytest

DIMS = [300, 512, 768, 1024, 1536]   # one per screened dpad class (384 ... 1536)
COUNTERS = ("hops_upper", "hops_base", "dist_evals", "visited_overflow")


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gaussian(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)


def gmm(n, d, seed, centres=64):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, d), dtype=np.float32) * 3
    return (c[rng.integers(0, centres, n)] + rng.standard_normal((n, d), dtype=np.float32)).astype(np.float32)


def make_index(x, metric, capacity=None):
    ix = _ehb().NativeIndex(x.shape[1], metric=metric, capacity=capacity or len(x))
    ix.add(x)
    ix.build()
    return ix


def run(ix, q, k, ef, screen):
    ix.set_option("walk_screen", screen)
    res = ix.search(q, k, ef=ef)
    return res, ix.stats(), ix.last_kernel_name()


def check_same(ix, q, k, ef, expect_screen=True):
    """Screen on vs off: identical results and walk counters; returns the screened run's stats."""
    (l0, d0, c0), s0, n0 = run(ix, q, k, ef, 0)
    (l1, d1, c1), s1, n1 = run(ix, q, k, ef, 1)
    ix.set_option("walk_screen", -1)
    assert n0 == n1
    assert np.array_equal(l0, l1)
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    assert np.array_equal(c0, c1)
    for c in COUNTERS:
        assert s0[c] == s1[c], (c, s0[c], s1[c])
    assert s0["screened_evals"] == 0 and s0["fp32_row_reads"] == s0["dist_evals"]
    ev, sc, fr = s1["dist_evals"], s1["screened_evals"], s1["fp32_row_reads"]
    assert 0 <= sc <= ev and fr <= ev
    assert ev - sc <= fr  # every unscreened evaluation reads its fp32 row; survivors add to them
    if expect_screen:
        assert sc > 0 and fr < ev, s1
        # the screen's bytes replace fp32 bytes: fp32_rows * 4d + screened * 2d
        assert s1["algorithmic_bytes"] < s0["algorithmic_bytes"]
    return s1


@pytest.mark.gpu
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_every_screened_dpad_class(d, metric):
    x = gaussian(20_000, d, 11)
    q = gaussian(300, d, 12)
    ix = make_index(x, metric)
    check_same(ix, q, 10, 128)


@pytest.mark.gpu
@pytest.mark.parametrize("ef", [40, 128, 256, 512])   # KPL 2, 4, 8, 16
@pytest.mark.parametrize("deleted", [False, True])
def test_every_kpl_with_and_without_tombstones(ef, deleted):
    d = 768
    x = gaussian(20_000, d, 21)
    q = gaussian(200, d, 22)
    ix = make_index(x, "ip")
    if deleted:
        ix.remove(np.arange(0, len(x), 7, dtype=np.uint64))
    _, _, name = run(ix, q, 10, ef, 1)
    assert ("HASDEL=1" in name) == deleted
    check_same(ix, q, 10, ef)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_gmm_data(metric):
    x = gmm(30_000, 1024, 31)
    q = gmm(300, 1024, 32)
    ix = make_index(x, metric)
    check_same(ix, q, 10, 128)


@pytest.mark.gpu
def test_adversarial_band():
    """Rows just below the bf16 rounding midpoints, errors aligned with the query's signs, and near-duplicate rows:
    many candidates land inside the bound's band, so both rejections and band survivors occur."""
    d, n = 768, 12_000
    rng = np.random.default_rng(41)
    b = rng.standard_normal((n // 40, d)).astype(np.float32)
    b = (b.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)            # exact bf16 values
    sign = np.where(rng.standard_normal(d) > 0, 1.0, -1.0).astype(np.float32)
    # x = b * (1 + 2^-9 (1 - 2^-12)) towards +sign: rounds back to b, the largest error bf16 keeps
    x = b * (1 + np.float32(2.0 ** -9 * (1 - 2.0 ** -12)) * np.sign(b) * sign)
    x = np.repeat(x, 40, axis=0) + rng.standard_normal((n, d)).astype(np.float32) * np.float32(1e-3)
    x = x.astype(np.float32)
    q = (np.abs(rng.standard_normal((200, d))) * sign).astype(np.float32)
    ix = make_index(x, "ip")
    s = check_same(ix, q, 10, 128)
    survivors = s["fp32_row_reads"] - (s["dist_evals"] - s["screened_evals"])
    assert 0 < survivors < s["screened_evals"], s


@pytest.mark.gpu
def test_default_rule():
    d = 768
    x = gaussian(20_000, d, 51)
    ix = make_index(x, "ip")
    big = gaussian(4 * sms(), d, 52)
    ix.search(big, 10, ef=128)
    assert ix.stats()["screened_evals"] > 0          # a batch of 4 queries per SM screens by default
    ix.search(big[:16], 10, ef=128)
    assert ix.stats()["screened_evals"] == 0         # a small batch does not
    ix.set_option("walk_screen", 0)
    ix.search(big, 10, ef=128)
    assert ix.stats()["screened_evals"] == 0
    lx = make_index(gaussian(5000, d, 53), "l2")     # L2 is never screened
    lx.set_option("walk_screen", 1)
    lx.search(big, 10, ef=128)
    assert lx.stats()["screened_evals"] == 0
    sx = make_index(gaussian(5000, 256, 54), "ip")   # nor are rows loaded directly (dpad <= 256)
    sx.set_option("walk_screen", 1)
    sx.search(gaussian(600, 256, 55), 10, ef=128)
    assert sx.stats()["screened_evals"] == 0


@pytest.mark.gpu
def test_after_add_remove_compact_save_load(tmp_path):
    d = 1024
    x = gaussian(8000, d, 61)
    q = gaussian(200, d, 62)
    ix = _ehb().NativeIndex(d, metric="cosine", capacity=2000)
    ix.add(x[:2000])
    ix.build()
    check_same(ix, q, 10, 128)                       # the shadow exists from here on
    before = ix.stats()["device_bytes"]
    ix.add(x[2000:])                                 # capacity 2000 -> 8192: the shadow grows with the rows
    assert ix.stats()["device_bytes"] > before
    check_same(ix, q, 10, 128)
    ix.remove(np.arange(0, 8000, 5, dtype=np.uint64))
    check_same(ix, q, 10, 128)
    ix.compact()
    check_same(ix, q, 10, 128)
    p = str(tmp_path / "ix.ehb")
    ix.save(p)
    lx = _ehb().NativeIndex.load(p)
    check_same(lx, q, 10, 128)
