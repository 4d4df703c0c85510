"""The int8 screen's survivors are read straight into registers, in batches whose size depends on the row length
(eight rows at dpad 384 down to two at dpad 1536), not through the TMA ring that unscreened hops use.  Their fp32
distances must keep the bits of the ring path: screen on vs off must give the same ids, distance bits, counts and
walk counters at both ends of the batch sizes for every result-set width, and with a visited table so small that it
overflows.
"""
import numpy as np
import pytest

from test_gpu_walk_screen import check_same, gaussian, make_index


@pytest.mark.gpu
@pytest.mark.parametrize("d", [300, 1536])            # dpad 384 (8 rows per batch) and 1536 (2 rows per batch)
@pytest.mark.parametrize("ef", [40, 128, 256, 512])   # KPL 2, 4, 8, 16
def test_batch_sizes_at_every_kpl(d, ef):
    x = gaussian(20_000, d, 41)
    q = gaussian(200, d, 42)
    ix = make_index(x, "ip")
    check_same(ix, q, 10, ef)


@pytest.mark.gpu
def test_overflowing_visited_table():
    x = gaussian(20_000, 768, 51)
    q = gaussian(200, 768, 52)
    ix = make_index(x, "cosine")
    ix.set_tuning(hash_bits=8)
    s = check_same(ix, q, 10, 128)
    assert s["visited_overflow"] > 0
