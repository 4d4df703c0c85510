"""The shard exchange's exported buffer layout (csrc/exchange_layout.cuh) without a GPU: every offset, stride and size
of ehb::ExchangeLayout equals the formula the ranks agree on, over worlds, capacities and row widths (max_dim 0, and
widths that are not a multiple of 4 included)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exchange_layout_host_only():
    exe = os.path.join(ROOT, "tests", "cpp", "exchange_layout")
    assert os.path.exists(exe), "tests/cpp/exchange_layout is built by make"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "OK" in out.stdout, out.stdout + out.stderr
