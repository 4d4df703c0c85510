"""Measures the bf16 graph search (ehb_index_search_ex, EHB_BF16) against the fp32 walk and prints one JSON line
per shape.

For each shape the index is built once; then fp32 and bf16 searches alternate, with the L2 flushed before every
timed call.  Reported per precision: queries/s from device events around the walk (and, for bf16, the re-rank;
ehb_index_last_kernel_ms covers both), the walk and re-rank kernel times from one torch.profiler pass of their own,
algorithmic bytes (ehb_stats) and their share of the 3.35 TB/s data-sheet HBM bandwidth, recall@10 against the
exact path, the bf16 walk's id overlap with the fp32 walk, the kernel names, and the card name and power limit
read in the same run.  At c2 (Q = 1000) the fp32 search picks the team walk and bf16 does not.

  python tools/bf16_walk_probe.py [--shapes c2,c3s,c5s,c3] [--reps 5] [--truth-queries 1000] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
# name: (N, d, metric, Q, k, ef)
SHAPES = {
    "c2": (1_000_000, 128, "l2", 1000, 10, 64),
    "c3s": (1_000_000, 768, "ip", 10_000, 10, 128),
    "c5s": (1_000_000, 128, "cosine", 10_000, 100, 256),
    "c3": (10_000_000, 768, "ip", 10_000, 10, 128),
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def add_gaussian(ix, n, d, seed=1234, chunk=1 << 20):
    rng = np.random.default_rng(seed)
    for i in range(0, n, chunk):
        ix.add(rng.standard_normal((min(chunk, n - i), d), dtype=np.float32))


def overlap(a, b, k):
    return float(np.mean([len(set(x[:k].tolist()) & set(y[:k].tolist())) / k for x, y in zip(a, b)]))


def kernel_times(ix, q, k, ef, precision):
    """Device time per kernel name of one search, from torch.profiler (a pass of its own)."""
    from torch.profiler import ProfilerActivity, profile

    import torch
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        ix.search(q, k, ef=ef, precision=precision)
        torch.cuda.synchronize()
    out = {}
    for e in p.key_averages():
        if "hnsw_search" in e.key or "rerank_kernel" in e.key:
            key = "rerank" if "rerank_kernel" in e.key else "walk"
            out[key] = out.get(key, 0.0) + e.device_time_total / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,c3s,c5s,c3")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--truth-queries", type=int, default=1000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    shapes = [s for s in a.shapes.split(",") if s]
    for s in shapes:
        if s not in SHAPES:
            raise SystemExit(f"unknown shape {s}: {sorted(SHAPES)}")
    import torch

    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import BF16, FP32

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures the GPU and has no CPU fallback")
    name, power = card()
    flush = torch.empty(256 << 18, dtype=torch.float32, device="cuda")   # 256 MB > the 50 MB L2
    lines = []
    for s in shapes:
        n, d, metric, nq, k, ef = SHAPES[s]
        ix = ehb.NativeIndex(d, metric=metric, capacity=n)
        add_gaussian(ix, n, d)
        ix.build()
        q = np.random.default_rng(4321).standard_normal((nq, d), dtype=np.float32)
        nt = min(a.truth_queries, nq)
        truth = ix.search_bruteforce(q[:nt], k)[0]
        res, best, stats, kname = {}, {FP32: float("inf"), BF16: float("inf")}, {}, {}
        for p in (FP32, BF16):                               # warm-up (the first bf16 search creates the shadow)
            ix.search(q, k, ef=ef, precision=p)
        for _ in range(a.reps):                              # fp32 and bf16 alternate
            for p in (FP32, BF16):
                flush.zero_()
                res[p] = ix.search(q, k, ef=ef, precision=p)
                best[p] = min(best[p], ix.last_kernel_ms())
                stats[p] = ix.stats()
                kname[p] = ix.last_kernel_name()
        kt = {p: kernel_times(ix, q, k, ef, p) for p in (FP32, BF16)}
        line = {"shape": s, "n": n, "dim": d, "metric": metric, "nq": nq, "k": k, "ef": ef, "gpu": name,
                "power_limit": power}
        for p, tag in ((FP32, "fp32"), (BF16, "bf16")):
            ms = best[p]
            ab = stats[p]["algorithmic_bytes"]
            line[tag] = {"qps": round(nq / ms * 1e3), "ms": round(ms, 3), "kernel": kname[p],
                         "walk_ms_profiled": round(kt[p].get("walk", 0.0), 3),
                         "rerank_ms_profiled": round(kt[p].get("rerank", 0.0), 3),
                         "algorithmic_GB": round(ab / 1e9, 3), "hbm_share": round(ab / (ms * 1e-3) / HBM, 3),
                         "dist_evals_per_query": round(stats[p]["dist_evals"] / nq, 1),
                         f"recall@{k}": round(overlap(res[p][0][:nt], truth, k), 4)}
        line["bf16_overlap_with_fp32"] = round(overlap(res[BF16][0], res[FP32][0], k), 4)
        line["bf16_speedup"] = round(best[FP32] / best[BF16], 3)
        print(json.dumps(line), flush=True)
        lines.append(line)
        ix.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bf16_walk_probe.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
