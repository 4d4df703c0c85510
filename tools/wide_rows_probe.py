"""Measures the graph walk over wide rows (dpad 3072 and 4096, the wide form) against the d = 2048 walk in the same
run, and the GPU build's throughput, and prints one JSON line per dimension.

Per d: N Gaussian rows (IP), built on the GPU (points/s over the whole build call, ended by a device synchronise),
then Q queries at k, ef walked over the fp32 rows and over the bf16 copy (then re-ranked in fp32), alternating, with
the L2 flushed before every timed call; the best of --reps device-event times (ehb_index_last_kernel_ms) is kept.
Reported per precision: time, queries/s, algorithmic bytes (ehb_stats) over the kernel time as a share of the
3.35 TB/s data-sheet HBM bandwidth, evaluations per query, and recall@k against the exact path over the first
--recall-queries queries.  The card name, power limit and max SM clock are read in the same run.

  python tools/wide_rows_probe.py [--dims 2048,3072,4096] [--n 1000000] [--nq 10000] [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def recall(a, b, k):
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="2048,3072,4096")
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--ef", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--recall-queries", type=int, default=1000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch

    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import BF16, FP32

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures the GPU and has no CPU fallback")
    name, power, clock = card()
    flush = torch.empty(256 << 18, dtype=torch.float32, device="cuda")   # 256 MB > the 50 MB L2
    lines = []
    for d in [int(s) for s in a.dims.split(",") if s]:
        ix = ehb.NativeIndex(d, metric="ip", capacity=a.n)
        rng = np.random.default_rng(1234)
        chunk = max(1, (1 << 30) // (4 * d))                               # 1 GB of host rows at a time
        for i in range(0, a.n, chunk):
            ix.add(rng.standard_normal((min(chunk, a.n - i), d), dtype=np.float32))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.build()
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        q = np.random.default_rng(4321).standard_normal((a.nq, d), dtype=np.float32)
        ix.set_search_width(1)
        for p in (FP32, BF16):                                             # warm-up (the bf16 copy is made here)
            ix.search(q, a.k, ef=a.ef, precision=p)
        best, res, st, kern = {FP32: float("inf"), BF16: float("inf")}, {}, {}, {}
        for _ in range(a.reps):
            for p in (FP32, BF16):
                flush.zero_()
                res[p] = ix.search(q, a.k, ef=a.ef, precision=p)
                best[p] = min(best[p], ix.last_kernel_ms())
                st[p] = ix.stats()
                kern[p] = ix.last_kernel_name()
        rq = min(a.recall_queries, a.nq)
        exact = ix.search_bruteforce(q[:rq], a.k)[0]
        line = {"dim": d, "n": a.n, "nq": a.nq, "k": a.k, "ef": a.ef, "metric": "ip", "gpu": name,
                "power_limit": power, "max_sm_clock": clock, "build_s": round(build_s, 2),
                "build_points_per_s": round(a.n / build_s)}
        for p, tag in ((FP32, "fp32"), (BF16, "bf16")):
            ab = st[p]["algorithmic_bytes"]
            ms = best[p]
            line[tag] = {"kernel": kern[p], "ms": round(ms, 3), "qps": round(a.nq / ms * 1e3),
                         "algorithmic_GB": round(ab / 1e9, 3), "hbm_share": round(ab / (ms * 1e-3) / HBM, 3),
                         "dist_evals_per_query": round(st[p]["dist_evals"] / a.nq, 1),
                         "recall_at_k": round(recall(res[p][0][:rq], exact, a.k), 4)}
        print(json.dumps(line), flush=True)
        lines.append(line)
        ix.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "wide_rows_probe.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
