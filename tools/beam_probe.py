"""Measures the wide-beam walk (ehb_index_search_beam, ef 513 .. 4096) against the register walk at ef = 512 and the
exact scans users fall back to today, and prints one JSON line per (N, k).

Per N: N Gaussian rows (d = 768, IP), built on the GPU; Q queries.  Per k (default 100 and 1000) and per
ef in --efs, the fp32 graph walk at beam max(ef, k) (the register walk when that is <= 512, else the wide-beam walk),
with the L2 flushed before every timed call; the best of --reps device-event times (ehb_index_last_kernel_ms) is kept.
Reported per walk: kernel, ms per batch, queries/s, hops and evaluations per query, queries whose visited table
overflowed, algorithmic bytes (ehb_stats: rows, adjacency rows, queries) and their share of the 3.35 TB/s data-sheet
HBM bandwidth, the visited-table traffic of the wide-beam walk listed separately (a model, not a measurement: one
32-byte sector per probed neighbour of every base-layer hop, plus clearing the 2 M0 beam + 64 entry table per query),
and recall@k against the exact fp32 scan over the first --recall-queries queries.  Then the fp32 and bf16 exact scans
of the whole batch at the same k.  The card name, power limit and max SM clock are read in the same run.

  python tools/beam_probe.py [--n 1000000,10000000] [--nq 10000] [--ks 100,1000] [--efs 512,513,1024,2048,4096]
                             [--reps 2] [--out DIR]
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
    ap.add_argument("--n", default="1000000,10000000")
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--ks", default="100,1000")
    ap.add_argument("--efs", default="512,513,1024,2048,4096")
    ap.add_argument("--reps", type=int, default=2)
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
    d, M0 = a.dim, 32
    lines = []
    for n in [int(s) for s in a.n.split(",") if s]:
        ix = ehb.NativeIndex(d, metric="ip", capacity=n)
        rng = np.random.default_rng(1234)
        chunk = max(1, (1 << 30) // (4 * d))
        for i in range(0, n, chunk):
            ix.add(rng.standard_normal((min(chunk, n - i), d), dtype=np.float32))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.build()
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        ix.set_option("combine", 0)
        q = np.random.default_rng(4321).standard_normal((a.nq, d), dtype=np.float32)
        rq = min(a.recall_queries, a.nq)
        for k in [int(s) for s in a.ks.split(",") if s]:
            line = {"n": n, "dim": d, "nq": a.nq, "k": k, "metric": "ip", "gpu": name, "power_limit": power,
                    "max_sm_clock": clock, "build_s": round(build_s, 1), "walks": []}
            exact = None
            scans = {}
            for p, tag in ((FP32, "fp32"), (BF16, "bf16")):
                ix.search_bruteforce(q[:rq], k, precision=p)                    # warm-up (bf16: the copy)
                flush.zero_()
                r = ix.search_bruteforce(q, k, precision=p)
                ms = ix.last_kernel_ms()
                if p == FP32:
                    exact = r[0][:rq]
                scans[tag] = {"ms": round(ms, 2), "qps": round(a.nq / ms * 1e3), "recall_at_k": None}
            scans["bf16"]["recall_at_k"] = round(recall(r[0][:rq], exact, k), 4)
            line["scans"] = scans
            for ef in [int(s) for s in a.efs.split(",") if s]:
                beam = max(ef, k)
                if ef < k and any(max(e, k) == beam for e in [int(s) for s in a.efs.split(",")] if e > ef):
                    continue                                                     # the same beam as a larger ef
                ix.search_beam(q[:256], k, ef=ef)                                # warm-up
                best, res, st = float("inf"), None, None
                for _ in range(a.reps):
                    flush.zero_()
                    res = ix.search_beam(q, k, ef=ef)
                    ms = ix.last_kernel_ms()
                    if ms < best:
                        best, st = ms, ix.stats()
                kern = ix.last_kernel_name()
                ab = st["algorithmic_bytes"]
                w = {"ef": ef, "beam": beam, "kernel": kern, "ms": round(best, 2), "qps": round(a.nq / best * 1e3),
                     "hops_per_query": round((st["hops_upper"] + st["hops_base"]) / a.nq, 1),
                     "evals_per_query": round(st["dist_evals"] / a.nq, 1),
                     "overflow_queries": st["visited_overflow"], "algorithmic_GB": round(ab / 1e9, 3),
                     "hbm_share": round(ab / (best * 1e-3) / HBM, 3),
                     "recall_at_k": round(recall(res[0][:rq], exact, k), 4)}
                if beam > 512:
                    vt = st["hops_base"] * M0 * 32 + a.nq * (2 * M0 * beam + 64) * 4
                    w["visited_table_GB_model"] = round(vt / 1e9, 3)
                line["walks"].append(w)
                print(json.dumps(w), flush=True)
            print(json.dumps(line), flush=True)
            lines.append(line)
        ix.close()
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "beam_probe.json"), "w") as f:
                json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
