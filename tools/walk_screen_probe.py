"""Measures the fp32 walk's int8 screen (option "walk_screen") against the unscreened walk and prints one JSON line
per shape.

For each shape the index is built once; then searches with the screen off (0) and at its default (-1) alternate
in one process, with the L2 flushed before every timed call, and the best of --reps device-event times
(ehb_index_last_kernel_ms) is kept for each.  Reported per setting: time, queries/s, algorithmic bytes (ehb_stats)
and their share of the 3.35 TB/s data-sheet HBM bandwidth, the share of evaluations that read an fp32 row, the
share that were screened and the share of screened candidates that survived the screen (ehb_index_screen_stats), and whether labels, distance bits, counts and the hop /
evaluation / overflow counters are identical.  For shapes the screen applies to, --small-batches also times the
screen forced on (1) against off at batches of a few queries per SM, where the default leaves it off.  The card
name and power limit are read in the same run.

  python tools/walk_screen_probe.py [--shapes c3s,d384,d512,d1024,d1536,d2048,c5s,c2] [--reps 5]
                                    [--small-batches 132,264,528] [--out DIR]
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
    "d384": (1_000_000, 384, "ip", 10_000, 10, 128),
    "d512": (1_000_000, 512, "ip", 10_000, 10, 128),
    "d1024": (1_000_000, 1024, "ip", 10_000, 10, 128),
    "d1536": (1_000_000, 1536, "cosine", 10_000, 10, 128),
    "d2048": (1_000_000, 2048, "ip", 10_000, 10, 128),
    "c3": (10_000_000, 768, "ip", 10_000, 10, 128),
}
COUNTERS = ("hops_upper", "hops_base", "dist_evals", "visited_overflow")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def add_gaussian(ix, n, d, seed=1234, chunk=1 << 20):
    rng = np.random.default_rng(seed)
    for i in range(0, n, chunk):
        ix.add(rng.standard_normal((min(chunk, n - i), d), dtype=np.float32))


def same(a, b):
    (la, da, ca), (lb, db, cb) = a, b
    return bool(np.array_equal(la, lb) and np.array_equal(da.view(np.uint32), db.view(np.uint32))
                and np.array_equal(ca, cb))


def timed(ix, flush, q, k, ef, opts, reps):
    """Alternates the option values; returns {value: (best ms, result, stats)}."""
    best = {o: float("inf") for o in opts}
    res, st = {}, {}
    for o in opts:                                           # warm-up (the first screened search creates the int8 copy)
        ix.set_option("walk_screen", o)
        ix.search(q, k, ef=ef)
    for _ in range(reps):
        for o in opts:
            ix.set_option("walk_screen", o)
            flush.zero_()
            res[o] = ix.search(q, k, ef=ef)
            best[o] = min(best[o], ix.last_kernel_ms())
            st[o] = ix.stats()
    return {o: (best[o], res[o], st[o]) for o in opts}


def describe(ms, st, nq):
    ab = st["algorithmic_bytes"]
    ev = max(st["dist_evals"], 1)
    return {"ms": round(ms, 3), "qps": round(nq / ms * 1e3), "algorithmic_GB": round(ab / 1e9, 3),
            "hbm_share": round(ab / (ms * 1e-3) / HBM, 3), "fp32_read_share": round(st["fp32_row_reads"] / ev, 4),
            "screened_share": round(st["screened_evals"] / ev, 4),
            "survivor_share": round((st["fp32_row_reads"] - st["dist_evals"] + st["screened_evals"])
                                    / max(st["screened_evals"], 1), 4),
            "dist_evals_per_query": round(st["dist_evals"] / nq, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3s,d384,d512,d1024,d1536,d2048,c5s,c2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--small-batches", default="132,264,528")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    shapes = [s for s in a.shapes.split(",") if s]
    for s in shapes:
        if s not in SHAPES:
            raise SystemExit(f"unknown shape {s}: {sorted(SHAPES)}")
    small = [int(x) for x in a.small_batches.split(",") if x]
    import torch

    import embeddinghub_b200 as ehb

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
        r = timed(ix, flush, q, k, ef, (0, -1), a.reps)
        (m0, r0, s0), (m1, r1, s1) = r[0], r[-1]
        line = {"shape": s, "n": n, "dim": d, "metric": metric, "nq": nq, "k": k, "ef": ef, "gpu": name,
                "power_limit": power, "kernel": ix.last_kernel_name(),
                "off": describe(m0, s0, nq), "default": describe(m1, s1, nq), "speedup": round(m0 / m1, 3),
                "identical": same(r0, r1) and all(s0[c] == s1[c] for c in COUNTERS)}
        if s1["screened_evals"] and small:
            line["small_batches"] = []
            for b in small:
                rb = timed(ix, flush, q[:b], k, ef, (0, 1), a.reps)
                (b0, x0, t0), (b1, x1, t1) = rb[0], rb[1]
                line["small_batches"].append({"nq": b, "off_ms": round(b0, 3), "on_ms": round(b1, 3),
                                              "speedup": round(b0 / b1, 3),
                                              "identical": same(x0, x1) and all(t0[c] == t1[c] for c in COUNTERS)})
        print(json.dumps(line), flush=True)
        lines.append(line)
        ix.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "walk_screen_probe.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
