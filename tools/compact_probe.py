"""Measures ehb_index_compact at the c3s / c5s shapes and prints one JSON line per case.

For each shape the index is built once and saved; each case loads it, deletes a fraction of the points and
reports: compaction seconds against a GPU rebuild of the surviving points, walk queries/s from device events
(L2 flushed before every timed call) before (tombstones) and after, recall@10 against the exact path before and
after, the walk kernel names, and the card name and power limit read in the same run.

  python tools/compact_probe.py [--shapes c3s,c5s] [--fracs 0.1,0.5] [--n N] [--nq Q] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"c3s": (768, "ip"), "c5s": (128, "cosine")}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def data(n, d, nq, seed=1234):
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.float32)
    for i in range(0, n, 1 << 18):
        x[i:i + (1 << 18)] = rng.standard_normal((min(1 << 18, n - i), d), dtype=np.float32)
    return x, np.random.default_rng(seed + 1).standard_normal((nq, d), dtype=np.float32)


def timed_walk(ix, q, k, ef, flush, reps=5):
    """Best of reps device-event times of the graph walk, L2 flushed before each call."""
    best, res = float("inf"), None
    for _ in range(reps):
        flush.zero_()
        res = ix.search(q, k, ef=ef)
        best = min(best, ix.last_kernel_ms())
    return best, res, ix.last_kernel_name()


def recall(l, truth, k):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(l, truth)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3s,c5s")
    ap.add_argument("--fracs", default="0.1,0.5")
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--ef", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    shapes = [s for s in a.shapes.split(",") if s]
    fracs = [float(f) for f in a.fracs.split(",") if f]
    for s in shapes:
        if s not in SHAPES:
            raise SystemExit(f"unknown shape {s}: {sorted(SHAPES)}")
    import torch
    import embeddinghub_b200 as ehb

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures the GPU and has no CPU fallback")
    name, power = card()
    flush = torch.empty(256 << 18, dtype=torch.float32, device="cuda")   # 256 MB > the 50 MB L2
    lines = []
    for s in shapes:
        d, metric = SHAPES[s]
        x, q = data(a.n, d, a.nq)
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, f"{s}.ehb")
            full = ehb.NativeIndex(d, metric=metric, capacity=a.n)
            full.add(x)
            full.build()
            full.save(path)
            full.close()
            for frac in fracs:
                ix = ehb.NativeIndex.load(path)
                dead = np.random.default_rng(int(frac * 1000)).choice(a.n, int(frac * a.n), replace=False)
                ix.remove(dead.astype(np.uint64))
                truth = ix.search_bruteforce(q, a.k)[0]
                ms0, (l0, _, _), k0 = timed_walk(ix, q, a.k, a.ef, flush)
                torch.cuda.synchronize()
                t = time.perf_counter()
                ix.compact()
                t_compact = time.perf_counter() - t
                ms1, (l1, _, _), k1 = timed_walk(ix, q, a.k, a.ef, flush)
                ix.close()
                live = np.setdiff1d(np.arange(a.n), dead)
                rb = ehb.NativeIndex(d, metric=metric, capacity=len(live))
                rb.add(x[live], live.astype(np.uint64))
                torch.cuda.synchronize()
                t = time.perf_counter()
                rb.build()
                t_rebuild = time.perf_counter() - t
                rb.close()
                line = {"shape": s, "n": a.n, "dim": d, "metric": metric, "deleted": frac, "nq": a.nq, "k": a.k,
                        "ef": a.ef, "compact_s": round(t_compact, 3), "rebuild_s": round(t_rebuild, 3),
                        "walk_qps_before": round(a.nq / ms0 * 1e3), "walk_qps_after": round(a.nq / ms1 * 1e3),
                        "recall_before": round(recall(l0, truth, a.k), 4),
                        "recall_after": round(recall(l1, truth, a.k), 4),
                        "kernel_before": k0, "kernel_after": k1, "gpu": name, "power_limit": power}
                print(json.dumps(line), flush=True)
                lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "compact_probe.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
