"""Measures key-mode search (ehb_index_search_by_label_ex) against the host composition it replaces, and prints one
JSON line per shape.

Per shape the index is built once; then, alternating, with the L2 flushed before every timed call and the best of
--reps kept:
  * by-label search of Q stored labels (k, ef) vs the host composition: get per label, search_ex(rows, k + 1),
    self-removal in Python (what EmbeddingHub.multi_nearest_neighbor(keys=...) does); wall time of the whole call
    and the device-event time of the walk (ehb_index_last_kernel_ms), results checked equal;
  * the per-key get loop vs get_batch for the same Q labels (wall);
  * the neighbour table (ehb_index_neighbor_table) of the index, or of a separate index of --table-points points:
    wall time and rows/s (one run; it is long).
The card name, power limit and SM clock are read in the same run.

  python tools/label_search_probe.py [--shapes c3s,c5s] [--reps 5] [--table-points 0 (= all)] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# name: (N, d, metric, Q, k, ef)
SHAPES = {
    "c3s": (1_000_000, 768, "ip", 10_000, 10, 128),
    "c5s": (1_000_000, 128, "cosine", 10_000, 100, 256),
    "tiny": (20_000, 64, "ip", 1000, 10, 64),
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power, sm, sm_max = (s.strip() for s in out.strip().splitlines()[0].split(","))
    return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def add_gaussian(ix, n, d, seed=1234, chunk=1 << 20):
    rng = np.random.default_rng(seed)
    for i in range(0, n, chunk):
        ix.add(rng.standard_normal((min(chunk, n - i), d), dtype=np.float32))


def host_key_mode(ix, labels, k, ef):
    """The host composition: one synchronous get per label, search at k + 1, self-removal in Python."""
    rows = np.stack([ix.get(int(l)) for l in labels])
    L, _, C = ix.search(rows, k + 1, ef)
    out = []
    for l, row, c in zip(labels, L, C):
        r = list(row[:c])
        if l in r:
            r.remove(l)
        elif len(r) > k:
            r = r[:-1]
        out.append(r[:k])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3s,c5s")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--table-points", type=int, default=0, help="table over an index of this many points (0: N)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch

    import embeddinghub_b200 as ehb

    flush = torch.empty(256 << 18, dtype=torch.float32, device="cuda")   # 256 MB > the 50 MB L2
    lines = []
    for name in a.shapes.split(","):
        N, d, metric, Q, k, ef = SHAPES[name]
        ix = ehb.NativeIndex(d, metric=metric, capacity=N)
        t0 = time.perf_counter()
        add_gaussian(ix, N, d)
        ix.build()
        build_s = time.perf_counter() - t0
        labels = np.random.default_rng(7).choice(N, Q, replace=False).astype(np.uint64)
        # warm every path once
        got = ix.search_by_label(labels, k, ef)
        ref = host_key_mode(ix, labels, k, ef)
        same = all(list(r[:c]) == h for r, c, h in zip(got[0], got[2], ref))
        ix.get_batch(labels)
        best = {"bylabel_wall": 1e9, "bylabel_walk": 1e9, "host_wall": 1e9, "host_walk": 1e9, "get_loop": 1e9,
                "get_batch": 1e9}
        for _ in range(a.reps):
            flush.zero_(); torch.cuda.synchronize()
            t = time.perf_counter(); ix.search_by_label(labels, k, ef); best["bylabel_wall"] = min(best["bylabel_wall"], time.perf_counter() - t)
            best["bylabel_walk"] = min(best["bylabel_walk"], ix.last_kernel_ms() / 1e3)
            flush.zero_(); torch.cuda.synchronize()
            t = time.perf_counter(); host_key_mode(ix, labels, k, ef); best["host_wall"] = min(best["host_wall"], time.perf_counter() - t)
            best["host_walk"] = min(best["host_walk"], ix.last_kernel_ms() / 1e3)
            t = time.perf_counter(); [ix.get(int(l)) for l in labels]; best["get_loop"] = min(best["get_loop"], time.perf_counter() - t)
            t = time.perf_counter(); ix.get_batch(labels); best["get_batch"] = min(best["get_batch"], time.perf_counter() - t)
        tp = a.table_points or N
        tix = ix
        if tp != N:
            tix = ehb.NativeIndex(d, metric=metric, capacity=tp)
            add_gaussian(tix, tp, d)
            tix.build()
        flush.zero_(); torch.cuda.synchronize()
        t = time.perf_counter()
        q, _, _, _ = tix.neighbor_table(k, ef)
        table_s = time.perf_counter() - t
        line = {"shape": name, "N": N, "d": d, "metric": metric, "Q": Q, "k": k, "ef": ef, "build_s": round(build_s, 2),
                "results_equal": bool(same),
                "bylabel_ms": round(best["bylabel_wall"] * 1e3, 3), "host_ms": round(best["host_wall"] * 1e3, 3),
                "bylabel_walk_ms": round(best["bylabel_walk"] * 1e3, 3),
                "host_walk_ms": round(best["host_walk"] * 1e3, 3),
                "speedup_wall": round(best["host_wall"] / best["bylabel_wall"], 2),
                "get_loop_ms": round(best["get_loop"] * 1e3, 3), "get_batch_ms": round(best["get_batch"] * 1e3, 3),
                "table_points": int(len(q)), "table_s": round(table_s, 3),
                "table_rows_per_s": round(len(q) / table_s, 1), **card()}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del ix, tix
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "label_search_probe.jsonl"), "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
