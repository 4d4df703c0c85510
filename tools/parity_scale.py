#!/usr/bin/env python
"""Recall parity at scale for the north-star shapes (SURVEY.md §8d parity gate: recall@k(GPU) >=
recall@k(oracle) at the same ef).  For each shape, on the prescribed iid-Gaussian data:
  * oracle-built graph, oracle walk                  (the reference's behaviour)
  * GPU-built graph (several wave fractions), GPU walk
  * GPU-built graph, oracle walk                     (isolates construction from the walk)
  * oracle-built graph, GPU walk                     (isolates the walk from construction)
Ground truth = the exact fp32 brute-force kernel.  One JSON line per shape -> stdout and
--out (default: parity_scale.jsonl in the temporary directory).  The oracle is used as the checker only.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import embeddinghub_b200 as ehb  # noqa: E402
from oracle import oracle as orc  # noqa: E402

SHAPES = {
    "c3": dict(d=768, k=10, ef=128, metric="ip"),
    "c5": dict(d=128, k=100, ef=256, metric="cosine"),
    "c2": dict(d=128, k=10, ef=64, metric="l2"),
}


def gen(n, d, seed):
    rng = np.random.default_rng(seed)
    out = np.empty((n, d), np.float32)
    for i in range(0, n, 1 << 20):
        m = min(1 << 20, n - i)
        out[i:i + m] = rng.standard_normal((m, d), dtype=np.float32)
    return out


def recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3,c5")
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--fracs", default="64,256,16")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "parity_scale.jsonl"))
    args = ap.parse_args()
    cores = len(os.sched_getaffinity(0))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    for name in args.shapes.split(","):
        sh = SHAPES[name]
        d, k, ef, metric = sh["d"], sh["k"], sh["ef"], sh["metric"]
        base, q = gen(args.n, d, 1234), gen(args.nq, d, 4321)
        res = {"shape": name, "n": args.n, "nq": args.nq, **sh, "cores": cores}
        # exact ground truth from the exact kernel
        gx = ehb.NativeIndex(d, metric=metric, capacity=args.n)
        gx.add(base)
        gt, _, _ = gx.search_bruteforce(q, k)
        # oracle-built graph
        t0 = time.time()
        o = orc.OracleHNSW(d, metric, args.n)
        o.add(base, threads=cores)
        res["oracle_build_s"] = time.time() - t0
        ol, od, _ = o.search(q, k, ef=ef, threads=cores)
        res["recall_oracle_graph_oracle_walk"] = recall(ol, gt)
        og = o.export_graph()
        gi = ehb.NativeIndex(d, metric=metric, capacity=args.n)
        gi.import_graph(og)
        gi.set_search_width(1)
        l1, d1, _ = gi.search(q, k, ef=ef)
        res["recall_oracle_graph_gpu_walk"] = recall(l1, gt)
        res["ids_equal_same_graph"] = float(np.mean(l1 == ol))
        m = l1 == ol
        res["max_rel_dist_err_same_graph"] = float(np.max(np.abs(d1[m] - od[m]) / np.maximum(np.abs(od[m]), 1e-6)))
        del gi
        for frac in [int(x) for x in args.fracs.split(",")]:
            ix = ehb.NativeIndex(d, metric=metric, capacity=args.n)
            ix.set_option("build_frac", frac)
            ix.add(base)
            t0 = time.time()
            ix.build()
            tb = time.time() - t0
            ix.set_search_width(1)
            gl, gd, _ = ix.search(q, k, ef=ef)
            r = {"build_s": tb, "recall_gpu_graph_gpu_walk": recall(gl, gt)}
            ix.set_search_width(0)
            gl2, _, _ = ix.search(q, k, ef=ef)
            r["recall_gpu_graph_gpu_walk_auto_width"] = recall(gl2, gt)
            if frac == 64:
                o2 = orc.OracleHNSW(d, metric, args.n)
                o2.import_graph(ix.export_graph())
                l2, _, _ = o2.search(q, k, ef=ef, threads=cores)
                r["recall_gpu_graph_oracle_walk"] = recall(l2, gt)
                del o2
            res[f"frac{frac}"] = r
            del ix
        line = json.dumps(res)
        print(line, flush=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
