"""Measures the GPU build at construction beams from 200 to 1024: the register form up to ef_construction 256 and the
wide form above (ehb_params.ef_construction up to 4096), and prints one JSON line per efc.

N rows of bench.py's seeded Gaussian stream (d = 768, inner product by default) are added to one index per efc and
built; the build time is the host clock around build(), which ends in a device synchronise.  Reported per efc: build
seconds, points per second, and recall@10 at ef 32 / 64 / 128 of the built graph against the exact fp32 scan, over
--nq of bench's seeded queries.  The 256 -> 257 pair is the same beam in the two forms.  The card name, power limit and
max SM clock are read in the same run.

  python tools/build_efc_probe.py [--n 1000000] [--dim 768] [--metric ip] [--efcs 200,256,257,512,1024] [--nq 2000]
                                  [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (the seeded data stream)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--metric", default="ip")
    ap.add_argument("--efcs", default="200,256,257,512,1024")
    ap.add_argument("--nq", type=int, default=2000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch

    import embeddinghub_b200 as ehb

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures the GPU and has no CPU fallback")
    name, power, clock = card()
    x = bench.gen(a.n, a.dim, bench.BASE_SEED)
    q = bench.gen(a.nq, a.dim, bench.QUERY_SEED)
    k, gt, lines = 10, None, []
    for efc in [int(v) for v in a.efcs.split(",")]:
        ix = ehb.NativeIndex(a.dim, metric=a.metric, capacity=a.n, ef_construction=efc)
        ix.add(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.build()
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        if gt is None:
            gt = ix.search_bruteforce(q, k)[0]   # exact fp32 scan: the same rows in every index
        rec = {ef: recall(ix.search(q, k, ef=ef)[0], gt) for ef in (32, 64, 128)}
        line = {"n": a.n, "dim": a.dim, "metric": a.metric, "ef_construction": efc,
                "form": "register" if efc <= 256 else "wide", "build_s": round(sec, 3),
                "points_per_s": round(a.n / sec), "recall10": {str(e): round(r, 4) for e, r in rec.items()},
                "queries": a.nq, "gpu": name, "power_limit": power, "max_sm_clock": clock}
        print(json.dumps(line), flush=True)
        lines.append(line)
        ix.close()
        del ix
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "build_efc_probe.jsonl"), "w") as f:
            f.writelines(json.dumps(v) + "\n" for v in lines)


if __name__ == "__main__":
    main()
