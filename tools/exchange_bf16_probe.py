"""fp32 against bf16 graph search in the fused shard exchange (ehb_exchange_search_ex_dev), two ranks.

One index of N Gaussian rows is split by label range into two shards, each with its own ehb_exchange; the two ranks
live in this process (ehb_exchange_attach_local), one per GPU when more than one is visible, else both on GPU 0 (they
then split its SMs, so the time is not that of a one-rank-per-GPU deployment).  Steps alternate fp32 and bf16, with L2
flushed on every rank's device before each timed step.  A step's time is the larger of the two ranks' device-event
spans (search + exchange + merge on that rank's stream); the best and the median over the timed steps are reported,
with recall@k of both precisions against the exact path and the card's name and power limit read in the same run.

    python tools/exchange_bf16_probe.py [--n 1000000] [--q 10000] [--steps 10] [--shapes c3s,c5s] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {  # name: (d, metric, k, ef)
    "c3s": (768, "ip", 10, 128),
    "c5s": (128, "cosine", 100, 256),
}


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"name": torch.cuda.get_device_name(0), "power_limit": pl, "gpus": torch.cuda.device_count()}


def recall(a, b):
    k = b.shape[1]
    return float(np.mean([len(set(x.tolist()) & set(y.tolist())) / k for x, y in zip(a, b)]))


def run_shape(name, n, nq, steps, seed=1234):
    import torch
    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import check, lib

    d, metric, k, ef = SHAPES[name]
    L = lib()
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    devs = [0, 1] if torch.cuda.device_count() > 1 else [0, 0]
    half = n // 2
    parts = [(0, half), (half, n)]
    ixs, exs = [], []
    for r, (lo, hi) in enumerate(parts):
        ix = ehb.NativeIndex(d, metric=metric, capacity=hi - lo, device=devs[r])
        ix.add(x[lo:hi], np.arange(lo, hi, dtype=np.uint64))
        ix.build()
        ixs.append(ix)
        h = C.c_void_p()
        check(L.ehb_exchange_create(devs[r], 2, r, nq, k, C.byref(h)))
        exs.append(h)
    check(L.ehb_exchange_attach_local(exs[0], 1, exs[1]))
    check(L.ehb_exchange_attach_local(exs[1], 0, exs[0]))
    # the exact path: each shard's exact top-k, merged on the host
    el, ed = [], []
    for ix in ixs:
        lab, dist, _ = ix.search_bruteforce(q, k)
        el.append(lab)
        ed.append(dist)
    cl, cd = np.concatenate(el, 1), np.concatenate(ed, 1)
    exact = np.take_along_axis(cl, np.argsort(cd, axis=1, kind="stable")[:, :k], 1)

    streams = [torch.cuda.Stream(device=dv) for dv in devs]
    dq = [torch.from_numpy(q).to(f"cuda:{dv}") for dv in devs]
    outs = [(torch.empty((nq, k), dtype=torch.int64, device=f"cuda:{dv}"),
             torch.empty((nq, k), dtype=torch.float32, device=f"cuda:{dv}"),
             torch.empty(nq, dtype=torch.int32, device=f"cuda:{dv}")) for dv in devs]
    flush = [torch.empty(256 << 20, dtype=torch.uint8, device=f"cuda:{dv}") for dv in devs]
    for dv in set(devs):
        torch.cuda.synchronize(dv)

    def step(precision):
        ev = []
        for r in range(2):
            torch.cuda.set_device(devs[r])
            with torch.cuda.stream(streams[r]):
                flush[r].zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(streams[r])
            ml, md, mc = outs[r]
            check(L.ehb_exchange_search_ex_dev(exs[r], ixs[r]._h, nq, C.c_void_p(dq[r].data_ptr()), k, ef, precision,
                                               C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                               C.c_void_p(mc.data_ptr()), None, C.c_void_p(streams[r].cuda_stream)))
            e1.record(streams[r])
            ev.append((e0, e1))
        for r in range(2):
            streams[r].synchronize()
        for r in range(2):
            t = C.c_uint32()
            check(L.ehb_exchange_timed_out(exs[r], C.byref(t)))
            if t.value:
                raise RuntimeError(f"rank {r} timed out waiting for its peer")
        return max(e0.elapsed_time(e1) for e0, e1 in ev)

    res = {}
    for precision, pname in ((0, "fp32"), (1, "bf16")):  # warm-up: shadow / screen copy, scratch, module loads
        step(precision)
        step(precision)
        res[pname] = {"ms": [],
                      "recall": recall(outs[0][0].cpu().numpy().view(np.uint64), exact),
                      "ranks_agree": bool(np.array_equal(outs[0][0].cpu().numpy(), outs[1][0].cpu().numpy())),
                      "walk_kernel": ixs[0].last_kernel_name()}
    for _ in range(steps):
        for precision, pname in ((0, "fp32"), (1, "bf16")):
            res[pname]["ms"].append(step(precision))
    for pname in res:
        ms = res[pname].pop("ms")
        res[pname]["best_ms"] = round(min(ms), 3)
        res[pname]["median_ms"] = round(float(np.median(ms)), 3)
        res[pname]["recall"] = round(res[pname]["recall"], 4)
    res["bf16_speedup_best"] = round(res["fp32"]["best_ms"] / res["bf16"]["best_ms"], 3)
    for h in exs:
        L.ehb_exchange_destroy(h)
    return {"shape": name, "n": n, "per_shard": half, "q": nq, "d": d, "metric": metric, "k": k, "ef": ef,
            "devices": devs, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--q", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--shapes", default="c3s,c5s")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("exchange_bf16_probe: needs a CUDA device")
    rep = {"card": card(), "results": []}
    for name in a.shapes.split(","):
        r = run_shape(name, a.n, a.q, a.steps)
        print(json.dumps(r), flush=True)
        rep["results"].append(r)
    rep["card_after"] = card()
    print(json.dumps(rep["card"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
