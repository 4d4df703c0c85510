"""Key mode in the shard exchange (ehb_exchange_search_by_label_ex_dev) against the host composition, two ranks.

One index of N Gaussian rows is split by label range into two shards, each with its own ehb_exchange (with a row region,
ehb_exchange_create_ex); the two ranks live in this process (ehb_exchange_attach_local), one per GPU when more than one
is visible, else both on GPU 0 (they then split its SMs, so the time is not that of a one-rank-per-GPU deployment).
Q stored labels drawn from both shards are the queries.  Two ways of answering them, each timed best of --steps with L2
flushed on every rank's device first:
  * by_label: one ehb_exchange_search_by_label_ex_dev step per rank, each rank on its own host thread; wall time from
    the first call to both ranks' streams being synchronised;
  * host composition: each owner's get_batch of the labels it holds, the rows assembled on the host and uploaded to
    every rank, the fused ehb_exchange_search_ex_dev step at k + 1, the results copied back and the self-removal rule
    applied on the host.
Also reported: the row kernel's device time (torch.profiler, in a separate profiled step), the bytes its push stores
(Q * d * 4 per destination), whether both ways agree output for output on both ranks, and the card's name and power
limit read in the same run.

    python tools/exchange_by_label_probe.py [--n 1000000] [--q 10000] [--steps 5] [--shapes c3s,c5s] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {  # name: (d, metric, k, ef)
    "c3s": (768, "ip", 10, 128),
    "c5s": (128, "cosine", 100, 256),
}
NO_LABEL = np.uint64(0xFFFFFFFFFFFFFFFF)


def card():
    import torch
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return {"name": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": out,
            "gpus": torch.cuda.device_count()}


def drop_self(self_labels, labels, dists, counts, k):
    """The reference's self-removal (server.cc:190-207) over [nq][k + 1] results, vectorised so the host composition
    is timed without a Python loop; tests/test_exchange_by_label_cpu.py holds it equal to tests/label_rule_model."""
    k1 = k + 1
    c = np.minimum(counts.astype(np.int64), k1)
    j = np.arange(k1)[None, :]
    hit = (labels[:, :k1] == self_labels[:, None]) & (j < c[:, None])
    has = hit.any(1)
    pos = np.where(has, hit.argmax(1), k1)
    i = np.arange(k)[None, :]
    src = np.minimum(i + (i >= pos[:, None]), k)
    cn = np.where(has, c - 1, np.minimum(c, k))
    live = i < cn[:, None]
    ol = np.where(live, np.take_along_axis(labels, src, 1), NO_LABEL)
    od = np.where(live, np.take_along_axis(dists, src, 1), np.float32(np.inf)).astype(np.float32)
    return ol, od, cn.astype(np.uint32)


def run_shape(name, n, nq, steps, seed=4321):
    import torch
    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import check, lib

    d, metric, k, ef = SHAPES[name]
    k1 = k + 1
    L = lib()
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d), dtype=np.float32)
    labels = rng.choice(n, nq, replace=False).astype(np.uint64)
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
        check(L.ehb_exchange_create_ex(devs[r], 2, r, nq, k1, d, C.byref(h)))
        exs.append(h)
    del x
    check(L.ehb_exchange_attach_local(exs[0], 1, exs[1]))
    check(L.ehb_exchange_attach_local(exs[1], 0, exs[0]))
    owner = (labels >= half).astype(np.int64)
    streams = [torch.cuda.Stream(device=dv) for dv in devs]
    dev = [f"cuda:{dv}" for dv in devs]
    outs = [(torch.empty((nq, k), dtype=torch.int64, device=dev[r]), torch.empty((nq, k), dtype=torch.float32,
             device=dev[r]), torch.empty(nq, dtype=torch.int32, device=dev[r])) for r in range(2)]
    outs1 = [(torch.empty((nq, k1), dtype=torch.int64, device=dev[r]), torch.empty((nq, k1), dtype=torch.float32,
              device=dev[r]), torch.empty(nq, dtype=torch.int32, device=dev[r])) for r in range(2)]
    dq = [torch.empty((nq, d), dtype=torch.float32, device=dev[r]) for r in range(2)]
    flush = [torch.empty(256 << 20, dtype=torch.uint8, device=dev[r]) for r in range(2)]

    def flush_all():
        for r in range(2):
            with torch.cuda.stream(streams[r]):
                flush[r].zero_()
        for r in range(2):
            streams[r].synchronize()

    def check_timeouts():
        for r in range(2):
            t = C.c_uint32()
            check(L.ehb_exchange_timed_out(exs[r], C.byref(t)))
            if t.value:
                raise RuntimeError(f"rank {r} timed out waiting for its peer")

    def host_composition():
        rows = np.empty((nq, d), np.float32)
        for r in range(2):
            m = owner == r
            rows[m] = ixs[r].get_batch(labels[m])
        for r in range(2):
            torch.cuda.set_device(devs[r])
            dq[r].copy_(torch.from_numpy(rows), non_blocking=False)
        for r in range(2):
            ml, md, mc = outs1[r]
            streams[r].wait_stream(torch.cuda.current_stream(devs[r]))
            check(L.ehb_exchange_search_ex_dev(exs[r], ixs[r]._h, nq, C.c_void_p(dq[r].data_ptr()), k1, ef, 0,
                                               C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                               C.c_void_p(mc.data_ptr()), None, C.c_void_p(streams[r].cuda_stream)))
        res = []
        for r in range(2):
            streams[r].synchronize()
            ml, md, mc = outs1[r]
            res.append(drop_self(labels, ml.cpu().numpy().view(np.uint64), md.cpu().numpy(), mc.cpu().numpy(), k))
        return res

    def by_label():
        rcs = [None, None]

        def one(r):
            torch.cuda.set_device(devs[r])
            ml, md, mc = outs[r]
            rcs[r] = L.ehb_exchange_search_by_label_ex_dev(exs[r], ixs[r]._h, nq, labels.ctypes.data_as(C.c_void_p), k,
                                                           ef, 0, C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                                           C.c_void_p(mc.data_ptr()), C.c_void_p(streams[r].cuda_stream))
            streams[r].synchronize()

        th = [threading.Thread(target=one, args=(r,)) for r in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for rc in rcs:
            check(rc)
        return [(outs[r][0].cpu().numpy().view(np.uint64), outs[r][1].cpu().numpy(),
                 outs[r][2].cpu().numpy().view(np.uint32)) for r in range(2)]

    def timed(fn):
        flush_all()
        t0 = time.perf_counter()
        out = fn()
        ms = (time.perf_counter() - t0) * 1e3
        check_timeouts()
        return ms, out

    # warm-up: scratch, screen copy, module loads (the host composition sizes every search slot first)
    hc = host_composition()
    bl = by_label()
    check_timeouts()
    agree = all(np.array_equal(bl[r][0], hc[r][0]) and np.array_equal(bl[r][1].view(np.uint32), hc[r][1].view(np.uint32))
                and np.array_equal(bl[r][2], hc[r][2]) for r in range(2))
    t_bl, t_hc = [], []
    for _ in range(steps):
        t_bl.append(timed(by_label)[0])
        t_hc.append(timed(host_composition)[0])
    # the row kernel's device time, from a profiled step of its own
    from torch.profiler import ProfilerActivity, profile
    flush_all()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        by_label()
    rows_us = [e.device_time_total for e in prof.key_averages() if "exchange_rows_kernel" in e.key]
    rows_calls = [e.count for e in prof.key_averages() if "exchange_rows_kernel" in e.key]
    for h in exs:
        L.ehb_exchange_destroy(h)
    return {"shape": name, "n": n, "per_shard": half, "q": nq, "d": d, "metric": metric, "k": k, "ef": ef,
            "devices": devs, "by_label_best_ms": round(min(t_bl), 3), "by_label_median_ms": round(float(np.median(t_bl)), 3),
            "host_composition_best_ms": round(min(t_hc), 3),
            "host_composition_median_ms": round(float(np.median(t_hc)), 3),
            "speedup_best": round(min(t_hc) / min(t_bl), 3),
            "row_kernel_ms_per_rank": round(rows_us[0] / 1e3 / max(rows_calls[0], 1), 3) if rows_us else None,
            "row_push_bytes_per_destination": nq * d * 4, "outputs_agree": bool(agree),
            "walk_kernel": ixs[0].last_kernel_name()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--q", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--shapes", default="c3s,c5s")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("exchange_by_label_probe: needs a CUDA device")
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
