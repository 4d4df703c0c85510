"""The fused wide-beam exchange step (ehb_exchange_search_beam_dev): walk, step and merge times.

Each base is split by label range into shards of --per-shard rows, one ehb_exchange per rank.  Without torchrun the
ranks live in this process (ehb_exchange_attach_local): one per GPU when enough are visible, else all on GPU 0.  On one
GPU the ranks split its SMs, so that figure checks that the step works and what it costs there; it is NOT the time of
a one-rank-per-GPU deployment and is labelled "mode": "one-gpu-functional".  Under torchrun (one process per GPU,
CUDA IPC between them) the mode is "ipc".

Per (k, ef) it reports, best and median over --steps timed steps after one warm-up step:
  * walk_ms: each rank's beam walk alone (ehb_index_last_kernel_ms of the step's search);
  * step_ms: device events around the whole fused call on each rank's stream (the larger over the ranks);
  * merge_ms: ehb_merge_topk_dev alone over the ranks' own ehb_index_search_beam_dev outputs, gathered on GPU 0;
and the card's name and power limit read in the same run.

    python tools/exchange_beam_probe.py [--per-shard 1000000] [--q 10000] [--steps 3] [--bases c5,d768] [--out FILE]
    torchrun --nproc-per-node 8 tools/exchange_beam_probe.py ...
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BASES = {"c5": (128, "cosine"), "d768": (768, "ip")}   # C5 rows; 768-d inner product
KEFS = [(100, 1024), (1000, 1024), (1000, 2048), (4096, 4096)]


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"name": torch.cuda.get_device_name(0), "power_limit": pl, "gpus": torch.cuda.device_count()}


def stats(ms):
    return {"best": round(min(ms), 3), "median": round(float(np.median(ms)), 3)}


def run_base(base, per_shard, nq, steps, world, rank, dist):
    import torch
    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import check, lib

    d, metric = BASES[base]
    L = lib()
    ipc = dist is not None
    mine = [rank] if ipc else list(range(world))
    devs = {r: (rank if ipc else (r if torch.cuda.device_count() >= world else 0)) for r in mine}
    q = np.random.default_rng(99).standard_normal((nq, d), dtype=np.float32)
    max_k = max(k for k, _ in KEFS)
    ixs, exs = {}, {}
    for r in mine:
        x = np.random.default_rng(1000 + r).standard_normal((per_shard, d), dtype=np.float32)
        ix = ehb.NativeIndex(d, metric=metric, capacity=per_shard, device=devs[r])
        ix.add(x, np.arange(r * per_shard, (r + 1) * per_shard, dtype=np.uint64))
        ix.build()
        ixs[r] = ix
        h = C.c_void_p()
        check(L.ehb_exchange_create(devs[r], world, r, nq, max_k, C.byref(h)))
        exs[r] = h
    if ipc:
        own = np.zeros(64, np.uint8)
        check(L.ehb_exchange_ipc_handle(exs[rank], own.ctypes.data_as(C.c_void_p)))
        send = torch.from_numpy(own).cuda(rank)
        recv = torch.empty(world * 64, dtype=torch.uint8, device=f"cuda:{rank}")
        dist.all_gather_into_tensor(recv, send)
        handles = np.ascontiguousarray(recv.cpu().numpy())
        check(L.ehb_exchange_open(exs[rank], handles.ctypes.data_as(C.c_void_p)))
        dist.barrier()
    else:
        for r in mine:
            for g in mine:
                if g != r:
                    check(L.ehb_exchange_attach_local(exs[r], g, exs[g]))
    streams = {r: torch.cuda.Stream(device=devs[r]) for r in mine}
    dq = {r: torch.from_numpy(q).to(f"cuda:{devs[r]}") for r in mine}
    out = []
    for k, ef in KEFS:
        outs = {r: (torch.empty((nq, k), dtype=torch.int64, device=f"cuda:{devs[r]}"),
                    torch.empty((nq, k), dtype=torch.float32, device=f"cuda:{devs[r]}"),
                    torch.empty(nq, dtype=torch.int32, device=f"cuda:{devs[r]}")) for r in mine}
        # each rank's own beam search (sizes its scratch before any step), gathered for the merge-alone timing
        own = {}
        for r in mine:
            torch.cuda.set_device(devs[r])
            l, dd, c = outs[r]
            ixs[r].search_beam_dev(dq[r].data_ptr(), nq, k, ef, l.data_ptr(), dd.data_ptr(), c.data_ptr(),
                                   streams[r].cuda_stream)
            streams[r].synchronize()
            own[r] = (l.clone(), dd.clone())
        merge_ms = []
        if ipc:
            gl = [torch.empty_like(own[rank][0]) for _ in range(world)]
            gd = [torch.empty_like(own[rank][1]) for _ in range(world)]
            dist.all_gather(gl, own[rank][0])
            dist.all_gather(gd, own[rank][1])
            mdev = rank
        else:
            gl = [own[r][0].to("cuda:0") for r in mine]
            gd = [own[r][1].to("cuda:0") for r in mine]
            mdev = 0
        torch.cuda.set_device(mdev)
        gl, gd = torch.stack(gl).contiguous(), torch.stack(gd).contiguous()
        ml, md = torch.empty((nq, k), dtype=torch.int64, device=f"cuda:{mdev}"), \
            torch.empty((nq, k), dtype=torch.float32, device=f"cuda:{mdev}")
        mc = torch.empty(nq, dtype=torch.int32, device=f"cuda:{mdev}")
        for i in range(steps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            check(L.ehb_merge_topk_dev(world, nq, k, C.c_void_p(gd.data_ptr()), C.c_void_p(gl.data_ptr()),
                                       C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                                       mdev, None))
            e1.record()
            torch.cuda.synchronize(mdev)
            if i:
                merge_ms.append(e0.elapsed_time(e1))
        step_ms, walk_ms = [], []
        for i in range(steps + 1):
            ev = {}
            if ipc:
                dist.barrier()
            for r in mine:
                torch.cuda.set_device(devs[r])
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(streams[r])
                l, dd, c = outs[r]
                check(L.ehb_exchange_search_beam_dev(exs[r], ixs[r]._h, nq, C.c_void_p(dq[r].data_ptr()), k, ef, 0,
                                                     C.c_void_p(dd.data_ptr()), C.c_void_p(l.data_ptr()),
                                                     C.c_void_p(c.data_ptr()), None,
                                                     C.c_void_p(streams[r].cuda_stream)))
                e1.record(streams[r])
                ev[r] = (e0, e1)
            for r in mine:
                streams[r].synchronize()
                t = C.c_uint32()
                check(L.ehb_exchange_timed_out(exs[r], C.byref(t)))
                if t.value:
                    raise RuntimeError(f"rank {r} timed out waiting for its peers")
            if i:
                step_ms.append(max(e0.elapsed_time(e1) for e0, e1 in ev.values()))
                walk_ms.append(max(ixs[r].last_kernel_ms() for r in mine))
        same = all(torch.equal(ml, outs[r][0].to(f"cuda:{mdev}")) for r in mine)
        out.append({"k": k, "ef": ef, "walk_ms": stats(walk_ms), "step_ms": stats(step_ms),
                    "merge_ms": stats(merge_ms), "merge_share_of_step": round(min(merge_ms) / min(step_ms), 4),
                    "step_equals_merge_of_own": bool(same), "walk_kernel": ixs[mine[0]].last_kernel_name()})
        del outs, own, gl, gd
    for h in exs.values():
        L.ehb_exchange_destroy(h)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-shard", type=int, default=1_000_000)
    ap.add_argument("--q", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--world", type=int, default=2, help="ranks in one process (ignored under torchrun)")
    ap.add_argument("--bases", default="c5,d768")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("exchange_beam_probe: needs a CUDA device")
    dist, world, rank = None, a.world, 0
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        import torch.distributed as dist
        rank = int(os.environ["RANK"])
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl")
        world = dist.get_world_size()
    mode = "ipc" if dist is not None else ("one-process-multi-gpu" if torch.cuda.device_count() >= world
                                           else "one-gpu-functional")
    rep = {"card": card(), "mode": mode, "world": world, "per_shard": a.per_shard, "q": a.q, "results": []}
    for base in a.bases.split(","):
        d, metric = BASES[base]
        for r in run_base(base, a.per_shard, a.q, a.steps, world, rank, dist):
            r = {"base": base, "d": d, "metric": metric, **r}
            if rank == 0:
                print(json.dumps(r), flush=True)
            rep["results"].append(r)
    rep["card_after"] = card()
    if rank == 0:
        print(json.dumps({"card": rep["card"], "mode": mode}))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(rep, f, indent=1)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
