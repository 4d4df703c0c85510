"""bf16 graph search in the one-process-per-GPU shard exchange (ehb_exchange_search_ex_dev with EHB_BF16): the bf16
walk of each rank's shard, then the fp32 re-rank, which stores each query's top-k into every peer's receive buffer
and raises the slice flags; one kernel per rank waits for the peers' flags and merges.

Both "ranks" live in this process (ehb_exchange_attach_local), on two devices when the box has them and both on
device 0 otherwise.  Held exactly:
  * the fused bf16 step is ehb_merge_topk_dev of each shard's own ehb_index_search_ex_dev(EHB_BF16) output: labels,
    distance bits and counts, on both ranks; shard_counts_dev is each shard's own counts;
  * on tie-free integer inner-product data the bf16 step equals the fp32 step and the merge of the oracle's per-shard
    searches;
  * fp32-fused, bf16-fused and push-after brute-force steps interleave on one exchange (parity and epochs carry
    across precisions), at nq = 1, 4, 5 and at the exchange's capacity, with a tombstoned shard;
  * a bad precision or ef fails before the step starts, and the next step still completes on both ranks.
After every step no rank's exchange has timed out.

Two ranks on one GPU share its SMs, and a merge kernel of rank 0 waits on the GPU for rank 1's search, which is
queued after it.  A call that frees device memory waits for the whole device, so every test sizes the search
scratch (by running the references first) before its fused steps.
"""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest

from oracle import oracle as orc  # test infrastructure

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_LABEL = np.uint64(0xFFFFFFFFFFFFFFFF)
EHB_FP32, EHB_BF16, EHB_ERR_INVALID = 0, 1, 1


def _ehb():
    import embeddinghub_b200 as ehb
    return ehb


def _lib():
    from embeddinghub_b200._native import lib
    return lib()


def _check(rc):
    from embeddinghub_b200._native import check
    check(rc)


def _devices(n):
    import torch
    have = torch.cuda.device_count()
    return [i % have for i in range(n)]


def gauss(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)


class Pair:
    """Two shards of one index (global labels) and two attached exchanges, one per 'rank'."""

    def __init__(self, parts, d, metric, max_nq, max_k, build=True):
        import torch
        self.torch = torch
        self.devs = _devices(2)
        self.ixs, self.exs = [], []
        L = _lib()
        lo = 0
        for r, x in enumerate(parts):
            ix = _ehb().NativeIndex(d, metric=metric, capacity=len(x), device=self.devs[r])
            ix.add(x, np.arange(lo, lo + len(x), dtype=np.uint64))
            if build:
                ix.build()
            lo += len(x)
            self.ixs.append(ix)
            h = C.c_void_p()
            _check(L.ehb_exchange_create(self.devs[r], 2, r, max_nq, max_k, C.byref(h)))
            self.exs.append(h)
        _check(L.ehb_exchange_attach_local(self.exs[0], 1, self.exs[1]))
        _check(L.ehb_exchange_attach_local(self.exs[1], 0, self.exs[0]))
        self.streams = [torch.cuda.Stream(device=dv) for dv in self.devs]

    def close(self):
        for r in range(2):
            self.streams[r].synchronize()
        for h in self.exs:
            _lib().ehb_exchange_destroy(h)

    def dev(self, r):
        return f"cuda:{self.devs[r]}"

    def _out(self, r, nq, k):
        t = self.torch
        return (t.empty((nq, k), dtype=t.int64, device=self.dev(r)), t.empty((nq, k), dtype=t.float32, device=self.dev(r)),
                t.empty(nq, dtype=t.int32, device=self.dev(r)))

    def own(self, q, k, ef, precision):
        """Each shard's own graph search (labels, dists, counts) on host, then their merge by ehb_merge_topk_dev."""
        t = self.torch
        nq = len(q)
        per = []
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(q).to(self.dev(r))
            l, d, c = self._out(r, nq, k)
            s = self.streams[r]
            s.wait_stream(t.cuda.current_stream(self.devs[r]))
            self.ixs[r].search_dev(dq.data_ptr(), nq, k, ef, l.data_ptr(), d.data_ptr(), c.data_ptr(), s.cuda_stream,
                                   precision)
            s.synchronize()
            per.append((l.cpu().numpy(), d.cpu().numpy(), c.cpu().numpy()))
        return self.merge(per, k), per

    def own_brute(self, q, k):
        t = self.torch
        nq = len(q)
        per = []
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(q).to(self.dev(r))
            l, d, c = self._out(r, nq, k)
            self.streams[r].wait_stream(t.cuda.current_stream(self.devs[r]))
            self.ixs[r].search_bruteforce_dev(dq.data_ptr(), nq, k, EHB_FP32, l.data_ptr(), d.data_ptr(),
                                              c.data_ptr(), self.streams[r].cuda_stream)
            self.streams[r].synchronize()
            per.append((l.cpu().numpy(), d.cpu().numpy(), c.cpu().numpy()))
        return self.merge(per, k), per

    def merge(self, per, k):
        t = self.torch
        nq = per[0][0].shape[0]
        t.cuda.set_device(self.devs[0])
        gl = t.from_numpy(np.stack([p[0] for p in per])).to(self.dev(0))
        gd = t.from_numpy(np.stack([p[1] for p in per])).to(self.dev(0))
        ml, md, mc = self._out(0, nq, k)
        _check(_lib().ehb_merge_topk_dev(2, nq, k, C.c_void_p(gd.data_ptr()), C.c_void_p(gl.data_ptr()),
                                         C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                                         self.devs[0], None))
        t.cuda.synchronize(self.devs[0])
        return ml.cpu().numpy(), md.cpu().numpy(), mc.cpu().numpy()

    def fused(self, q, k, ef, precision):
        """One fused exchange step on both ranks (both queued before anyone synchronises): per rank the merged
        (labels, dists, counts) and the shard's own counts."""
        t = self.torch
        nq = len(q)
        res = []
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(q).to(self.dev(r))
            ml, md, mc = self._out(r, nq, k)
            sc = t.full((nq,), -1, dtype=t.int32, device=self.dev(r))
            self.streams[r].wait_stream(t.cuda.current_stream(self.devs[r]))
            _check(_lib().ehb_exchange_search_ex_dev(
                self.exs[r], self.ixs[r]._h, nq, C.c_void_p(dq.data_ptr()), k, ef, precision,
                C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                C.c_void_p(sc.data_ptr()), C.c_void_p(self.streams[r].cuda_stream)))
            res.append((ml, md, mc, sc, dq))
        return self._collect(res)

    def push_after_brute(self, q, k):
        t = self.torch
        nq = len(q)
        res = []
        L = _lib()
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(q).to(self.dev(r))
            sc = t.full((nq,), -1, dtype=t.int32, device=self.dev(r))
            self.streams[r].wait_stream(t.cuda.current_stream(self.devs[r]))
            lp, dp = C.c_void_p(), C.c_void_p()
            _check(L.ehb_exchange_begin(self.exs[r], nq, k, C.byref(lp), C.byref(dp)))
            self.ixs[r].search_bruteforce_dev(dq.data_ptr(), nq, k, EHB_FP32, lp.value, dp.value, sc.data_ptr(),
                                              self.streams[r].cuda_stream)
            res.append((*self._out(r, nq, k), sc, dq))
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            ml, md, mc = res[r][:3]
            _check(L.ehb_exchange_merge_dev(self.exs[r], C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                            C.c_void_p(mc.data_ptr()), C.c_void_p(self.streams[r].cuda_stream)))
        return self._collect(res)

    def _collect(self, res):
        out = []
        for r in range(2):
            self.streams[r].synchronize()
            ml, md, mc, sc, _ = res[r]
            out.append((ml.cpu().numpy().view(np.uint64), md.cpu().numpy(), mc.cpu().numpy(), sc.cpu().numpy()))
        self.assert_no_timeout()
        return out

    def assert_no_timeout(self):
        for r in range(2):
            v = C.c_uint32()
            _check(_lib().ehb_exchange_timed_out(self.exs[r], C.byref(v)))
            assert v.value == 0, r


def assert_equal_results(got, want, what):
    gl, gd, gc = got[:3]
    wl, wd, wc = want
    assert np.array_equal(np.asarray(gl).view(np.uint64), np.asarray(wl).view(np.uint64)), what
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), what
    assert np.array_equal(gc, wc), what


def assert_step(out, ref, per, what):
    """Both ranks hold the reference merge, and each rank's shard counts are its shard's own."""
    for r in range(2):
        assert_equal_results(out[r], ref, (what, r))
        assert np.array_equal(out[r][3], per[r][2]), (what, r)


# ---- 1. bitwise against each shard's own bf16 search, merged ----------------------------------------------------
KEFS = [(1, 64), (10, 64), (64, 64), (10, 128), (64, 128)]


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("d", [128, 768])
def test_fused_bf16_step_equals_merge_of_own_bf16_searches(d, metric):
    """d = 128: bf16 rows of 256 B (direct loads); d = 768: 1.5 KB (the bf16 TMA ring).  nq = 333: ragged slices."""
    n, nq = 6000, 333
    x, q = gauss(2 * n, d, 11 + d), gauss(nq, d, 12 + d)
    p = Pair([x[:n], x[n:]], d, metric, nq, 64)
    try:
        refs = {kef: p.own(q, kef[0], kef[1], EHB_BF16) for kef in sorted(KEFS, key=lambda t: -t[1])}
        for step in range(2):
            for k, ef in KEFS:
                ref, per = refs[(k, ef)]
                assert_step(p.fused(q, k, ef, EHB_BF16), ref, per, (step, k, ef))
                assert np.all(ref[2] == k)
    finally:
        p.close()


# ---- 2. exact against the oracle on tie-free data ---------------------------------------------------------------
def split_tiefree(n, d, nq, seed=7):
    """x_i = (B u_i, 256 floor((i+1)/256), (i+1) mod 256), q = (v, 1, 1): q.x_i = B (u_i.v) + i + 1, all distinct,
    every coordinate exact in bf16 and every partial sum an integer below 2^24 (DESIGN.md §2)."""
    B = 1 << (n + 1).bit_length()
    assert B * (d + 1) <= 1 << 24
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.int64)
    x[:, :d - 2] = B * rng.integers(-1, 2, (n, d - 2))
    x[:, d - 2] = 256 * (np.arange(1, n + 1) // 256)
    x[:, d - 1] = np.arange(1, n + 1) % 256
    q = np.ones((nq, d), np.int64)
    q[:, :d - 2] = rng.integers(-1, 2, (nq, d - 2))
    return x, q


@pytest.mark.parametrize("d", [64, 768])
def test_fused_bf16_step_equals_fp32_step_and_oracle(d):
    n, nq = 6000, 160
    x, q = split_tiefree(n, d, nq)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    half = n // 2
    p = Pair([xf[:half], xf[half:]], d, "ip", nq, 100)
    for ix in p.ixs:
        ix.set_search_width(1)                    # the fp32 walk in hnswlib's order (no team walk)
    try:
        oracles = []
        for r in range(2):
            o = orc.OracleHNSW(d, "ip", half)
            o.import_graph(p.ixs[r].export_graph())
            oracles.append(o)
        cases = [(10, 128), (100, 257), (10, 64)]
        for k, ef in cases:                       # size the scratch for the largest ef of either precision
            p.own(qf, k, ef, EHB_BF16)
            p.own(qf, k, ef, EHB_FP32)
        for k, ef in cases:
            per = []
            for o in oracles:
                ol, od, oc = o.search(qf, k, ef=ef, threads=8)
                per.append((ol.view(np.int64), od, oc.astype(np.int32)))
            want = p.merge(per, k)
            D = (1 - q @ x.T).astype(np.float32)
            assert np.array_equal(want[1].view(np.uint32),
                                  np.take_along_axis(D, want[0].view(np.uint64).astype(np.int64), 1).view(np.uint32))
            b = p.fused(qf, k, ef, EHB_BF16)
            f = p.fused(qf, k, ef, EHB_FP32)
            for r in range(2):
                assert_equal_results(b[r], want, ("bf16", k, ef, r))
                assert_equal_results(f[r], want, ("fp32", k, ef, r))
                assert np.array_equal(b[r][3], per[r][2]) and np.array_equal(f[r][3], per[r][2])
    finally:
        p.close()


# ---- 3. protocol: precisions, push-after steps, tiny batches, capacity, tombstones -----------------------------
def test_steps_alternate_precisions_and_push_after():
    d, n, k, ef, cap = 128, 5000, 10, 64, 333
    x, q = gauss(2 * n, d, 31), gauss(cap, d, 32)
    p = Pair([x[:n], x[n:]], d, "cosine", cap, k)
    try:
        st = p.ixs[0].stats()
        rng = np.random.default_rng(33)
        dead = np.union1d(rng.choice(n, n // 10, replace=False), [st["entry_point"]]).astype(np.uint64)
        p.ixs[0].remove(dead)                   # shard 0 walks with HASDEL; its labels are 0 .. n-1
        sizes = [cap, 1, 4, 5, cap]             # cap * k == the exchange's capacity; the largest batch first
        refs = {}
        for nq in sizes:
            qq = np.ascontiguousarray(q[:nq])
            refs[nq] = (p.own(qq, k, ef, EHB_FP32), p.own(qq, k, ef, EHB_BF16), p.own_brute(qq, k))
        for step, nq in enumerate(sizes):
            qq = np.ascontiguousarray(q[:nq])
            rf, rb, rx = refs[nq]
            for kind in ("fp32", "bf16", "brute", "bf16"):
                if kind == "brute":
                    out = p.push_after_brute(qq, k)
                    ref, per = rx
                else:
                    out = p.fused(qq, k, ef, EHB_BF16 if kind == "bf16" else EHB_FP32)
                    ref, per = rb if kind == "bf16" else rf
                assert_step(out, ref, per, (step, nq, kind))
                assert not np.isin(out[0][0], dead).any()
    finally:
        p.close()


# ---- 4. errors fail before the step starts -----------------------------------------------------------------------
def test_rejected_calls_leave_the_ranks_in_phase():
    import torch
    d, n, nq, k = 64, 3000, 40, 10
    x, q = gauss(2 * n, d, 41), gauss(nq, d, 42)
    p = Pair([x[:n], x[n:]], d, "l2", nq, k)
    L = _lib()
    try:
        ref, per = p.own(q, k, 64, EHB_BF16)
        p.own(q, k, 64, EHB_FP32)
        for prec, ef in [(7, 64), (-1, 64), (EHB_BF16, 513), (EHB_FP32, 600)]:
            for r in range(2):
                torch.cuda.set_device(p.devs[r])
                dq = torch.from_numpy(q).to(p.dev(r))
                ml, md, mc = p._out(r, nq, k)
                rc = L.ehb_exchange_search_ex_dev(p.exs[r], p.ixs[r]._h, nq, C.c_void_p(dq.data_ptr()), k, ef, prec,
                                                  C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                                  C.c_void_p(mc.data_ptr()), None,
                                                  C.c_void_p(p.streams[r].cuda_stream))
                assert rc == EHB_ERR_INVALID, (prec, ef, r)
            assert_step(p.fused(q, k, 64, EHB_BF16), ref, per, (prec, ef))
        # the fp32 entry point rejects ef > 512 before the step starts too
        for r in range(2):
            torch.cuda.set_device(p.devs[r])
            dq = torch.from_numpy(q).to(p.dev(r))
            ml, md, mc = p._out(r, nq, k)
            rc = L.ehb_exchange_search_dev(p.exs[r], p.ixs[r]._h, nq, C.c_void_p(dq.data_ptr()), k, 600,
                                           C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                           C.c_void_p(mc.data_ptr()), None, C.c_void_p(p.streams[r].cuda_stream))
            assert rc == EHB_ERR_INVALID
        assert_step(p.fused(q, k, 64, EHB_BF16), ref, per, "after fp32 rejection")
    finally:
        p.close()


# ---- 5. the first bf16 step creates the bf16 copy of the rows ------------------------------------------------------
def test_first_bf16_step_creates_the_shadow():
    d, n, nq, k, ef = 128, 4000, 333, 10, 64
    x, q = gauss(2 * n, d, 51), gauss(nq, d, 52)
    p = Pair([x[:n], x[n:]], d, "ip", nq, k)
    try:
        before = [ix.stats()["device_bytes"] for ix in p.ixs]
        out = p.fused(q, k, ef, EHB_BF16)
        after = [ix.stats()["device_bytes"] for ix in p.ixs]
        for r in range(2):                       # bf16 rows (2 B per padded element) + one norm per row
            assert after[r] - before[r] >= n * 2 * 128, (before, after)
        ref, per = p.own(q, k, ef, EHB_BF16)
        assert_step(out, ref, per, "first step")
        assert "ROW=bf16" in p.ixs[0].last_kernel_name()
    finally:
        p.close()


# ---- 6. the Python searcher passes the precision through ---------------------------------------------------------
def test_sharded_searcher_world1_bf16_equals_native_bf16():
    import torch
    from embeddinghub_b200._native import BF16
    from embeddinghub_b200.sharded import ShardedSearcher
    d, n, nq, k, ef = 128, 6000, 300, 10, 32
    x, q = gauss(n, d, 61), gauss(nq, d, 62)
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n)
    ix.add(x)
    ix.build()
    ix.set_search_width(1)
    want = ix.search(q, k, ef=ef, precision=BF16)
    s = ShardedSearcher(ix, 1, 0)
    dq = torch.from_numpy(q).cuda()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    ml, md, mc = s.search_dev(dq, k, ef, stream.cuda_stream, precision=BF16)
    stream.synchronize()
    assert "ROW=bf16" in ix.last_kernel_name()
    assert_equal_results((ml.cpu().numpy(), md.cpu().numpy(), mc.cpu().numpy()), want, "world 1")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _peer_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    import embeddinghub_b200 as ehb
    from embeddinghub_b200._native import BF16
    from embeddinghub_b200.sharded import ShardedSearcher, route_rows

    d, n, nq, k, ef = 128, 8000, 333, 10, 64
    x = np.random.default_rng(71).standard_normal((n, d), dtype=np.float32)
    q = np.random.default_rng(72).standard_normal((nq, d), dtype=np.float32)
    mv, ml = route_rows(x, np.arange(n, dtype=np.uint64), n, world, rank)
    ix = ehb.NativeIndex(d, metric="ip", capacity=len(mv), device=rank)
    ix.add(mv, ml)
    ix.build()
    dq = torch.from_numpy(q).cuda(rank)
    stream = torch.cuda.Stream(device=rank)
    res = {}
    for ex in ("peer", "nccl"):
        s = ShardedSearcher(ix, world, rank, exchange=ex)
        stream.wait_stream(torch.cuda.current_stream(rank))
        l, dd, c = s.search_dev(dq, k, ef, stream.cuda_stream, precision=BF16)
        stream.synchronize()
        res[ex] = (l.cpu().numpy(), dd.cpu().numpy(), c.cpu().numpy())
        s.close()
    (pl, pd, pc), (nl, nd, nc) = res["peer"], res["nccl"]
    ok = np.array_equal(pl, nl) and np.array_equal(pd.view(np.uint32), nd.view(np.uint32)) and np.array_equal(pc, nc)
    out.put((rank, ok))
    dist.barrier()
    dist.destroy_process_group()


def test_two_process_peer_exchange_bf16():
    """torchrun-style: one process per GPU, the peer (CUDA IPC) exchange's bf16 step equals the NCCL exchange's."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, port, out)) for r in range(2)]
    for pr in procs:
        pr.start()
    for pr in procs:
        pr.join(600)
    got = sorted(out.get(timeout=5) for _ in range(2))
    assert got == [(0, True), (1, True)]
    assert all(pr.exitcode == 0 for pr in procs)
