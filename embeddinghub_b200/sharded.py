"""Range-sharded multi-GPU search (SURVEY.md §8e): one process per GPU, base vectors partitioned
by contiguous label range, every rank owns an independent graph over its range, every rank
searches all queries, ONE all-gather of the per-shard top-k, then the merge kernel
(ehb_merge_topk_dev).  There is no collective on the write path: inserts route by label.

torch.distributed is only the plumbing (process group + the all-gather over NCCL/NVLink).
"""
import ctypes as C

import numpy as np

from ._native import check, lib


def shard_bounds(n_total, world):
    """Contiguous label ranges [lo, hi) per rank: rank g owns [g*N/G, (g+1)*N/G)."""
    return [(n_total * g) // world for g in range(world + 1)]


def owner_of(labels, n_total, world):
    """Rank that owns each label (vectorised)."""
    b = np.asarray(shard_bounds(n_total, world)[1:], dtype=np.uint64)
    return np.searchsorted(b, np.asarray(labels, dtype=np.uint64), side="right").astype(np.int64)


def route_rows(vecs, labels, n_total, world, rank):
    """Rows of an insert batch that belong to this rank (no communication needed)."""
    mine = owner_of(labels, n_total, world) == rank
    return np.asarray(vecs)[mine], np.asarray(labels)[mine]


def gather_topk(local_labels, local_dists, world, group=None):
    """The single exchange step: all ranks contribute [nq, k] (int64-viewed u64 labels, f32
    distances) and receive [world, nq, k] of each.  Labels and distances travel in ONE all-gather
    (packed per rank as [labels bytes | distance bytes]).  Works on CUDA tensors (NCCL) and CPU
    tensors (gloo)."""
    import torch
    import torch.distributed as dist

    nq, k = local_labels.shape
    if world == 1:
        return local_labels.unsqueeze(0), local_dists.unsqueeze(0)
    nl, nd = nq * k * 8, nq * k * 4
    send = torch.empty(nl + nd, dtype=torch.uint8, device=local_labels.device)
    send[:nl].view(torch.int64).copy_(local_labels.contiguous().view(-1))
    send[nl:].view(torch.float32).copy_(local_dists.contiguous().view(-1))
    recv = torch.empty((world, nl + nd), dtype=torch.uint8, device=local_labels.device)
    dist.all_gather_into_tensor(recv.view(-1), send, group=group)
    gl = recv[:, :nl].contiguous().view(torch.int64).view(world, nq, k)
    gd = recv[:, nl:].contiguous().view(torch.float32).view(world, nq, k)
    return gl, gd


class ShardedSearcher:
    """Search over a range-sharded index, one process per GPU.  `index` is this rank's NativeIndex (global
    labels).  exchange="peer" (default on GPUs): the library's peer-memory exchange (ehb_exchange_*: CUDA IPC
    mappings, one push + flag + merge kernel per step, no collective); exchange="nccl": one
    all_gather_into_tensor of the packed per-shard top-k + the merge kernel (kept as the comparison baseline
    and for process groups without peer access)."""

    def __init__(self, index, world, device, group=None, exchange="peer"):
        import torch

        self.ix, self.world, self.device, self.group = index, world, device, group
        self._torch = torch
        self._buf = {}
        self.exchange = exchange if world > 1 else "none"
        self._ex, self._ex_cap = None, (0, 0, 0)

    def close(self):
        if self._ex is not None:
            lib().ehb_exchange_destroy(self._ex)
            self._ex = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ensure_exchange(self, nq, k, dim=0):
        """(Re)creates the exchange when (nq, k) outgrow it, or when a key-mode step needs room for rows of `dim`
        floats that it lacks.  Collective: every rank takes the same decision because every rank searches the same
        batch.  The 64-byte IPC handles travel in one all_gather."""
        import torch.distributed as dist

        t = self._torch
        if self._ex is not None and nq <= self._ex_cap[0] and k <= self._ex_cap[1] and dim <= self._ex_cap[2]:
            return
        t.cuda.synchronize()
        if self._ex is not None:
            dist.barrier(group=self.group)   # no peer may still be storing into the buffer that is about to go
        self.close()
        cap = (max(nq, self._ex_cap[0]), max(k, self._ex_cap[1]), max(dim, self._ex_cap[2]))
        rank = dist.get_rank(self.group)
        h = C.c_void_p()
        check(lib().ehb_exchange_create_ex(self.device, self.world, rank, cap[0], cap[1], cap[2], C.byref(h)))
        mine = np.zeros(64, np.uint8)
        check(lib().ehb_exchange_ipc_handle(h, mine.ctypes.data_as(C.c_void_p)))
        dev = t.device("cuda", self.device)
        send = t.from_numpy(mine).to(dev)
        recv = t.empty(self.world * 64, dtype=t.uint8, device=dev)
        dist.all_gather_into_tensor(recv, send, group=self.group)
        handles = np.ascontiguousarray(recv.cpu().numpy())
        check(lib().ehb_exchange_open(h, handles.ctypes.data_as(C.c_void_p)))
        dist.barrier(group=self.group)   # every rank has mapped every peer before the first push
        self._ex, self._ex_cap = h, cap

    def _bufs(self, nq, k):
        t = self._torch
        key = (nq, k)
        if key not in self._buf:
            dev = t.device("cuda", self.device)
            nl, nd = nq * k * 8, nq * k * 4
            send = t.empty(nl + nd, dtype=t.uint8, device=dev)     # [labels | distances], written by the kernels
            self._buf[key] = dict(
                send=send, l=send[:nl].view(t.int64).view(nq, k), d=send[nl:].view(t.float32).view(nq, k),
                recv=t.empty((self.world, nl + nd), dtype=t.uint8, device=dev) if self.exchange == "nccl" else None,
                c=t.empty(nq, dtype=t.int32, device=dev), ml=t.empty((nq, k), dtype=t.int64, device=dev),
                md=t.empty((nq, k), dtype=t.float32, device=dev), mc=t.empty(nq, dtype=t.int32, device=dev))
        return self._buf[key]

    def _local(self, q, nq, k, ef, stream_ptr, bruteforce, precision, lp, dp, cp, beam=False):
        if bruteforce:
            self.ix.search_bruteforce_dev(q.data_ptr(), nq, k, precision, lp, dp, cp, stream_ptr)
        elif beam:
            self.ix.search_beam_dev(q.data_ptr(), nq, k, ef, lp, dp, cp, stream_ptr, precision)
        else:
            self.ix.search_dev(q.data_ptr(), nq, k, ef, lp, dp, cp, stream_ptr, precision)

    def search_dev(self, q, k, ef, stream_ptr, bruteforce=False, precision=0):
        """q: CUDA float32 tensor [nq, dim].  Returns (labels int64-viewed-u64, dists, counts) CUDA tensors
        holding the global top-k on every rank.  precision (FP32 or BF16) applies to graph searches and brute force
        alike, on every exchange.  Nothing synchronises the host."""
        return self._search_dev(q, k, ef, stream_ptr, bruteforce, precision, False)

    def search_beam_dev(self, q, k, ef, stream_ptr, precision=0):
        """search_dev() of the graph walk with max(ef, k) up to 4096: the wide-beam walk above 512.  World 1:
        NativeIndex.search_beam_dev; the peer exchange: one ehb_exchange_search_beam_dev step; exchange="nccl": the
        local beam search, then the same all-gather and merge."""
        return self._search_dev(q, k, ef, stream_ptr, False, precision, True)

    def _search_dev(self, q, k, ef, stream_ptr, bruteforce, precision, beam):
        nq = q.shape[0]
        b = self._bufs(nq, k)
        if self.world == 1:
            self._local(q, nq, k, ef, stream_ptr, bruteforce, precision, b["l"].data_ptr(), b["d"].data_ptr(),
                        b["c"].data_ptr(), beam)
            return b["l"], b["d"], b["c"]
        if self.exchange == "peer":
            self._ensure_exchange(nq, k)
            if not bruteforce:
                # fused: the search's last kernel (the fp32 walk's epilogue, or the re-rank after a bf16 walk)
                # stores each query's top-k into every peer's receive buffer and raises the slice flags; one kernel
                # waits for the peers' flags and merges
                step = lib().ehb_exchange_search_beam_dev if beam else lib().ehb_exchange_search_ex_dev
                check(step(self._ex, self.ix._h, nq, C.c_void_p(q.data_ptr()), k, ef, int(precision),
                           C.c_void_p(b["md"].data_ptr()), C.c_void_p(b["ml"].data_ptr()),
                           C.c_void_p(b["mc"].data_ptr()), C.c_void_p(b["c"].data_ptr()), C.c_void_p(stream_ptr)))
                return b["ml"], b["md"], b["mc"]
            lp, dp = C.c_void_p(), C.c_void_p()
            check(lib().ehb_exchange_begin(self._ex, nq, k, C.byref(lp), C.byref(dp)))
            # the shard's kernels write straight into this rank's block of its own receive buffer ...
            self._local(q, nq, k, ef, stream_ptr, bruteforce, precision, lp.value, dp.value, b["c"].data_ptr())
            # ... and one kernel pushes it to the peers, flags, waits for theirs and merges
            check(lib().ehb_exchange_merge_dev(self._ex, C.c_void_p(b["md"].data_ptr()), C.c_void_p(b["ml"].data_ptr()),
                                               C.c_void_p(b["mc"].data_ptr()), C.c_void_p(stream_ptr)))
            return b["ml"], b["md"], b["mc"]
        import torch.distributed as dist

        self._local(q, nq, k, ef, stream_ptr, bruteforce, precision, b["l"].data_ptr(), b["d"].data_ptr(),
                    b["c"].data_ptr(), beam)
        dist.all_gather_into_tensor(b["recv"].view(-1), b["send"], group=self.group)
        check(lib().ehb_merge_topk_packed_dev(self.world, nq, k, C.c_void_p(b["recv"].data_ptr()),
                                              b["recv"].shape[1], C.c_void_p(b["md"].data_ptr()),
                                              C.c_void_p(b["ml"].data_ptr()), C.c_void_p(b["mc"].data_ptr()),
                                              self.device, C.c_void_p(stream_ptr)))
        return b["ml"], b["md"], b["mc"]

    def search_by_label_dev(self, labels, k, ef, stream_ptr, precision=0):
        """Key mode (server.cc:190-207): the k nearest other points of stored points named by label.  `labels` (u64,
        the same on every rank) may live on any rank; each is searched with its stored row at k + 1 and its own label
        is removed, or the last hit dropped when it is absent.  Returns (labels int64-viewed-u64, dists, counts) CUDA
        tensors [nq][k] holding the global result on every rank.  On the peer exchange this is one
        ehb_exchange_search_by_label_ex_dev step: the owners push their rows to every rank, every rank agrees that
        each label has exactly one owner (one 4-byte copy to the host), then the fused k + 1 step runs.  Raises
        EhbError with the library's status, the same on every rank: 1 (different label lists), else 5 (not found),
        else 4 (a label on two ranks).  At world 1 it is NativeIndex.search_by_label (KeyError for an unknown label),
        which synchronises the host, with the results copied into CUDA tensors on stream_ptr.  exchange="nccl" raises
        ValueError: it has no row exchange."""
        return self._by_label_dev(labels, k, ef, stream_ptr, precision, False)

    def search_by_label_beam_dev(self, labels, k, ef, stream_ptr, precision=0):
        """search_by_label_dev() with max(ef, k + 1) up to 4096: one ehb_exchange_search_by_label_beam_dev step on
        the peer exchange, NativeIndex.search_by_label_beam at world 1; exchange="nccl" raises ValueError."""
        return self._by_label_dev(labels, k, ef, stream_ptr, precision, True)

    def _by_label_dev(self, labels, k, ef, stream_ptr, precision, beam):
        if self.exchange == "nccl":
            raise ValueError("search_by_label_dev needs the peer exchange (exchange='peer'); the NCCL path only "
                             "exchanges result lists")
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        nq = lab.shape[0]
        if self.world == 1:
            # a host search (it synchronises); the results are allocated and copied on stream_ptr, so work queued
            # there afterwards reads them in order
            search = self.ix.search_by_label_beam if beam else self.ix.search_by_label
            ol, od, oc = search(lab, k, ef=ef, precision=precision)
            t = self._torch
            dev = t.device("cuda", self.device)
            s = t.cuda.ExternalStream(stream_ptr, device=dev) if stream_ptr else t.cuda.current_stream(dev)
            with t.cuda.stream(s):
                return tuple(t.from_numpy(a).to(dev, non_blocking=False)
                             for a in (ol.view(np.int64), od, oc.view(np.int32)))
        b = self._bufs(nq, k)
        self._ensure_exchange(nq, k + 1, self.ix.dim)
        step = lib().ehb_exchange_search_by_label_beam_dev if beam else lib().ehb_exchange_search_by_label_ex_dev
        check(step(self._ex, self.ix._h, nq, lab.ctypes.data_as(C.c_void_p), k, ef, int(precision),
                   C.c_void_p(b["md"].data_ptr()), C.c_void_p(b["ml"].data_ptr()), C.c_void_p(b["mc"].data_ptr()),
                   C.c_void_p(stream_ptr)))
        return b["ml"], b["md"], b["mc"]
