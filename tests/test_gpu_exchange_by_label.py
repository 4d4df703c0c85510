"""Key mode in the one-process-per-GPU shard exchange (ehb_exchange_search_by_label_ex_dev): the owners push the stored
rows of the query labels into every rank's row region, every rank agrees that each label has exactly one owner, then
the fused k + 1 step runs over those rows, the lists are merged and each query's own label is removed.

Both "ranks" live in this process (ehb_exchange_attach_local), on two devices when the box has them and both on
device 0 otherwise.  A by-label step synchronises the host once (the verdict of its row step), so each rank's calls
run on a host thread of their own.  Held exactly (labels, distance bits, counts, on both ranks):
  * the step equals tests/label_rule_model.drop_self applied to the fused ehb_exchange_search_ex_dev step at k + 1
    over the rows each owner's get_batch returns: fp32 and bf16, L2 / IP / cosine, d = 128 and 768 (the screened walk
    at 4 queries per SM), nq = 1, 4, 5 (the team walk, pushed after) and the capacity, k up to ef - 1, labels from one
    shard, from both, and repeated within a batch;
  * it equals ehb_sharded_search_by_label_ex over the same two shards;
  * on tie-free IP data it equals the oracle's per-shard searches, merged, then the rule (both branches occur);
  * after a compaction of one shard and with tombstones in the other.
Every lockstep failure (different lists, also of different lengths, first; then no owner, two owners) and every check before the step returns the same
status on both ranks, leaves the sentinel-filled outputs untouched, and the next fused fp32, bf16 and by-label steps
complete on both ranks.  After every step no rank's exchange has timed out.

A call that frees device memory waits for the whole device, and with two ranks on one GPU that would wait for a
peer's spinning exchange kernel; so can the first launch of a kernel under lazy module loading.  Every test runs its
reference searches first, which size the search scratch and load every kernel a step launches.
"""
import ctypes as C
import os
import socket
import sys
import threading

import numpy as np
import pytest

from label_rule_model import drop_self
from oracle import oracle as orc  # test infrastructure

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EHB_FP32, EHB_BF16 = 0, 1
EHB_OK, EHB_ERR_INVALID, EHB_ERR_STATE, EHB_ERR_NOT_FOUND = 0, 1, 4, 5
SENTINEL_L, SENTINEL_D, SENTINEL_C = 0x1234, 7.5, 77


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


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gauss(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)


class Pair:
    """Two shards (global labels) and two attached exchanges with row regions, one per 'rank'."""

    def __init__(self, parts, d, metric, max_nq, max_k, max_dim=None, ixs=None, labels=None):
        import torch
        self.torch = torch
        self.devs = _devices(2)
        self.d = d
        self.exs = []
        L = _lib()
        if ixs is None:
            ixs, lo = [], 0
            for r, x in enumerate(parts):
                ix = _ehb().NativeIndex(d, metric=metric, capacity=len(x), device=self.devs[r])
                lab = labels[r] if labels is not None else np.arange(lo, lo + len(x), dtype=np.uint64)
                ix.add(x, lab)
                ix.build()
                lo += len(x)
                ixs.append(ix)
        self.ixs = ixs
        for r in range(2):
            h = C.c_void_p()
            _check(L.ehb_exchange_create_ex(self.devs[r], 2, r, max_nq, max_k, d if max_dim is None else max_dim,
                                            C.byref(h)))
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
        return (t.full((nq, k), SENTINEL_L, dtype=t.int64, device=self.dev(r)),
                t.full((nq, k), SENTINEL_D, dtype=t.float32, device=self.dev(r)),
                t.full((nq,), SENTINEL_C, dtype=t.int32, device=self.dev(r)))

    def rows(self, labels):
        """Each label's stored row from its owner's get_batch (the owner: the shard whose get_batch finds it)."""
        labels = np.asarray(labels, np.uint64)
        out = np.empty((len(labels), self.d), np.float32)
        found = np.zeros(len(labels), bool)
        for ix in self.ixs:
            held = np.array([self._holds(ix, l) for l in labels])
            if held.any():
                out[held] = ix.get_batch(labels[held])
                found |= held
        assert found.all()
        return out

    @staticmethod
    def _holds(ix, label):
        try:
            ix.get_batch([label])
            return True
        except KeyError:
            return False

    def warm(self, labels, k, ef, precision):
        """Sizes every search slot for this (nq, k + 1, ef, precision) with each shard's own search, and loads the
        kernels of a key-mode search before any step (a first launch can wait for the kernels already running)."""
        t = self.torch
        q = self.rows(labels)
        nq = len(q)
        for ix in self.ixs:
            own = [l for l in labels if self._holds(ix, l)]
            if own:
                ix.search_by_label(own[:1], 1, ef, precision)
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(q).to(self.dev(r))
            l, d, c = self._out(r, nq, k + 1)
            s = self.streams[r]
            s.wait_stream(t.cuda.current_stream(self.devs[r]))
            self.ixs[r].search_dev(dq.data_ptr(), nq, k + 1, ef, l.data_ptr(), d.data_ptr(), c.data_ptr(),
                                   s.cuda_stream, precision)
            s.synchronize()

    def fused(self, q, k, ef, precision):
        """One fused step on both ranks (queued from this thread; the fused step never synchronises)."""
        t = self.torch
        nq = len(q)
        res = []
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            dq = t.from_numpy(np.ascontiguousarray(q)).to(self.dev(r))
            ml, md, mc = self._out(r, nq, k)
            self.streams[r].wait_stream(t.cuda.current_stream(self.devs[r]))
            _check(_lib().ehb_exchange_search_ex_dev(
                self.exs[r], self.ixs[r]._h, nq, C.c_void_p(dq.data_ptr()), k, ef, precision,
                C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()), None,
                C.c_void_p(self.streams[r].cuda_stream)))
            res.append((ml, md, mc, dq))
        return self._collect(res)

    def reference(self, labels, k, ef, precision):
        """The rule over the fused k + 1 step fed with the owners' rows."""
        out = self.fused(self.rows(labels), k + 1, ef, precision)
        lab = np.asarray(labels, np.uint64)
        for r in range(2):
            assert np.array_equal(out[r][0], out[0][0]) and np.array_equal(out[r][2], out[0][2])
        l, d, c = out[0]
        return drop_self(lab, l, d, c, k)

    def by_label(self, labels, k, ef, precision, labels1=None):
        """One by-label step, each rank on its own host thread: per rank (status, labels, dists, counts)."""
        t = self.torch
        labs = [np.ascontiguousarray(labels, np.uint64),
                np.ascontiguousarray(labels if labels1 is None else labels1, np.uint64)]
        outs = []
        for r in range(2):
            t.cuda.set_device(self.devs[r])
            outs.append(self._out(r, len(labs[r]), k))
            self.streams[r].wait_stream(t.cuda.current_stream(self.devs[r]))
        rcs = [None, None]

        def run(r):
            t.cuda.set_device(self.devs[r])
            ml, md, mc = outs[r]
            rcs[r] = _lib().ehb_exchange_search_by_label_ex_dev(
                self.exs[r], self.ixs[r]._h, len(labs[r]), labs[r].ctypes.data_as(C.c_void_p), k, ef, precision,
                C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                C.c_void_p(self.streams[r].cuda_stream))
            self.streams[r].synchronize()

        th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        got = self._collect([(*outs[r], None) for r in range(2)])
        return [(rcs[r], *got[r]) for r in range(2)]

    def _collect(self, res):
        out = []
        for r in range(2):
            self.streams[r].synchronize()
            ml, md, mc, _ = res[r]
            out.append((ml.cpu().numpy().view(np.uint64), md.cpu().numpy(), mc.cpu().numpy().view(np.uint32)))
        self.assert_no_timeout()
        return out

    def assert_no_timeout(self):
        for r in range(2):
            v = C.c_uint32()
            _check(_lib().ehb_exchange_timed_out(self.exs[r], C.byref(v)))
            assert v.value == 0, r


def assert_same(got, want, what):
    gl, gd, gc = got
    wl, wd, wc = want
    assert np.array_equal(np.asarray(gc).astype(np.uint32), np.asarray(wc).astype(np.uint32)), what
    assert np.array_equal(np.asarray(gl).view(np.uint64), np.asarray(wl).view(np.uint64)), what
    assert np.array_equal(np.asarray(gd).view(np.uint32), np.asarray(wd).view(np.uint32)), what


def assert_held(out, want, what):
    for r in range(2):
        assert out[r][0] == EHB_OK, (what, r, out[r][0])
        assert_same(out[r][1:], want, (what, r))


def assert_failed(out, status, what):
    for r in range(2):
        assert out[r][0] == status, (what, r, out[r][0])
        l, d, c = out[r][1:]
        assert (l == SENTINEL_L).all() and (d == np.float32(SENTINEL_D)).all() and (c == SENTINEL_C).all(), (what, r)


def batches(n, cap, seed):
    """Label batches of nq = cap, 1, 4, 5, cap (the largest first): shard 1 only, shard 0 only, both with repeats."""
    rng = np.random.default_rng(seed)
    return [rng.choice(2 * n, cap, replace=True).astype(np.uint64),
            rng.choice(np.arange(n, 2 * n), 1).astype(np.uint64),
            rng.choice(n, 4, replace=False).astype(np.uint64),
            np.array([3, n + 7, 3, 2 * n - 1, n + 7], np.uint64),
            rng.choice(2 * n, cap, replace=False).astype(np.uint64)]


# ---- 1. bitwise against the rule over the fused k + 1 step ----------------------------------------------------------
KS, EF = (1, 10, 63), 64


@pytest.mark.parametrize("precision", [EHB_FP32, EHB_BF16])
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("d", [128, 768])
def test_by_label_equals_rule_over_fused_step(d, metric, precision):
    n, cap = 3000, 150
    x = gauss(2 * n, d, 101 + d)
    p = Pair([x[:n], x[n:]], d, metric, cap, EF)
    try:
        bs = batches(n, cap, 102)
        for k in KS:
            p.warm(bs[0], k, EF, precision)
        for labels in bs:
            for k in KS:
                want = p.reference(labels, k, EF, precision)
                assert_held(p.by_label(labels, k, EF, precision), want, (len(labels), k))
                if len(labels) == cap and k == 10:
                    assert (want[2] == k).all()
    finally:
        p.close()


@pytest.mark.parametrize("precision", [EHB_FP32, EHB_BF16])
def test_by_label_screened_walk(precision):
    """d = 768, IP, nq = 4 queries per SM: the fp32 step walks with the int8 screen."""
    d, n, k, ef = 768, 4000, 10, 64
    nq = 4 * sms()
    x = gauss(2 * n, d, 111)
    p = Pair([x[:n], x[n:]], d, "ip", nq, k + 1)
    try:
        labels = np.random.default_rng(112).choice(2 * n, nq, replace=False).astype(np.uint64)
        p.warm(labels, k, ef, precision)
        want = p.reference(labels, k, ef, precision)
        assert_held(p.by_label(labels, k, ef, precision), want, "screened")
        if precision == EHB_FP32:
            assert p.ixs[0].stats()["screened_evals"] > 0 and p.ixs[1].stats()["screened_evals"] > 0
    finally:
        p.close()


# ---- 2. equal to the single-process sharded index --------------------------------------------------------------------
@pytest.mark.parametrize("precision", [EHB_FP32, EHB_BF16])
def test_by_label_equals_sharded_by_label(precision):
    d, n, nq, k, ef = 128, 3000, 200, 10, 64
    x = gauss(2 * n, d, 121)
    sh = _ehb().ShardedIndex(d, _devices(2), metric="cosine", capacity=n, shard_span=n)
    sh.add(x, np.arange(2 * n, dtype=np.uint64))
    sh.build()
    p = Pair(None, d, "cosine", nq, k + 1, ixs=[sh.shard(0), sh.shard(1)])
    try:
        labels = np.random.default_rng(122).choice(2 * n, nq, replace=False).astype(np.uint64)
        want = sh.search_by_label(labels, k, ef, precision)
        p.warm(labels, k, ef, precision)
        assert_held(p.by_label(labels, k, ef, precision), want, "sharded")
    finally:
        p.close()
        sh.close()


# ---- 3. exact against the oracle on tie-free data --------------------------------------------------------------------
def test_by_label_equals_oracle_on_tie_free_data():
    """x_i = (B u_i, i + 1): x_i . x_j = B^2 (u_i . u_j) + (i + 1)(j + 1), exact in fp32 and distinct over j."""
    n, d, B = 400, 8, 512
    assert B * B * (d - 1) + (n + 1) ** 2 < 1 << 24
    rng = np.random.default_rng(131)
    x = np.empty((n, d), np.int64)
    x[:, :d - 1] = B * rng.integers(-1, 2, (n, d - 1))
    x[:, d - 1] = np.arange(1, n + 1)
    xf = x.astype(np.float32)
    half = n // 2
    p = Pair([xf[:half], xf[half:]], d, "ip", n, 16)
    try:
        for ix in p.ixs:
            ix.set_search_width(1)
        oracles = []
        for r in range(2):
            o = orc.OracleHNSW(d, "ip", half)
            o.import_graph(p.ixs[r].export_graph())
            oracles.append(o)
        labels = np.arange(n, dtype=np.uint64)
        for k in (1, 10):
            p.warm(labels, k, 16, EHB_FP32)
            per = [o.search(xf, k + 1, ef=16, threads=8) for o in oracles]
            # merge the two shards' lists (tie-free: distance order alone), then the rule
            ml =np.concatenate([per[0][0].astype(np.uint64), per[1][0].astype(np.uint64)], 1)
            md = np.concatenate([per[0][1].astype(np.float32), per[1][1].astype(np.float32)], 1)
            mc = per[0][2].astype(np.int64) + per[1][2].astype(np.int64)
            key = np.where(ml == np.uint64(0xFFFFFFFFFFFFFFFF), np.inf, md)
            order = np.lexsort((ml, key), axis=1)
            ml, md = np.take_along_axis(ml, order, 1)[:, :k + 1], np.take_along_axis(md, order, 1)[:, :k + 1]
            mc = np.minimum(mc, k + 1)
            want = drop_self(labels, ml, md, mc, k)
            assert_held(p.by_label(labels, k, 16, EHB_FP32), want, ("oracle", k))
            present = np.array([l in row[:c] for l, row, c in zip(labels, ml, mc)])
            assert present.any() and (~present).any()
    finally:
        p.close()


# ---- 3b. a row region whose parity parts are not whole rows apart ---------------------------------------------------
@pytest.mark.parametrize("d,max_dim,max_nq", [(128, 130, 33), (768, 2047, 17)])
def test_by_label_with_max_dim_above_dim(d, max_dim, max_nq):
    """max_nq * max_dim is not a multiple of 4 floats, yet both parity parts of the row region take 16-byte stores
    at 16-byte aligned rows.  A by-label step spends two epochs and a fused step one, so the row steps of
    by-label, fused, by-label, by-label use parities p, 1 - p, 1 - p: both parts, and two consecutive steps."""
    n, k, ef = 1500, 10, 32
    x = gauss(2 * n, d, 135 + d)
    p = Pair([x[:n], x[n:]], d, "ip", max_nq, k + 1, max_dim=max_dim)
    try:
        rng = np.random.default_rng(136)
        bs = [rng.choice(2 * n, max_nq, replace=False).astype(np.uint64) for _ in range(3)]
        p.warm(bs[0], k, ef, EHB_FP32)
        wants = [p.reference(b, k, ef, EHB_FP32) for b in bs]
        assert_held(p.by_label(bs[0], k, ef, EHB_FP32), wants[0], "parity p")
        p.fused(p.rows(bs[2][:5]), k, ef, EHB_FP32)
        assert_held(p.by_label(bs[1], k, ef, EHB_FP32), wants[1], "parity 1 - p")
        assert_held(p.by_label(bs[2], k, ef, EHB_FP32), wants[2], "parity 1 - p again")
    finally:
        p.close()


# ---- 4. after a compaction and with tombstones -----------------------------------------------------------------------
def test_by_label_after_compaction_and_tombstones():
    d, n, nq, k, ef = 64, 3000, 120, 10, 32
    x = gauss(2 * n, d, 141)
    p = Pair([x[:n], x[n:]], d, "ip", nq, k + 1)
    try:
        rng = np.random.default_rng(142)
        dead0 = np.union1d(rng.choice(n, n // 4, replace=False), [p.ixs[0].stats()["entry_point"]]).astype(np.uint64)
        dead1 = (n + rng.choice(n, n // 10, replace=False)).astype(np.uint64)
        p.ixs[0].remove(dead0)
        p.ixs[0].compact()
        p.ixs[1].remove(dead1)
        live = np.setdiff1d(np.arange(2 * n, dtype=np.uint64), np.union1d(dead0, dead1))
        labels = rng.choice(live, nq, replace=False).astype(np.uint64)
        for precision in (EHB_FP32, EHB_BF16):
            p.warm(labels, k, ef, precision)
            want = p.reference(labels, k, ef, precision)
            out = p.by_label(labels, k, ef, precision)
            assert_held(out, want, precision)
            assert not np.isin(out[0][1], np.union1d(dead0, dead1)).any()
    finally:
        p.close()


# ---- 5. lockstep failures and checks before the step -----------------------------------------------------------------
def _after_failure(p, labels, q, k, ef, refs, what):
    """The next fused fp32, bf16 and by-label steps complete on both ranks."""
    for prec in (EHB_FP32, EHB_BF16):
        out = p.fused(q, k, ef, prec)
        for r in range(2):
            assert_same(out[r], refs[prec], (what, "fused", prec, r))
    assert_held(p.by_label(labels, k, ef, EHB_FP32), refs["label"], (what, "by-label"))


def test_lockstep_failures_leave_the_ranks_in_phase():
    import torch
    d, n, nq, k, ef = 64, 2000, 40, 10, 64
    x = gauss(2 * n, d, 151)
    lab1 = np.arange(n, 2 * n, dtype=np.uint64)
    lab1[-1] = 5                                  # label 5 is stored on both shards
    p = Pair([x[:n], x[n:]], d, "l2", nq, k + 1, labels=[np.arange(n, dtype=np.uint64), lab1])
    L = _lib()
    try:
        rng = np.random.default_rng(152)
        labels = rng.choice(np.setdiff1d(np.arange(6, 2 * n - 1), [n + 1]), nq, replace=False).astype(np.uint64)
        q = gauss(nq, d, 153)
        p.ixs[1].remove(np.array([n + 1], np.uint64))
        for prec in (EHB_FP32, EHB_BF16):
            p.warm(labels, k, ef, prec)
        refs = {EHB_FP32: p.fused(q, k, ef, EHB_FP32)[0], EHB_BF16: p.fused(q, k, ef, EHB_BF16)[0],
                "label": p.reference(labels, k, ef, EHB_FP32)}
        # rank 1's list differs only where rank 0 is the owner, by a label rank 0 owns: one owner per query, so only
        # the digests tell the lists apart
        j = int(np.flatnonzero(labels < n)[0])
        other = np.setdiff1d(np.arange(6, n), labels)[0]
        swapped = labels.copy()
        swapped[j] = other
        cases = [("unknown", np.r_[labels[:-1], [10 ** 9]], None, EHB_ERR_NOT_FOUND),
                 ("tombstoned", np.r_[labels[:-1], [n + 1]], None, EHB_ERR_NOT_FOUND),
                 ("two owners", np.r_[labels[:-1], [5]], None, EHB_ERR_STATE),
                 ("different lists", labels, swapped, EHB_ERR_INVALID),
                 # lists that also disagree on the owners: the digests decide first, on both ranks
                 ("rotated lists", labels, np.r_[labels[1:], labels[:1]], EHB_ERR_INVALID),
                 # lists of different lengths: the longer one's last marks were never written in this step
                 ("different lengths", labels[:-1], labels, EHB_ERR_INVALID),
                 ("different lengths, unknown label", np.r_[labels[:-1], [10 ** 9]], labels[:-2], EHB_ERR_INVALID)]
        for what, l0, l1, status in cases:
            out = p.by_label(l0.astype(np.uint64), k, ef, EHB_FP32, None if l1 is None else l1.astype(np.uint64))
            assert_failed(out, status, what)
            _after_failure(p, labels, q, k, ef, refs, what)
        # checks before the epoch advances: each rank is called once, from this thread
        too_many = np.arange(nq + 1, dtype=np.uint64)
        pre = [("precision", labels, k, ef, 7), ("ef", labels, k, 513, EHB_FP32), ("k + 1 > 512", labels, 512, 0, 0),
               ("nq > max_nq", too_many, 1, ef, EHB_FP32), ("nq * (k + 1)", labels, k + 1, ef, EHB_FP32)]
        for what, l0, kk, e, prec in pre:
            for r in range(2):
                torch.cuda.set_device(p.devs[r])
                ml, md, mc = p._out(r, len(l0), kk)
                rc = L.ehb_exchange_search_by_label_ex_dev(p.exs[r], p.ixs[r]._h, len(l0), l0.ctypes.data_as(C.c_void_p),
                                                           kk, e, prec, C.c_void_p(md.data_ptr()),
                                                           C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                                                           C.c_void_p(p.streams[r].cuda_stream))
                assert rc == EHB_ERR_INVALID, (what, r)
                p.streams[r].synchronize()
                assert (ml == SENTINEL_L).all().item() and (mc == SENTINEL_C).all().item(), (what, r)
            _after_failure(p, labels, q, k, ef, refs, what)
        for r in range(2):
            torch.cuda.set_device(p.devs[r])
            ml, md, mc = p._out(r, nq, k)
            ptrs = [C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr())]
            for what, lp, outs, kk, status in [("null labels", None, ptrs, k, EHB_ERR_INVALID),
                                               ("null dists", labels.ctypes.data_as(C.c_void_p), [None] + ptrs[1:], k,
                                                EHB_ERR_INVALID),
                                               ("k == 0", labels.ctypes.data_as(C.c_void_p), ptrs, 0, EHB_OK)]:
                rc = L.ehb_exchange_search_by_label_ex_dev(p.exs[r], p.ixs[r]._h, nq, lp, kk, ef, EHB_FP32, *outs,
                                                           C.c_void_p(p.streams[r].cuda_stream))
                assert rc == status, (what, r)
            p.streams[r].synchronize()
            assert (ml == SENTINEL_L).all().item() and (mc == SENTINEL_C).all().item(), r
        _after_failure(p, labels, q, k, ef, refs, "null and k == 0")
    finally:
        p.close()


def test_exchange_without_rows_rejects_key_mode():
    import torch
    d, n, nq, k, ef = 64, 2000, 30, 10, 64
    x = gauss(2 * n, d, 161)
    p = Pair([x[:n], x[n:]], d, "ip", nq, k + 1, max_dim=0)
    L = _lib()
    try:
        q = gauss(nq, d, 162)
        for prec in (EHB_FP32, EHB_BF16):
            p.warm(np.arange(nq, dtype=np.uint64), k, ef, prec)
        want = p.fused(q, k, ef, EHB_FP32)[0]
        labels = np.arange(nq, dtype=np.uint64)
        for r in range(2):
            torch.cuda.set_device(p.devs[r])
            ml, md, mc = p._out(r, nq, k)
            rc = L.ehb_exchange_search_by_label_ex_dev(p.exs[r], p.ixs[r]._h, nq, labels.ctypes.data_as(C.c_void_p), k,
                                                       ef, EHB_FP32, C.c_void_p(md.data_ptr()),
                                                       C.c_void_p(ml.data_ptr()), C.c_void_p(mc.data_ptr()),
                                                       C.c_void_p(p.streams[r].cuda_stream))
            assert rc == EHB_ERR_INVALID
        out = p.fused(q, k, ef, EHB_FP32)
        for r in range(2):
            assert_same(out[r], want, r)
        # peers must agree on max_dim
        h0, h1 = C.c_void_p(), C.c_void_p()
        _check(L.ehb_exchange_create_ex(p.devs[0], 2, 0, nq, k, 0, C.byref(h0)))
        _check(L.ehb_exchange_create_ex(p.devs[1], 2, 1, nq, k, d, C.byref(h1)))
        assert L.ehb_exchange_attach_local(h0, 1, h1) == EHB_ERR_INVALID
        L.ehb_exchange_destroy(h0)
        L.ehb_exchange_destroy(h1)
    finally:
        p.close()


# ---- 6. by-label, fused and push-after steps interleave --------------------------------------------------------------
def test_by_label_interleaves_with_fused_and_push_after_steps():
    d, n, k, ef, cap = 128, 3000, 10, 64, 150
    x = gauss(2 * n, d, 171)
    p = Pair([x[:n], x[n:]], d, "cosine", cap, k + 1)
    L = _lib()
    t = p.torch
    try:
        bs = batches(n, cap, 172)
        q = gauss(cap, d, 173)
        for prec in (EHB_FP32, EHB_BF16):
            p.warm(bs[0], k, ef, prec)
        sc = []
        for r in range(2):                        # sizes the brute-force scratch before any step
            t.cuda.set_device(p.devs[r])
            dq = t.from_numpy(q).to(p.dev(r))
            l, dd, c = p._out(r, cap, k)
            sc.append(t.empty(cap, dtype=t.int32, device=p.dev(r)))
            p.ixs[r].search_bruteforce_dev(dq.data_ptr(), cap, k, EHB_FP32, l.data_ptr(), dd.data_ptr(), c.data_ptr(),
                                           p.streams[r].cuda_stream)
            p.streams[r].synchronize()
        refs = {}
        for i, labels in enumerate(bs):
            nq = len(labels)
            refs[i] = (p.reference(labels, k, ef, EHB_FP32), p.reference(labels, k, ef, EHB_BF16),
                       p.fused(q[:nq], k, ef, EHB_FP32)[0])
        # the push-after brute-force reference: each shard's own brute force, merged by the exchange itself below
        for i, labels in enumerate(bs):
            nq = len(labels)
            rl, rb, rf = refs[i]
            assert_held(p.by_label(labels, k, ef, EHB_FP32), rl, (i, "label fp32"))
            out = p.fused(q[:nq], k, ef, EHB_FP32)
            for r in range(2):
                assert_same(out[r], rf, (i, "fused", r))
            assert_held(p.by_label(labels, k, ef, EHB_BF16), rb, (i, "label bf16"))
            # a push-after brute-force step: begin, each shard's exact brute force, merge
            res = []
            for r in range(2):
                t.cuda.set_device(p.devs[r])
                dq = t.from_numpy(np.ascontiguousarray(q[:nq])).to(p.dev(r))
                p.streams[r].wait_stream(t.cuda.current_stream(p.devs[r]))
                lp, dp = C.c_void_p(), C.c_void_p()
                _check(L.ehb_exchange_begin(p.exs[r], nq, k, C.byref(lp), C.byref(dp)))
                p.ixs[r].search_bruteforce_dev(dq.data_ptr(), nq, k, EHB_FP32, lp.value, dp.value, sc[r].data_ptr(),
                                               p.streams[r].cuda_stream)
                res.append((*p._out(r, nq, k), dq))
            for r in range(2):
                t.cuda.set_device(p.devs[r])
                ml, md, mc = res[r][:3]
                _check(L.ehb_exchange_merge_dev(p.exs[r], C.c_void_p(md.data_ptr()), C.c_void_p(ml.data_ptr()),
                                                C.c_void_p(mc.data_ptr()), C.c_void_p(p.streams[r].cuda_stream)))
            out = p._collect(res)
            assert_same(out[1], out[0], (i, "brute"))
            assert_held(p.by_label(labels, k, ef, EHB_FP32), rl, (i, "label after brute"))
    finally:
        p.close()


# ---- 7. the Python searcher ------------------------------------------------------------------------------------------
def test_sharded_searcher_world1_by_label_equals_native():
    import torch
    from embeddinghub_b200.sharded import ShardedSearcher
    d, n, nq, k, ef = 128, 4000, 200, 10, 32
    ix = _ehb().NativeIndex(d, metric="ip", capacity=n)
    ix.add(gauss(n, d, 181))
    ix.build()
    labels = np.random.default_rng(182).choice(n, nq, replace=False).astype(np.uint64)
    for prec in (EHB_FP32, EHB_BF16):
        want = ix.search_by_label(labels, k, ef, prec)
        s = ShardedSearcher(ix, 1, 0)
        stream = torch.cuda.Stream()
        ml, md, mc = s.search_by_label_dev(labels, k, ef, stream.cuda_stream, precision=prec)
        torch.cuda.synchronize()
        assert_same((ml.cpu().numpy(), md.cpu().numpy(), mc.cpu().numpy()), want, prec)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _peer_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    import embeddinghub_b200 as ehb
    from embeddinghub_b200.sharded import ShardedSearcher, route_rows
    from label_rule_model import drop_self as rule

    d, n, nq, k, ef = 128, 8000, 333, 10, 64
    x = np.random.default_rng(191).standard_normal((n, d), dtype=np.float32)
    labels = np.random.default_rng(192).choice(n, nq, replace=False).astype(np.uint64)
    mv, ml = route_rows(x, np.arange(n, dtype=np.uint64), n, world, rank)
    ix = ehb.NativeIndex(d, metric="ip", capacity=len(mv), device=rank)
    ix.add(mv, ml)
    ix.build()
    stream = torch.cuda.Stream(device=rank)
    s = ShardedSearcher(ix, world, rank)
    dq = torch.from_numpy(x[labels.astype(np.int64)]).cuda(rank)
    stream.wait_stream(torch.cuda.current_stream(rank))
    l1, d1, c1 = s.search_dev(dq, k + 1, ef, stream.cuda_stream)
    stream.synchronize()
    want = rule(labels, l1.cpu().numpy().view(np.uint64), d1.cpu().numpy(), c1.cpu().numpy(), k)
    l, dd, c = s.search_by_label_dev(labels, k, ef, stream.cuda_stream)
    stream.synchronize()
    ok = (np.array_equal(l.cpu().numpy().view(np.uint64), want[0]) and
          np.array_equal(dd.cpu().numpy().view(np.uint32), want[1].view(np.uint32)) and
          np.array_equal(c.cpu().numpy().astype(np.uint32), want[2]))
    s.close()
    out.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_process_peer_by_label():
    """torchrun-style: one process per GPU; the peer step equals search_dev(x[labels], k + 1) plus the rule."""
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
