"""Wide-beam graph search (max(ef, k) 513 .. 4096) across shards: the one-process-per-GPU exchange
(ehb_exchange_search_beam_dev, ehb_exchange_search_by_label_beam_dev), the one-process sharded index
(ehb_sharded_search_beam, ehb_sharded_search_by_label_beam) and ShardedSearcher.

The "ranks" live in this process (ehb_exchange_attach_local), two or three of them, on as many devices as the box has
and otherwise all on device 0.  Each rank's calls run on a host thread of their own (a by-label step synchronises the
host once).  Held exactly (labels, distance bits, counts, on every rank):
  * the fused beam step is ehb_merge_topk_dev over every rank's own ehb_index_search_beam_dev output, fp32 and bf16,
    L2 / IP / cosine, d = 64, 768 and 3072, ef 513 .. 4096 with k = 1, 600 and ef, and with a shard smaller than k;
    shard_counts_dev is the shard's own counts and the shard's last kernel is the wide-beam walk;
  * on tie-free IP data it is the merge of the oracle's per-shard searchKnn at the same beam;
  * with 10 % tombstones (the entry point included) on one shard;
  * by label it is the rule of tests/label_rule_model.drop_self over the fused beam step at k + 1 fed with the owners'
    get_batch rows; different lists, a missing label and a label on two ranks fail alike on every rank;
  * up to 512 every new call equals its _ex counterpart;
  * beam, _ex, by-label beam and push-after brute-force steps interleave on one exchange of three ranks;
  * every rejection fails before the step starts with the outputs untouched, and the next step pairs.
After every step no rank's exchange has timed out.

A call that frees device memory waits for the whole device, and with several ranks on one GPU that would wait for a
peer's spinning merge kernel, itself waiting for this rank.  So every test runs the per-rank reference beam searches,
which size the index's wide-beam scratch and the search slots and load the kernels, before any fused step.
"""
import ctypes as C
import threading

import numpy as np
import pytest

from label_rule_model import drop_self
from oracle import oracle as orc  # test infrastructure
from test_gpu_walk_exact import ip_dist, tiefree

pytestmark = pytest.mark.gpu
EHB_FP32, EHB_BF16 = 0, 1
EHB_OK, EHB_ERR_INVALID, EHB_ERR_STATE, EHB_ERR_NOT_FOUND = 0, 1, 4, 5
SENTINEL_L, SENTINEL_D, SENTINEL_C = 0x1234, 7.5, 77
EFS = [513, 1057, 2049, 4096]


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


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class Ranks:
    """One shard (global labels) and one attached exchange with row regions per 'rank'."""

    def __init__(self, parts, d, metric, max_nq, max_k, max_dim=None, labels=None):
        import torch
        self.torch = torch
        self.W = len(parts)
        self.devs = _devices(self.W)
        self.d = d
        self.ixs, self.exs = [], []
        L = _lib()
        lo = 0
        for r, x in enumerate(parts):
            ix = _ehb().NativeIndex(d, metric=metric, capacity=len(x), device=self.devs[r])
            ix.add(x, labels[r] if labels is not None else np.arange(lo, lo + len(x), dtype=np.uint64))
            ix.build()
            ix.set_option("combine", 0)
            lo += len(x)
            self.ixs.append(ix)
            h = C.c_void_p()
            _check(L.ehb_exchange_create_ex(self.devs[r], self.W, r, max_nq, max_k, d if max_dim is None else max_dim,
                                            C.byref(h)))
            self.exs.append(h)
        for r in range(self.W):
            for g in range(self.W):
                if g != r:
                    _check(L.ehb_exchange_attach_local(self.exs[r], g, self.exs[g]))
        self.streams = [torch.cuda.Stream(device=dv) for dv in self.devs]

    def close(self):
        for s in self.streams:
            s.synchronize()
        for h in self.exs:
            _lib().ehb_exchange_destroy(h)

    def dev(self, r):
        return f"cuda:{self.devs[r]}"

    def out(self, r, nq, k):
        t = self.torch
        return (t.full((nq, k), SENTINEL_L, dtype=t.int64, device=self.dev(r)),
                t.full((nq, k), SENTINEL_D, dtype=t.float32, device=self.dev(r)),
                t.full((nq,), SENTINEL_C, dtype=t.int32, device=self.dev(r)))

    def _on_ranks(self, call, outs):
        """call(r) on W host threads; then (status, labels, dists, counts, shard counts or None) per rank."""
        rcs = [None] * self.W
        self._settle()

        def run(r):
            self.torch.cuda.set_device(self.devs[r])
            rcs[r] = call(r)
            self.streams[r].synchronize()

        th = [threading.Thread(target=run, args=(r,)) for r in range(self.W)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        res = []
        for r in range(self.W):
            ml, md, mc, sc = outs[r]
            res.append((rcs[r], ml.cpu().numpy().view(np.uint64), md.cpu().numpy(), mc.cpu().numpy().view(np.uint32),
                        None if sc is None else sc.cpu().numpy().view(np.uint32)))
        self.assert_no_timeout()
        return res

    def _settle(self):
        """The inputs and sentinel-filled outputs made on the current streams are in place before any call."""
        for dv in sorted(set(self.devs)):
            self.torch.cuda.synchronize(dv)

    def _queries(self, q):
        return [self.torch.from_numpy(np.ascontiguousarray(q, np.float32)).to(self.dev(r)) for r in range(self.W)]

    def fused(self, q, k, ef, precision, step="ehb_exchange_search_beam_dev", null_out=False):
        nq = len(q)
        dqs = self._queries(q)
        outs = [(*self.out(r, nq, k), self.torch.full((nq,), -1, dtype=self.torch.int32, device=self.dev(r)))
                for r in range(self.W)]
        fn = getattr(_lib(), step)

        def call(r):
            ml, md, mc, sc = outs[r]
            return fn(self.exs[r], self.ixs[r]._h, nq, _vp(dqs[r]), k, ef, precision, _vp(md),
                      None if null_out else _vp(ml), _vp(mc), _vp(sc), C.c_void_p(self.streams[r].cuda_stream))
        return self._on_ranks(call, outs)

    def by_label(self, labels, k, ef, precision, step="ehb_exchange_search_by_label_beam_dev", per_rank=None):
        labs = [np.ascontiguousarray(labels if per_rank is None else per_rank[r], np.uint64) for r in range(self.W)]
        outs = [(*self.out(r, len(labs[r]), k), None) for r in range(self.W)]
        fn = getattr(_lib(), step)

        def call(r):
            ml, md, mc, _ = outs[r]
            return fn(self.exs[r], self.ixs[r]._h, len(labs[r]), labs[r].ctypes.data_as(C.c_void_p), k, ef, precision,
                      _vp(md), _vp(ml), _vp(mc), C.c_void_p(self.streams[r].cuda_stream))
        return self._on_ranks(call, outs)

    def brute(self, q, k):
        """A push-after step: begin, the exact brute force into this rank's block, merge_dev."""
        nq = len(q)
        dqs = self._queries(q)
        outs = [(*self.out(r, nq, k), self.torch.full((nq,), -1, dtype=self.torch.int32, device=self.dev(r)))
                for r in range(self.W)]
        L = _lib()

        def call(r):
            ml, md, mc, sc = outs[r]
            lp, dp = C.c_void_p(), C.c_void_p()
            rc = L.ehb_exchange_begin(self.exs[r], nq, k, C.byref(lp), C.byref(dp))
            if rc:
                return rc
            self.ixs[r].search_bruteforce_dev(dqs[r].data_ptr(), nq, k, EHB_FP32, lp.value, dp.value, sc.data_ptr(),
                                              self.streams[r].cuda_stream)
            return L.ehb_exchange_merge_dev(self.exs[r], _vp(md), _vp(ml), _vp(mc),
                                            C.c_void_p(self.streams[r].cuda_stream))
        return self._on_ranks(call, outs)

    def own(self, q, k, ef, precision, brute=False):
        """Each shard's own beam search (or exact brute force), then ehb_merge_topk_dev: (merged, per-shard)."""
        t = self.torch
        nq = len(q)
        dqs = self._queries(q)
        per = []
        for r in range(self.W):
            t.cuda.set_device(self.devs[r])
            l, d, c = self.out(r, nq, k)
            self._settle()
            s = self.streams[r]
            if brute:
                self.ixs[r].search_bruteforce_dev(dqs[r].data_ptr(), nq, k, EHB_FP32, l.data_ptr(), d.data_ptr(),
                                                  c.data_ptr(), s.cuda_stream)
            else:
                self.ixs[r].search_beam_dev(dqs[r].data_ptr(), nq, k, ef, l.data_ptr(), d.data_ptr(), c.data_ptr(),
                                            s.cuda_stream, precision)
            s.synchronize()
            per.append((l.cpu().numpy().view(np.uint64), d.cpu().numpy(), c.cpu().numpy().view(np.uint32)))
        return self.merge(per, k), per

    def merge(self, per, k):
        t = self.torch
        nq = per[0][0].shape[0]
        t.cuda.set_device(self.devs[0])
        gl = t.from_numpy(np.stack([p[0].view(np.int64) for p in per])).to(self.dev(0))
        gd = t.from_numpy(np.stack([p[1] for p in per])).to(self.dev(0))
        ml, md, mc = self.out(0, nq, k)
        _check(_lib().ehb_merge_topk_dev(len(per), nq, k, _vp(gd), _vp(gl), _vp(md), _vp(ml), _vp(mc), self.devs[0],
                                         None))
        t.cuda.synchronize(self.devs[0])
        return ml.cpu().numpy().view(np.uint64), md.cpu().numpy(), mc.cpu().numpy().view(np.uint32)

    def rows(self, labels):
        """Each label's stored row from the shard that holds it."""
        labels = np.asarray(labels, np.uint64)
        out = np.empty((len(labels), self.d), np.float32)
        for i, lab in enumerate(labels):
            for ix in self.ixs:
                try:
                    out[i] = ix.get(int(lab))
                    break
                except KeyError:
                    pass
            else:
                raise AssertionError(lab)
        return out

    def by_label_reference(self, labels, k, ef, precision):
        """The rule over the fused beam step at k + 1 fed with the owners' rows (which itself is checked against the
        merge of the per-rank beam searches)."""
        rows = self.rows(labels)
        ref, per = self.own(rows, k + 1, ef, precision)
        out = self.fused(rows, k + 1, ef, precision)
        assert_step(out, ref, per, ("by-label reference", k, ef))
        return drop_self(np.asarray(labels, np.uint64), *ref, k)

    def assert_no_timeout(self):
        for r in range(self.W):
            v = C.c_uint32()
            _check(_lib().ehb_exchange_timed_out(self.exs[r], C.byref(v)))
            assert v.value == 0, r


def assert_same(got, want, what):
    gl, gd, gc = got
    wl, wd, wc = want
    assert np.array_equal(np.asarray(gc).astype(np.uint32), np.asarray(wc).astype(np.uint32)), what
    assert np.array_equal(np.asarray(gl).view(np.uint64), np.asarray(wl).view(np.uint64)), what
    assert np.array_equal(np.asarray(gd).view(np.uint32), np.asarray(wd).view(np.uint32)), what


def assert_step(out, ref, per, what):
    """Every rank returned EHB_OK and holds the reference merge; each rank's shard counts are its shard's own."""
    for r, o in enumerate(out):
        assert o[0] == EHB_OK, (what, r, o[0])
        assert_same(o[1:4], ref, (what, r))
        if per is not None and o[4] is not None:
            assert np.array_equal(o[4], per[r][2].astype(np.uint32)), (what, r)


def assert_failed(out, status, what):
    for r, o in enumerate(out):
        assert o[0] == status, (what, r, o[0])
        l, d, c = o[1:4]
        assert (l == SENTINEL_L).all() and (d == np.float32(SENTINEL_D)).all() and (c == SENTINEL_C).all(), (what, r)


def beam_name(ix, bf16):
    name = ix.last_kernel_name()
    assert name.startswith("hnsw_search_beam_kernel<"), name
    assert ("ROW=bf16" in name) == bf16, name


GRID = [(ef, k) for ef in EFS for k in sorted({1, 600, ef})]


# ---- 1. the fused beam step against each rank's own beam search, merged ----------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("d", [64, 768, 3072])
def test_fused_beam_step_equals_merge_of_own_beam_searches(d, metric):
    n, nq = 10000, 37                               # nq = 37: ragged slices
    x, q = gauss(2 * n, d, 11 + d), gauss(nq, d, 12 + d)
    p = Ranks([x[:n], x[n:]], d, metric, nq, 4096)
    try:
        for prec in (EHB_FP32, EHB_BF16):
            refs = {(ef, k): p.own(q, k, ef, prec) for ef, k in sorted(GRID, reverse=True)}
            for ef, k in GRID:
                ref, per = refs[(ef, k)]
                assert_step(p.fused(q, k, ef, prec), ref, per, (prec, ef, k))
                for ix in p.ixs:
                    beam_name(ix, prec == EHB_BF16)
    finally:
        p.close()


def test_fused_beam_step_pads_a_shard_smaller_than_k():
    d, nq = 64, 20
    x, q = gauss(12700, d, 21), gauss(nq, d, 22)
    p = Ranks([x[:12000], x[12000:]], d, "ip", nq, 2049)
    try:
        for prec in (EHB_FP32, EHB_BF16):
            for ef, k in [(2049, 2049), (1057, 1000)]:
                ref, per = p.own(q, k, ef, prec)
                assert np.all(per[1][2] == 700) and np.all(per[1][0][:, 700:] == np.uint64(2**64 - 1))
                assert_step(p.fused(q, k, ef, prec), ref, per, (prec, ef, k))
    finally:
        p.close()


# ---- 2. exact against the oracle on tie-free data ---------------------------------------------------------------------
def test_fused_beam_step_equals_oracle_merge():
    d, n, nq = 64, 16000, 24
    x, q = tiefree(n, d, nq)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    half = n // 2
    p = Ranks([xf[:half], xf[half:]], d, "ip", nq, 4096)
    try:
        oracles = []
        for ix in p.ixs:
            o = orc.OracleHNSW(d, "ip", half)
            o.import_graph(ix.export_graph())
            oracles.append(o)
        cases = [(4096, 4096), (1057, 600), (2049, 1)]
        for ef, k in cases:
            p.own(qf, k, ef, EHB_FP32)
        D = ip_dist(x, q)
        for ef, k in cases:
            per = []
            for o in oracles:
                ol, od, oc = o.search(qf, k, ef=ef, threads=8)
                per.append((ol, od, oc.astype(np.uint32)))
            want = p.merge(per, k)
            ok = want[0] != np.uint64(2**64 - 1)
            exact = np.take_along_axis(D, np.where(ok, want[0], 0).astype(np.int64), 1)
            assert np.array_equal(want[1][ok].view(np.uint32), exact[ok].view(np.uint32))
            assert_step(p.fused(qf, k, ef, EHB_FP32), want, per, (ef, k))
    finally:
        p.close()


# ---- 3. tombstones ----------------------------------------------------------------------------------------------------
def test_fused_beam_step_with_tombstones():
    d, n, nq = 128, 10000, 30
    x, q = gauss(2 * n, d, 31), gauss(nq, d, 32)
    p = Ranks([x[:n], x[n:]], d, "cosine", nq, 2049)
    try:
        rng = np.random.default_rng(33)
        entry = p.ixs[0].stats()["entry_point"]
        dead = np.union1d(rng.choice(n, n // 10, replace=False), [entry]).astype(np.uint64)
        p.ixs[0].remove(dead)                       # shard 0's labels are its internal ids 0 .. n-1
        for prec in (EHB_FP32, EHB_BF16):
            refs = {kef: p.own(q, kef[1], kef[0], prec) for kef in [(2049, 2049), (1057, 600)]}
            for (ef, k), (ref, per) in refs.items():
                out = p.fused(q, k, ef, prec)
                assert_step(out, ref, per, (prec, ef, k))
                assert not np.isin(out[0][1], dead).any()
                assert "HASDEL=1" in p.ixs[0].last_kernel_name()
    finally:
        p.close()


# ---- 4. by label --------------------------------------------------------------------------------------------------------
def test_by_label_beam_step_equals_composition_and_fails_alike():
    d, n = 64, 8000
    x = gauss(2 * n, d, 41)
    # label 5 is stored on both ranks (rank 1's first row), label 2n + 9 nowhere
    labels = [np.arange(n, dtype=np.uint64), np.concatenate([[5], np.arange(n + 1, 2 * n)]).astype(np.uint64)]
    p = Ranks([x[:n], x[n:]], d, "l2", 16, 4096, labels=labels)
    rng = np.random.default_rng(42)
    batch = np.concatenate([rng.choice(np.arange(6, n), 6, replace=False),
                            rng.choice(np.arange(n + 1, 2 * n), 6, replace=False), [7, n + 3]]).astype(np.uint64)
    try:
        for prec in (EHB_FP32, EHB_BF16):             # the scratch of the widest beam at the largest batch below
            p.own(gauss(16, d, 43), 4096, 4096, prec)
        cases = [(4095, 4095, EHB_FP32), (1057, 600, EHB_BF16), (2049, 1, EHB_FP32)]
        refs = {}
        for ef, k, prec in cases:
            refs[(ef, k, prec)] = p.by_label_reference(batch, k, ef, prec)
        for ef, k, prec in cases:
            assert_step(p.by_label(batch, k, ef, prec), refs[(ef, k, prec)], None, (ef, k, prec))
        ef, k, prec = cases[1]
        other = batch.copy()
        other[0] = 9
        assert_failed(p.by_label(batch, k, ef, prec, per_rank=[batch, other]), EHB_ERR_INVALID, "lists differ")
        assert_failed(p.by_label(np.append(batch, 2 * n + 9), k, ef, prec), EHB_ERR_NOT_FOUND, "missing")
        assert_failed(p.by_label(np.append(batch, 5), k, ef, prec), EHB_ERR_STATE, "two owners")
        assert_step(p.by_label(batch, k, ef, prec), refs[(ef, k, prec)], None, "after the failures")
    finally:
        p.close()


# ---- 5. up to 512 the new calls are their _ex counterparts ------------------------------------------------------------
def test_up_to_512_every_beam_call_equals_its_ex_counterpart():
    d, n, nq = 128, 6000, 40
    x, q = gauss(2 * n, d, 51), gauss(nq, d, 52)
    p = Ranks([x[:n], x[n:]], d, "ip", nq, 512)
    batch = np.random.default_rng(53).choice(2 * n, 12, replace=False).astype(np.uint64)
    try:
        for prec in (EHB_FP32, EHB_BF16):
            for k, ef in [(10, 64), (100, 512), (512, 0), (1, 300)]:
                p.own(q, k, ef, prec)
                ex = p.fused(q, k, ef, prec, step="ehb_exchange_search_ex_dev")
                names = [ix.last_kernel_name() for ix in p.ixs]
                bm = p.fused(q, k, ef, prec)
                assert names == [ix.last_kernel_name() for ix in p.ixs]
                assert not names[0].startswith("hnsw_search_beam_kernel")
                assert_step(bm, ex[0][1:4], [(None, None, o[4]) for o in ex], (prec, k, ef))
                if k < 512:
                    p.by_label_reference(batch, k, ef, prec)          # sizes the k + 1 searches
                    ex = p.by_label(batch, k, ef, prec, step="ehb_exchange_search_by_label_ex_dev")
                    assert_step(p.by_label(batch, k, ef, prec), ex[0][1:4], None, ("by label", prec, k, ef))
    finally:
        p.close()


# ---- 6. step kinds interleave on one exchange of three ranks ----------------------------------------------------------
def test_step_kinds_interleave_on_three_ranks():
    d, n, nq, k, ef = 64, 7000, 24, 700, 1057
    x, q = gauss(3 * n, d, 61), gauss(nq, d, 62)
    p = Ranks([x[:n], x[n:2 * n], x[2 * n:]], d, "l2", nq, 4096)
    batch = np.random.default_rng(63).choice(3 * n, nq, replace=False).astype(np.uint64)
    try:
        beam = p.own(q, k, ef, EHB_BF16)
        narrow = p.own(q, 50, 128, EHB_FP32)
        brute = p.own(q, 100, 0, EHB_FP32, brute=True)
        label = p.by_label_reference(batch, k, ef, EHB_FP32)
        for step in range(2):
            assert_step(p.fused(q, k, ef, EHB_BF16), *beam, ("beam", step))
            assert_step(p.fused(q, 50, 128, EHB_FP32, step="ehb_exchange_search_ex_dev"), *narrow, ("ex", step))
            assert_step(p.by_label(batch, k, ef, EHB_FP32), label, None, ("by label", step))
            assert_step(p.brute(q, 100), *brute, ("brute", step))
    finally:
        p.close()


# ---- 7. rejections fail before the step starts ---------------------------------------------------------------------------
def test_rejections_leave_outputs_untouched_and_ranks_in_phase():
    d, n, nq = 64, 5000, 20
    x, q = gauss(2 * n, d, 71), gauss(nq, d, 72)
    p = Ranks([x[:n], x[n:]], d, "l2", nq, 1024, max_dim=d - 4)   # no room for rows of dim d: by label is rejected
    try:
        ref = p.own(q, 1024, 1057, EHB_FP32)
        for what, kw in [("precision", dict(precision=7)), ("null", dict(null_out=True)),
                         ("ef", dict(ef=4097)), ("capacity", dict(k=1025, ef=2049))]:
            args = dict(k=1024, ef=1057, precision=EHB_FP32)
            args.update(kw)
            null_out = args.pop("null_out", False)
            out = p.fused(q, args["k"], args["ef"], args["precision"], null_out=null_out)
            assert_failed(out, EHB_ERR_INVALID, what)
            assert_step(p.fused(q, 1024, 1057, EHB_FP32), *ref, ("after", what))
        assert_failed(p.fused(q[:1], 4097, 0, EHB_FP32), EHB_ERR_INVALID, "k 4097")
        lab = np.arange(4, dtype=np.uint64)
        for what, (k, ef, prec) in [("precision", (10, 600, 7)), ("k 4096", (4096, 0, EHB_FP32)),
                                    ("ef 4097", (10, 4097, EHB_FP32)), ("max_dim", (10, 600, EHB_FP32))]:
            assert_failed(p.by_label(lab, k, ef, prec), EHB_ERR_INVALID, ("by label", what))
            assert_step(p.fused(q, 1024, 1057, EHB_FP32), *ref, ("after by label", what))
    finally:
        p.close()


# ---- 8. the one-process sharded index -------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [EHB_FP32, EHB_BF16])
def test_sharded_index_beam_equals_merge_of_shard_beams(prec):
    d, n, nq = 96, 16000, 30
    x, q = gauss(n, d, 81), gauss(nq, d, 82)
    sh = _ehb().ShardedIndex(d, _devices(2), metric="ip", capacity=n)
    sh.add(x, np.arange(n, dtype=np.uint64))
    sh.build()
    p = Ranks.__new__(Ranks)                        # only its merge
    import torch
    p.torch, p.devs, p.W = torch, _devices(2), 2
    try:
        for ef, k in [(1057, 600), (4096, 4096), (2049, 1)]:
            per = [sh.shard(i).search_beam(q, k, ef=ef, precision=prec) for i in range(2)]
            want = p.merge(per, k)
            assert_same(sh.search_beam(q, k, ef=ef, precision=prec), want, (ef, k))
        batch = np.random.default_rng(83).choice(n, 10, replace=False).astype(np.uint64)
        for ef, k in [(1057, 600), (4096, 4095)]:
            rows = sh.get_batch(batch)
            want = drop_self(batch, *sh.search_beam(rows, k + 1, ef=ef, precision=prec), k)
            assert_same(sh.search_by_label_beam(batch, k, ef=ef, precision=prec), want, ("by label", ef, k))
        for ef, k in [(64, 10), (512, 100)]:
            assert_same(sh.search_beam(q, k, ef=ef, precision=prec), sh.search(q, k, ef=ef, precision=prec), (ef, k))
            assert_same(sh.search_by_label_beam(batch, k, ef=ef, precision=prec),
                        sh.search_by_label(batch, k, ef=ef, precision=prec), ("by label", ef, k))
        with pytest.raises(_ehb().EhbError):
            sh.search_beam(q, 10, ef=4097, precision=prec)
        with pytest.raises(_ehb().EhbError):
            sh.search_by_label_beam(batch, 4096, ef=0, precision=prec)
    finally:
        sh.close()


# ---- 9. ShardedSearcher at world 1 ---------------------------------------------------------------------------------------
def test_sharded_searcher_world1_beam_equals_native_beam():
    import torch
    from embeddinghub_b200.sharded import ShardedSearcher
    d, n, nq, k, ef = 128, 12000, 40, 700, 2049
    x, q = gauss(n, d, 91), gauss(nq, d, 92)
    ix = _ehb().NativeIndex(d, metric="l2", capacity=n)
    ix.add(x)
    ix.build()
    s = ShardedSearcher(ix, 1, 0)
    dq = torch.from_numpy(q).cuda()
    stream = torch.cuda.Stream()
    batch = np.arange(0, n, n // 9, dtype=np.uint64)
    for prec in (EHB_FP32, EHB_BF16):
        want = ix.search_beam(q, k, ef=ef, precision=prec)
        stream.wait_stream(torch.cuda.current_stream())
        ml, md, mc = s.search_beam_dev(dq, k, ef, stream.cuda_stream, precision=prec)
        stream.synchronize()
        beam_name(ix, prec == EHB_BF16)
        assert_same((ml.cpu().numpy(), md.cpu().numpy(), mc.cpu().numpy()), want, ("world 1", prec))
        want = ix.search_by_label_beam(batch, k, ef=ef, precision=prec)
        ml, md, mc = s.search_by_label_beam_dev(batch, k, ef, stream.cuda_stream, precision=prec)
        stream.synchronize()
        assert_same((ml.cpu().numpy(), md.cpu().numpy(), mc.cpu().numpy()), want, ("world 1 by label", prec))
