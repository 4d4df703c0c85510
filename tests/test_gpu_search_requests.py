"""Every search entry point checks its request the same way, before it touches the index: an unknown precision, then a
null buffer, then k == 0 or nq == 0 (nothing to do), then the width (max(ef or the index default, k) <= 512 for the
graph walk, k <= 2048 for the brute force, k + 1 for the by-label forms).  Each rejected call returns
EHB_ERR_INVALID and leaves the output buffers as they were; the by-label forms reject before they look up a label."""
import ctypes as C
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import embeddinghub_b200 as ehb  # noqa: E402
from embeddinghub_b200._native import BF16, FP32, _p, lib  # noqa: E402
from test_gpu_exchange_bf16 import Pair  # noqa: E402

EHB_ERR_INVALID = 1
N, D, NQ = 600, 64, 4

# entry point -> (engine, queries are labels, where the results go)
ENTRIES = {
    "search_ex": ("walk", False, "host"),
    "search_ex_dev": ("walk", False, "dev"),
    "search_by_label_ex": ("walk", True, "host"),
    "neighbor_table": ("walk", True, "table"),
    "exchange_search_ex_dev": ("walk", False, "exchange"),
    "sharded_search_ex": ("walk", False, "sharded"),
    "sharded_search_by_label_ex": ("walk", True, "sharded"),
    "search_bruteforce": ("brute", False, "host"),
    "search_bruteforce_dev": ("brute", False, "dev"),
    "search_bruteforce_by_label": ("brute", True, "host"),
    "sharded_search_bruteforce": ("brute", False, "sharded"),
}
CASES = ["precision", "precision_k0", "null_query", "null_out", "ef513", "k_over_limit", "ef0_default600"]
PARAMS = [(e, c) for e, c in itertools.product(ENTRIES, CASES) if ENTRIES[e][0] == "walk" or not c.startswith("ef")]


@pytest.fixture(scope="module")
def env():
    x = np.random.default_rng(1).standard_normal((2 * N, D), dtype=np.float32)
    ix = ehb.NativeIndex(D, capacity=N)
    ix.add(x[:N])
    ix.build()
    sh = ehb.ShardedIndex(D, [0, 0], capacity=N)
    sh.add(x[:N])
    sh.build()
    pair = Pair([x[:N], x[N:]], D, "l2", NQ, 600)
    yield ix, sh, pair, x[:NQ] + 0.01
    pair.close()
    sh.close()
    ix.close()


def request(entry, case):
    """(precision, k, ef, query pointer present, output pointer present) of one case."""
    engine, by_label = ENTRIES[entry][:2]
    k = 5
    if case == "k_over_limit":
        k = (512 if engine == "walk" else 2048) + 1 - by_label
    return (7 if case.startswith("precision") else FP32, 0 if case == "precision_k0" else k,
            {"ef513": 513}.get(case, 0 if case == "ef0_default600" else 32), case != "null_query", case != "null_out")


def set_default_ef(ix, sh, pair, ef):
    for i in [ix] + pair.ixs:
        i.set_ef(ef)
    lib().ehb_sharded_set_ef(sh._h, ef)


@pytest.mark.parametrize("entry,case", PARAMS)
def test_rejected_request_leaves_outputs_untouched(env, entry, case):
    import torch
    ix, sh, pair, q = env
    engine, by_label, where = ENTRIES[entry]
    precision, k, ef, has_q, has_out = request(entry, case)
    L = lib()
    rows = N if where == "table" else NQ
    w = max(k, 1)
    hl, hd, hc = np.full((rows, w), 77, np.uint64), np.full((rows, w), 7.5, np.float32), np.full(rows, 9, np.uint32)
    hq = np.full(rows, 55, np.uint64)
    # one label is not stored: a call that resolved or gathered the rows before its checks would fail with
    # EHB_ERR_NOT_FOUND instead
    labels = np.array([1, 2, 3, 10 ** 9], np.uint64)
    qp = (_p(labels) if by_label else _p(q)) if has_q else None
    ol, od, oc = (_p(hl) if has_out else None), _p(hd), _p(hc)
    if case == "ef0_default600":
        set_default_ef(ix, sh, pair, 600)
    try:
        if where in ("dev", "exchange"):
            ranks = [0, 1] if where == "exchange" else [0]
            outs = []
            for r in ranks:
                dev = f"cuda:{pair.devs[r]}"
                torch.cuda.set_device(dev)
                dq = torch.from_numpy(q).to(dev)
                t = (torch.full((NQ, w), 77, dtype=torch.int64, device=dev),
                     torch.full((NQ, w), 7.5, dtype=torch.float32, device=dev),
                     torch.full((NQ,), 9, dtype=torch.int32, device=dev))
                outs.append(t)
                dqp = C.c_void_p(dq.data_ptr()) if has_q else None
                dl = C.c_void_p(t[0].data_ptr()) if has_out else None
                dd, dc = C.c_void_p(t[1].data_ptr()), C.c_void_p(t[2].data_ptr())
                if where == "exchange":
                    rc = L.ehb_exchange_search_ex_dev(pair.exs[r], pair.ixs[r]._h, NQ, dqp, k, ef, precision, dd, dl,
                                                      dc, None, C.c_void_p(pair.streams[r].cuda_stream))
                elif engine == "walk":
                    rc = L.ehb_index_search_ex_dev(ix._h, NQ, dqp, k, ef, precision, dl, dd, dc, None)
                else:
                    rc = L.ehb_index_search_bruteforce_dev(ix._h, NQ, dqp, k, precision, dl, dd, dc, None)
                assert rc == EHB_ERR_INVALID, (entry, case, r)
            torch.cuda.synchronize()
            for t in outs:
                assert (t[0] == 77).all() and (t[1] == 7.5).all() and (t[2] == 9).all(), (entry, case)
            return
        if where == "table":
            got = C.c_uint64(N)
            rc = L.ehb_index_neighbor_table(ix._h, k, ef, precision, _p(hq) if has_q else None, ol, od, oc,
                                            C.byref(got))
            assert got.value == N and (hq == 55).all()
        else:
            fn = {"search_ex": lambda: L.ehb_index_search_ex(ix._h, NQ, qp, k, ef, precision, ol, od, oc),
                  "search_by_label_ex": lambda: L.ehb_index_search_by_label_ex(ix._h, NQ, qp, k, ef, precision, ol, od,
                                                                               oc),
                  "search_bruteforce": lambda: L.ehb_index_search_bruteforce(ix._h, NQ, qp, k, precision, ol, od, oc),
                  "search_bruteforce_by_label": lambda: L.ehb_index_search_bruteforce_by_label(ix._h, NQ, qp, k,
                                                                                               precision, ol, od, oc),
                  "sharded_search_ex": lambda: L.ehb_sharded_search_ex(sh._h, NQ, qp, k, ef, precision, ol, od, oc),
                  "sharded_search_by_label_ex": lambda: L.ehb_sharded_search_by_label_ex(sh._h, NQ, qp, k, ef,
                                                                                         precision, ol, od, oc),
                  "sharded_search_bruteforce": lambda: L.ehb_sharded_search_bruteforce(sh._h, NQ, qp, k, precision, ol,
                                                                                       od, oc)}[entry]
            rc = fn()
        assert rc == EHB_ERR_INVALID, (entry, case)
        assert (hl == 77).all() and (hd == 7.5).all() and (hc == 9).all(), (entry, case)
    finally:
        if case == "ef0_default600":
            set_default_ef(ix, sh, pair, 10)


def test_rejected_bf16_dev_search_creates_no_bf16_copy():
    import torch
    ix = ehb.NativeIndex(D, metric="ip", capacity=N)
    ix.add(np.random.default_rng(2).standard_normal((N, D), dtype=np.float32))
    ix.build()
    q = np.random.default_rng(3).standard_normal((NQ, D), dtype=np.float32)
    before = ix.stats()["device_bytes"]
    dq = torch.from_numpy(q).cuda()
    dl = torch.empty((NQ, 5), dtype=torch.int64, device="cuda")
    rc = lib().ehb_index_search_ex_dev(ix._h, NQ, C.c_void_p(dq.data_ptr()), 5, 513, BF16,
                                       C.c_void_p(dl.data_ptr()), None, None, None)
    assert rc == EHB_ERR_INVALID
    assert ix.stats()["device_bytes"] == before
    ix.search(q, 5, 64, BF16)  # an accepted bf16 search does create it
    assert ix.stats()["device_bytes"] > before
