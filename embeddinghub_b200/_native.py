"""ctypes binding of the ehb200 C ABI (include/ehb200.h).

There is no CPU fallback: importing works anywhere (so the ABI can be checked on
a CPU-only box), but every compute call raises EhbError when the CUDA library is
missing or no H100-class (sm_90) device is present.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("EHB200_LIB") or os.path.join(_HERE, "libehb200.so")  # EHB200_LIB: A/B builds (tools/)

NO_LABEL = np.uint64(0xFFFFFFFFFFFFFFFF)
METRICS = {"l2": 0, "ip": 1, "cosine": 2}
FP32, BF16 = 0, 1


class EhbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"ehb200 error {code}: {msg}")
        self.code = code


class Params(C.Structure):
    _fields_ = [
        ("dim", C.c_uint32),
        ("metric", C.c_int32),
        ("capacity", C.c_uint64),
        ("M", C.c_uint32),
        ("ef_construction", C.c_uint32),
        ("ef_search", C.c_uint32),
        ("seed", C.c_uint64),
        ("device", C.c_int32),
        ("build_batch", C.c_uint32),
        ("reserved", C.c_uint32 * 6),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("queries", C.c_uint64),
        ("hops_upper", C.c_uint64),
        ("hops_base", C.c_uint64),
        ("dist_evals", C.c_uint64),
        ("visited_overflow", C.c_uint64),
        ("algorithmic_bytes", C.c_uint64),
        ("size", C.c_uint64),
        ("capacity", C.c_uint64),
        ("upper_rows", C.c_uint64),
        ("dim", C.c_uint32),
        ("M", C.c_uint32),
        ("max_level", C.c_uint32),
        ("entry_point", C.c_uint32),
        ("device_bytes", C.c_uint64),
        ("deleted", C.c_uint64),
        ("combined_batches", C.c_uint64),
        ("combined_queries", C.c_uint64),
        ("metric", C.c_uint32),
        ("reserved_", C.c_uint32),
    ]


# name -> (restype, argtypes); every symbol include/ehb200.h declares
_VP, _U64, _U32, _I32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32
SYMBOLS = {
    "ehb_last_error": (C.c_char_p, []),
    "ehb_abi_version": (_U32, []),
    "ehb_params_default": (None, [C.POINTER(Params), _U32]),
    "ehb_device_count": (C.c_int, [C.POINTER(_I32)]),
    "ehb_index_create": (C.c_int, [C.POINTER(Params), C.POINTER(_VP)]),
    "ehb_index_destroy": (C.c_int, [_VP]),
    "ehb_index_add": (C.c_int, [_VP, _U64, _VP, _VP]),
    "ehb_index_add_dev": (C.c_int, [_VP, _U64, _VP, _VP]),
    "ehb_index_build": (C.c_int, [_VP]),
    "ehb_index_remove": (C.c_int, [_VP, _U64, _VP]),
    "ehb_index_compact": (C.c_int, [_VP]),
    "ehb_index_set_ef": (C.c_int, [_VP, _U32]),
    "ehb_index_size": (C.c_int, [_VP, C.POINTER(_U64)]),
    "ehb_index_get": (C.c_int, [_VP, _U64, _VP]),
    "ehb_index_search": (C.c_int, [_VP, _U64, _VP, _U32, _U32, _VP, _VP, _VP]),
    "ehb_index_search_dev": (C.c_int, [_VP, _U64, _VP, _U32, _U32, _VP, _VP, _VP, _VP]),
    "ehb_index_search_ex": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_search_ex_dev": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP]),
    "ehb_index_search_bruteforce": (C.c_int, [_VP, _U64, _VP, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_search_bruteforce_dev": (C.c_int, [_VP, _U64, _VP, _U32, C.c_int, _VP, _VP, _VP, _VP]),
    "ehb_index_get_batch": (C.c_int, [_VP, _U64, _VP, _VP]),
    "ehb_index_search_by_label_ex": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_search_bruteforce_by_label": (C.c_int, [_VP, _U64, _VP, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_search_beam": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_search_beam_dev": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP]),
    "ehb_index_search_by_label_beam": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_index_neighbor_table": (C.c_int, [_VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP, C.POINTER(_U64)]),
    "ehb_index_stats": (C.c_int, [_VP, C.POINTER(Stats)]),
    "ehb_index_screen_stats": (C.c_int, [_VP, C.POINTER(_U64), C.POINTER(_U64)]),
    "ehb_index_last_kernel_ms": (C.c_int, [_VP, C.POINTER(C.c_float)]),
    "ehb_index_last_kernel_name": (C.c_int, [_VP, C.c_char_p, _U32]),
    "ehb_index_export_graph": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, C.POINTER(_U32), C.POINTER(_I32)]),
    "ehb_index_import_graph": (C.c_int, [_VP, _U64, _VP, _VP, _VP, _VP, _VP, _U64, _VP, _U32, _I32]),
    "ehb_index_save": (C.c_int, [_VP, C.c_char_p]),
    "ehb_index_load": (C.c_int, [C.c_char_p, _I32, C.POINTER(_VP)]),
    "ehb_merge_topk_dev": (C.c_int, [_U32, _U64, _U32, _VP, _VP, _VP, _VP, _VP, _I32, _VP]),
    "ehb_merge_topk_packed_dev": (C.c_int, [_U32, _U64, _U32, _VP, _U64, _VP, _VP, _VP, _I32, _VP]),
    "ehb_index_set_tuning": (C.c_int, [_VP, _U32, _U32, _U32, _U32]),
    "ehb_index_set_search_width": (C.c_int, [_VP, _U32]),
    "ehb_index_set_option": (C.c_int, [_VP, C.c_char_p, C.c_int64]),
    "ehb_sharded_create": (C.c_int, [C.POINTER(Params), C.POINTER(_I32), _U32, _U64, C.POINTER(_VP)]),
    "ehb_sharded_destroy": (C.c_int, [_VP]),
    "ehb_sharded_n_shards": (C.c_int, [_VP, C.POINTER(_U32)]),
    "ehb_sharded_shard": (C.c_int, [_VP, _U32, C.POINTER(_VP)]),
    "ehb_sharded_add": (C.c_int, [_VP, _U64, _VP, _VP]),
    "ehb_sharded_remove": (C.c_int, [_VP, _U64, _VP]),
    "ehb_sharded_get": (C.c_int, [_VP, _U64, _VP]),
    "ehb_sharded_size": (C.c_int, [_VP, C.POINTER(_U64)]),
    "ehb_sharded_build": (C.c_int, [_VP]),
    "ehb_sharded_compact": (C.c_int, [_VP]),
    "ehb_sharded_set_ef": (C.c_int, [_VP, _U32]),
    "ehb_sharded_search": (C.c_int, [_VP, _U64, _VP, _U32, _U32, _VP, _VP, _VP]),
    "ehb_sharded_search_ex": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_sharded_search_bruteforce": (C.c_int, [_VP, _U64, _VP, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_sharded_get_batch": (C.c_int, [_VP, _U64, _VP, _VP]),
    "ehb_sharded_search_by_label_ex": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_sharded_search_beam": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_sharded_search_by_label_beam": (C.c_int, [_VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP]),
    "ehb_exchange_create": (C.c_int, [_I32, _U32, _U32, _U64, _U32, C.POINTER(_VP)]),
    "ehb_exchange_create_ex": (C.c_int, [_I32, _U32, _U32, _U64, _U32, _U32, C.POINTER(_VP)]),
    "ehb_exchange_destroy": (C.c_int, [_VP]),
    "ehb_exchange_ipc_handle": (C.c_int, [_VP, _VP]),
    "ehb_exchange_open": (C.c_int, [_VP, _VP]),
    "ehb_exchange_attach_local": (C.c_int, [_VP, _U32, _VP]),
    "ehb_exchange_begin": (C.c_int, [_VP, _U64, _U32, C.POINTER(_VP), C.POINTER(_VP)]),
    "ehb_exchange_merge_dev": (C.c_int, [_VP, _VP, _VP, _VP, _VP]),
    "ehb_exchange_search_dev": (C.c_int, [_VP, _VP, _U64, _VP, _U32, _U32, _VP, _VP, _VP, _VP, _VP]),
    "ehb_exchange_search_ex_dev": (C.c_int, [_VP, _VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP, _VP]),
    "ehb_exchange_search_by_label_ex_dev": (C.c_int, [_VP, _VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP]),
    "ehb_exchange_search_beam_dev": (C.c_int, [_VP, _VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP, _VP, _VP]),
    "ehb_exchange_search_by_label_beam_dev": (C.c_int, [_VP, _VP, _U64, _VP, _U32, _U32, C.c_int, _VP, _VP, _VP,
                                                        _VP]),
    "ehb_exchange_timed_out": (C.c_int, [_VP, C.POINTER(_U32)]),
}

_LIB = None


def lib():
    """Loads libehb200.so (built in-tree by `make` / __graft_entry__.build())."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise EhbError(-1, f"{LIB_PATH} is missing: run `make` (nvcc, sm_90a). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc):
    if rc != 0:
        raise EhbError(rc, lib().ehb_last_error().decode(errors="replace"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _check_key(rc, labels):
    if rc == 5:
        raise KeyError(labels)
    check(rc)


def _alloc(nq, k):
    """Result buffers of nq queries at k; the counts start at 0, which is what a call with k == 0 leaves them."""
    return np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32), np.zeros(nq, np.uint32)


class NativeIndex:
    """Thin owner of an ehb_index handle; numpy in / numpy out (host entry points)."""

    def __init__(self, dim, metric="l2", capacity=128, M=16, ef_construction=200, ef_search=10, seed=100, device=0,
                 build_batch=0, _handle=None):
        L = lib()
        self.dim = int(dim)
        self.metric = metric
        self.M = int(M)
        if _handle is not None:
            self._h = _handle
            return
        p = Params()
        L.ehb_params_default(C.byref(p), self.dim)
        p.metric = METRICS[metric]
        p.capacity = int(capacity)
        p.M = int(M)
        p.ef_construction = int(ef_construction)
        p.ef_search = int(ef_search)
        p.seed = int(seed)
        p.device = int(device)
        p.build_batch = int(build_batch)
        h = C.c_void_p()
        check(L.ehb_index_create(C.byref(p), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            if getattr(self, "_owned", True):
                lib().ehb_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- mutation ---------------------------------------------------------------
    def add(self, vecs, labels=None):
        v = np.ascontiguousarray(vecs, dtype=np.float32).reshape(-1, self.dim)
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.uint64)
        if lab is not None and lab.shape[0] != v.shape[0]:
            raise ValueError("labels/vectors length mismatch")
        check(lib().ehb_index_add(self._h, v.shape[0], _p(v), _p(lab)))

    def add_dev(self, dev_ptr, n, labels=None):
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.uint64)
        check(lib().ehb_index_add_dev(self._h, int(n), C.c_void_p(int(dev_ptr)), _p(lab)))

    def build(self):
        check(lib().ehb_index_build(self._h))

    def remove(self, labels):
        """Tombstones (hnswlib markDelete): KeyError for an unknown label."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        _check_key(lib().ehb_index_remove(self._h, lab.shape[0], _p(lab)), labels)

    def compact(self):
        """Drops every tombstone and repairs the graph on the GPU: size() counts the survivors, labels and vectors
        are kept, internal ids change, capacity is kept (ehb_index_compact)."""
        check(lib().ehb_index_compact(self._h))

    def set_ef(self, ef):
        check(lib().ehb_index_set_ef(self._h, int(ef)))

    def set_tuning(self, stage_slots=0, stage_groups=0, hash_bits=0, warps_per_block=0):
        check(lib().ehb_index_set_tuning(self._h, stage_slots, stage_groups, hash_bits, warps_per_block))

    def set_option(self, name, value):
        check(lib().ehb_index_set_option(self._h, name.encode(), int(value)))

    def set_search_width(self, warps_per_query):
        check(lib().ehb_index_set_search_width(self._h, int(warps_per_query)))

    # -- queries ------------------------------------------------------------------
    @property
    def size(self):
        n = C.c_uint64()
        check(lib().ehb_index_size(self._h, C.byref(n)))
        return n.value

    def get(self, label):
        out = np.empty(self.dim, np.float32)
        _check_key(lib().ehb_index_get(self._h, int(label), _p(out)), label)
        return out

    def get_batch(self, labels):
        """The stored rows of `labels` ([n][dim]), each exactly as get() returns it; KeyError for an unknown or
        deleted label (ehb_index_get_batch)."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out = np.empty((lab.shape[0], self.dim), np.float32)
        _check_key(lib().ehb_index_get_batch(self._h, lab.shape[0], _p(lab), _p(out)), labels)
        return out

    def search(self, q, k, ef=0, precision=FP32):
        """Graph search.  precision=BF16 walks the bf16 copy of the rows and re-ranks the walk's whole result set
        in fp32: every distance is the exact fp32 one (ehb_index_search_ex)."""
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_index_search_ex(self._h, q.shape[0], _p(q), k, ef, int(precision), _p(labels), _p(dists),
                                        _p(counts)))
        return labels, dists, counts

    def search_beam(self, q, k, ef=0, precision=FP32):
        """search() with max(ef, k) up to EHB_MAX_BEAM = 4096: above 512 the wide-beam walk, which keeps hnswlib's
        order and stop rule (ehb_index_search_beam); up to 512 exactly search()."""
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_index_search_beam(self._h, q.shape[0], _p(q), k, ef, int(precision), _p(labels), _p(dists),
                                          _p(counts)))
        return labels, dists, counts

    def search_beam_dev(self, q_ptr, nq, k, ef, labels_ptr, dists_ptr, counts_ptr, stream=0, precision=FP32):
        """search_dev() with max(ef, k) up to 4096 (ehb_index_search_beam_dev)."""
        check(lib().ehb_index_search_beam_dev(self._h, nq, C.c_void_p(q_ptr), k, ef, int(precision),
                                              C.c_void_p(labels_ptr),
                                              C.c_void_p(dists_ptr) if dists_ptr else None,
                                              C.c_void_p(counts_ptr) if counts_ptr else None,
                                              C.c_void_p(stream) if stream else None))

    def search_by_label_beam(self, labels, k, ef=0, precision=FP32):
        """search_by_label() with max(ef, k + 1) up to 4096 (ehb_index_search_by_label_beam)."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out_l, out_d, out_c = _alloc(lab.shape[0], k)
        _check_key(lib().ehb_index_search_by_label_beam(self._h, lab.shape[0], _p(lab), k, ef, int(precision),
                                                        _p(out_l), _p(out_d), _p(out_c)), labels)
        return out_l, out_d, out_c

    def search_bruteforce(self, q, k, precision=FP32):
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_index_search_bruteforce(self._h, q.shape[0], _p(q), k, precision, _p(labels), _p(dists),
                                                _p(counts)))
        return labels, dists, counts

    def search_by_label(self, labels, k, ef=0, precision=FP32):
        """Key mode of the reference's NearestNeighbor (server.cc:190-207): each stored point's k nearest other points.
        The point's row is searched at k + 1; its own label is removed, or the last hit dropped when it is absent
        (ehb_index_search_by_label_ex).  KeyError for an unknown or deleted label."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out_l, out_d, out_c = _alloc(lab.shape[0], k)
        _check_key(lib().ehb_index_search_by_label_ex(self._h, lab.shape[0], _p(lab), k, ef, int(precision), _p(out_l),
                                                      _p(out_d), _p(out_c)), labels)
        return out_l, out_d, out_c

    def search_bruteforce_by_label(self, labels, k, precision=FP32):
        """search_by_label over the exact (or bf16) brute force at k + 1 (ehb_index_search_bruteforce_by_label)."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out_l, out_d, out_c = _alloc(lab.shape[0], k)
        _check_key(lib().ehb_index_search_bruteforce_by_label(self._h, lab.shape[0], _p(lab), k, int(precision),
                                                              _p(out_l), _p(out_d), _p(out_c)), labels)
        return out_l, out_d, out_c

    def neighbor_table(self, k, ef=0, precision=FP32):
        """(query_labels, labels, dists, counts): search_by_label of every live point, rows in internal-id order
        (ehb_index_neighbor_table; option "table_chunk" sets the batch)."""
        st = self.stats()
        rows = st["size"] - st["deleted"]
        q = np.empty(rows, np.uint64)
        out_l, out_d, out_c = _alloc(rows, k)
        got = C.c_uint64(rows)
        check(lib().ehb_index_neighbor_table(self._h, k, ef, int(precision), _p(q), _p(out_l), _p(out_d), _p(out_c),
                                             C.byref(got)))
        n = got.value if k else 0
        return q[:n], out_l[:n], out_d[:n], out_c[:n]

    def search_dev(self, q_ptr, nq, k, ef, labels_ptr, dists_ptr, counts_ptr, stream=0, precision=FP32):
        check(lib().ehb_index_search_ex_dev(self._h, nq, C.c_void_p(q_ptr), k, ef, int(precision),
                                            C.c_void_p(labels_ptr),
                                            C.c_void_p(dists_ptr) if dists_ptr else None,
                                            C.c_void_p(counts_ptr) if counts_ptr else None,
                                            C.c_void_p(stream) if stream else None))

    def search_bruteforce_dev(self, q_ptr, nq, k, precision, labels_ptr, dists_ptr, counts_ptr, stream=0):
        check(lib().ehb_index_search_bruteforce_dev(self._h, nq, C.c_void_p(q_ptr), k, precision,
                                                    C.c_void_p(labels_ptr),
                                                    C.c_void_p(dists_ptr) if dists_ptr else None,
                                                    C.c_void_p(counts_ptr) if counts_ptr else None,
                                                    C.c_void_p(stream) if stream else None))

    def stats(self):
        s = Stats()
        check(lib().ehb_index_stats(self._h, C.byref(s)))
        out = {f: getattr(s, f) for f, _ in Stats._fields_}
        screened, fp32_rows = C.c_uint64(), C.c_uint64()
        check(lib().ehb_index_screen_stats(self._h, C.byref(screened), C.byref(fp32_rows)))
        out["screened_evals"], out["fp32_row_reads"] = screened.value, fp32_rows.value
        return out

    def last_kernel_ms(self):
        ms = C.c_float()
        check(lib().ehb_index_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def last_kernel_name(self):
        buf = C.create_string_buffer(96)
        check(lib().ehb_index_last_kernel_name(self._h, buf, 96))
        return buf.value.decode()

    # -- graph exchange -------------------------------------------------------------
    def export_graph(self):
        self.build()
        st = self.stats()
        n, rows, M = st["size"], st["upper_rows"], self.M
        g = {
            "vectors": np.empty((n, self.dim), np.float32),
            "labels": np.empty(n, np.uint64),
            "levels": np.empty(n, np.uint8),
            "links0": np.empty((n, 2 * M), np.uint32),
            "up_off": np.empty(n, np.uint32),
            "links_up": np.empty((max(rows, 1), M), np.uint32),
        }
        e, ml = C.c_uint32(), C.c_int32()
        check(lib().ehb_index_export_graph(self._h, _p(g["vectors"]), _p(g["labels"]), _p(g["levels"]),
                                           _p(g["links0"]), _p(g["up_off"]), _p(g["links_up"]), C.byref(e),
                                           C.byref(ml)))
        g["links_up"] = g["links_up"][:rows]
        g["entry"], g["maxlevel"] = e.value, ml.value
        return g

    def import_graph(self, g):
        v = np.ascontiguousarray(g["vectors"], np.float32)
        lu = np.ascontiguousarray(g["links_up"], np.uint32)
        rows = lu.shape[0] if lu.size else 0
        check(lib().ehb_index_import_graph(
            self._h, v.shape[0], _p(v), _p(np.ascontiguousarray(g["labels"], np.uint64)),
            _p(np.ascontiguousarray(g["levels"], np.uint8)), _p(np.ascontiguousarray(g["links0"], np.uint32)),
            _p(np.ascontiguousarray(g["up_off"], np.uint32)), rows, _p(lu) if rows else None, int(g["entry"]),
            int(g["maxlevel"])))

    def save(self, path):
        check(lib().ehb_index_save(self._h, os.fsencode(path)))

    @classmethod
    def load(cls, path, device=0):
        h = C.c_void_p()
        check(lib().ehb_index_load(os.fsencode(path), device, C.byref(h)))
        ix = cls.__new__(cls)
        ix._h = h
        st = Stats()
        check(lib().ehb_index_stats(h, C.byref(st)))
        ix.dim, ix.M, ix.metric = st.dim, st.M, {v: k for k, v in METRICS.items()}[st.metric]
        return ix


class ShardedIndex:
    """ehb_sharded: one process, several GPUs of one box, behind the same host entry points."""

    def __init__(self, dim, devices, metric="l2", capacity=128, M=16, ef_construction=200, ef_search=10, seed=100,
                 shard_span=0, build_batch=0):
        L = lib()
        self.dim, self.metric, self.M = int(dim), metric, int(M)
        p = Params()
        L.ehb_params_default(C.byref(p), self.dim)
        p.metric, p.capacity, p.M = METRICS[metric], int(capacity), int(M)
        p.ef_construction, p.ef_search, p.seed, p.build_batch = int(ef_construction), int(ef_search), int(seed), int(build_batch)
        devs = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        check(L.ehb_sharded_create(C.byref(p), devs, len(devices), int(shard_span), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            lib().ehb_sharded_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, vecs, labels=None):
        v = np.ascontiguousarray(vecs, dtype=np.float32).reshape(-1, self.dim)
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.uint64)
        check(lib().ehb_sharded_add(self._h, v.shape[0], _p(v), _p(lab)))

    def remove(self, labels):
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        _check_key(lib().ehb_sharded_remove(self._h, lab.shape[0], _p(lab)), labels)

    def build(self):
        check(lib().ehb_sharded_build(self._h))

    def compact(self):
        check(lib().ehb_sharded_compact(self._h))

    def get(self, label):
        out = np.empty(self.dim, np.float32)
        _check_key(lib().ehb_sharded_get(self._h, int(label), _p(out)), label)
        return out

    def get_batch(self, labels):
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out = np.empty((lab.shape[0], self.dim), np.float32)
        _check_key(lib().ehb_sharded_get_batch(self._h, lab.shape[0], _p(lab), _p(out)), labels)
        return out

    def search_by_label(self, labels, k, ef=0, precision=FP32):
        """NativeIndex.search_by_label on the sharded index (ehb_sharded_search_by_label_ex)."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out_l, out_d, out_c = _alloc(lab.shape[0], k)
        _check_key(lib().ehb_sharded_search_by_label_ex(self._h, lab.shape[0], _p(lab), k, ef, int(precision),
                                                        _p(out_l), _p(out_d), _p(out_c)), labels)
        return out_l, out_d, out_c

    def search_by_label_beam(self, labels, k, ef=0, precision=FP32):
        """search_by_label() with max(ef, k + 1) up to 4096 (ehb_sharded_search_by_label_beam)."""
        lab = np.ascontiguousarray(np.atleast_1d(labels), dtype=np.uint64)
        out_l, out_d, out_c = _alloc(lab.shape[0], k)
        _check_key(lib().ehb_sharded_search_by_label_beam(self._h, lab.shape[0], _p(lab), k, ef, int(precision),
                                                          _p(out_l), _p(out_d), _p(out_c)), labels)
        return out_l, out_d, out_c

    @property
    def size(self):
        n = C.c_uint64()
        check(lib().ehb_sharded_size(self._h, C.byref(n)))
        return n.value

    def shard(self, i):
        h = C.c_void_p()
        check(lib().ehb_sharded_shard(self._h, i, C.byref(h)))
        ix = NativeIndex.__new__(NativeIndex)
        ix._h, ix.dim, ix.M, ix.metric = h, self.dim, self.M, self.metric
        ix._owned = False   # borrowed: the sharded index destroys it
        return ix

    def search(self, q, k, ef=0, precision=FP32):
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_sharded_search_ex(self._h, q.shape[0], _p(q), k, ef, int(precision), _p(labels), _p(dists),
                                          _p(counts)))
        return labels, dists, counts

    def search_beam(self, q, k, ef=0, precision=FP32):
        """search() with max(ef, k) up to 4096: the wide-beam walk on every shard above 512, then the same merge
        (ehb_sharded_search_beam); up to 512 exactly search()."""
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_sharded_search_beam(self._h, q.shape[0], _p(q), k, ef, int(precision), _p(labels), _p(dists),
                                            _p(counts)))
        return labels, dists, counts

    def search_bruteforce(self, q, k, precision=FP32):
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, self.dim)
        labels, dists, counts = _alloc(q.shape[0], k)
        check(lib().ehb_sharded_search_bruteforce(self._h, q.shape[0], _p(q), k, precision, _p(labels), _p(dists),
                                                  _p(counts)))
        return labels, dists, counts
