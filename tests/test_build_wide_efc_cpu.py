"""ef_construction up to 4096 without a GPU: the parameter and file-header limits, and the wave model anchored to
hnswlib at construction beams the register build cannot hold (efc > 256), which the GPU tier then holds the wide
build to."""
import ctypes as C
import struct

import numpy as np
import pytest

import embeddinghub_b200 as ehb
from embeddinghub_b200 import _native
from oracle import oracle as orc  # test infrastructure
from test_build_wave_model_cpu import assert_same_graph_sets
from wave_model import WaveModel, ip_matrix, tiefree_ip

EHB_OK, EHB_ERR_INVALID, EHB_ERR_CUDA, EHB_ERR_IO = 0, 1, 2, 6


def _has_device():
    n = C.c_int(0)
    return ehb.lib().ehb_device_count(C.byref(n)) == EHB_OK and n.value > 0


def _create(efc):
    p = _native.Params()
    ehb.lib().ehb_params_default(C.byref(p), 8)
    p.ef_construction = efc
    h = C.c_void_p()
    rc = ehb.lib().ehb_index_create(C.byref(p), C.byref(h))
    if rc == EHB_OK:
        ehb.lib().ehb_index_destroy(h)
    return rc, ehb.lib().ehb_last_error().decode()


def test_create_rejects_ef_construction_above_4096():
    rc, msg = _create(4097)
    assert (rc, msg) == (EHB_ERR_INVALID, "ef_construction must be <= 4096")
    # 4096 passes the parameter checks: without a device the create then fails at the device check
    rc, msg = _create(4096)
    assert rc == (EHB_OK if _has_device() else EHB_ERR_CUDA), msg


def _index_file(path, efc):
    """An index file of no points whose header says ef_construction = efc (size as its header implies)."""
    p = _native.Params()
    ehb.lib().ehb_params_default(C.byref(p), 8)
    p.ef_construction = efc
    with open(path, "wb") as f:
        f.write(b"EHB200\x00\x02")
        f.write(bytes(p))
        f.write(struct.pack("<6Q", 0, 0, 0, 0, 0, 0))


def _load(path):
    h = C.c_void_p()
    rc = ehb.lib().ehb_index_load(str(path).encode(), 0, C.byref(h))
    if rc == EHB_OK:
        ehb.lib().ehb_index_destroy(h)
    return rc, ehb.lib().ehb_last_error().decode()


def test_load_accepts_headers_up_to_4096(tmp_path):
    _index_file(tmp_path / "a.ehb", 4097)
    assert _load(tmp_path / "a.ehb") == (EHB_ERR_IO, "corrupt header")
    _index_file(tmp_path / "b.ehb", 4096)
    rc, msg = _load(tmp_path / "b.ehb")
    assert rc == (EHB_OK if _has_device() else EHB_ERR_CUDA), msg


# ---- the wave model at wide beams ------------------------------------------------------------------------------
def _oracle(x, M, efc):
    o = orc.OracleHNSW(x.shape[1], "ip", x.shape[0], M=M, ef_construction=efc)
    o.add(x.astype(np.float32), threads=1)
    return o


@pytest.mark.parametrize("efc,n,d,nnz,M", [(300, 400, 16, None, 4), (300, 400, 32, None, 16), (1000, 1100, 16, 3, 8)])
def test_model_waves_of_one_equal_oracle_wide_efc(efc, n, d, nnz, M):
    """n > efc: the construction result set fills, and the heuristic walks all of it."""
    x, _ = tiefree_ip(n, d, nnz=nnz)
    og = _oracle(x, M, efc).export_graph()
    m = WaveModel(ip_matrix(x), og["levels"], M, ef_construction=efc).build(build_batch=1)
    assert m.trace["waves"] == [1] * n
    assert_same_graph_sets(m.export(), og)


@pytest.mark.parametrize("M", [4, 16])
def test_model_single_moves_equal_oracle_wide_efc(M):
    """updatePoint at efc 1100: keep = min(efc, |sCand| - 1) is all of sCand (|sCand| <= 1 + 2M + 4M^2 = 1057)."""
    n, d, efc = 400, 16, 1100
    x, B = tiefree_ip(n, d)
    o = _oracle(x, M, efc)
    m = WaveModel(ip_matrix(x), o.export_graph()["levels"], M, ef_construction=efc).build(build_batch=1)
    rng = np.random.default_rng(M * 5 + 1)
    moved = rng.choice(n, 30, replace=False)
    moved = np.concatenate([moved, moved[:6]])
    for lab in moved.tolist():
        x[lab, :d - 1] = B * rng.integers(-1, 2, d - 1)
        o.add(x[lab:lab + 1].astype(np.float32), np.array([lab], np.uint64), threads=1)
        m.set_distances(ip_matrix(x))
        m.update([lab])
    og = o.export_graph()
    assert np.array_equal(og["vectors"], x.astype(np.float32))
    assert_same_graph_sets(m.export(), og)


@pytest.mark.parametrize("efc", [300, 600])
def test_model_inserts_after_tombstones_equal_oracle_wide_efc(efc):
    """Tombstones are traversed but never results at wide beams too (n0 = 400 < 600: the set never fills there)."""
    n0, n, d, M = 400, 500, 32, 8
    x, _ = tiefree_ip(n, d)
    o = orc.OracleHNSW(d, "ip", n, M=M, ef_construction=efc)
    o.add(x[:n0].astype(np.float32), threads=1)
    dead = np.random.default_rng(efc).choice(n0, n0 // 10, replace=False)
    for lab in dead.tolist():
        o.mark_delete(lab)
    o.add(x[n0:].astype(np.float32), np.arange(n0, n, dtype=np.uint64), threads=1)
    og = o.export_graph()
    m = WaveModel(ip_matrix(x), og["levels"], M, ef_construction=efc).build(n0, build_batch=1)
    m.mark_deleted(dead)
    m.build(build_batch=1)
    assert_same_graph_sets(m.export(), og)
    dset = set(dead.tolist())
    assert not any(v in dset for p in range(n0, n) for v in m.row(p, 0))
