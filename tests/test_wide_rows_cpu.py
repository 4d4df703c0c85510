"""Row-width limits of the C ABI that hold without a GPU: dim 1..4096 passes the argument check of ehb_index_create,
4097 is EHB_ERR_INVALID (the check comes before any device is touched)."""
import ctypes as C

import pytest

import embeddinghub_b200 as ehb
from embeddinghub_b200 import _native

EHB_ERR_INVALID = 1


def _create(dim):
    p = _native.Params()
    ehb.lib().ehb_params_default(C.byref(p), dim)
    out = C.c_void_p()
    rc = ehb.lib().ehb_index_create(C.byref(p), C.byref(out))
    if rc == 0:
        ehb.lib().ehb_index_destroy(out)
    return rc, ehb.lib().ehb_last_error().decode()


def test_dim_above_4096_is_invalid():
    rc, msg = _create(4097)
    assert rc == EHB_ERR_INVALID and "1..4096" in msg, (rc, msg)
    rc, msg = _create(0)
    assert rc == EHB_ERR_INVALID and "1..4096" in msg, (rc, msg)


@pytest.mark.parametrize("dim", [2049, 3072, 4096])
def test_wide_dims_pass_the_argument_check(dim):
    rc, msg = _create(dim)
    assert rc != EHB_ERR_INVALID, msg
