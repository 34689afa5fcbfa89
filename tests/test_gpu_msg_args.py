"""The message arguments of the hashing calls are checked in an order that never reads past the caller's offsets: with
n >= 2^31 the call returns SBV_ERR_ARG before it looks at msg_off[n], even when msgs is NULL and msg_off is short.  The
outputs stay untouched (a fault is never a verdict)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

P8, P32, P64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(n_devices=1)
    yield e
    e.close()


@pytest.mark.parametrize("name", ["sbv_sha256_batch", "sbv_hash_verify_batch", "sbv_hash_verify_registered", "sbv_ed25519_verify_batch",
                                  "sbv_ed25519_verify_registered"])
def test_huge_n_with_null_msgs_is_rejected_before_msg_off_is_read(eng, name):
    import consensus_b200 as sbv
    n = C.c_size_t(1 << 31)
    off = np.array([0, 10, 20, 30], np.uint64)  # 4 entries: msg_off[n] lies 16 GiB past the array
    field = np.zeros(2 * 48, np.uint8)           # r, s, keys, slots and signatures are never read either
    out = np.full(4096, 0x5A, np.uint8)
    offp, fp, op = off.ctypes.data_as(P64), field.ctypes.data_as(P8), out.ctypes.data_as(P8)
    args = {
        "sbv_sha256_batch": (n, None, offp, op),
        "sbv_hash_verify_batch": (C.c_uint8(sbv.P256), n, None, offp, fp, fp, fp, fp, op, op),
        "sbv_hash_verify_registered": (C.c_uint8(sbv.P256), n, None, offp, field.ctypes.data_as(P32), fp, fp, op),
        "sbv_ed25519_verify_batch": (n, None, offp, fp, fp, op),
        "sbv_ed25519_verify_registered": (n, None, offp, field.ctypes.data_as(P32), fp, op),
    }[name]
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) < 0
    assert (out == 0x5A).all(), "a rejected call must not write its outputs"
    assert eng.kernel_launches == before
    assert b"n too large" in eng._lib.sbv_last_error(eng._h)
