"""The P-256 comb build as libsbv.so runs it — a warp per key, lane = chain (k_comb_fill_warp, k_kt_inv over the key-major
scratch, k_comb_final), the warps in lockstep in the CPU simulation (tools/hostsim) — against the one-thread-per-chain
kernels (k_comb_fill, k_kt_inv and k_kt_final over the window tables' scratch layout) on the same keys: the Jacobian
entries and Z ratios of the fill, the inverted top Z's and the affine table, word for word."""
import ctypes as C

import numpy as np
import pytest

import ecdsa_keys as ek
import oracle
from oracle import corpus
from oracle import ecdsa_ref as ref
from test_hostsim import _p8, hs  # noqa: F401  (hs: the simulation library fixture)

N, CHAINS, ENT = 8, 32, 16


def _u32(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def _build(hs, warp, kxy, cap):
    n = kxy.shape[0]
    qx, qy = np.ascontiguousarray(kxy[:, :32]), np.ascontiguousarray(kxy[:, 32:])
    kt = np.zeros(cap * CHAINS * ENT * 2 * N, np.uint32)
    jac = np.zeros_like(kt)
    hz = np.zeros(cap * CHAINS * (ENT - 1) * N, np.uint32)
    zt = np.zeros(cap * CHAINS * N, np.uint32)
    fl = np.zeros(cap, np.uint8)
    assert hs.hs_comb_build(C.c_int(warp), C.c_size_t(n), C.c_size_t(cap), _p8(qx), _p8(qy), _u32(kt), _u32(jac), _u32(hz), _u32(zt), _p8(fl)) == 0
    return {"ktab": kt, "jac": jac, "hs": hz, "ztop": zt, "flags": fl}


def _keys(n, seed):
    c = ref.CURVES[oracle.P256]
    _, kxy = corpus.make_keys(oracle.P256, n, seed=seed)
    kxy = kxy.copy()
    if n > 1:
        kxy[1, 32 + 8] ^= 1                                                      # off the curve
    if n > 2:
        kxy[2, :32] = np.frombuffer(int(c.p + 2).to_bytes(32, "big"), np.uint8)  # x >= p
    return kxy


@pytest.mark.parametrize("nkeys,cap", [(5, 5), (3, 8), (1, 1)])
def test_warp_build_equals_thread_per_chain_build(hs, nkeys, cap):
    """Key counts that are not a multiple of the two keys of a block, and a build capacity above the key count: every
    intermediate and the table agree word for word, and the invalid keys get no table on either path."""
    kxy = _keys(nkeys, seed=70 + nkeys)
    ref_ = _build(hs, 0, kxy, cap)
    got = _build(hs, 1, kxy, cap)
    want_flags = [1] * nkeys + [0] * (cap - nkeys)
    for bad in (1, 2)[:max(0, nkeys - 1)]:
        want_flags[bad] = 0
    assert ref_["flags"].tolist() == got["flags"].tolist() == want_flags
    for what in ("jac", "hs", "ztop", "ktab"):
        bad = np.nonzero(ref_[what] != got[what])[0]
        assert bad.size == 0, f"{what}: {bad.size} words differ, first {bad[:8].tolist()}"
    assert ref_["jac"].any() and ref_["hs"].any() and ref_["ztop"].any()


def test_warp_build_equals_python_integers(hs):
    """The table of the warp path equals the Python-integer model for a valid key, and is zero for the keys without one."""
    kxy = _keys(3, seed=81)
    got = _build(hs, 1, kxy, 3)
    tabs = got["ktab"].reshape(3, -1)
    Q = (int.from_bytes(kxy[0, :32].tobytes(), "big"), int.from_bytes(kxy[0, 32:].tobytes(), "big"))
    assert np.array_equal(tabs[0], ek.comb_table(Q))
    assert not tabs[1].any() and not tabs[2].any()
