"""k_kt_bases2 — the doubling chain of the P-256 comb tables with two lanes per key (both lanes multiplying at every level,
pair exchanges between them) — in the CPU simulation of the device code (tools/hostsim), its 32 lanes run in lockstep
with one OS thread per lane meeting at every shuffle."""
import ctypes as C

import numpy as np

import oracle
from oracle import corpus
from oracle import ecdsa_ref as ref
from test_hostsim import _p8, hs  # noqa: F401  (hs: the simulation library fixture)
from test_hostsim_comb import _comb_tables

NBASE = 16  # CombTab<P256>: bases P_c = 2^(16c) * Q


def _bases(hs, kxy, four):
    n = kxy.shape[0]
    qx, qy = np.ascontiguousarray(kxy[:, :32]), np.ascontiguousarray(kxy[:, 32:])
    out, fl = np.zeros(NBASE * 3 * 8 * n, np.uint32), np.zeros(n, np.uint8)
    assert hs.hs_comb_bases(C.c_size_t(n), _p8(qx), _p8(qy), C.c_int(four), out.ctypes.data_as(C.POINTER(C.c_uint32)), _p8(fl)) == 0
    return out.reshape(NBASE, 3, 8, n), fl


def test_two_lane_bases_equal_one_thread_chain(hs):
    """The 16 Jacobian bases of every key equal those of the one-thread-per-key k_kt_bases word for word, the validity
    flags too (an off-curve key and a key with x >= p among them, whose bases stay unwritten), and the tables built
    from them are bit-identical; base c of key 0 is 2^(16c) * Q."""
    c = ref.CURVES[oracle.P256]
    _, kxy = corpus.make_keys(oracle.P256, 6, seed=23)
    kxy = kxy.copy()
    kxy[1, 32 + 8] ^= 1                                                      # off the curve
    kxy[4, :32] = np.frombuffer(int(c.p + 2).to_bytes(32, "big"), np.uint8)  # x >= p
    want, fw = _bases(hs, kxy, four=0)
    got, fg = _bases(hs, kxy, four=2)
    assert fw.tolist() == fg.tolist() == [1, 0, 1, 1, 0, 1]
    assert np.array_equal(got, want)
    assert not got[:, :, :, [1, 4]].any()
    ta, fa = _comb_tables(hs, 0, kxy, four=0)
    tb, fb = _comb_tables(hs, 0, kxy, four=2)
    assert fa.tolist() == fb.tolist() and np.array_equal(ta, tb)
    Q = (int.from_bytes(kxy[0, :32].tobytes(), "big"), int.from_bytes(kxy[0, 32:].tobytes(), "big"))
    Rm = 1 << 256
    val = lambda w: sum(int(x) << (32 * i) for i, x in enumerate(w))
    for base in range(NBASE):
        X, Y, Z = (val(got[base, j, :, 0]) * pow(Rm, -1, c.p) % c.p for j in range(3))
        zi = pow(Z, -1, c.p)
        assert (X * zi * zi % c.p, Y * zi * zi * zi % c.p) == ref.scalar_mult(c, 1 << (16 * base), Q), base
