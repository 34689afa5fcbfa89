"""CPU simulation of the Ed25519 device code (tools/hostsim: ed25519.cuh, sha512.cuh, ed25519_verify.cuh compiled with g++)
against Python integers, hashlib and the oracle.  The `-m gpu` tests (test_gpu_ed25519.py) run the same checks on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ed25519_cases as cases
import oracle_ed25519 as oe
from oracle_ed25519 import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _runner(hs):
    def run(op, inp):
        inp = np.ascontiguousarray(inp, np.uint32)
        out = np.zeros_like(inp)
        assert hs.hs_ed25519_op(C.c_int(op), C.c_size_t(inp.shape[0]), _p(inp), _p(out)) == 0
        return out
    return run


def test_field_ops(hs):
    """mul / sqr / add / sub / canon / inverse against Python integers, operands across [0, 2^256) ([p, 2^256) included)."""
    assert cases.check_field(_runner(hs), np.random.default_rng(1)) > 400


def test_sqrt_ratio(hs):
    cases.check_sqrt_ratio(_runner(hs), np.random.default_rng(2))


def test_decode_every_edge_key(hs):
    cases.check_decode(_runner(hs), np.random.default_rng(3))


def test_reduce_mod_L(hs):
    """0, L-1, L, kL +- 1, 2^512 - 1 and random 512-bit values."""
    cases.check_reduce(_runner(hs), np.random.default_rng(4))


@pytest.mark.parametrize("sorted_order", [False, True])
def test_sha512_of_R_A_M_and_k(hs, sorted_order):
    """SHA-512(R || A || M) on a ragged, misaligned batch crossing every block boundary, against hashlib; k = digest mod L.
    sorted_order: threads take the items in a permuted order (as after the length sort), results land by item."""
    rng = np.random.default_rng(5)
    msgs, off, sig, pub = cases.ragged_batch(rng)
    n = off.size - 1
    perm = rng.permutation(n).astype(np.uint32) if sorted_order else None
    k = np.zeros(8 * n, np.uint32)
    dig = np.zeros(16 * n, np.uint32)
    assert hs.hs_ed25519_sha512(C.c_size_t(n), _p(msgs), _p(off), C.c_uint64(0), _p(sig), _p(pub),
                                _p(perm) if perm is not None else None, _p(k), _p(dig)) == 0
    want = cases.expected_digests(msgs, off, sig, pub)
    got = dig.reshape(n, 16)
    kk = k.reshape(8, n)
    for i in range(n):
        assert got[i].astype("<u4").tobytes() == want[i], i
        kv = sum(int(kk[w, i]) << (32 * w) for w in range(8))
        assert kv == int.from_bytes(want[i], "little") % cases.L


def test_fixed_base_table(hs):
    """Entries of the table of B (affine Niels: y + x, y - x, 2dxy) against Python integers."""
    from oracle_ed25519 import ref
    tab = np.zeros(32 * 128 * 24, np.uint32)
    assert hs.hs_ed25519_btab(_p(tab)) == 0
    tab = tab.reshape(32, 128, 24)
    for win, j in [(0, 1), (0, 2), (0, 128), (1, 1), (5, 77), (31, 1), (31, 128), (17, 3)]:
        x, y = ref.affine(ref.mul(j * 256**win, ref.B))
        row = tab[win, j - 1]
        assert cases.val(row, 0) == (y + x) % ref.p
        assert cases.val(row, 8) == (y - x) % ref.p
        assert cases.val(row, 16) == 2 * ref.d * x * y % ref.p


def test_pipeline_matches_oracle(hs):
    """Hash -> verify over a corrupted corpus with every class, against OpenSSL."""
    c = corpus.make_corpus(400, seed=7)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    ok = np.zeros(400, np.uint8)
    assert hs.hs_ed25519_verify(C.c_size_t(400), _p(c["msgs"]), _p(c["off"]), _p(c["sig"]), _p(c["pub"]), _p(ok)) == 0
    assert np.array_equal(ok, want)
    assert 0 < want.sum() < want.size
