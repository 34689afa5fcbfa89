"""The Ed25519 edge sets of tests/ed25519_edges.py on the CPU simulation of the device code (tools/hostsim): the S < L
boundary, every B-loop digit, small-order R', crafted k, B-loop collisions, every entry of the table of B and the batch
shapes around the block sizes.  tests/test_gpu_ed25519_edges.py runs the same sets on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ed25519_edges as edges
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


def _verify(hs):
    def run(a):
        n = a["off"].size - 1
        ok = np.zeros(n, np.uint8)
        assert hs.hs_ed25519_verify(C.c_size_t(n), _p(a["msgs"]), _p(a["off"]), _p(a["sig"]), _p(a["pub"]), _p(ok)) == 0
        return ok
    return run


def _verify_k(hs):
    def run(a):
        n = a["off"].size - 1
        ok = np.zeros(n, np.uint8)
        assert hs.hs_ed25519_verify_k(C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) == 0
        return ok
    return run


def test_every_entry_of_the_table_of_B(hs):
    """All 32 x 128 entries of k_ed_btab_init's table, 24 words each, against the table the model walks in Python."""
    tab = np.zeros(32 * 128 * 24, np.uint32)
    assert hs.hs_ed25519_btab(_p(tab)) == 0
    assert np.array_equal(tab.reshape(32, 128, 24), edges.btab_words())


def test_S_boundary(hs):
    """S in {0, 1, L-2, L-1} accepts under the three encodings of the identity; L, L+1, 2L-1, s + mL and 2^256-1 reject."""
    acc, n = edges.check(edges.s_boundary(), verify=_verify(hs), seed=1)
    assert 0 < acc < n


def test_every_B_loop_digit(hs):
    """One S per reachable (window, 8-bit digit), A = identity or a small-order key with [k]A = O."""
    acc, n = edges.check(edges.digit_sweep(), verify=_verify(hs), seed=2)
    assert acc == 7954


def test_small_order_R(hs):
    """R' of order 1, 2, 4 and 8 with its canonical and every non-canonical R; R' = O under full- and mixed-order keys."""
    acc, n = edges.check(edges.small_order_r(), verify=_verify(hs), seed=3)
    assert 0 < acc < n


def test_crafted_k(hs):
    """k = 0, 1, 2, L-2, L-1, all nibbles 8, all nibbles 7, every single nibble and +8 at every window, every kind of key."""
    acc, n = edges.check(edges.crafted_k(), verify_k=_verify_k(hs), seed=4)
    assert 0 < acc < n and acc == len(edges.crafted_k_keys()) * len(edges.crafted_ks())


def test_B_loop_collisions(hs):
    """The B loop's affine addition with P = Q, with P = -Q (O partway, then from O), and R' = O at the end."""
    acc, n = edges.check(edges.collisions(), verify_k=_verify_k(hs), seed=5)
    assert 0 < acc < n


def test_verify_k_rejects_k_at_least_L(hs):
    rows = edges.crafted_k()
    a = edges._subset(rows, range(4)).arrays()
    for bad in (edges.L, 2**256 - 1):
        a["k"][2] = np.frombuffer(bad.to_bytes(32, "little"), "<u4")
        ok = np.zeros(4, np.uint8)
        assert hs.hs_ed25519_verify_k(C.c_size_t(4), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) != 0


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 127, 128, 129, 2047, 2048, 2049])
def test_batch_shapes(hs, n):
    c = corpus.make_corpus(n, seed=300 + n, crafted_max=16)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(_verify(hs)(c), want)


def test_long_messages_among_short_ones(hs):
    """Messages of 70 KB and 1 MiB among 4,090 short ones."""
    b = edges.mixed_length_batch()
    want = oe.verify_batch(b["msgs"], b["off"], b["sig"], b["pub"])
    assert np.array_equal(_verify(hs)(b), want)
    assert want[b["long"][2:]].all() and not want[b["long"][:2]].any() and 0 < want.sum() < want.size
