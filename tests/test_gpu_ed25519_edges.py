"""The Ed25519 edge sets of tests/ed25519_edges.py on the H100: production-path rows through sbv_ed25519_verify_batch
(in calls below 2048 items, and repeated past 2048 so that the length sort runs), crafted-k rows through the
sbv_debug_ed25519_verify_k hook (the production k_ed_verify with the caller's k), every entry of the device's table of B
(sbv_debug_ed25519_btab) and batch shapes around the block sizes and the sort threshold.
tests/test_hostsim_ed25519_edges.py runs the same sets on the CPU simulation."""
import ctypes as C

import numpy as np
import pytest

import ed25519_edges as edges
import oracle_ed25519 as oe
from oracle_ed25519 import corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _verify(eng):
    def run(a):
        return eng.ed25519_verify_batch(a["msgs"], a["off"], a["sig"], a["pub"])
    return run


def _verify_k(eng):
    def run(a):
        n = a["off"].size - 1
        ok = np.full(n, 7, np.uint8)
        assert eng._lib.sbv_debug_ed25519_verify_k(eng._h, C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) == 0
        return ok
    return run


def test_every_entry_of_the_table_of_B(eng):
    """All 32 x 128 entries of the table k_ed_btab_init builds on the device, 24 words each, against the model's table."""
    got = np.zeros((32, 128, 24), np.uint32)
    assert eng._lib.sbv_debug_ed25519_btab(eng._h, C.c_size_t(0), C.c_size_t(32 * 128), _p(got)) == 0
    assert np.array_equal(got, edges.btab_words())
    part = np.zeros((5, 24), np.uint32)
    assert eng._lib.sbv_debug_ed25519_btab(eng._h, C.c_size_t(17 * 128 + 99), C.c_size_t(5), _p(part)) == 0
    assert np.array_equal(part, edges.btab_words()[17, 99:104])
    assert eng._lib.sbv_debug_ed25519_btab(eng._h, C.c_size_t(4095), C.c_size_t(2), _p(part)) < 0


def test_S_boundary(eng):
    """S in {0, 1, L-2, L-1} accepts under the three encodings of the identity; L, L+1, 2L-1, s + mL and 2^256-1 reject."""
    acc, n = edges.check(edges.s_boundary(), verify=_verify(eng), sort_pass=True, seed=1)
    assert 0 < acc < n


def test_every_B_loop_digit(eng):
    """One S per reachable (window, 8-bit digit), A = identity or a small-order key with [k]A = O."""
    acc, n = edges.check(edges.digit_sweep(), verify=_verify(eng), sort_pass=True, seed=2)
    assert acc == 7954


def test_small_order_R(eng):
    """R' of order 1, 2, 4 and 8 with its canonical and every non-canonical R; R' = O under full- and mixed-order keys."""
    acc, n = edges.check(edges.small_order_r(), verify=_verify(eng), sort_pass=True, seed=3)
    assert 0 < acc < n


def test_crafted_k(eng):
    """k = 0, 1, 2, L-2, L-1, all nibbles 8, all nibbles 7, every single nibble and +8 at every window, every kind of key."""
    acc, n = edges.check(edges.crafted_k(), verify_k=_verify_k(eng), seed=4)
    assert 0 < acc < n and acc == len(edges.crafted_k_keys()) * len(edges.crafted_ks())


def test_B_loop_collisions(eng):
    """The B loop's affine addition with P = Q, with P = -Q (O partway, then from O), and R' = O at the end."""
    acc, n = edges.check(edges.collisions(), verify_k=_verify_k(eng), seed=5)
    assert 0 < acc < n


def test_verify_k_rejects_k_at_least_L(eng):
    a = edges._subset(edges.crafted_k(), range(4)).arrays()
    for bad in (edges.L, 2**256 - 1):
        a["k"][2] = np.frombuffer(bad.to_bytes(32, "little"), "<u4")
        ok = np.full(4, 7, np.uint8)
        assert eng._lib.sbv_debug_ed25519_verify_k(eng._h, C.c_size_t(4), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) < 0
        assert (ok == 7).all()


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 127, 128, 129, 2047, 2048, 2049])
def test_batch_shapes(eng, n):
    """ED_BLOCK = 32, the SHA-512 block of 128 threads and the length sort from 2048 items on."""
    c = corpus.make_corpus(n, seed=300 + n, crafted_max=16)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(_verify(eng)(c), want)


def test_long_messages_among_short_ones(eng):
    """Messages of 70 KB and 1 MiB among 4,090 short ones: the length sort's bin is clamped at 1023 blocks."""
    b = edges.mixed_length_batch()
    want = oe.verify_batch(b["msgs"], b["off"], b["sig"], b["pub"])
    assert np.array_equal(_verify(eng)(b), want)
    assert want[b["long"][2:]].all() and not want[b["long"][:2]].any() and 0 < want.sum() < want.size
