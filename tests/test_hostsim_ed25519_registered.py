"""Registered Ed25519 keys on the CPU simulation of the device code (tools/hostsim): the per-key tables k_ed_ktab_build
builds, and k_ed_key_gather + k_ed_sha512 + k_ed_verify_keyed against OpenSSL and the constructions of
tests/ed25519_registered.py, at sizes a CPU affords.  tests/test_gpu_ed25519_registered.py runs the same sets on the
device through sbv_ed25519_set_keys / sbv_ed25519_verify_registered."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ed25519_edges as edges
import ed25519_registered as reg
import oracle_ed25519 as oe
from oracle_ed25519 import corpus, ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _set_keys(hs, chunk=0):
    def run(pub):
        pub = np.ascontiguousarray(pub, np.uint8)
        assert hs.hs_ed25519_set_keys(C.c_size_t(pub.size // 32), _p(pub), C.c_uint32(chunk)) == 0
    return run


def _verify(hs):
    def run(a, slot):
        n = a["off"].size - 1
        slot = np.ascontiguousarray(slot, np.uint32)
        ok = np.full(n, 7, np.uint8)
        assert hs.hs_ed25519_verify_registered(C.c_size_t(n), _p(a["msgs"]), _p(a["off"]), _p(slot), _p(a["sig"]), _p(ok)) == 0
        return ok
    return run


def _verify_k(hs):
    def run(a, slot):
        n = a["off"].size - 1
        slot = np.ascontiguousarray(slot, np.uint32)
        ok = np.full(n, 7, np.uint8)
        assert hs.hs_ed25519_verify_registered_k(C.c_size_t(n), _p(slot), _p(a["sig"]), _p(a["k"]), _p(ok)) == 0
        return ok
    return run


def _ktab(hs, slot):
    out = np.zeros((32, 128, 24), np.uint32)
    return out if hs.hs_ed25519_ktab(C.c_uint32(slot), _p(out)) == 0 else None


def test_table_of_the_encoding_of_B_is_the_table_of_B(hs):
    _set_keys(hs)(np.frombuffer(ref.encode(ref.B), np.uint8))
    b = np.zeros(32 * 128 * 24, np.uint32)
    assert hs.hs_ed25519_btab(_p(b)) == 0
    assert np.array_equal(_ktab(hs, 0), b.reshape(32, 128, 24))


def test_every_entry_of_every_kind_of_key(hs):
    """A random, a small-order, a y >= p and a mixed-order key against the model tables; an off-curve slot has none."""
    keys = reg.table_keys()
    bad = corpus.off_curve_encodings(np.random.default_rng(5), 1)[0]
    _set_keys(hs)(np.frombuffer(b"".join(keys[:2] + [bad] + keys[2:]), np.uint8))
    for slot, A in zip((0, 1, 3, 4), keys):
        assert np.array_equal(_ktab(hs, slot), reg.ktab_words(A)), reg.key_class(A)
    assert _ktab(hs, 2) is None and _ktab(hs, 5) is None


def test_tables_built_in_chunks(hs):
    """The build split into launches of 3 keys, as the device splits it into launches of 1,024 (a shorter last chunk, an
    off-curve key between chunks): every table equals the model's."""
    keys = reg.table_keys() + [ref.encode(ref.B)]
    bad = corpus.off_curve_encodings(np.random.default_rng(6), 1)[0]
    order = keys[:3] + [bad] + keys[3:] + [keys[0]]
    _set_keys(hs, chunk=3)(np.frombuffer(b"".join(order), np.uint8))
    for slot, A in enumerate(order):
        if A == bad:
            assert _ktab(hs, slot) is None
        else:
            assert np.array_equal(_ktab(hs, slot), reg.ktab_words(A)), (slot, reg.key_class(A))


def test_unknown_slots_reject_in_the_kernel(hs):
    """Rows that accept under slot 0's key with their k reject by slot n and 2^32 - 1, and in an empty registry: the
    kernel's own slot check, with no gather involved."""
    A0, rows = reg.slot0_rows()
    a, n = rows.arrays(), len(rows)
    others = reg.table_keys()[1:]
    _set_keys(hs)(np.frombuffer(b"".join([A0] + others), np.uint8))
    verify_k = _verify_k(hs)
    assert verify_k(a, np.zeros(n, np.uint32)).all()
    for bad in (len(others) + 1, 2**32 - 1):
        assert not verify_k(a, np.full(n, bad, np.uint32)).any(), bad
    _set_keys(hs)(np.zeros(0, np.uint8))
    assert not verify_k(a, np.zeros(n, np.uint32)).any()


def test_S_boundary(hs):
    acc, n = reg.check(edges.s_boundary(), _set_keys(hs), verify=_verify(hs), seed=1)
    assert 0 < acc < n


def test_every_B_loop_digit(hs):
    """One S per reachable (window, 8-bit digit) of the B loop, after the key loop (identity and small-order keys)."""
    acc, n = reg.check(edges.digit_sweep(), _set_keys(hs), verify=_verify(hs), seed=2)
    assert acc == 7954


def test_small_order_R(hs):
    """R' of small order under every R encoding; R' = O under full- and mixed-order keys."""
    acc, n = reg.check(edges.small_order_r(), _set_keys(hs), verify=_verify(hs), seed=3)
    assert 0 < acc < n


def test_every_key_loop_digit(hs):
    """One k per reachable (window, 8-bit digit) of k < L through the k hook, every kind of key in turn."""
    acc, n = reg.check(reg.k_sweep(), _set_keys(hs), verify_k=_verify_k(hs), seed=4)
    assert acc == len(reg.k_sweep_ks())


def test_collisions(hs):
    """The B loop meeting +entry, -entry and ending at O after the key loop; the key loop's P = Q at window 31."""
    acc, n = reg.check(reg.collisions(), _set_keys(hs), verify_k=_verify_k(hs), seed=5)
    assert 0 < acc < n


def test_verify_k_rejects_k_at_least_L(hs):
    rows = edges._subset(reg.k_sweep(), range(4))
    pub, slot = reg.registry(rows.A)
    _set_keys(hs)(pub)
    a = rows.arrays()
    for bad in (edges.L, 2**256 - 1):
        a["k"][2] = np.frombuffer(bad.to_bytes(32, "little"), "<u4")
        ok = np.zeros(4, np.uint8)
        assert hs.hs_ed25519_verify_registered_k(C.c_size_t(4), _p(slot), _p(a["sig"]), _p(a["k"]), _p(ok)) != 0


def _corpus(n, seed, n_keys):
    return reg.merge(corpus.make_corpus(n, seed=seed, n_keys=n_keys, crafted_max=64), reg.class_rows())


def test_corpus_every_class(hs):
    """A corpus with every corruption class plus the edge rows: verdicts equal OpenSSL's and the keys-per-item path's, and
    y >= p, "-0", small-order and mixed-order keys and non-canonical R each have accepts and rejects."""
    c = _corpus(1500, 31, 24)
    pub, slot = reg.corpus_registry(c)
    _set_keys(hs)(pub)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(_verify(hs)(c, slot), want)
    n = want.size
    per_item = np.zeros(n, np.uint8)
    assert hs.hs_ed25519_verify(C.c_size_t(n), _p(c["msgs"]), _p(c["off"]), _p(c["sig"]), _p(c["pub"]), _p(per_item)) == 0
    assert np.array_equal(per_item, want)
    cls = np.array([reg.key_class(bytes(A)) for A in c["pub"]])
    for name in ("y>=p", "-0", "small order", "mixed order"):
        assert 0 < want[cls == name].sum() < (cls == name).sum(), name
    assert (cls == "off-curve").any() and not want[cls == "off-curve"].any()
    m = c["cls"] == corpus.R_NONCANON
    assert 0 < want[m].sum() < m.sum()


def test_registry_semantics(hs):
    c = corpus.make_corpus(300, seed=32, n_keys=8, crafted_max=0)
    pub, slot = reg.corpus_registry(c)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert want.sum() > 100
    verify, set_keys = _verify(hs), _set_keys(hs)
    # unknown slots reject
    set_keys(pub)
    for bad in (pub.shape[0], 2**32 - 1):
        s2 = slot.copy()
        s2[::3] = bad
        got = verify(c, s2)
        assert not got[::3].any() and np.array_equal(np.delete(got, np.s_[::3]), np.delete(want, np.s_[::3]))
    # an empty registry rejects everything
    set_keys(np.zeros(0, np.uint8))
    assert not verify(c, slot).any()
    # the same key in two slots
    set_keys(np.concatenate([pub, pub]))
    assert np.array_equal(verify(c, slot + pub.shape[0]), want) and np.array_equal(verify(c, slot), want)
    # replacing the registry re-points the old slots to the new keys
    new = pub[::-1].copy()
    set_keys(new)
    assert np.array_equal(verify(c, pub.shape[0] - 1 - slot), want)
    want_new = oe.verify_batch(c["msgs"], c["off"], c["sig"], new[slot])
    assert np.array_equal(verify(c, slot), want_new) and want_new.sum() < want.sum() // 2


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 2047, 2048, 2049])
def test_batch_shapes(hs, n):
    c = corpus.make_corpus(n, seed=300 + n, n_keys=16, crafted_max=16)
    pub, slot = reg.corpus_registry(c)
    _set_keys(hs)(pub)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(_verify(hs)(c, slot), want)
