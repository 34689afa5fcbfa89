"""The Ed25519 oracle pair: OpenSSL (oracle_ed25519/ed25519_oracle.c) and the pure-Python restatement of the accept set
(oracle_ed25519/ref.py) agree on a corpus with every corruption class, on RFC 8032 TEST 1 and on the edge keys."""
import numpy as np
import pytest

import oracle_ed25519 as oe
from oracle_ed25519 import corpus, ref

RFC_A = bytes.fromhex("d75a980182b10ab7d54bfed3c964073a0ee172f3daa62325af021a68f707511a")
RFC_SIG = bytes.fromhex("e5564300c360ac729086e2cc806e828a84877f1eb8e5d974d873e065224901555fb8821590a33bacc61e39701cf9b46bd25bf5f0595bbe24655141438e7a100b")


def _one(A, M, sig):
    msgs = np.frombuffer(M + bytes(16), np.uint8)
    off = np.array([0, len(M)], np.uint64)
    return int(oe.verify_batch(msgs, off, np.frombuffer(sig, np.uint8), np.frombuffer(A, np.uint8))[0])


def test_rfc8032_test1():
    assert ref.verify(RFC_A, b"", RFC_SIG)
    assert _one(RFC_A, b"", RFC_SIG) == 1
    assert _one(RFC_A, b"x", RFC_SIG) == 0


def test_corpus_every_class_both_oracles_agree():
    c = corpus.make_corpus(700, seed=3)
    got = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    want = corpus.ref_verdicts(c)
    assert np.array_equal(got, want)
    for k, name in enumerate(corpus.CLASS_NAMES):
        assert (c["cls"] == k).sum() > 0, name
    # the corrupted classes never accept; the crafted ones accept sometimes and reject sometimes
    for k in (corpus.MSG_FLIP, corpus.R_FLIP, corpus.S_FLIP, corpus.S_PLUS_L, corpus.S_TOP, corpus.A_OFF_CURVE):
        assert got[c["cls"] == k].sum() == 0, corpus.CLASS_NAMES[k]
    assert got[c["cls"] == corpus.VALID].all()
    for k in (corpus.SMALL_ORDER, corpus.MIXED_ORDER, corpus.R_NONCANON):
        m = c["cls"] == k
        assert 0 < got[m].sum() < m.sum(), corpus.CLASS_NAMES[k]
    lens = np.diff(c["off"].astype(np.int64))
    assert set(corpus.EDGE_LENGTHS) <= set(lens.tolist())
    assert (c["off"] % 4 != 0).any()


def test_identity_keys_accept_forged_signatures():
    """A = identity in its canonical, y = 1 + p and "-0" encodings: [S]B - [k]A = [S]B for every k."""
    rng = np.random.default_rng(1)
    for A in (corpus._enc_y(1), corpus._enc_y(1 + ref.p), corpus._enc_y(1, 1)):
        s = int(rng.integers(1, 2**62)) ** 3 % ref.L
        sig = ref.encode(ref.mul(s, ref.B)) + s.to_bytes(32, "little")
        assert ref.verify(A, b"msg", sig)
        assert _one(A, b"msg", sig) == 1


def test_mixed_order_keys_accept_exactly_when_8_divides_k():
    rng = np.random.default_rng(2)
    T = ref.point_from_affine(*[pt for pt in ref.small_order_points() if pt[0] and pt[1]][0])  # order 8
    seen = set()
    for i in range(40):
        a = int(rng.integers(1, 2**62)) ** 3 % ref.L
        A = ref.encode(ref.add(ref.mul(a, ref.B), T))
        M = bytes([i])
        sig = ref.sign_with_scalar(a, A, M, int(rng.integers(1, 2**62)) ** 3 % ref.L)
        k = ref.challenge(sig[:32], A, M)
        want = k % 8 == 0
        assert ref.verify(A, M, sig) == want
        assert _one(A, M, sig) == int(want)
        seen.add(want)
    assert seen == {True, False}


def test_s_plus_l_and_noncanonical_r_reject():
    A, M, sig = RFC_A, b"", RFC_SIG
    s = int.from_bytes(sig[32:], "little") + ref.L
    bad = sig[:32] + s.to_bytes(32, "little")
    assert not ref.verify(A, M, bad) and _one(A, M, bad) == 0
    ident, zero = corpus._enc_y(1), bytes(32)
    assert ref.verify(ident, M, ident + zero) and _one(ident, M, ident + zero) == 1
    for R in (corpus._enc_y(1 + ref.p), corpus._enc_y(1, 1)):
        assert not ref.verify(ident, M, R + zero) and _one(ident, M, R + zero) == 0


@pytest.mark.parametrize("enc", corpus.small_order_encodings())
def test_small_order_keys_decode(enc):
    P = ref.decode(enc)
    assert P is not None
    assert ref.affine(ref.mul(8, P)) == (0, 1)
