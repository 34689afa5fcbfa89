"""The split of keys-per-item mixed shards (k_mix_split<true>, consensus_b200/csrc/mixed.cuh) compiled into the CPU
simulation, against numpy; and the whole simulated pipeline of sbv_mixed_verify_batch against OpenSSL, every bad key
included."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mixed_keys_cases as mk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
PATTERNS = ["p256", "p384", "ed", "alternating", "random", "runs"]
SENTINEL = 0xEE


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _split(hs, tag, key96, sig96, off):
    """hs_mixed_split_keys into arrays with one spare row each, filled with SENTINEL: the spare rows show a copy that is
    too wide."""
    n = tag.size
    m = [int((tag == f).sum()) for f in range(3)]
    idx = np.full(n + 1, 0xFFFFFFFF, np.uint32)
    rows = lambda k, w: np.full((k + 1, w), SENTINEL, np.uint8)
    r0, s0, qx0, qy0 = rows(m[0], 32), rows(m[0], 32), rows(m[0], 32), rows(m[0], 32)
    r1, s1, qx1, qy1 = rows(m[1], 48), rows(m[1], 48), rows(m[1], 48), rows(m[1], 48)
    sig2, pub2 = rows(m[2], 64), rows(m[2], 32)
    fo = np.full(n + 3, 2**64 - 1, np.uint64)
    assert hs.hs_mixed_split_keys(C.c_size_t(n), _p(tag), _p(key96), _p(sig96), _p(off), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(idx), _p(r0), _p(s0),
                                  _p(r1), _p(s1), _p(sig2), _p(qx0), _p(qy0), _p(qx1), _p(qy1), _p(pub2), _p(fo)) == 0
    return m, idx, dict(r0=r0, s0=s0, qx0=qx0, qy0=qy0, r1=r1, s1=s1, qx1=qx1, qy1=qy1, sig2=sig2, pub2=pub2), fo


@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("n", [1, 15, 16, 17, 31, 32, 33, 700])
def test_split_with_keys_matches_numpy(hs, kind, n):
    rng = np.random.default_rng(hash((kind, n, "keys")) % 2**32)
    tag = mk.tag_pattern(kind, n, rng)
    lens = rng.integers(0, 90, n)
    lens[rng.random(n) < 0.2] = 0
    off = (np.concatenate([[0], np.cumsum(lens)]) + int(rng.integers(1, 40))).astype(np.uint64)
    sig96 = rng.integers(0, 256, (n, 96), dtype=np.uint8)  # every byte random: the ignored ones too
    key96 = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    m, idx, a, fo = _split(hs, tag, key96, sig96, off)
    want = [np.flatnonzero(tag == f) for f in range(3)]
    assert m == [i.size for i in want]
    assert np.array_equal(idx[:n], np.concatenate(want)) and idx[n] == 0xFFFFFFFF  # stable: item order inside every family
    i0, i1, i2 = want
    expect = dict(r0=sig96[i0, :32], s0=sig96[i0, 32:64], qx0=key96[i0, :32], qy0=key96[i0, 32:64],
                  r1=sig96[i1, :48], s1=sig96[i1, 48:96], qx1=key96[i1, :48], qy1=key96[i1, 48:96],
                  sig2=sig96[i2, :64], pub2=key96[i2, :32])
    for name, w in expect.items():
        got = a[name]
        assert np.array_equal(got[:-1], w), name
        assert (got[-1] == SENTINEL).all(), name  # nothing written past the family's last row
    lens_all = (off[1:] - off[:-1]).astype(np.int64)
    B = [int(lens_all[i].sum()) for i in want]
    al16 = lambda x: (x + 15) & ~15
    start = [0, al16(B[0] + 16)]
    start.append(start[1] + al16(B[1] + 16))
    at = [0, m[0] + 1, m[0] + m[1] + 2]
    for f in range(3):
        wo = np.concatenate([[0], np.cumsum(lens_all[want[f]])]).astype(np.uint64) + np.uint64(start[f])
        assert np.array_equal(fo[at[f]:at[f] + m[f] + 1], wo), f


def _verify(hs, cp, T=4, max_keys=8192):
    n = cp["scheme"].size
    ok = np.full(n, 7, np.uint8)
    assert hs.hs_mixed_verify_batch(C.c_size_t(n), _p(cp["scheme"]), _p(cp["msgs"]), _p(cp["off"]), _p(cp["sig96"]), _p(cp["key96"]), C.c_uint32(T),
                                    C.c_uint32(max_keys), _p(ok)) == 0
    return ok


@pytest.fixture(scope="module")
def pools():
    return mk.key_pools(k256=3, k384=3, k_ed=3, seed=41)


@pytest.mark.parametrize("kind", PATTERNS)
def test_simulated_pipeline_matches_openssl(hs, pools, kind):
    tag = mk.tag_pattern(kind, 90, np.random.default_rng(17))
    cp = mk.make_corpus(tag, pools, seed=18, hi=150, corrupt=0.4, junk=True)
    got = _verify(hs, cp)
    want = mk.expected_ok(cp)
    assert np.array_equal(got, want), np.flatnonzero(got != want)
    assert 0 < want.sum() < want.size
    # T = 0: no grouping, every item on the generic path of its family; the verdicts do not change
    assert np.array_equal(_verify(hs, cp, T=0), want)


def test_every_bad_key_class_rejects_as_openssl_does(hs, pools):
    tag = mk.tag_pattern("alternating", 120, None)
    cp = mk.make_corpus(tag, pools, seed=19, hi=60, corrupt=0.6, classes=mk.BAD_KEY_CLASSES)
    present = set(cp["cls"][cp["cls"] >= 0].tolist())
    assert present == set(mk.BAD_KEY_CLASSES), present
    got = _verify(hs, cp)
    want = mk.expected_ok(cp)
    assert np.array_equal(got, want), np.flatnonzero(got != want)
    bad = cp["cls"] >= 0
    assert not got[bad].any() and got[~bad].all()


def test_every_signature_class(hs, pools):
    tag = mk.tag_pattern("random", 150, np.random.default_rng(20))
    sig_classes = sorted(set(mk.EC_CLASSES + mk.ED_CLASSES) - set(mk.BAD_KEY_CLASSES))
    cp = mk.make_corpus(tag, pools, seed=21, hi=80, corrupt=0.6, classes=sig_classes)
    assert set(cp["cls"][cp["cls"] >= 0].tolist()) == set(sig_classes)
    got = _verify(hs, cp)
    assert np.array_equal(got, mk.expected_ok(cp))


def test_junk_in_ignored_bytes_changes_nothing(hs, pools):
    tag = mk.tag_pattern("alternating", 60, None)
    clean = mk.make_corpus(tag, pools, seed=22, hi=40, corrupt=0.3)
    junk = dict(clean, sig96=clean["sig96"].copy(), key96=clean["key96"].copy())
    rng = np.random.default_rng(23)
    for c, sig_end, key_end in ((mk.P256, 64, 64), (mk.ED, 64, 32)):
        idx = np.flatnonzero(tag == c)
        junk["sig96"][idx, sig_end:] = rng.integers(0, 256, (idx.size, 96 - sig_end), dtype=np.uint8)
        junk["key96"][idx, key_end:] = rng.integers(0, 256, (idx.size, 96 - key_end), dtype=np.uint8)
    got = _verify(hs, junk)
    assert np.array_equal(got, _verify(hs, clean))
    assert np.array_equal(got, mk.expected_ok(clean))


def test_equal_bytes_under_two_schemes_are_two_keys(hs, pools):
    """The 32 bytes of an Ed25519 key as the X of a P-256 item: each item is verified under its own scheme."""
    tag = np.array([mk.ED, mk.P256] * 20, np.uint8)
    cp = mk.make_corpus(tag, pools, seed=24, hi=40, corrupt=0, key_idx=np.zeros(40, np.int64))
    p256 = np.flatnonzero(tag == mk.P256)
    cp["key96"][p256[::2], :32] = cp["key96"][0, :32]  # X = the Ed25519 key's bytes: not a P-256 key any more
    got = _verify(hs, cp, T=2)
    want = mk.expected_ok(cp)
    assert np.array_equal(got, want)
    assert got[tag == mk.ED].all() and not got[p256[::2]].any() and got[p256[1::2]].all()
