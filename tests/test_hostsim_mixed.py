"""The split, compaction and scatter kernels of mixed ECDSA / Ed25519 shards (consensus_b200/csrc/mixed.cuh), compiled into
the CPU simulation, against numpy; and the whole simulated pipeline of sbv_mixed_verify_registered against OpenSSL."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mixed_cases as mc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _al16(x):
    return (x + 15) & ~15


def _model(tag, slot, sig96, msgs, off):
    """What the split and the compaction must produce, restated with numpy."""
    lens = (off[1:] - off[:-1]).astype(np.int64)
    idx = [np.flatnonzero(tag == f) for f in range(3)]
    B = [int(lens[i].sum()) for i in idx]
    start = [0, _al16(B[0] + 16)]
    start.append(start[1] + _al16(B[1] + 16))
    offs = [np.concatenate([[0], np.cumsum(lens[i])]).astype(np.uint64) + np.uint64(start[f]) for f, i in enumerate(idx)]
    regions = [mc.gather(msgs, off, i)[0][:B[f]] for f, i in enumerate(idx)]
    return idx, offs, regions, start


def _split(hs, tag, slot, sig96, msgs, off):
    n = tag.size
    m = [int((tag == f).sum()) for f in range(3)]
    idx, slo = np.full(n + 1, 0xFFFFFFFF, np.uint32), np.full(n + 1, 0xFFFFFFFF, np.uint32)
    r0, s0 = np.zeros((m[0] + 1, 32), np.uint8), np.zeros((m[0] + 1, 32), np.uint8)
    r1, s1 = np.zeros((m[1] + 1, 48), np.uint8), np.zeros((m[1] + 1, 48), np.uint8)
    sig2 = np.zeros((m[2] + 1, 64), np.uint8)
    fo = np.full(n + 3, 2**64 - 1, np.uint64)
    assert hs.hs_mixed_split(C.c_size_t(n), _p(tag), _p(slot), _p(sig96), _p(off), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(idx), _p(slo), _p(r0), _p(s0),
                             _p(r1), _p(s1), _p(sig2), _p(fo)) == 0
    total = int(off[-1] - off[0])
    blob = np.full(total + 128, 0xEE, np.uint8)
    src = np.concatenate([msgs[int(off[0]):int(off[-1])], np.zeros(16, np.uint8)])
    assert hs.hs_mixed_compact(C.c_size_t(n), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(src), _p(off), C.c_uint64(int(off[0])), _p(idx), _p(fo),
                               _p(blob)) == 0
    return m, idx[:n], slo[:n], (r0[:m[0]], s0[:m[0]], r1[:m[1]], s1[:m[1]], sig2[:m[2]]), fo, blob


PATTERNS = ["p256", "p384", "ed", "alternating", "random", "runs"]


@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("n", [1, 15, 16, 17, 700])
def test_split_and_compaction_match_numpy(hs, kind, n):
    rng = np.random.default_rng(hash((kind, n)) % 2**32)
    tag = mc.tag_pattern(kind, n, rng)
    lens = rng.integers(0, 90, n)
    lens[rng.random(n) < 0.2] = 0  # empty messages
    first = int(rng.integers(1, 40))
    off = (np.concatenate([[0], np.cumsum(lens)]) + first).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    slot = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    sig96 = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    m, idx, slo, (r0, s0, r1, s1, sig2), fo, blob = _split(hs, tag, slot, sig96, msgs, off)
    want_idx, want_off, regions, start = _model(tag, slot, sig96, msgs, off)
    assert m == [i.size for i in want_idx]
    assert np.array_equal(idx, np.concatenate(want_idx))  # stable: item order inside every family
    assert np.array_equal(slo, slot[idx])
    i0, i1, i2 = want_idx
    assert np.array_equal(r0, sig96[i0, :32]) and np.array_equal(s0, sig96[i0, 32:64])
    assert np.array_equal(r1, sig96[i1, :48]) and np.array_equal(s1, sig96[i1, 48:96])
    assert np.array_equal(sig2, sig96[i2, :64])
    at = [0, m[0] + 1, m[0] + m[1] + 2]
    for f in range(3):
        assert np.array_equal(fo[at[f]:at[f] + m[f] + 1], want_off[f]), f
        assert start[f] % 16 == 0
        assert np.array_equal(blob[start[f]:start[f] + regions[f].size], regions[f]), f
    # nothing outside the three regions is written
    written = np.zeros(blob.size, bool)
    for f in range(3):
        written[start[f]:start[f] + regions[f].size] = True
    assert (blob[~written] == 0xEE).all()


def test_family_regions_keep_sixteen_bytes_of_slack(hs):
    tag = np.array([0, 1, 2, 0, 1, 2], np.uint8)
    off = np.array([3, 20, 20, 53, 70, 71, 100], np.uint64)
    msgs = np.arange(116, dtype=np.uint8)
    _, _, _, _, fo, _ = _split(hs, tag, np.zeros(6, np.uint32), np.zeros((6, 96), np.uint8), msgs, off)
    ends = [int(fo[2]), int(fo[5]), int(fo[8])]
    starts = [int(fo[0]), int(fo[3]), int(fo[6])]
    assert starts == [0, _al16(ends[0] + 16), starts[1] + _al16(ends[1] - starts[1] + 16)]
    assert starts[1] - ends[0] >= 16 and starts[2] - ends[1] >= 16


@pytest.mark.parametrize("kind", PATTERNS)
def test_scatter_puts_verdicts_back_in_item_order(hs, kind):
    rng = np.random.default_rng(5)
    n = 777
    tag = mc.tag_pattern(kind, n, rng)
    idx = np.concatenate([np.flatnonzero(tag == f) for f in range(3)]).astype(np.uint32)
    m = [int((tag == f).sum()) for f in range(3)]
    ok_fam = rng.integers(0, 2, n).astype(np.uint8)
    ok = np.full(n, 7, np.uint8)
    assert hs.hs_mixed_scatter(C.c_size_t(n), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(idx), _p(ok_fam), _p(ok)) == 0
    want = np.zeros(n, np.uint8)
    want[idx] = ok_fam
    assert np.array_equal(ok, want)


def _verify(hs, cp, reg, ed_pub=None, ecdsa=None):
    ed_pub = reg["ed_pub"] if ed_pub is None else ed_pub
    curve, xy = ecdsa if ecdsa is not None else (reg["ecdsa_curve"], reg["ecdsa_xy"])
    curve, xy, ed_pub = (np.ascontiguousarray(a, np.uint8) for a in (curve, xy, ed_pub))
    assert hs.hs_ed25519_set_keys(C.c_size_t(ed_pub.size // 32), _p(ed_pub) if ed_pub.size else None, C.c_uint32(0)) == 0
    n = cp["scheme"].size
    ok = np.full(n, 7, np.uint8)
    assert hs.hs_mixed_verify_registered(C.c_size_t(n), _p(cp["scheme"]), _p(cp["msgs"]), _p(cp["off"]), _p(cp["key_slot"]), _p(cp["sig96"]),
                                         C.c_size_t(curve.size), _p(curve), _p(xy), _p(ok)) == 0
    return ok


@pytest.mark.parametrize("kind", ["alternating", "random", "runs"])
def test_simulated_pipeline_matches_openssl(hs, kind):
    reg = mc.registries(n256=2, n384=2, n_ed=3, seed=3)
    rng = np.random.default_rng(11)
    tag = mc.tag_pattern(kind, 96, rng)
    cp = mc.make_corpus(tag, reg, seed=12, hi=150, junk=True)
    got = _verify(hs, cp, reg)
    want = mc.expected_ok(cp, reg["ecdsa_curve"], reg["ecdsa_xy"], reg["ed_pub"])
    assert np.array_equal(got, want), np.flatnonzero(got != want)
    assert 0 < want.sum() < want.size
    classes = set(cp["cls"][cp["cls"] >= 0].tolist())
    assert len(classes) >= 8, classes


def test_simulated_pipeline_with_bad_and_missing_keys(hs):
    reg = mc.registries(n256=2, n384=1, n_ed=3, seed=4)
    tag = mc.tag_pattern("alternating", 48, np.random.default_rng(0))
    cp = mc.make_corpus(tag, reg, seed=13, hi=40, corrupt=False)
    # small-order and y >= p keys in Ed25519 slots 1 and 2: their items reject
    ed_pub = reg["ed_pub"].copy()
    ed_pub[1], ed_pub[2] = mc.small_order_key(), mc.y_ge_p_key()
    got = _verify(hs, cp, reg, ed_pub=ed_pub)
    want = mc.expected_ok(cp, reg["ecdsa_curve"], reg["ecdsa_xy"], ed_pub)
    assert np.array_equal(got, want)
    ed_items = cp["scheme"] == mc.ED
    assert not got[ed_items & (cp["key_slot"] >= 1)].any() and got[ed_items & (cp["key_slot"] == 0)].all()
    # either registry empty: its items reject, the others are unaffected
    for ecdsa, edp in (((np.zeros(0, np.uint8), np.zeros((0, 96), np.uint8)), reg["ed_pub"]), ((reg["ecdsa_curve"], reg["ecdsa_xy"]), np.zeros((0, 32), np.uint8))):
        got = _verify(hs, cp, reg, ed_pub=edp, ecdsa=ecdsa)
        assert np.array_equal(got, mc.expected_ok(cp, ecdsa[0], ecdsa[1], edp))
