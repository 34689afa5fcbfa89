"""The hash and mixed-split kernels past 32 bits, in the CPU simulation (tools/hostsim): bit lengths of 2^32 and more,
message offsets past 2^32 both as the kernels see them with base 0 and as the engine hands them over (base = the first
offset, over a small staged copy), and per-family byte sums past 2^32 in the split and the compaction of mixed shards.

Offsets past 2^32 live in sparse buffers (tests/wide_messages.py), so they cost no memory.  The long messages take about
8 s each in the simulation and come last, so that `pytest -x` meets the cheap tests first.  The GPU twin of this file is
test_gpu_wide.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import wide_messages as wm
from oracle_ed25519 import ref

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


def _sha256(hs, buf, off, base=0, perm=None):
    n = off.size - 1
    dig = np.zeros((n, 32), np.uint8)
    assert hs.hs_sha256(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(base), _p(perm) if perm is not None else None, _p(dig)) == 0
    return [bytes(d) for d in dig]


def _sha512(hs, buf, off, sig, pub, base=0):
    n = off.size - 1
    k = np.zeros(8 * n, np.uint32)
    dig = np.zeros(16 * n, np.uint32)
    assert hs.hs_ed25519_sha512(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(base), _p(sig), _p(pub), None, _p(k), _p(dig)) == 0
    kk = k.reshape(8, n)
    return [dig.reshape(n, 16)[i].astype("<u4").tobytes() for i in range(n)], [sum(int(kk[w, i]) << (32 * w) for w in range(8)) for i in range(n)]


def _length_sort(off):
    """The order the device's counting sort gives: most SHA-256 blocks first, input order among equals."""
    nb = np.minimum((np.diff(off.astype(np.int64)) + 9 + 63) // 64, 1023)
    return np.argsort(-nb, kind="stable").astype(np.uint32)


def _far_probes(arrangement, seed):
    """The probe set past 2^32: base 0 over a sparse buffer that holds it at wm.FAR, or base = the first offset over a copy
    of just its bytes (what the engine stages)."""
    lay = wm.probe_layout()
    buf = wm.sparse(wm.FAR + lay.bytes + 64)
    off = wm.fill(buf, wm.FAR, lay, seed)
    assert int(off[0]) > 2**32
    if arrangement == "base0":
        return lay, buf, off, buf, 0
    return lay, buf, off, np.concatenate([buf[int(off[0]):int(off[-1])], np.zeros(16, np.uint8)]), int(off[0])


@pytest.mark.parametrize("arrangement", ["base0", "staged"])
def test_sha256_probe_set_past_2_32(hs, arrangement):
    lay, buf, off, src, base = _far_probes(arrangement, 11)
    want = wm.sha256_ref(buf, off)
    assert _sha256(hs, src, off, base) == want
    twins = np.flatnonzero(lay.kind == wm.TWIN)
    assert all(want[t] != want[lay.twin_of[t]] for t in twins if lay.lens[t])


@pytest.mark.parametrize("arrangement", ["base0", "staged"])
def test_sha512_probe_set_past_2_32(hs, arrangement):
    lay, buf, off, src, base = _far_probes(arrangement, 12)
    rng = np.random.default_rng(13)
    sig = rng.integers(0, 256, (lay.n, 64), dtype=np.uint8)
    pub = rng.integers(0, 256, (lay.n, 32), dtype=np.uint8)
    dig, k = _sha512(hs, src, off, sig, pub, base)
    want = wm.sha512_ref(buf, off, sig, pub)
    assert dig == want
    assert k == [int.from_bytes(w, "little") % ref.L for w in want]


def _split_model(tag, off):
    lens = np.diff(off.astype(np.int64))
    idx = [np.flatnonzero(tag == f) for f in range(3)]
    B = [int(lens[i].sum()) for i in idx]
    start = [0, _al16(B[0] + 16)]
    start.append(start[1] + _al16(B[1] + 16))
    offs = [[start[f] + int(v) for v in np.concatenate([[0], np.cumsum(lens[i])])] for f, i in enumerate(idx)]
    return idx, offs


def test_mixed_split_with_family_byte_sums_past_2_32(hs):
    """Count, scan and split read offsets only: items of 1.5 GiB put a tile's P-256 bytes, every family's total and the
    split's running positions past 2^32.  Family offsets and the split against a Python model."""
    rng = np.random.default_rng(21)
    n = 100
    tag = (np.arange(n) % 3).astype(np.uint8)
    tag[:3] = wm.P256
    lens = rng.integers(0, 200, n).astype(np.int64)
    lens[:3] = 3 * 2**29                                   # tile 0: 4.5 GiB of P-256 bytes
    big = rng.choice(np.arange(16, n), 12, replace=False)
    lens[big] = 3 * 2**29 + rng.integers(0, 16, big.size)  # every family's running sum passes 2^32 again later
    off = (np.concatenate([[0], np.cumsum(lens)]) + 2**33 + 5).astype(np.uint64)
    slot = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    sig96 = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    m = [int((tag == f).sum()) for f in range(3)]
    idx, slo = np.full(n + 1, 0xFFFFFFFF, np.uint32), np.full(n + 1, 0xFFFFFFFF, np.uint32)
    r0, s0 = np.zeros((m[0] + 1, 32), np.uint8), np.zeros((m[0] + 1, 32), np.uint8)
    r1, s1 = np.zeros((m[1] + 1, 48), np.uint8), np.zeros((m[1] + 1, 48), np.uint8)
    sig2 = np.zeros((m[2] + 1, 64), np.uint8)
    fo = np.full(n + 3, 2**64 - 1, np.uint64)
    assert hs.hs_mixed_split(C.c_size_t(n), _p(tag), _p(slot), _p(sig96), _p(off), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(idx), _p(slo), _p(r0),
                             _p(s0), _p(r1), _p(s1), _p(sig2), _p(fo)) == 0
    want_idx, want_off = _split_model(tag, off)
    assert max(max(o) for o in want_off) > 2**34
    assert np.array_equal(idx[:n], np.concatenate(want_idx))
    assert np.array_equal(slo[:n], slot[idx[:n]])
    assert np.array_equal(r0[:m[0]], sig96[want_idx[0], :32]) and np.array_equal(s1[:m[1]], sig96[want_idx[1], 48:])
    assert np.array_equal(sig2[:m[2]], sig96[want_idx[2], :64])
    at = [0, m[0] + 1, m[0] + m[1] + 2]
    for f in range(3):
        assert [int(v) for v in fo[at[f]:at[f] + m[f] + 1]] == want_off[f], f


@pytest.mark.parametrize("arrangement", ["base0", "staged"])
def test_mixed_compaction_past_2_32(hs, arrangement):
    """k_mix_compact with source offsets past 2^32 (base 0) or a staged copy (base = the first offset), into family regions
    that start past 2^32.  Every destination residue mod 16 and source residue mod 4 occurs; the regions must be byte-exact
    and the bytes around and between them untouched."""
    lay, buf, off, src, base = _far_probes(arrangement, 31)
    n = lay.n
    idx = [np.flatnonzero(lay.tag == f) for f in range(3)]
    m = [i.size for i in idx]
    B = [int(lay.lens[i].sum()) for i in idx]
    start = [wm.FAR + 2**20]
    start += [start[0] + _al16(B[0] + 16), start[0] + _al16(B[0] + 16) + _al16(B[1] + 16)]
    fo = np.concatenate([np.concatenate([[0], np.cumsum(lay.lens[i])]) + start[f] for f, i in enumerate(idx)]).astype(np.uint64)
    for f, i in enumerate(idx):  # the probes and twins of a family cover every residue mod 16 of its region
        pt = np.isin(lay.kind[i], (wm.PROBE, wm.TWIN))
        assert set((fo[np.flatnonzero(pt) + sum(m[:f]) + f] % 16).tolist()) == set(range(16))
    end = start[2] + B[2]
    blob = wm.sparse(end + 4096)
    blob[start[0] - 64:] = 0xEE
    assert hs.hs_mixed_compact(C.c_size_t(n), C.c_uint32(m[0]), C.c_uint32(m[1]), _p(src), _p(off), C.c_uint64(base),
                               _p(np.concatenate(idx).astype(np.uint32)), _p(fo), _p(blob)) == 0
    written = np.zeros(blob.size - (start[0] - 64), bool)
    for f, i in enumerate(idx):
        want = np.concatenate([buf[int(off[j]):int(off[j + 1])] for j in i])
        assert np.array_equal(blob[start[f]:start[f] + B[f]], want), f
        written[start[f] - (start[0] - 64):start[f] - (start[0] - 64) + B[f]] = True
    assert (blob[start[0] - 64:][~written] == 0xEE).all()


@pytest.mark.parametrize("which", [0, 1])
def test_sha256_bit_length_past_32_bits(hs, which):
    """2^29 - 1 bytes (bit length 2^32 - 8: high word 0) and 2^29 + 56 bytes (high word 1, the length in a block of its own),
    among short messages; the first in input order, the second in the length sort's order."""
    huge = wm.HUGE_SHA[which]
    short = [0, 1, 55, 56, 64, 119, 120, 200]
    lens = short + [huge] if which == 0 else [huge] + short
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    buf = wm.pattern(int(off[-1]) + 16, seed=which)
    perm = _length_sort(off) if which == 1 else None
    if perm is not None:
        assert perm[0] == 0  # the long message is hashed by thread 0
    assert _sha256(hs, buf, off, perm=perm) == wm.sha256_ref(buf, off)


def test_sha512_bit_length_past_32_bits(hs):
    """M = 2^29 - 63 bytes: 64 + M bytes hashed, so the bit length is 2^32 + 8.  Digest against hashlib, k = digest mod L."""
    rng = np.random.default_rng(3)
    off = np.array([0, 5, 5 + wm.HUGE_ED, 5 + wm.HUGE_ED + 1], np.uint64)
    buf = wm.pattern(int(off[-1]) + 16, seed=2)
    sig = rng.integers(0, 256, (3, 64), dtype=np.uint8)
    pub = rng.integers(0, 256, (3, 32), dtype=np.uint8)
    dig, k = _sha512(hs, buf, off, sig, pub)
    want = wm.sha512_ref(buf, off, sig, pub)
    assert dig == want
    assert k == [int.from_bytes(w, "little") % ref.L for w in want]
