"""The kernels of mixed_hash.cuh in the CPU simulation (tools/hostsim): k_mix_alg against numpy, and k_sha2_sel against
hashlib in both family layouts (P-256: 32-byte slots, P-384: 48-byte slots), with flags read through the family's shard
indices, in length-sorted and shuffled processing orders, with SHA-256 and SHA-384 items side by side in one warp.
The GPU twin of this file is test_gpu_mixed384.py."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
JUNK = 0xA5


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _mix_alg(hs, tag):
    t = np.ascontiguousarray(tag, dtype=np.uint8).copy()
    flag = np.full(t.size, JUNK, np.uint8)
    assert hs.hs_mix_alg(C.c_size_t(t.size), _p(t), _p(flag)) == 0
    return t, flag


@pytest.mark.parametrize("pattern", ["random", "runs", "alternating", "ecdsa_only", "sha384_only"])
def test_mix_alg_maps_tags_to_families_and_flags_sha384(hs, pattern):
    rng = np.random.default_rng(1)
    n = 1000  # not a multiple of the 256-thread block: the grid guard is crossed
    if pattern == "random":
        tag = rng.integers(0, 5, n)
    elif pattern == "runs":
        tag = np.repeat(rng.integers(0, 5, 40), rng.integers(1, 60, 40))[:n]
    elif pattern == "alternating":
        tag = np.tile([3, 0, 4, 1, 2], n // 5)
    elif pattern == "ecdsa_only":
        tag = rng.integers(0, 2, n)
    else:
        tag = rng.integers(3, 5, n)
    tag = tag.astype(np.uint8)
    fam, flag = _mix_alg(hs, tag)
    np.testing.assert_array_equal(fam, np.where(tag >= 3, tag - 3, tag))
    np.testing.assert_array_equal(flag, (tag >= 3).astype(np.uint8))


def _family(lens, lead, seed):
    """Messages of the given lengths back to back after `lead` bytes (readable 16 bytes past the last one)."""
    rng = np.random.default_rng(seed)
    off = (np.concatenate([[0], np.cumsum(lens)]) + lead).astype(np.uint64)
    buf = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    return buf, off


def _want(buf, off, wide, dlen):
    """e as k_prep reads it: dlen 32 = SHA-256 or the first 32 bytes of SHA-384; dlen 48 = SHA-384 or 16 zeros || SHA-256."""
    out = []
    for j in range(off.size - 1):
        m = memoryview(buf[int(off[j]):int(off[j + 1])])
        if wide[j]:
            out.append(hashlib.sha384(m).digest()[:dlen])
        else:
            out.append(bytes(dlen - 32) + hashlib.sha256(m).digest())
    return out


def _sel(hs, buf, off, idx, flags, dlen, perm=None, base=0):
    n = off.size - 1
    guard = 64
    dig = np.full(n * dlen + guard, JUNK, np.uint8)  # junk: every byte of every slot must be written, and nothing past them
    assert hs.hs_sha2_sel(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(base), _p(idx), _p(flags), C.c_uint32(dlen),
                          _p(perm) if perm is not None else None, _p(dig)) == 0
    assert (dig[n * dlen:] == JUNK).all(), "k_sha2_sel wrote past the family's digest slots"
    return [bytes(dig[j * dlen:(j + 1) * dlen]) for j in range(n)]


def _length_sort(off):
    """The order of the device's block-count sort (longest first, stable)."""
    nb = (np.diff(off.astype(np.int64)) + 9 + 63) // 64
    return np.argsort(-nb, kind="stable").astype(np.uint32)


def _case(lens, lead, seed, wide_rate=0.5, shard_extra=37):
    """A family of len(lens) items inside a shard of len(lens) + shard_extra items: idx maps family item j to its shard
    index (increasing, as the split makes them, but not the identity), and the shard's flags hold the other items' flags
    too (set to the opposite of what a misread would need to pass)."""
    rng = np.random.default_rng(seed)
    n = len(lens)
    buf, off = _family(lens, lead, seed)
    idx = np.sort(rng.choice(n + shard_extra, n, replace=False)).astype(np.uint32)
    wide = (rng.random(n) < wide_rate).astype(np.uint8)
    flags = (rng.random(n + shard_extra) < 0.5).astype(np.uint8)
    flags[idx] = wide
    return buf, off, idx, flags, wide


EDGES = [0, 1, 55, 56, 63, 64, 65, 111, 112, 119, 120, 127, 128, 129, 239, 240, 255, 256]


@pytest.mark.parametrize("dlen", [32, 48])
@pytest.mark.parametrize("lead", [0, 1, 2, 3])
def test_padding_edges_both_hashes_both_layouts(hs, dlen, lead):
    """Every edge length under both hashes: the SHA-256 padding edges 55/56/64 and the SHA-384 edges 111/112/128, each
    message at every start offset mod 4 over the four leads."""
    lens = EDGES * 2
    buf, off = _family(lens, lead, seed=10 + lead)
    n = len(lens)
    wide = np.array([0] * len(EDGES) + [1] * len(EDGES), np.uint8)
    idx = np.arange(n, dtype=np.uint32)[::-1].copy()  # family item j is shard item n - 1 - j
    flags = wide[::-1].copy()
    assert _sel(hs, buf, off, idx, flags, dlen) == _want(buf, off, wide, dlen)


@pytest.mark.parametrize("dlen", [32, 48])
@pytest.mark.parametrize("order", ["identity", "length_sort", "shuffled"])
def test_ragged_family_with_hashes_mixed_inside_warps(hs, dlen, order):
    """300 items with ragged lengths up to 4 KiB, SHA-256 and SHA-384 at random inside every 32-item warp, flags read
    through idx from a larger shard."""
    rng = np.random.default_rng(7 + dlen)
    lens = list(rng.integers(0, 4097, 300))
    lens[:len(EDGES)] = EDGES
    buf, off, idx, flags, wide = _case(lens, lead=3, seed=dlen)
    for w in range(0, 300, 32):  # both hashes inside every warp of the identity order
        assert 0 < wide[w:w + 32].sum() < len(wide[w:w + 32])
    perm = None
    if order == "length_sort":
        perm = _length_sort(off)
    elif order == "shuffled":
        perm = rng.permutation(300).astype(np.uint32)
    assert _sel(hs, buf, off, idx, flags, dlen, perm) == _want(buf, off, wide, dlen)


@pytest.mark.parametrize("dlen", [32, 48])
@pytest.mark.parametrize("rate", [0.0, 1.0])
def test_single_hash_family_matches_the_single_hash_kernels(hs, dlen, rate):
    """A family of one hash only: every slot is what k_sha256 (rate 0) or k_sha384 (rate 1) writes, laid out for dlen."""
    rng = np.random.default_rng(int(rate) + dlen)
    lens = list(rng.integers(0, 700, 130))
    buf, off, idx, flags, wide = _case(lens, lead=1, seed=5, wide_rate=rate)
    n = len(lens)
    got = _sel(hs, buf, off, idx, flags, dlen, _length_sort(off))
    if rate:
        ref = np.zeros((n, 48), np.uint8)
        assert hs.hs_sha384(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(0), None, _p(ref)) == 0
        assert got == [bytes(r[:dlen]) for r in ref]
    else:
        ref = np.zeros((n, 32), np.uint8)
        assert hs.hs_sha256(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(0), None, _p(ref)) == 0
        assert got == [bytes(dlen - 32) + bytes(r) for r in ref]


def test_offsets_relative_to_base(hs):
    """The family's offsets are read relative to base, as for k_sha256 (the engine passes 0: a family's offsets are
    positions in the shared buffer)."""
    lens = [5, 130, 0, 64, 200]
    buf, off, idx, flags, wide = _case(lens, lead=2, seed=3, wide_rate=0.5)
    base = 1 << 20
    got = _sel(hs, buf, off + np.uint64(base), idx, flags, 48, base=base)
    assert got == _want(buf, off, wide, 48)
