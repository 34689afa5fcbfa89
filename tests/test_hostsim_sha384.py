"""k_sha384 in the CPU simulation (tools/hostsim: sha384.cuh over the SHA-512 core of sha512_core.cuh) against hashlib:
every length from 0 to 400 bytes at every start offset mod 4, the FIPS 180-4 vectors, and a message whose bit length
needs more than 32 bits.  Also checks that k_ed_sha512, which shares the core, still hashes R || A || M as hashlib does.
The GPU twin of this file is test_gpu_sha384.py."""
import ctypes as C
import hashlib
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


def _sha384(hs, buf, off, base=0, perm=None):
    n = off.size - 1
    dig = np.zeros((n, 48), np.uint8)
    assert hs.hs_sha384(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(base), _p(perm) if perm is not None else None, _p(dig)) == 0
    return [bytes(d) for d in dig]


def _ref(buf, off):
    return [hashlib.sha384(memoryview(buf[int(off[i]):int(off[i + 1])])).digest() for i in range(off.size - 1)]


def _ragged(lens, lead, seed):
    """Messages of the given lengths back to back after `lead` bytes, in a buffer readable 8 bytes past the last one."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(lead)
    buf = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    return buf, off


@pytest.mark.parametrize("base", [0, 2**20 + 4 * 1234 + 3])
@pytest.mark.parametrize("start", [0, 1, 2, 3])
def test_every_length_to_400_at_every_start_mod_4(hs, start, base):
    """Lengths 0..400 back to back cross every padding boundary (111/112, 127/128, 239/240, 255/256, 367/368).  The first
    message starts `start` bytes into the blob, so over the four starts every length meets every residue mod 4.  The
    offsets are the caller's, `base` on from 0: the kernel reads message i at off[i] - base (the engine passes the first
    offset of the shard it staged)."""
    buf, off = _ragged(list(range(401)), start, seed=start)
    residues = [set() for _ in range(401)]
    for s in range(4):
        o = np.concatenate([[0], np.cumsum(range(401))]) + s
        for ln in range(401):
            residues[ln].add(int(o[ln]) % 4)
    assert all(r == {0, 1, 2, 3} for r in residues)
    assert _sha384(hs, buf, off + np.uint64(base), base=base) == _ref(buf, off)


def test_permuted_order(hs):
    """Thread t hashes item perm[t]; each digest still lands at its item's slot."""
    buf, off = _ragged(list(range(0, 401, 3)) + [128, 111, 112, 0], 5, seed=7)
    n = off.size - 1
    perm = np.random.default_rng(8).permutation(n).astype(np.uint32)
    assert _sha384(hs, buf, off, perm=perm) == _ref(buf, off)


def test_fips_180_4_vectors(hs):
    msgs = [b"abc", b"abcdefghbcdefghicdefghijdefghijkefghijklfghijklmghijklmnhijklmnoijklmnopjklmnopqklmnopqrlmnopqrsmnopqrstnopqrstu",
            b"a" * 1_000_000, b""]
    want = ["cb00753f45a35e8bb5a03d699ac65007272c32ab0eded1631a8b605a43ff5bed8086072ba1e7cc2358baeca134c825a7",
            "09330c33f71147e83d192fc782cd1b4753111b173b3b05d22fa08086e3b0f712fcc7c71a557e2db966c3e9fa91746039",
            "9d0e1809716474cb086e834e310a4a1ced149e9c00f248527972cec5704c2a5b07b8b3dc38ecc4ebae97ddd87f3d8985",
            "38b060a751ac96384cd9327eb1b1e36a21fdb71114be07434c0cc7bf63f6e1da274edebfe76f65fbd51ad2f14898b95b"]
    off = np.concatenate([[0], np.cumsum([len(m) for m in msgs])]).astype(np.uint64)
    buf = np.frombuffer(b"".join(msgs) + bytes(16), np.uint8).copy()
    assert [d.hex() for d in _sha384(hs, buf, off)] == want


@pytest.mark.parametrize("pre", [[0, 1, 111, 112], [127, 128, 129]])
def test_ed25519_sha512_is_unchanged(hs, pre):
    """k_ed_sha512 runs on the same compression and message loader: its digests of R || A || M (lengths around its own
    block boundaries, which count the 64-byte R || A prefix) still equal hashlib's, and k = digest mod L."""
    lens = pre + list(range(40, 200, 7))
    buf, off = _ragged(lens, 3, seed=11)
    n = off.size - 1
    rng = np.random.default_rng(12)
    sig = rng.integers(0, 256, (n, 64), dtype=np.uint8)
    pub = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    k = np.zeros(8 * n, np.uint32)
    dig = np.zeros(16 * n, np.uint32)
    assert hs.hs_ed25519_sha512(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(0), _p(sig), _p(pub), None, _p(k), _p(dig)) == 0
    want = [hashlib.sha512(bytes(sig[i, :32]) + bytes(pub[i]) + buf[int(off[i]):int(off[i + 1])].tobytes()).digest() for i in range(n)]
    assert [dig.reshape(n, 16)[i].astype("<u4").tobytes() for i in range(n)] == want
    kk = k.reshape(8, n)
    assert [sum(int(kk[w, i]) << (32 * w) for w in range(8)) for i in range(n)] == [int.from_bytes(w, "little") % ref.L for w in want]


def test_bit_length_past_32_bits(hs):
    """2^29 + 56 bytes: the bit length 2^32 + 448 needs the upper half of the low 64-bit length word.  Among short
    messages, hashed in the order of the device's length sort (the long message first).  About 10 s; last, so that
    `pytest -x` meets the cheap tests first."""
    huge = wm.HUGE_SHA[1]
    assert huge * 8 >= 2**32
    lens = [0, 1, 111, 112, huge, 127, 128]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    buf = wm.pattern(int(off[-1]) + 16, seed=5)
    nb = np.minimum((np.diff(off.astype(np.int64)) + 9 + 63) // 64, 1023)
    perm = np.argsort(-nb, kind="stable").astype(np.uint32)
    assert perm[0] == 4
    assert _sha384(hs, buf, off, perm=perm) == _ref(buf, off)
