"""The RSA device code (rsa.cuh) and k_sha512 (sha512_batch.cuh) in the CPU simulation (tools/hostsim), a group of 16
lanes per item run in lockstep, one OS thread per lane:

- Montgomery products against Python integers for 0, 1, N - 1, operands near R and random operands, on moduli at both
  ends (an all-ones top limb, and 2^(8k-8) + 1) and on real keys, for every size;
- S - N and its borrow, n0' = -N^-1 mod 2^32 and R^2 mod N for every size;
- the carry resolution that ends a product, on redundant forms that reach every branch of its ballot;
- a handful of whole verifications per class of tests/rsa_cases.py, against oracle_rsa.ref;
- k_sha512 against hashlib at the padding boundaries and unaligned starts.
The GPU twin of this file is test_gpu_rsa.py."""
import ctypes as C
import hashlib
import os
import random
import subprocess

import numpy as np
import pytest

import rsa_cases as rc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows(vals, k):
    return np.frombuffer(b"".join(v.to_bytes(k, "big") for v in vals), np.uint8).reshape(len(vals), k).copy()


def _op(hs, k, op, a, b, n):
    cnt = len(n)
    A, B, N = _rows(a, k), _rows(b, k), _rows(n, k)
    out, ninv = np.zeros((cnt, k), np.uint8), np.zeros(cnt, np.uint32)
    assert hs.hs_rsa_op(C.c_int(k // 64), C.c_int(op), C.c_size_t(cnt), _p(A), _p(B), _p(N), _p(out), _p(ninv)) == 0
    return [int.from_bytes(r.tobytes(), "big") for r in out], [int(x) for x in ninv]


def _moduli(k):
    """Odd moduli at both ends of the size: an all-ones top limb, 2^(8k-8) + 1 (the smallest with a nonzero leading byte),
    a random one with the top bit set, and a real key."""
    rng = random.Random(k)
    return [2 ** (8 * k) - 1 - 2 * rng.getrandbits(8 * k - 40), 2 ** (8 * k - 8) + 1, rng.getrandbits(8 * k) | 1 | (1 << (8 * k - 1)), rc.key(8 * k).n]


def _ragged(lens, lead, seed):
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(lead)
    buf = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    return buf, off


@pytest.mark.parametrize("start", [0, 1, 2, 3])
def test_sha512_lengths_and_offsets(hs, start):
    lens = list(range(0, 300)) + [383, 384, 495, 496, 1000]
    buf, off = _ragged(lens, start, seed=start)
    n = len(lens)
    dig = np.zeros((n, 64), np.uint8)
    perm = np.random.default_rng(start).permutation(n).astype(np.uint32)
    assert hs.hs_sha512(C.c_size_t(n), _p(buf), _p(off), C.c_uint64(0), _p(perm), _p(dig)) == 0
    for i in range(n):
        assert dig[i].tobytes() == hashlib.sha512(buf[int(off[i]):int(off[i + 1])].tobytes()).digest(), lens[i]


@pytest.mark.parametrize("k", rc.SIZES)
def test_montgomery_products(hs, k):
    R = 2 ** (8 * k)
    rng = random.Random(100 + k)
    a, b, n = [], [], []
    for N in _moduli(k):
        near_r = [N - 1, N - 2, (R - 1) % N, (R - 2**32) % N]
        ops = [0, 1, N - 1, rng.randrange(N), rng.randrange(N)] + near_r
        pairs = [(0, rng.randrange(N)), (1, 1), (N - 1, N - 1), (N - 1, 1), (ops[3], ops[4]), (near_r[2], near_r[2]), (near_r[3], near_r[0]),
                 (rng.randrange(N), rng.randrange(N))]
        for x, y in pairs:
            a.append(x); b.append(y); n.append(N)
    got, ninv = _op(hs, k, 0, a, b, n)
    rinv = {N: pow(R, -1, N) for N in set(n)}
    for i, (x, y, N) in enumerate(zip(a, b, n)):
        assert got[i] == x * y * rinv[N] % N, (i, hex(N)[:12])
        assert ninv[i] == (-pow(N, -1, 2**32)) % 2**32


@pytest.mark.parametrize("k", rc.SIZES)
def test_r2_and_ninv(hs, k):
    ns = _moduli(k)
    got, ninv = _op(hs, k, 1, [0] * len(ns), [0] * len(ns), ns)
    for N, r2, ni in zip(ns, got, ninv):
        assert r2 == 2 ** (16 * k) % N
        assert ni == (-pow(N, -1, 2**32)) % 2**32


@pytest.mark.parametrize("k", rc.SIZES)
def test_subtraction_borrow(hs, k):
    """S - N with its borrows resolved across the group: the range check S < N."""
    N = rc.key(8 * k).n
    R = 2 ** (8 * k)
    a = [0, 1, N - 1, N, N + 1, R - 1, N + (1 << 200), N - (1 << 300), (N >> 64) << 64]
    got, bo = _op(hs, k, 2, a, [0] * len(a), [N] * len(a))
    for x, d, b in zip(a, got, bo):
        assert d == (x - N) % R and b == (1 if x < N else 0), hex(x)[:20]


@pytest.mark.parametrize("k", rc.SIZES)
def test_carry_resolution(hs, k):
    """The end of a product (rsa_resolve) on redundant forms built to reach every branch of the ballot: lanes that are all
    ones after the lazy word below lands (propagate), lanes whose add carries out (generate), chains of both up to and
    out of the top lane, and values on both sides of N.  A form is limbs t plus a lazy word cz_l <= 3 per lane at the
    weight of lane l + 1's first limb; the value is below 2N, and the result must be that value mod N."""
    K = k // 4
    NL = K // 16
    W = 32 * NL  # bits per lane
    R = 2 ** (8 * k)
    rng = random.Random(200 + k)
    N = 2 ** (8 * k) - 1 - 2 * rng.getrandbits(8 * k - 40)  # top 40 bits all ones, so R - small < 2N
    lane_ones = (1 << W) - 1
    forms = []

    def add(t, cz):
        v = t + sum(c << (W * (l + 1)) for l, c in enumerate(cz))
        if 0 <= t < R and v < 2 * N:
            forms.append((t, cz, v))

    add(R - 4, [0] * 16)                           # no lazy words: lanes 1..15 all ones, nothing moves
    add(R - 3, [2] + [0] * 15)                     # lane 1 overflows; lanes 2..15 propagate; the carry leaves the top
    add(R - 1 - (3 << W), [3] + [0] * 15)          # lane 1 becomes all ones: it propagates, nothing to propagate
    add(R - (3 << W), [3] + [0] * 15)              # value R: lane 1 overflows and the carry leaves the top
    add(R - (1 << (W * 15)), [0] * 14 + [1, 0])    # lane 15 overflows on its lazy word alone
    add(N - 1, [0] * 16)
    add(N, [0] * 16)
    add(N - (2 << (W * 3)), [0, 0, 2] + [0] * 13)
    for _ in range(40):
        cz = [rng.randrange(4) if rng.random() < 0.7 else 0 for _ in range(15)] + [0]
        # limbs mostly all ones, so that carries meet propagating lanes
        t = 0
        for l in range(16):
            t |= (lane_ones - (rng.randrange(4) if rng.random() < 0.3 else 0)) << (W * l)
        add(t - rng.randrange(2 ** 20), cz)
        add(rng.randrange(2 * N) - sum(c << (W * (l + 1)) for l, c in enumerate(cz)), cz)
    assert len(forms) > 40
    A = _rows([f[0] for f in forms], k)
    B = np.array([f[1] for f in forms], np.uint32)
    Nr = _rows([N] * len(forms), k)
    out, dummy = np.zeros((len(forms), k), np.uint8), np.zeros(len(forms), np.uint32)
    assert hs.hs_rsa_op(C.c_int(NL), C.c_int(3), C.c_size_t(len(forms)), _p(A), _p(B), _p(Nr), _p(out), _p(dummy)) == 0
    for (t, cz, v), o in zip(forms, out):
        assert int.from_bytes(o.tobytes(), "big") == v % N, (hex(t)[:20], cz)


def _verify(hs, c, idx):
    k, hl = c["k"], 32 + 16 * c["hash"]
    sel = lambda a: np.ascontiguousarray(a[idx])  # noqa: E731
    sig, mod, exp, dig = sel(c["sig"]), sel(c["mod"]), sel(c["exp"]), sel(c["digest"])
    ok = np.full(len(idx), 7, np.uint8)
    assert hs.hs_rsa_verify(C.c_int(k // 64), C.c_size_t(len(idx)), C.c_uint32(c["hash"]), _p(sig), _p(mod), _p(exp), _p(dig), _p(ok)) == 0
    assert dig.shape[1] == hl
    return ok


@pytest.mark.parametrize("k,hash", [(k, h) for k in rc.SIZES for h in rc.HASHES if (k, h) != (512, 1)])
def test_whole_verifications_per_class(hs, k, hash):
    """One item of every class (tests/rsa_cases.py) per size and hash; the 4096-bit keys only over SHA-256 and SHA-512, the
    two ends of the encoding's width (the GPU file runs every pair)."""
    c = rc.make_cases(k, hash, seed=1, short=True)
    seen, idx = set(), []
    for i, cl in enumerate(c["cls"]):
        if cl not in seen:
            seen.add(cl)
            idx.append(i)
    ok = _verify(hs, c, np.array(idx))
    want = c["want"][idx]
    bad = [c["cls"][i] for i, g, w in zip(idx, ok, want) if g != w]
    assert not bad, bad
    assert 0 < want.sum() < len(idx)
