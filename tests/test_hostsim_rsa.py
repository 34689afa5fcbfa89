"""The RSA device code (rsa.cuh) and k_sha512 (sha512_batch.cuh) in the CPU simulation (tools/hostsim), a group of 16
lanes per item run in lockstep, one OS thread per lane:

- the arithmetic sets of tests/rsa_arith.py through hs_rsa_debug (k_rsa_debug of rsa_debug.cuh, as sbv_debug_rsa runs it on
  the device): Montgomery products through every outcome of the final subtraction, R^2 mod N and n0', S - N with its
  borrow generated in every lane, the carry resolution that ends a product in every lane, and S^e mod N; the products,
  R^2 and S^e on a subset of the modulus shapes (test_gpu_rsa_arith.py runs every shape);
- a handful of whole verifications per class of tests/rsa_cases.py, against oracle_rsa.ref;
- one item of every class of tests/rsa_edges.py per size (test_gpu_rsa_edges.py runs every item);
- k_sha512 against hashlib at the padding boundaries and unaligned starts.
The GPU twins of this file are test_gpu_rsa.py, test_gpu_rsa_arith.py and test_gpu_rsa_edges.py."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

import rsa_arith as arith
import rsa_cases as rc
import rsa_edges as edges

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _call(hs):
    return lambda mb, op, n, *bufs: hs.hs_rsa_debug(C.c_uint32(mb), C.c_int(op), C.c_size_t(n), *map(_p, bufs))


@pytest.fixture(scope="module")
def run(hs):
    return arith.runner(_call(hs))


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
def test_montgomery_products(run, k):
    arith.check_products(run, k, full=False)


@pytest.mark.parametrize("k", rc.SIZES)
def test_r2_and_ninv(run, k):
    arith.check_r2_ninv(run, k, full=False)


@pytest.mark.parametrize("k", rc.SIZES)
def test_subtraction_borrow(run, k):
    arith.check_sub(run, k)


@pytest.mark.parametrize("k", rc.SIZES)
def test_carry_resolution(run, k):
    assert arith.check_resolve(run, k) > 150


@pytest.mark.parametrize("k", rc.SIZES)
def test_pow_chains(run, k):
    arith.check_pow(run, k, full=False)


def test_hook_refuses_bad_calls(hs):
    arith.check_refused(_call(hs))


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


# one hash per size, so that the three pairs cover every hash and the 4096-bit size meets SHA-384
EDGE_HASH = {256: edges.ref.SHA256, 384: edges.ref.SHA512, 512: edges.ref.SHA384}


@pytest.mark.parametrize("k", rc.SIZES)
def test_edge_classes(hs, k):
    """One item of every class of tests/rsa_edges.py: the shortest key's valid and corrupted signatures, the longest odd
    exponent with alternating bits, an even exponent accepted (S and N - S) and refused (-EM), a changed DigestInfo
    byte, the separator, a digest byte and one changed byte in a middle lane."""
    h = EDGE_HASH[k]
    K, NL = k // 4, k // 64
    sets = [(edges.bitlen(k, h), [f"bitlen{8 * k - 7}_valid", f"bitlen{8 * k - 7}_valid_bit", f"bitlen{8 * k - 4}_n-1"]),
            (edges.oddexp(k, h), ["oddexp_0x55555555"]),
            (edges.evenexp(k, h), ["evenexp_0x2_n-s", "evenexp_0x7ffffffe_s", "evenexp_0x4_minus_em"]),
            (edges.encoding(k, h, limbs=[7 * NL + 2]), ["encoding_good", "encoding_digest_info9", "encoding_separator", "encoding_digest17",
                                                         f"encoding_limb{7 * NL + 2}"])]
    for c, names in sets:
        idx = np.array([c["cls"].index(nm) for nm in names])
        ok = _verify(hs, c, idx)
        assert list(ok) == list(c["want"][idx]), list(zip(names, ok))
    assert K > 7 * NL + 2
