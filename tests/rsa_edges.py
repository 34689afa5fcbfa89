"""Verdict sets for RSA PKCS #1 v1.5 that reach what tests/rsa_cases.py does not, judged by oracle_rsa.ref: keys of
several bit lengths, odd exponents of every bit length, accepted even exponents, and the encoding changed at every
position the kernel compares.  Kept out of rsa_cases.py, whose corpus test_oracle_rsa.py also checks against OpenSSL,
which may refuse some of these keys (a 2041-bit modulus, e = 2).  Shared by test_hostsim_rsa.py (one item per class) and
test_gpu_rsa_edges.py (every item).

The keys come from tests/golden/rsa_keys.npz (made by tests/golden/make_rsa_keys.py):
  std_<b>   oracle_rsa.ref.Key(b, 1) for b = 8k, 8k - 1, 8k - 4, 8k - 7
  blum_<b>  a Blum key of b = 8k bits, p = q = 3 (mod 4)

Sets, per size k and hash (each returns a dict like rsa_cases.make_cases, digests given per item):
  bitlen    per key of every bit length: a valid signature, N - 1, and a one-bit corruption of each (e = 65537);
            messages included, so the set also goes through the fused hash-and-verify call
  oddexp    for every bit length j from 2 to 31 the smallest odd e of that length prime to lambda, and e = 2^j - 1 where
            it is invertible; 0x55555555 and the smallest invertible e from 0x2AAAAAAB up: a valid signature each
  evenexp   a Blum key: S with S^e = EM for e in {2, 4, 2^30, 2 * 65537, 2^31 - 2} and an EM that is a square mod p and q,
            both S and N - S; and per e an S with S^e = -EM for an EM that is a square mod neither (rejected)
  encoding  the intact encoding; every digest byte flipped (the valid signature, the digest changed); every DigestInfo
            byte, the separator and bytes 0 and 1 changed in an EM signed with d; and (SHA-256 only) one byte changed
            in every limb, at position 4L + (L mod 4) from the end for limb L, so that all four byte positions of a word
            occur in every lane
"""
from __future__ import annotations

import functools
import math
import os
import random

import numpy as np

from oracle_rsa import ref

SIZES = (256, 384, 512)
HASHES = (ref.SHA256, ref.SHA384, ref.SHA512)
E = 65537
EVEN_EXPONENTS = (2, 4, 2**30, 2 * 65537, 2**31 - 2)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rsa_keys.npz")


@functools.lru_cache(maxsize=None)
def _golden():
    with np.load(GOLDEN) as z:
        return {name: int.from_bytes(z[name].tobytes(), "big") for name in z.files}


@functools.lru_cache(maxsize=None)
def key(name: str) -> ref.Key:
    """A key of the golden file: std_<bits> or blum_<bits>."""
    g = _golden()
    K = ref.Key.from_primes(g[name + "_p"], g[name + "_q"])
    assert K.bits == int(name.split("_")[1]) and K.p != K.q, name
    if name.startswith("blum"):
        assert K.p % 4 == 3 and K.q % 4 == 3, name
    return K


class _Set:
    def __init__(self, k, hash, name):
        self.k, self.hash, self.hl = k, hash, ref.HLEN[hash]
        self.rng = random.Random(f"rsa-edges-{name}-{k}-{hash}")
        self.msgs, self.dig, self.sig, self.mod, self.exp, self.cls = [], [], [], [], [], []

    def msg(self):
        return self.rng.randbytes(self.rng.randrange(1, 200))

    def digest(self, m):
        return ref.HASHLIB[self.hash](m).digest()

    def add(self, cls, digest, sig, N, e, msg=b""):
        if isinstance(sig, int):
            sig = sig.to_bytes(self.k, "big")
        assert len(sig) == self.k and len(digest) == self.hl
        self.msgs.append(bytes(msg)); self.dig.append(bytes(digest)); self.sig.append(bytes(sig))
        self.mod.append(N.to_bytes(self.k, "big")); self.exp.append(e); self.cls.append(cls)

    def done(self):
        k, n = self.k, len(self.cls)
        off = np.concatenate([[0], np.cumsum([len(m) for m in self.msgs])]).astype(np.uint64)
        out = dict(k=k, hash=self.hash, n=n, msgs=np.frombuffer(b"".join(self.msgs) + b"\0", np.uint8)[:-1].copy(), off=off,
                   digest=np.frombuffer(b"".join(self.dig), np.uint8).reshape(n, self.hl).copy(),
                   sig=np.frombuffer(b"".join(self.sig), np.uint8).reshape(n, k).copy(),
                   mod=np.frombuffer(b"".join(self.mod), np.uint8).reshape(n, k).copy(), exp=np.array(self.exp, np.uint32), cls=list(self.cls))
        out["want"] = ref.verify_batch(k, self.hash, out["digest"], out["sig"], out["mod"], out["exp"])
        return out


def bitlen(k, hash):
    s = _Set(k, hash, "bitlen")
    for b in (8 * k, 8 * k - 1, 8 * k - 4, 8 * k - 7):
        K = key(f"std_{b}")
        m = s.msg()
        h = s.digest(m)
        sig = int.from_bytes(K.sign(k, hash, h, E), "big")
        flip = 1 << s.rng.randrange(b - 1)
        s.add(f"bitlen{b}_valid", h, sig, K.n, E, m)
        s.add(f"bitlen{b}_n-1", h, K.n - 1, K.n, E, m)
        s.add(f"bitlen{b}_valid_bit", h, sig ^ flip, K.n, E, m)
        s.add(f"bitlen{b}_n-1_bit", h, (K.n - 1) ^ flip, K.n, E, m)
    out = s.done()
    assert list(out["want"]) == [1, 0, 0, 0] * 4
    return out


def odd_exponents(lam):
    """The odd exponents of the oddexp set for a key with lambda = lam."""
    es = []
    for j in range(2, 32):
        e = 2 ** (j - 1) + 1
        while math.gcd(e, lam) != 1:
            e += 2
        assert e.bit_length() == j
        es.append(e)
        if math.gcd(2**j - 1, lam) == 1:
            es.append(2**j - 1)
    e = 0x2AAAAAAB
    while math.gcd(e, lam) != 1:
        e += 2
    es += [0x55555555, e]
    assert all(math.gcd(e, lam) == 1 for e in es)
    return sorted(set(es))


def oddexp(k, hash):
    s = _Set(k, hash, "oddexp")
    K = key(f"std_{8 * k}")
    for e in odd_exponents(K.lam):
        h = s.digest(s.msg())
        s.add(f"oddexp_{e:#x}", h, K.sign(k, hash, h, e), K.n, e)
    out = s.done()
    assert out["want"].all()
    return out


def _sqrt_root(K, x, e):
    """S with S^e = x (mod N) for even e and x a square mod p and q (p = q = 3 mod 4): with d_p = e^-1 mod (p - 1) / 2,
    (x^d_p)^e = x^(1 + j (p - 1) / 2) = x mod p, and likewise mod q."""
    p, q = K.p, K.q
    sp = pow(x % p, pow(e, -1, (p - 1) // 2), p)
    sq = pow(x % q, pow(e, -1, (q - 1) // 2), q)
    return sp + p * ((sq - sp) * pow(p, -1, q) % q)


def _is_square(x, p):
    return pow(x % p, (p - 1) // 2, p) == 1


def evenexp(k, hash):
    s = _Set(k, hash, "evenexp")
    K = key(f"blum_{8 * k}")
    for e in EVEN_EXPONENTS:
        while True:  # an EM that is a square mod p and mod q
            h = s.digest(s.msg())
            em = int.from_bytes(ref.encode(k, hash, h), "big")
            if _is_square(em, K.p) and _is_square(em, K.q):
                break
        S = _sqrt_root(K, em, e)
        for name, sv in (("s", S), ("n-s", K.n - S)):
            assert pow(sv, e, K.n) == em
            assert ref.verify(k, hash, h, sv.to_bytes(k, "big"), K.mod_bytes(k), e)
            s.add(f"evenexp_{e:#x}_{name}", h, sv, K.n, e)
        while True:  # an EM that is a square mod neither: -EM is a square mod both (-1 is not, for Blum primes)
            h = s.digest(s.msg())
            em = int.from_bytes(ref.encode(k, hash, h), "big")
            if not _is_square(em, K.p) and not _is_square(em, K.q):
                break
        S = _sqrt_root(K, K.n - em, e)
        assert pow(S, e, K.n) == K.n - em
        s.add(f"evenexp_{e:#x}_minus_em", h, S, K.n, e)
    out = s.done()
    assert list(out["want"]) == [1, 1, 0] * len(EVEN_EXPONENTS)
    return out


def encoding(k, hash, limbs=None):
    """limbs: the limbs that get a changed byte (default: every limb for SHA-256, none for the other hashes)."""
    s = _Set(k, hash, "encoding")
    K = key(f"std_{8 * k}")
    m = s.msg()
    h = s.digest(m)
    em = ref.encode(k, hash, h)
    sig = K.sign(k, hash, h, E)
    s.add("encoding_good", h, sig, K.n, E, m)
    hl = len(h)
    for i in range(hl):
        d = bytearray(h)
        d[i] ^= 1 << (i % 8)
        s.add(f"encoding_digest{i}", d, sig, K.n, E)
    tl = hl + len(ref.DIGEST_INFO[hash])

    def changed(cls, r):  # the EM with its byte r (counted from the end) changed, signed with d
        b = bytearray(em)
        b[k - 1 - r] ^= 1  # bit 0: byte 0 changed still leaves EM < N
        s.add(cls, h, K.sign_em(bytes(b), E, k), K.n, E)

    for r in range(hl, tl):
        changed(f"encoding_digest_info{tl - 1 - r}", r)
    changed("encoding_separator", tl)
    changed("encoding_byte1", k - 2)
    changed("encoding_byte0", k - 1)
    if limbs is None:
        limbs = range(k // 4) if hash == ref.SHA256 else ()
    for L in limbs:
        changed(f"encoding_limb{L}", 4 * L + L % 4)
    out = s.done()
    assert out["want"][0] == 1 and not out["want"][1:].any()
    return out


SETS = {"bitlen": bitlen, "oddexp": oddexp, "evenexp": evenexp, "encoding": encoding}


def shifted(c):
    """The set c with one item in front (a copy of its last item), so that every item lands in the other half of its
    warp and, past the first block, in the neighbouring block position."""
    idx = np.concatenate([[c["n"] - 1], np.arange(c["n"])])
    parts = [c["msgs"][int(c["off"][i]):int(c["off"][i + 1])] for i in idx]
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)
    return dict(k=c["k"], hash=c["hash"], n=c["n"] + 1, msgs=np.concatenate(parts), off=off, digest=c["digest"][idx].copy(), sig=c["sig"][idx].copy(),
                mod=c["mod"][idx].copy(), exp=c["exp"][idx].copy(), want=c["want"][idx].copy(), cls=[c["cls"][i] for i in idx])
