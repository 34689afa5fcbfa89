"""Go's crypto/rsa.VerifyPKCS1v15 and crypto/rsa.VerifyPSS restated in Python integers (the accept sets of include/sbv.h),
a seeded RSA key generator and a CRT signer.  TEST INFRASTRUCTURE ONLY.

verify(k, hash, H, S, N, e):
  1. key: N odd, N's leading byte (of k) nonzero, 2 <= e <= 2^31 - 1;
  2. range: S < N;
  3. EM = S^e mod N as k bytes, big-endian;
  4. accept iff EM == 00 || 01 || FF * (k - tLen - 3) || 00 || DigestInfo(hash) || H.

pss_verify(k, hash, H, S, N, e, salt_len): steps 1-3 as above, then the EMSA-PSS decoding of RFC 8017 §9.1.2 as Go's
emsaPSSVerify writes it, MGF1 over the message hash; salt_len as Go's PSSOptions.SaltLength (-1: hLen, 0: auto).
"""
from __future__ import annotations

import hashlib
import math
import random

import numpy as np

SHA256, SHA384, SHA512 = 0, 1, 2
HLEN = {SHA256: 32, SHA384: 48, SHA512: 64}
HASHLIB = {SHA256: hashlib.sha256, SHA384: hashlib.sha384, SHA512: hashlib.sha512}
# RFC 8017 §9.2 note 1, with the NULL parameters
DIGEST_INFO = {
    SHA256: bytes.fromhex("3031300d060960864801650304020105000420"),
    SHA384: bytes.fromhex("3041300d060960864801650304020205000430"),
    SHA512: bytes.fromhex("3051300d060960864801650304020305000440"),
}
E_MAX = 2**31 - 1


def encode(k: int, hash: int, digest: bytes) -> bytes:
    """EMSA-PKCS1-v1_5 encoding of a digest into k bytes."""
    t = DIGEST_INFO[hash] + bytes(digest)
    return b"\x00\x01" + b"\xff" * (k - len(t) - 3) + b"\x00" + t


def verify(k: int, hash: int, digest: bytes, sig: bytes, mod: bytes, e: int) -> bool:
    mod, sig = bytes(mod), bytes(sig)
    assert len(mod) == k and len(sig) == k and len(digest) == HLEN[hash]
    n = int.from_bytes(mod, "big")
    if n % 2 == 0 or mod[0] == 0 or not 2 <= e <= E_MAX:
        return False
    s = int.from_bytes(sig, "big")
    if s >= n:
        return False
    return pow(s, e, n).to_bytes(k, "big") == encode(k, hash, digest)


def verify_batch(k, hash, digest, sig, mod, exp) -> np.ndarray:
    n = len(exp)
    digest = np.asarray(digest, np.uint8).reshape(n, HLEN[hash])
    sig, mod = np.asarray(sig, np.uint8).reshape(n, k), np.asarray(mod, np.uint8).reshape(n, k)
    return np.array([verify(k, hash, digest[i].tobytes(), sig[i].tobytes(), mod[i].tobytes(), int(exp[i])) for i in range(n)], np.uint8)


# ---- RSA-PSS ----------------------------------------------------------------------------------------------------------
SALT_EQUALS_HASH, SALT_AUTO = -1, 0


def mgf1(seed: bytes, length: int, hash: int) -> bytes:
    """MGF1 (RFC 8017 §B.2.1): Hash(seed || BE32(c)) for c = 0, 1, ... cut to length bytes."""
    out = b"".join(HASHLIB[hash](seed + c.to_bytes(4, "big")).digest() for c in range(-(-length // HLEN[hash])))
    return out[:length]


def pss_encode(em_bits: int, hash: int, digest: bytes, salt: bytes) -> bytes:
    """EMSA-PSS-ENCODE (RFC 8017 §9.1.1) of a digest with the given salt: emLen = ceil(emBits / 8) bytes."""
    hl, em_len = HLEN[hash], (em_bits + 7) // 8
    assert em_len >= hl + len(salt) + 2
    h = HASHLIB[hash](bytes(8) + bytes(digest) + bytes(salt)).digest()
    db = bytes(em_len - len(salt) - hl - 2) + b"\x01" + bytes(salt)
    masked = bytearray(x ^ y for x, y in zip(db, mgf1(h, len(db), hash)))
    masked[0] &= 0xFF >> (8 * em_len - em_bits)
    return bytes(masked) + h + b"\xbc"


def pss_verify(k: int, hash: int, digest: bytes, sig: bytes, mod: bytes, e: int, salt_len: int) -> bool:
    assert salt_len >= SALT_EQUALS_HASH, "salt_len < -1 is an argument error, not a verdict"
    mod, sig = bytes(mod), bytes(sig)
    assert len(mod) == k and len(sig) == k and len(digest) == HLEN[hash]
    n = int.from_bytes(mod, "big")
    if n % 2 == 0 or mod[0] == 0 or not 2 <= e <= E_MAX:
        return False
    s = int.from_bytes(sig, "big")
    if s >= n:
        return False
    em = pow(s, e, n).to_bytes(k, "big")
    em_bits = n.bit_length() - 1
    em_len = (em_bits + 7) // 8
    while len(em) > em_len:  # Go's "strip leading zeroes"
        if em[0] != 0:
            return False
        em = em[1:]
    hl = HLEN[hash]
    s_len = hl if salt_len == SALT_EQUALS_HASH else salt_len
    if em_len < hl + s_len + 2:
        return False
    if em[-1] != 0xBC:
        return False
    db_len = em_len - hl - 1
    masked, h = em[:db_len], em[db_len:db_len + hl]
    keep = 0xFF >> (8 * em_len - em_bits)
    if masked[0] & ~keep & 0xFF:
        return False
    db = bytearray(x ^ y for x, y in zip(masked, mgf1(h, db_len, hash)))
    db[0] &= keep
    if salt_len == SALT_AUTO:  # Go: the first 01 byte is the separator
        ps_len = db.find(b"\x01")
        if ps_len < 0:
            return False
        s_len = db_len - ps_len - 1
    ps_len = em_len - hl - s_len - 2
    if any(db[:ps_len]) or db[ps_len] != 0x01:
        return False
    salt = bytes(db[db_len - s_len:])
    return HASHLIB[hash](bytes(8) + bytes(digest) + salt).digest() == h


def pss_verify_batch(k, hash, digest, sig, mod, exp, salt_len) -> np.ndarray:
    n = len(exp)
    digest = np.asarray(digest, np.uint8).reshape(n, HLEN[hash])
    sig, mod = np.asarray(sig, np.uint8).reshape(n, k), np.asarray(mod, np.uint8).reshape(n, k)
    return np.array([pss_verify(k, hash, digest[i].tobytes(), sig[i].tobytes(), mod[i].tobytes(), int(exp[i]), salt_len) for i in range(n)],
                    np.uint8)


# ---- keys and signatures ----------------------------------------------------------------------------------------------
_SMALL = math.prod(p for p in range(3, 5000, 2) if all(p % q for q in range(3, int(p**0.5) + 1, 2)))


def _probable_prime(x: int, rng: random.Random) -> bool:
    d, s = x - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for _ in range(8):
        y = pow(rng.randrange(2, x - 1), d, x)
        if y in (1, x - 1):
            continue
        for _ in range(s - 1):
            y = y * y % x
            if y == x - 1:
                break
        else:
            return False
    return True


def _prime(bits: int, rng: random.Random) -> int:
    """A prime of exactly `bits` bits with its top two bits set and p - 1 prime to 3, 65537, 2^31 - 1 and 2^32 - 1 (= 3 * 5 *
    17 * 257 * 65537): one prime pair serves every exponent the tests sign with, e = 2^32 - 1 included."""
    while True:
        x = rng.getrandbits(bits) | (3 << (bits - 2))
        x += (5 - x % 6) % 6  # = 5 mod 6: odd and 2 mod 3
        for _ in range(2000):
            if x.bit_length() != bits:
                break
            if math.gcd(x, _SMALL) == 1 and math.gcd(x - 1, (2**32 - 1) * E_MAX) == 1 and _probable_prime(x, rng):
                return x
            x += 6


class Key:
    """An RSA key of `bits` bits from a seed: n, the primes and the CRT exponents for any public exponent."""

    def __init__(self, bits: int, seed: int):
        rng = random.Random(f"rsa-{bits}-{seed}")
        while True:
            p, q = _prime((bits + 1) // 2, rng), _prime(bits // 2, rng)
            if p != q and (p * q).bit_length() == bits:
                break
        self._set(p, q)

    @classmethod
    def from_primes(cls, p: int, q: int) -> "Key":
        """The key of two given primes (a committed fixture, or primes of a special form)."""
        key = cls.__new__(cls)
        key._set(p, q)
        return key

    def _set(self, p: int, q: int) -> None:
        self.p, self.q, self.n, self.bits = p, q, p * q, (p * q).bit_length()
        self.lam = math.lcm(p - 1, q - 1)

    def mod_bytes(self, k: int) -> bytes:
        return self.n.to_bytes(k, "big")

    def sign_int(self, m: int, e: int) -> int:
        """m^d mod n, d = e^-1 mod lcm(p-1, q-1), by CRT."""
        d = pow(e, -1, self.lam)
        p, q = self.p, self.q
        mp, mq = pow(m % p, d % (p - 1), p), pow(m % q, d % (q - 1), q)
        h = (mq - mp) * pow(p, -1, q) % q
        return mp + p * h

    def sign_em(self, em: bytes, e: int, k: int) -> bytes:
        return self.sign_int(int.from_bytes(em, "big"), e).to_bytes(k, "big")

    def sign(self, k: int, hash: int, digest: bytes, e: int = 65537) -> bytes:
        return self.sign_em(encode(k, hash, digest), e, k)

    def sign_pss(self, k: int, hash: int, digest: bytes, salt: bytes, e: int = 65537) -> bytes:
        """An RSA-PSS signature (k bytes) of the digest with the given salt: emBits = bitlen(N) - 1."""
        return self.sign_em(pss_encode(self.bits - 1, hash, digest, salt).rjust(k, b"\0"), e, k)
