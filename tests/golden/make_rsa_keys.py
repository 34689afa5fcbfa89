#!/usr/bin/env python3
"""Generates tests/golden/rsa_keys.npz, the RSA keys of the edge sets in tests/rsa_edges.py, so that no test session
spends a minute of CPU on key generation.  Run from the repo root:  python tests/golden/make_rsa_keys.py

  std_<b>   oracle_rsa.ref.Key(b, seed=1) for b = 8k, 8k - 1, 8k - 4, 8k - 7 and k = 256, 384, 512 bytes: every leading byte
            shape from 0xff down to 0x01 over the three sizes
  blum_<b>  a Blum key of b = 8k bits: p = q = 3 (mod 4), (p - 1) / 2 and (q - 1) / 2 prime to 65537 and 2^30 - 1, so that
            every even exponent e = 2^t * m with m in {1, 65537, 2^30 - 1} has an inverse mod (p - 1) / 2 and (q - 1) / 2
Each key is stored as its primes p and q, big-endian bytes."""
import math
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle_rsa import ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = (256, 384, 512)
STD_BITS = [8 * k - j for k in SIZES for j in (0, 1, 4, 7)]
BLUM_ODD = 65537 * (2**30 - 1)  # the odd parts of the even exponents the tests sign with


def blum_prime(bits: int, rng: random.Random) -> int:
    """A prime of `bits` bits with its top two bits set, = 3 mod 4, and (p - 1) / 2 prime to BLUM_ODD."""
    while True:
        x = rng.getrandbits(bits) | (3 << (bits - 2)) | 3
        for _ in range(4000):
            if x.bit_length() != bits:
                break
            if math.gcd(x, ref._SMALL) == 1 and math.gcd((x - 1) // 2, BLUM_ODD) == 1 and ref._probable_prime(x, rng):
                return x
            x += 4


def blum_key(bits: int) -> ref.Key:
    rng = random.Random(f"blum-{bits}")
    while True:
        p, q = blum_prime(bits // 2, rng), blum_prime(bits // 2, rng)
        if p != q and (p * q).bit_length() == bits:
            return ref.Key.from_primes(p, q)


def main():
    out = {}
    for name, key in [(f"std_{b}", ref.Key(b, 1)) for b in STD_BITS] + [(f"blum_{8 * k}", blum_key(8 * k)) for k in SIZES]:
        plen = (key.p.bit_length() + 7) // 8
        out[name + "_p"] = np.frombuffer(key.p.to_bytes(plen, "big"), np.uint8)
        out[name + "_q"] = np.frombuffer(key.q.to_bytes((key.q.bit_length() + 7) // 8, "big"), np.uint8)
        print(name, key.bits, "bits", flush=True)
    np.savez_compressed(os.path.join(HERE, "rsa_keys.npz"), **out)


if __name__ == "__main__":
    main()
