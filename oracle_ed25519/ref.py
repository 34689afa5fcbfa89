"""Independent pure-Python restatement of Ed25519 verification with the accept set of Go's crypto/ed25519.Verify
(pure Ed25519, no context).  TEST INFRASTRUCTURE ONLY; slow (big integers), for corpora of a few hundred items.

1. reject if S >= L (S little-endian; covers sig[63] & 0xE0 != 0);
2. A decodes as edwards25519 Point.SetBytes: y = low 255 bits, values in [p, 2^255) accepted and reduced;
   x = sqrt((y^2-1)/(d y^2+1)), reject if none; negative root when bit 255 is set (x = 0 with the bit set accepted);
   no subgroup check;
3. k = SHA-512(R || A || M) mod L over the caller's bytes;
4. accept iff the canonical encoding of [S]B - [k]A equals R byte for byte (cofactorless).
"""
from __future__ import annotations

import hashlib

p = 2**255 - 19
L = 2**252 + 27742317777372353535851937790883648493
d = (-121665 * pow(121666, -1, p)) % p
SQRT_M1 = pow(2, (p - 1) // 4, p)
IDENTITY = (0, 1, 1, 0)


def _recover_x(y: int, sign: int):
    """x with x^2 = (y^2-1)/(d y^2+1) and parity `sign` (x = 0 keeps 0), or None."""
    u = (y * y - 1) % p
    v = (d * y * y + 1) % p
    x2 = u * pow(v, p - 2, p) % p
    x = pow(x2, (p + 3) // 8, p)
    if (x * x - x2) % p:
        x = x * SQRT_M1 % p
    if (x * x - x2) % p:
        return None
    if (x & 1) != sign:
        x = (-x) % p
    return x


def decode(enc: bytes):
    """Point.SetBytes: extended point or None."""
    v = int.from_bytes(enc, "little")
    y = (v & ((1 << 255) - 1)) % p
    x = _recover_x(y, v >> 255)
    if x is None:
        return None
    return (x, y, 1, x * y % p)


def add(P, Q):
    X1, Y1, Z1, T1 = P
    X2, Y2, Z2, T2 = Q
    A = (Y1 - X1) * (Y2 - X2) % p
    B = (Y1 + X1) * (Y2 + X2) % p
    C = T1 * 2 * d * T2 % p
    D = Z1 * 2 * Z2 % p
    E, F, G, H = B - A, D - C, D + C, B + A
    return (E * F % p, G * H % p, F * G % p, E * H % p)


def neg(P):
    X, Y, Z, T = P
    return ((-X) % p, Y, Z, (-T) % p)


def mul(k: int, P):
    Q = IDENTITY
    for bit in bin(k)[2:] if k else "":
        Q = add(Q, Q)
        if bit == "1":
            Q = add(Q, P)
    return Q


def encode(P) -> bytes:
    X, Y, Z, _ = P
    zi = pow(Z, p - 2, p)
    x, y = X * zi % p, Y * zi % p
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


def affine(P):
    X, Y, Z, _ = P
    zi = pow(Z, p - 2, p)
    return X * zi % p, Y * zi % p


_By = 4 * pow(5, -1, p) % p
B = (_recover_x(_By, 0), _By, 1, _recover_x(_By, 0) * _By % p)


def challenge(R: bytes, A: bytes, M: bytes) -> int:
    return int.from_bytes(hashlib.sha512(R + A + M).digest(), "little") % L


def verify(A: bytes, M: bytes, sig: bytes) -> bool:
    if len(sig) != 64 or len(A) != 32:
        return False
    R, S = sig[:32], int.from_bytes(sig[32:], "little")
    if S >= L:
        return False
    Ap = decode(A)
    if Ap is None:
        return False
    k = challenge(R, A, M)
    return encode(add(mul(S, B), neg(mul(k, Ap)))) == R


def sign_with_scalar(a: int, A: bytes, M: bytes, r: int) -> bytes:
    """R || S for secret scalar a, public encoding A (taken as given) and nonce r: S = r + k a mod L."""
    R = encode(mul(r, B))
    return R + ((r + challenge(R, A, M) * a) % L).to_bytes(32, "little")


def _sqrt(v):
    v %= p
    x = pow(v, (p + 3) // 8, p)
    if (x * x - v) % p:
        x = x * SQRT_M1 % p
    return x if (x * x - v) % p == 0 else None


def small_order_points():
    """The 8 points of order dividing 8 (affine): (0, 1), (0, -1), (+-sqrt(-1), 0), and the four of order 8, whose
    doubles are (+-sqrt(-1), 0): y^2 = -x^2 with x^2 = t a root of d t^2 - 2t - 1 = 0."""
    pts = {(0, 1), (0, p - 1), (SQRT_M1, 0), (p - SQRT_M1, 0)}
    s = _sqrt(1 + d)
    for root in (s, p - s):
        t = (1 + root) * pow(d, p - 2, p) % p
        x = _sqrt(t)
        if x is None:
            continue
        for xx in (x, p - x):
            for yy in (SQRT_M1 * xx % p, (p - SQRT_M1) * xx % p):
                if (-xx * xx + yy * yy - 1 - d * xx * xx * yy * yy) % p == 0:
                    pts.add((xx, yy))
    assert len(pts) == 8, len(pts)
    return sorted(pts)


def point_from_affine(x, y):
    return (x, y, 1, x * y % p)


def comb_table(A: bytes):
    """The comb table of a key grouped inside a launch, or None when A does not decode: entry b * 255 + m - 1 (b = 0, 1;
    m = 1..255) is the affine sum of 2^(16 (8b + t)) A over the set bits t of m."""
    P = decode(A)
    if P is None:
        return None
    bases = [P]
    for _ in range(15):
        Q = bases[-1]
        for _ in range(16):
            Q = add(Q, Q)
        bases.append(Q)
    out = []
    for b in range(2):
        for m in range(1, 256):
            S = IDENTITY
            for t in range(8):
                if (m >> t) & 1:
                    S = add(S, bases[8 * b + t])
            out.append(affine(S))
    return out
