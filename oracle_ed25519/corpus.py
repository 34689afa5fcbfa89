"""Seeded Ed25519 corpora with every corruption class (TEST INFRASTRUCTURE).

make_corpus(n, seed) -> dict(msgs, off, sig, pub, cls): messages in one blob from a random off[0] > 0 on (so with
the odd lengths offsets are misaligned), the blob padded by 16 bytes; signatures by OpenSSL over n_keys seeded keys; then a
share of the items corrupted or replaced by crafted ones.  cls names the class of each item; the verdicts come from
the oracles, not from the class.
"""
from __future__ import annotations

import numpy as np

from . import ref, sign_batch, pubkey

VALID, MSG_FLIP, R_FLIP, S_FLIP, S_PLUS_L, S_TOP, A_OFF_CURVE, A_BIG_Y, SMALL_ORDER, MIXED_ORDER, R_NONCANON = range(11)
CLASS_NAMES = ["valid", "msg_flip", "r_flip", "s_flip", "s_plus_l", "s_top_bits", "a_off_curve", "a_y_ge_p", "small_order_a",
               "mixed_order_a", "r_noncanonical"]
# Message lengths at the edges of k_ed_sha512.  SHA-512 hashes 64 + len bytes plus at least 17 of padding in 128-byte
# blocks: 47 / 48, 175 / 176 and 303 / 304 are the one / two, two / three and three / four block boundaries.  The kernel
# loads the message in 64-byte halves of a block, taking a fast path for halves that lie wholly inside the message:
# 63 / 64 and 127 / 128 are where a half stops or starts being whole.  10 KiB = RequestMaxBytes.
EDGE_LENGTHS = [0, 1, 47, 48, 63, 64, 127, 128, 175, 176, 303, 304, 10240]


def _enc_y(y: int, sign: int = 0) -> bytes:
    return (y | (sign << 255)).to_bytes(32, "little")


def small_order_encodings():
    """Every encoding of a point of order dividing 8 that decodes: canonical ones, the sign-bit variants of the x = 0
    points ("-0"), and the non-canonical y + p of y = 0 and y = 1."""
    out = []
    for x, y in ref.small_order_points():
        out.append(_enc_y(y, x & 1))
        if x == 0:
            out.append(_enc_y(y, 1))
        if y + ref.p < 2**255:
            out.append(_enc_y(y + ref.p, x & 1))
    return out


def off_curve_encodings(rng, k=8):
    out = []
    while len(out) < k:
        enc = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
        if ref.decode(enc) is None:
            out.append(enc)
    return out


def big_y_encodings():
    """y in [p, 2^255) with both sign bits; some decode (y - p = 1: the identity), some do not."""
    return [_enc_y(ref.p + t, s) for t in range(19) for s in (0, 1)]


def _crafted(kind, M: bytes, rng):
    """(pub, sig) of a crafted item over message M."""
    if kind == SMALL_ORDER:
        encs = small_order_encodings()
        A = encs[int(rng.integers(len(encs)))]
        s = int(rng.integers(1, 2**62)) * int(rng.integers(1, 2**62)) % ref.L
        return A, ref.encode(ref.mul(s, ref.B)) + s.to_bytes(32, "little")  # accepts iff [k]A = O
    if kind == MIXED_ORDER:
        pts = ref.small_order_points()
        T = ref.point_from_affine(*pts[int(rng.integers(len(pts)))])
        a = int(rng.integers(1, 2**62)) * int(rng.integers(1, 2**62)) % ref.L
        A = ref.encode(ref.add(ref.mul(a, ref.B), T))
        r = int(rng.integers(1, 2**62)) * int(rng.integers(1, 2**62)) % ref.L
        return A, ref.sign_with_scalar(a, A, M, r)  # accepts iff [k]T = O
    # R_NONCANON: A = identity and S = 0, so R' = O for every k: the canonical R accepts, the others must not
    A = _enc_y(1)
    R = [_enc_y(1), _enc_y(1 + ref.p), _enc_y(1, 1)][int(rng.integers(3))]
    return A, R + bytes(32)


def make_corpus(n: int, seed: int, n_keys: int = 64, fixed_len=None, lo: int = 0, hi: int = 300, corrupt: bool = True,
                crafted_max: int = 256):
    rng = np.random.default_rng(seed)
    if fixed_len is not None:
        lens = np.full(n, fixed_len, np.int64)
    else:
        lens = rng.integers(lo, hi + 1, n)
        edge = rng.random(n) < 0.15
        lens[edge] = rng.choice(EDGE_LENGTHS, int(edge.sum()))
        if n >= len(EDGE_LENGTHS):  # every edge length at least once
            lens[: len(EDGE_LENGTHS)] = EDGE_LENGTHS
    first = int(rng.integers(1, 8)) if fixed_len is None else 0  # off[0] > 0; odd lengths misalign the rest
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(first)
    msgs = rng.integers(0, 256, int(off[n]) + 16, dtype=np.uint8) if n else np.zeros(16, np.uint8)
    seeds = rng.integers(0, 256, (n_keys, 32), dtype=np.uint8)
    pubs = np.frombuffer(b"".join(pubkey(bytes(s)) for s in seeds), np.uint8).reshape(n_keys, 32)
    kidx = rng.integers(0, n_keys, n).astype(np.uint32)
    sig = sign_batch(seeds, kidx, msgs, off)
    pub = pubs[kidx].copy()
    cls = np.full(n, VALID, np.uint8)
    if corrupt and n:
        cls = rng.choice(np.arange(11, dtype=np.uint8), n, p=[0.5, 0.05, 0.05, 0.05, 0.05, 0.05, 0.05, 0.05, 0.05, 0.05, 0.05])
        crafted = np.flatnonzero(np.isin(cls, [SMALL_ORDER, MIXED_ORDER, R_NONCANON]))
        cls[crafted[crafted_max:]] = VALID  # the crafted classes cost big-integer arithmetic in Python: cap them
        off_curve, big_y = off_curve_encodings(rng), big_y_encodings()
        for i in np.flatnonzero(cls != VALID):
            c = int(cls[i])
            if c == MSG_FLIP:
                if lens[i] == 0:
                    cls[i] = VALID
                    continue
                msgs[int(off[i]) + int(rng.integers(lens[i]))] ^= np.uint8(1 << int(rng.integers(8)))
            elif c == R_FLIP:
                sig[i, int(rng.integers(32))] ^= np.uint8(1 << int(rng.integers(8)))
            elif c == S_FLIP:
                sig[i, 32 + int(rng.integers(32))] ^= np.uint8(1 << int(rng.integers(8)))
            elif c == S_PLUS_L:
                s = int.from_bytes(bytes(sig[i, 32:]), "little") + ref.L
                sig[i, 32:] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
            elif c == S_TOP:
                sig[i, 63] |= np.uint8(0x20 << int(rng.integers(3)))
            elif c == A_OFF_CURVE:
                pub[i] = np.frombuffer(off_curve[int(rng.integers(len(off_curve)))], np.uint8)
            elif c == A_BIG_Y:
                pub[i] = np.frombuffer(big_y[int(rng.integers(len(big_y)))], np.uint8)
            else:
                M = bytes(msgs[int(off[i]): int(off[i]) + int(lens[i])])
                A, sg = _crafted(c, M, rng)
                pub[i] = np.frombuffer(A, np.uint8)
                sig[i] = np.frombuffer(sg, np.uint8)
    return {"msgs": msgs, "off": off, "sig": sig, "pub": pub, "cls": cls}


def item(c, i):
    """(A, M, sig) bytes of item i of corpus c."""
    o0, o1 = int(c["off"][i]), int(c["off"][i + 1])
    return bytes(c["pub"][i]), bytes(c["msgs"][o0:o1]), bytes(c["sig"][i])


def ref_verdicts(c) -> np.ndarray:
    n = c["off"].size - 1
    return np.array([ref.verify(*item(c, i)) for i in range(n)], np.uint8)
