"""Seeded mixed ECDSA / Ed25519 corpora with the key of each item carried in the call, for sbv_mixed_verify_batch (TEST /
BENCH INFRASTRUCTURE).

A corpus item carries a scheme tag, a message, a 96-byte signature row and a 96-byte key row (P-256 X || Y in [0, 64),
P-384 X || Y, Ed25519 encoding in [0, 32)), drawn from a pool of keys per scheme so that keys repeat.  Expected verdicts
always come from the oracles (OpenSSL through oracle/ and oracle_ed25519/), never from the corruption labels.  Tag
patterns, the signature corruptions and message gathering come from tests/mixed_cases.py.
"""
from __future__ import annotations

import numpy as np

import oracle
import oracle_ed25519 as oe
from oracle import corpus as ecorpus
from oracle.ecdsa_ref import CURVES
from oracle_ed25519 import corpus as edcorpus
from oracle_ed25519 import ref, votes

from mixed_cases import ED, L, P256, P384, gather, tag_pattern  # noqa: F401  (re-exported for the tests)

# corruption classes: the signature and message classes of mixed_cases, then the bad keys
FLIP_SIG, FLIP_MSG, WRONG_KEY, R_ZERO, S_ZERO, R_EQ_N, HIGH_S, S_PLUS_L, NONCANON_R = range(9)
EC_OFF_CURVE, EC_X_GE_P, EC_Y_GE_P, EC_ZERO = range(9, 13)
ED_NO_DECODE, ED_SMALL_ORDER, ED_Y_GE_P, ED_NEG_ZERO = range(13, 17)
EC_CLASSES = [FLIP_SIG, FLIP_MSG, WRONG_KEY, R_ZERO, S_ZERO, R_EQ_N, HIGH_S, EC_OFF_CURVE, EC_X_GE_P, EC_Y_GE_P, EC_ZERO]
ED_CLASSES = [FLIP_SIG, FLIP_MSG, WRONG_KEY, S_PLUS_L, NONCANON_R, ED_NO_DECODE, ED_SMALL_ORDER, ED_Y_GE_P, ED_NEG_ZERO]
BAD_KEY_CLASSES = list(range(EC_OFF_CURVE, ED_NEG_ZERO + 1))


def key_pools(k256=8, k384=8, k_ed=8, seed=1):
    """Private and public keys per scheme: {P256: (d (k, 32), xy (k, 64)), P384: (d, xy (k, 96)), ED: (seeds, pub (k, 32))}."""
    return {P256: ecorpus.make_keys(P256, k256, seed) if k256 else None, P384: ecorpus.make_keys(P384, k384, seed + 1) if k384 else None,
            ED: votes.consenter_keys(k_ed, seed + 2) if k_ed else None}


def sign(scheme, msgs, off, key_idx, pools, rng, junk=False):
    """(sig96, key96): every item signed under key key_idx[i] of its scheme's pool; junk: random bytes past the signature
    and past the key instead of zeros."""
    n = scheme.size
    mk = (lambda: rng.integers(0, 256, (n, 96), dtype=np.uint8)) if junk else (lambda: np.zeros((n, 96), np.uint8))
    sig96, key96 = mk(), mk()
    dig = oracle.sha256_batch(msgs, off) if n else np.zeros((0, 32), np.uint8)
    for c in (P256, P384):
        idx = np.flatnonzero(scheme == c)
        if idx.size == 0:
            continue
        d, xy = pools[c]
        nonces = rng.integers(0, 256, (idx.size, L[c]), dtype=np.uint8)
        nonces[:, 0] &= 0x7F
        nonces[:, -1] |= 1
        r, s = oracle.sign_batch(c, d, key_idx[idx].astype(np.uint32), dig[idx], nonces)
        sig96[idx, :L[c]] = r
        sig96[idx, L[c]:2 * L[c]] = s
        key96[idx, :2 * L[c]] = xy[key_idx[idx]]
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        seeds, pub = pools[ED]
        m, o = gather(msgs, off, idx)
        sig96[idx, :64] = oe.sign_batch(seeds, key_idx[idx].astype(np.uint32), m, o)
        key96[idx, :32] = pub[key_idx[idx]]
    return sig96, key96


def make_corpus(scheme, pools, seed=0, lo=0, hi=200, lens=None, corrupt=0.25, junk=False, key_idx=None, classes=None):
    """Items of the given scheme tags: random messages (off[0] > 0), a random key of the item's pool each (or key_idx),
    signed; a `corrupt` share of them fall in one corruption class each (cls: -1 = untouched; classes: the classes to
    draw from, per scheme those that apply)."""
    rng = np.random.default_rng(seed)
    scheme = np.asarray(scheme, np.uint8)
    n = scheme.size
    if lens is None:
        lens = rng.integers(lo, hi + 1, n)
    first = int(rng.integers(1, 8))
    off = (np.concatenate([[0], np.cumsum(lens)]) + first).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    if key_idx is None:
        key_idx = np.zeros(n, np.int64)
        for c in (P256, P384, ED):
            idx = np.flatnonzero(scheme == c)
            if idx.size:
                key_idx[idx] = rng.integers(0, pools[c][1].shape[0], idx.size)
    key_idx = np.asarray(key_idx, np.int64)
    sig96, key96 = sign(scheme, msgs, off, key_idx, pools, rng, junk)
    cls = np.full(n, -1, np.int16)
    cp = {"scheme": scheme, "msgs": msgs, "off": off, "sig96": sig96, "key96": key96, "key_idx": key_idx, "cls": cls}
    if corrupt:
        for i in np.flatnonzero(rng.random(n) < corrupt):
            own = EC_CLASSES if scheme[i] != ED else ED_CLASSES
            pick = [c for c in own if classes is None or c in classes]
            if pick:
                corrupt_item(cp, i, int(rng.choice(pick)), pools, rng)
    return cp


def tile(cp, k, seed=0):
    """k copies of every item of cp, shuffled: a large corpus for the price of signing a small one."""
    n = cp["scheme"].size
    order = np.random.default_rng(seed).permutation(np.tile(np.arange(n), k))
    msgs, off = gather(cp["msgs"], cp["off"], order)
    return dict({key: cp[key][order] for key in ("scheme", "sig96", "key96", "key_idx", "cls")}, msgs=msgs, off=off)


def _be(v, n):
    return np.frombuffer(int(v).to_bytes(n, "big"), np.uint8)


def corrupt_item(cp, i, c, pools, rng):
    """Puts item i in class c (a FLIP_MSG of an empty message becomes a FLIP_SIG)."""
    t = int(cp["scheme"][i])
    sig, key, msgs, off = cp["sig96"], cp["key96"], cp["msgs"], cp["off"]
    ln = int(off[i + 1] - off[i])
    if c == FLIP_MSG and ln == 0:
        c = FLIP_SIG
    cp["cls"][i] = c
    Lt = 32 if t == ED else L[t]
    w = 64 if t == ED else 2 * Lt
    if c == FLIP_SIG:
        b = int(rng.integers(0, 8 * w))
        sig[i, b >> 3] ^= 1 << (b & 7)
    elif c == FLIP_MSG:
        msgs[int(off[i]) + int(rng.integers(0, ln))] ^= 1 << int(rng.integers(0, 8))
    elif c == WRONG_KEY:
        pool = pools[t][1]
        other = (int(cp["key_idx"][i]) + 1 + int(rng.integers(0, max(pool.shape[0] - 1, 1)))) % pool.shape[0]
        key[i, :pool.shape[1]] = pool[other]
    elif c == R_ZERO:
        sig[i, :Lt] = 0
    elif c == S_ZERO:
        sig[i, Lt:2 * Lt] = 0
    elif c == R_EQ_N:
        sig[i, :Lt] = _be(CURVES[t].n, Lt)
    elif c == HIGH_S:  # still valid: Go has no low-S rule
        sig[i, Lt:2 * Lt] = _be(CURVES[t].n - int.from_bytes(bytes(sig[i, Lt:2 * Lt]), "big"), Lt)
    elif c == S_PLUS_L:
        s = int.from_bytes(bytes(sig[i, 32:64]), "little") + ref.L
        if s < 2**256:
            sig[i, 32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
    elif c == NONCANON_R:
        sig[i, :32] = np.frombuffer((1 + ref.p).to_bytes(32, "little"), np.uint8)
    elif c == EC_OFF_CURVE:
        b = int(rng.integers(0, 8 * Lt))
        key[i, Lt + (b >> 3)] ^= 1 << (b & 7)
    elif c in (EC_X_GE_P, EC_Y_GE_P):  # v + p where it fits (the same point mod p), else p + a small value
        at = 0 if c == EC_X_GE_P else Lt
        v = int.from_bytes(bytes(key[i, at:at + Lt]), "big")
        p = CURVES[t].p
        key[i, at:at + Lt] = _be(v + p if v + p < 2**(8 * Lt) else p + int(rng.integers(0, 3)), Lt)
    elif c == EC_ZERO:
        key[i, :2 * Lt] = 0
    elif c == ED_NO_DECODE:
        key[i, :32] = np.frombuffer(edcorpus.off_curve_encodings(rng, 1)[0], np.uint8)
    elif c == ED_SMALL_ORDER:
        encs = edcorpus.small_order_encodings()
        key[i, :32] = np.frombuffer(encs[int(rng.integers(0, len(encs)))], np.uint8)
    elif c == ED_Y_GE_P:
        encs = edcorpus.big_y_encodings()
        key[i, :32] = np.frombuffer(encs[int(rng.integers(0, len(encs)))], np.uint8)
    elif c == ED_NEG_ZERO:  # x = 0 with the sign bit set: y = 1 or y = p - 1
        y = 1 if rng.random() < 0.5 else ref.p - 1
        key[i, :32] = np.frombuffer((y | (1 << 255)).to_bytes(32, "little"), np.uint8)
    else:
        raise ValueError(c)


def expected_ok(cp) -> np.ndarray:
    """OpenSSL's verdict of every item under the key its row carries."""
    scheme, msgs, off, sig96, key96 = cp["scheme"], cp["msgs"], cp["off"], cp["sig96"], cp["key96"]
    n = scheme.size
    ok = np.zeros(n, np.uint8)
    dig = oracle.sha256_batch(msgs, off) if n else None
    for c in (P256, P384):
        idx = np.flatnonzero(scheme == c)
        if idx.size:
            Lc = L[c]
            ok[idx] = oracle.verify_batch(c, sig96[idx, :Lc], sig96[idx, Lc:2 * Lc], key96[idx, :Lc], key96[idx, Lc:2 * Lc], dig[idx])
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        m, o = gather(msgs, off, idx)
        ok[idx] = oe.verify_batch(m, o, sig96[idx, :64], key96[idx, :32])
    return ok


def family_arrays(cp, c):
    """The items of scheme c as the single-scheme keys-per-item calls take them: (idx, msgs, off, sig fields, key fields);
    ECDSA: (r, s) and (qx, qy), Ed25519: (sig,) and (pub,)."""
    idx = np.flatnonzero(cp["scheme"] == c)
    m, o = gather(cp["msgs"], cp["off"], idx)
    if c == ED:
        return idx, m, o, (np.ascontiguousarray(cp["sig96"][idx, :64]),), (np.ascontiguousarray(cp["key96"][idx, :32]),)
    Lc = L[c]
    s, k = cp["sig96"][idx], cp["key96"][idx]
    return (idx, m, o, (np.ascontiguousarray(s[:, :Lc]), np.ascontiguousarray(s[:, Lc:2 * Lc])),
            (np.ascontiguousarray(k[:, :Lc]), np.ascontiguousarray(k[:, Lc:2 * Lc])))
