"""Seeded mixed corpora whose ECDSA items are signed over SHA-256 or SHA-384, for the sbv_mixed384_* calls (TEST / BENCH
INFRASTRUCTURE).

Scheme tags 0 to 4: P-256 and P-384 over SHA-256, Ed25519, P-256 and P-384 over SHA-384.  Keys come from a registry pair
of mixed_cases.registries; an item carries a slot of its curve's registry, and key96 holds the same key as a 96-byte row,
so one corpus serves the registered, keys-per-item and quorum calls.  Expected verdicts always come from the oracles
(OpenSSL over the item's own digest, through oracle/ and oracle_ed25519/), never from the corruption labels.
"""
from __future__ import annotations

import hashlib

import numpy as np

import oracle
import oracle_ed25519 as oe
from mixed_cases import gather, registries  # noqa: F401  (registries: re-exported for the tests)

P256, P384, ED, P256_SHA384, P384_SHA384 = 0, 1, 2, 3, 4
CURVE = {P256: P256, P384: P384, P256_SHA384: P256, P384_SHA384: P384}
L = {P256: 32, P384: 48}
SWAP = np.array([3, 4, 2, 0, 1], np.uint8)  # the same curve under the other hash (Ed25519 stays)


def digests(tag, msgs, off, idx):
    """The digest each ECDSA item is signed over: SHA-256 (tags 0, 1) or the whole SHA-384 (tags 3, 4; OpenSSL truncates
    it to the field for P-256)."""
    h = hashlib.sha384 if tag >= P256_SHA384 else hashlib.sha256
    return np.array([np.frombuffer(h(memoryview(msgs[int(off[i]):int(off[i + 1])])).digest(), np.uint8) for i in idx], np.uint8).reshape(
        len(idx), h().digest_size)


def key_rows(reg, scheme, key_slot):
    """key96 as sbv_mixed_verify_batch takes it: X || Y of the item's slot (P-256 in bytes [0, 64)), the Ed25519 encoding in
    [0, 32)."""
    n = scheme.size
    rows = np.zeros((n, 96), np.uint8)
    for t, c in CURVE.items():
        idx = np.flatnonzero(scheme == t)
        xy = reg["ecdsa_xy"][key_slot[idx]]
        rows[idx, :L[c]] = xy[:, 48 - L[c]:48]
        rows[idx, L[c]:2 * L[c]] = xy[:, 96 - L[c]:]
    idx = np.flatnonzero(scheme == ED)
    rows[idx, :32] = reg["ed_pub"][key_slot[idx]]
    return rows


def sign(scheme, msgs, off, key_slot, reg, rng):
    rows = np.zeros((scheme.size, 96), np.uint8)
    for t, c in CURVE.items():
        idx = np.flatnonzero(scheme == t)
        if idx.size == 0:
            continue
        slots_c = np.flatnonzero(reg["ecdsa_curve"] == c)
        local = np.searchsorted(slots_c, key_slot[idx].astype(np.int64))
        d = np.ascontiguousarray(reg["ecdsa_priv"][slots_c][:, 48 - L[c]:])
        nonces = rng.integers(0, 256, (idx.size, L[c]), dtype=np.uint8)
        nonces[:, 0] &= 0x7F
        nonces[:, -1] |= 1
        r, s = oracle.sign_batch(c, d, local.astype(np.uint32), digests(t, msgs, off, idx), nonces)
        rows[idx, :L[c]] = r
        rows[idx, L[c]:2 * L[c]] = s
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        m, o = gather(msgs, off, idx)
        rows[idx, :64] = oe.sign_batch(reg["ed_seeds"], key_slot[idx].astype(np.uint32), m, o)
    return rows


def make_corpus(scheme, reg, seed=0, lo=0, hi=300, lens=None, corrupt=0.2, key_choice=None, key_slot=None):
    """Items of the given tags: random messages (off[0] > 0), a slot of the item's own curve (or Ed25519) registry each
    (key_choice: how many of each registry's keys to draw from, to make keys repeat; key_slot: the caller's slots), signed;
    with corrupt, that share of the items gets one flipped signature or message bit."""
    rng = np.random.default_rng(seed)
    scheme = np.asarray(scheme, np.uint8)
    n = scheme.size
    if lens is None:
        lens = rng.integers(lo, hi + 1, n)
    first = int(rng.integers(1, 8))
    off = (np.concatenate([[0], np.cumsum(lens)]) + first).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    given = key_slot is not None
    key_slot = np.zeros(n, np.uint32) if not given else np.asarray(key_slot, np.uint32)
    for c in (P256, P384) if not given else ():
        own = np.flatnonzero(reg["ecdsa_curve"] == c)[:key_choice]
        idx = np.flatnonzero(np.isin(scheme, [c, c + P256_SHA384]))
        key_slot[idx] = own[rng.integers(0, own.size, idx.size)]
    idx = np.flatnonzero(scheme == ED)
    if not given:
        key_slot[idx] = rng.integers(0, reg["ed_pub"].shape[0] if key_choice is None else key_choice, idx.size)
    sig96 = sign(scheme, msgs, off, key_slot, reg, rng)
    for i in np.flatnonzero(rng.random(n) < corrupt):
        ln = int(off[i + 1] - off[i])
        if ln and rng.random() < 0.5:
            msgs[int(off[i]) + int(rng.integers(0, ln))] ^= 1 << int(rng.integers(0, 8))
        else:
            w = 64 if scheme[i] == ED else 2 * L[CURVE[int(scheme[i])]]
            b = int(rng.integers(0, 8 * w))
            sig96[i, b >> 3] ^= 1 << (b & 7)
    return {"scheme": scheme, "msgs": msgs, "off": off, "key_slot": key_slot, "sig96": sig96, "key96": key_rows(reg, scheme, key_slot)}


def with_scheme(cp, scheme):
    """The corpus with other tags (keys, messages and signatures as they are)."""
    out = dict(cp)
    out["scheme"] = np.asarray(scheme, np.uint8)
    return out


def concat(a, b):
    """Corpus a followed by corpus b, as one call's items."""
    ma = a["msgs"][:int(a["off"][-1])]
    mb = b["msgs"][int(b["off"][0]):int(b["off"][-1])]
    off = np.concatenate([a["off"], (b["off"][1:] - b["off"][0] + a["off"][-1])]).astype(np.uint64)
    out = {"msgs": np.concatenate([ma, mb, np.zeros(16, np.uint8)]), "off": off}
    for k in ("scheme", "key_slot", "sig96", "key96"):
        out[k] = np.concatenate([a[k], b[k]])
    return out


def expected_ok(cp, reg):
    """OpenSSL's verdict for every item over its own digest and key."""
    scheme, msgs, off, slot, sig96 = cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"]
    ok = np.zeros(scheme.size, np.uint8)
    for t, c in CURVE.items():
        idx = np.flatnonzero(scheme == t)
        if idx.size == 0:
            continue
        xy = reg["ecdsa_xy"][slot[idx]]
        ok[idx] = oracle.verify_batch(c, np.ascontiguousarray(sig96[idx, :L[c]]), np.ascontiguousarray(sig96[idx, L[c]:2 * L[c]]),
                                      np.ascontiguousarray(xy[:, 48 - L[c]:48]), np.ascontiguousarray(xy[:, 96 - L[c]:]),
                                      digests(t, msgs, off, idx))
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        m, o = gather(msgs, off, idx)
        ok[idx] = oe.verify_batch(m, o, np.ascontiguousarray(sig96[idx, :64]), np.ascontiguousarray(reg["ed_pub"][slot[idx]]))
    return ok


def set_keys(eng, reg):
    eng.set_keys(reg["ecdsa_curve"], reg["ecdsa_xy"])
    eng.ed25519_set_keys(reg["ed_pub"])


def vote_stream(tags, n_inst, seed):
    """A commit-vote stream of a consenter set whose consenter k signs with scheme tags[k] (C4's shape: every consenter
    votes once per instance, in a shuffled order, plus a few repeated votes and votes whose signer is not their sender).
    Returns (scheme per vote, consenter per vote, instance, sender, signer, digest_match)."""
    rng = np.random.default_rng(seed)
    K = len(tags)
    inst, who, sender, signer = [], [], [], []
    for i in range(n_inst):
        order = list(rng.permutation(K)) + list(rng.integers(0, K, 2))
        for k in order:
            inst.append(i)
            who.append(int(k))
            sender.append(int(k) + 1)
            signer.append(int(k) + 1 if rng.random() < 0.95 else int(rng.integers(1, K + 1)))
    who = np.array(who)
    n = who.size
    dm = (rng.random(n) < 0.9).astype(np.uint8)
    return (np.asarray(tags, np.uint8)[who], who, np.array(inst, np.uint32), np.array(sender, np.uint16), np.array(signer, np.uint16), dm)
