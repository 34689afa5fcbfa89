"""Seeded mixed ECDSA / Ed25519 corpora and commit-vote streams for sbv_mixed_verify_registered and
sbv_mixed_verify_quorum (TEST / BENCH INFRASTRUCTURE).

A registry pair: the ECDSA registry of sbv_set_keys (P-256 and P-384 keys in alternating slots) and the Ed25519 registry
of sbv_ed25519_set_keys.  A corpus item carries a scheme tag, a message, a slot of its scheme's registry and a 96-byte
signature row.  Expected verdicts always come from the oracles (OpenSSL through oracle/ and oracle_ed25519/), never from
the corruption labels.
"""
from __future__ import annotations

import numpy as np

import oracle
import oracle_ed25519 as oe
from oracle import corpus as ecorpus
from oracle.ecdsa_ref import CURVES
from oracle_ed25519 import corpus as edcorpus
from oracle_ed25519 import ref, votes

P256, P384, ED = 0, 1, 2
L = {P256: 32, P384: 48}
UNKNOWN = 2**32 - 1


def registries(n256=3, n384=2, n_ed=4, seed=1):
    """dict: ecdsa_curve (k,), ecdsa_xy (k, 96) as sbv_set_keys takes it, ecdsa_priv (k, 48) right-aligned, ed_seeds and
    ed_pub (n_ed, 32)."""
    d256, k256 = ecorpus.make_keys(P256, n256, seed)
    d384, k384 = ecorpus.make_keys(P384, n384, seed + 1)
    curves, xy, priv = [], [], []
    order = sorted([(2 * i, P256, i) for i in range(n256)] + [(2 * i + 1, P384, i) for i in range(n384)])
    for _, c, i in order:
        d, k = (d256, k256) if c == P256 else (d384, k384)
        row = np.zeros((2, 48), np.uint8)
        row[:, 48 - L[c]:] = k[i].reshape(2, L[c])
        p = np.zeros(48, np.uint8)
        p[48 - L[c]:] = d[i]
        curves.append(c)
        xy.append(row.reshape(96))
        priv.append(p)
    seeds, pubs = votes.consenter_keys(n_ed, seed + 2)
    return {"ecdsa_curve": np.array(curves, np.uint8), "ecdsa_xy": np.array(xy, np.uint8).reshape(-1, 96),
            "ecdsa_priv": np.array(priv, np.uint8).reshape(-1, 48), "ed_seeds": seeds, "ed_pub": pubs}


def tag_pattern(kind: str, n: int, rng) -> np.ndarray:
    if kind in ("p256", "p384", "ed"):
        return np.full(n, {"p256": P256, "p384": P384, "ed": ED}[kind], np.uint8)
    if kind == "alternating":
        return (np.arange(n) % 3).astype(np.uint8)
    if kind == "random":
        return rng.integers(0, 3, n).astype(np.uint8)
    if kind == "runs":  # runs of 1 to 300 items of one scheme
        out, t = [], 0
        while sum(len(r) for r in out) < n:
            t = (t + int(rng.integers(1, 3))) % 3
            out.append(np.full(int(rng.integers(1, 301)), t, np.uint8))
        return np.concatenate(out)[:n]
    raise ValueError(kind)


def gather(msgs, off, idx):
    """The messages idx of (msgs, off) as their own compact (msgs, off)."""
    idx = np.asarray(idx, np.int64)
    lens = (off[idx + 1] - off[idx]).astype(np.int64)
    o = np.zeros(idx.size + 1, np.uint64)
    o[1:] = np.cumsum(lens)
    if int(o[-1]) == 0:
        return np.zeros(16, np.uint8), o
    starts = off[idx].astype(np.int64)
    pos = np.repeat(starts - o[:-1].astype(np.int64), lens) + np.arange(int(o[-1]))
    return np.concatenate([msgs[pos], np.zeros(16, np.uint8)]), o


def sign_rows(scheme, msgs, off, key_slot, reg, rng, junk=False) -> np.ndarray:
    """96-byte rows: every item signed under the key of its slot (items whose slot is outside the registry get a signature
    under slot 0 of their scheme).  junk: random bytes past the signature instead of zeros."""
    n = scheme.size
    rows = rng.integers(0, 256, (n, 96), dtype=np.uint8) if junk else np.zeros((n, 96), np.uint8)
    dig = oracle.sha256_batch(msgs, off) if n else np.zeros((0, 32), np.uint8)
    for c in (P256, P384):
        idx = np.flatnonzero(scheme == c)
        if idx.size == 0:
            continue
        slots_c = np.flatnonzero(reg["ecdsa_curve"] == c)
        slot = key_slot[idx].astype(np.int64)
        own = np.isin(slot, slots_c)
        local = np.searchsorted(slots_c, np.where(own, slot, slots_c[0]))
        d = np.ascontiguousarray(reg["ecdsa_priv"][slots_c][:, 48 - L[c]:])
        nonces = rng.integers(0, 256, (idx.size, L[c]), dtype=np.uint8)
        nonces[:, 0] &= 0x7F
        nonces[:, -1] |= 1
        r, s = oracle.sign_batch(c, d, local.astype(np.uint32), dig[idx], nonces)
        rows[idx, :L[c]] = r
        rows[idx, L[c]:2 * L[c]] = s
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        slot = key_slot[idx].astype(np.int64)
        k = np.where(slot < reg["ed_seeds"].shape[0], slot, 0).astype(np.uint32)
        m, o = gather(msgs, off, idx)
        rows[idx, :64] = oe.sign_batch(reg["ed_seeds"], k, m, o)
    return rows


def make_corpus(scheme, reg, seed=0, lo=0, hi=200, lens=None, corrupt=True, junk=False):
    """Items of the given scheme tags: random messages (off[0] > 0, odd lengths), a random own-scheme slot each, signed;
    with corrupt, about a quarter of them fall in one corruption class each (cls: -1 = untouched)."""
    rng = np.random.default_rng(seed)
    scheme = np.asarray(scheme, np.uint8)
    n = scheme.size
    if lens is None:
        lens = rng.integers(lo, hi + 1, n)
    first = int(rng.integers(1, 8))
    off = (np.concatenate([[0], np.cumsum(lens)]) + first).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    key_slot = np.zeros(n, np.uint32)
    for c in (P256, P384):
        own = np.flatnonzero(reg["ecdsa_curve"] == c)
        idx = np.flatnonzero(scheme == c)
        key_slot[idx] = own[rng.integers(0, own.size, idx.size)]
    idx = np.flatnonzero(scheme == ED)
    key_slot[idx] = rng.integers(0, reg["ed_pub"].shape[0], idx.size)
    sig96 = sign_rows(scheme, msgs, off, key_slot, reg, rng, junk)
    cls = np.full(n, -1, np.int16)
    if corrupt:
        corrupt_items(scheme, msgs, off, key_slot, sig96, reg, cls, rng)
    return {"scheme": scheme, "msgs": msgs, "off": off, "key_slot": key_slot, "sig96": sig96, "cls": cls}


# corruption classes (both schemes unless noted)
FLIP_SIG, FLIP_MSG, UNKNOWN_SLOT, MAX_SLOT, WRONG_KEY, OTHER_CURVE, R_ZERO, S_ZERO, R_EQ_N, HIGH_S, S_PLUS_L, NONCANON_R = range(12)


def corrupt_items(scheme, msgs, off, key_slot, sig96, reg, cls, rng):
    n = scheme.size
    for i in np.flatnonzero(rng.random(n) < 0.25):
        t = int(scheme[i])
        c = int(rng.integers(0, 12))
        ln = int(off[i + 1] - off[i])
        if c == FLIP_MSG and ln == 0:
            c = FLIP_SIG
        if t == ED and c in (OTHER_CURVE, R_ZERO, S_ZERO, R_EQ_N, HIGH_S):
            c = [S_PLUS_L, NONCANON_R, FLIP_SIG, WRONG_KEY, UNKNOWN_SLOT][c - OTHER_CURVE]
        if t != ED and c in (S_PLUS_L, NONCANON_R):
            c = HIGH_S
        cls[i] = c
        w = 64 if t == ED else 2 * L[t]
        if c == FLIP_SIG:
            b = int(rng.integers(0, 8 * w))
            sig96[i, b >> 3] ^= 1 << (b & 7)
        elif c == FLIP_MSG:
            msgs[int(off[i]) + int(rng.integers(0, ln))] ^= 1 << int(rng.integers(0, 8))
        elif c == UNKNOWN_SLOT:
            key_slot[i] = (reg["ed_pub"].shape[0] if t == ED else reg["ecdsa_curve"].size) + int(rng.integers(0, 3))
        elif c == MAX_SLOT:
            key_slot[i] = UNKNOWN
        elif c == WRONG_KEY:
            if t == ED:
                key_slot[i] = (int(key_slot[i]) + 1) % reg["ed_pub"].shape[0]
            else:
                own = np.flatnonzero(reg["ecdsa_curve"] == t)
                key_slot[i] = own[(int(np.searchsorted(own, key_slot[i])) + 1) % own.size]
        elif c == OTHER_CURVE:
            key_slot[i] = np.flatnonzero(reg["ecdsa_curve"] != t)[0]
        elif c == R_ZERO:
            sig96[i, :L[t]] = 0
        elif c == S_ZERO:
            sig96[i, L[t]:2 * L[t]] = 0
        elif c == R_EQ_N:
            sig96[i, :L[t]] = np.frombuffer(CURVES[t].n.to_bytes(L[t], "big"), np.uint8)
        elif c == HIGH_S:  # still valid: Go has no low-S rule
            s = CURVES[t].n - int.from_bytes(bytes(sig96[i, L[t]:2 * L[t]]), "big")
            sig96[i, L[t]:2 * L[t]] = np.frombuffer(s.to_bytes(L[t], "big"), np.uint8)
        elif c == S_PLUS_L:
            s = int.from_bytes(bytes(sig96[i, 32:64]), "little") + ref.L
            if s < 2**256:
                sig96[i, 32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
        elif c == NONCANON_R:
            sig96[i, :32] = np.frombuffer((1 + ref.p).to_bytes(32, "little"), np.uint8)


def expected_ok(cp, ecdsa_curve, ecdsa_xy, ed_pub) -> np.ndarray:
    """OpenSSL's verdict of every item under the key its slot holds in its own scheme's registry (a slot outside the
    registry, or an ECDSA slot of the other curve, rejects)."""
    scheme, msgs, off, slot, sig96 = cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"].astype(np.int64), cp["sig96"]
    n = scheme.size
    ok = np.zeros(n, np.uint8)
    ecdsa_curve = np.asarray(ecdsa_curve, np.uint8)
    ecdsa_xy = np.asarray(ecdsa_xy, np.uint8).reshape(-1, 96)
    ed_pub = np.asarray(ed_pub, np.uint8).reshape(-1, 32)
    dig = oracle.sha256_batch(msgs, off) if n else None
    for c in (P256, P384):
        idx = np.flatnonzero(scheme == c)
        if idx.size == 0:
            continue
        s = slot[idx]
        known = s < ecdsa_curve.size
        good = known.copy()
        good[known] = ecdsa_curve[s[known]] == c
        kk = np.where(good, s, 0)
        xy = ecdsa_xy[kk] if ecdsa_curve.size else np.zeros((idx.size, 96), np.uint8)
        v = oracle.verify_batch(c, sig96[idx, :L[c]], sig96[idx, L[c]:2 * L[c]], xy[:, 48 - L[c]:48], xy[:, 96 - L[c]:], dig[idx])
        ok[idx] = v & good.astype(np.uint8)
    idx = np.flatnonzero(scheme == ED)
    if idx.size:
        s = slot[idx]
        known = s < ed_pub.shape[0]
        pub = np.zeros((idx.size, 32), np.uint8)
        pub[known] = ed_pub[s[known]]
        m, o = gather(msgs, off, idx)
        ok[idx] = oe.verify_batch(m, o, sig96[idx, :64], pub) & known.astype(np.uint8)
    return ok


def small_order_key():
    return np.frombuffer(edcorpus.small_order_encodings()[0], np.uint8)


def y_ge_p_key():
    return np.frombuffer(edcorpus.big_y_encodings()[0], np.uint8)


def make_votes(n_instances, schemes, seed=0, pad=0, byzantine=True, aux_lo=0, aux_hi=64):
    """A commit-vote stream of len(schemes) consenters (consenter id k + 1 holds a key of schemes[k]) in the layout of
    oracle_ed25519.votes.make_stream, re-signed under each signer's own scheme.  Returns (stream, registries): consenter k's
    key sits in slot k of its scheme's registry (the ECDSA registry holds the ECDSA consenters in id order, the Ed25519
    registry the Ed25519 ones); inert votes carry the Ed25519 tag and slot 2^32 - 1."""
    schemes = np.asarray(schemes, np.uint8)
    N = schemes.size
    rng = np.random.default_rng(seed + 7)
    ec = np.flatnonzero(schemes != ED)
    edc = np.flatnonzero(schemes == ED)
    seeds, pubs = votes.consenter_keys(N, seed + 1)
    reg = {"ed_seeds": seeds[edc], "ed_pub": pubs[edc]}
    curves, xy, priv = [], [], []
    for j, k in enumerate(ec):
        c = int(schemes[k])
        d, kxy = ecorpus.make_keys(c, 1, seed * 1000 + 10 + int(k))
        row = np.zeros((2, 48), np.uint8)
        row[:, 48 - L[c]:] = kxy[0].reshape(2, L[c])
        p = np.zeros(48, np.uint8)
        p[48 - L[c]:] = d[0]
        curves.append(c)
        xy.append(row.reshape(96))
        priv.append(p)
    reg["ecdsa_curve"] = np.array(curves, np.uint8)
    reg["ecdsa_xy"] = np.array(xy, np.uint8).reshape(-1, 96)
    reg["ecdsa_priv"] = np.array(priv, np.uint8).reshape(-1, 48)
    slot_of = np.zeros(N, np.uint32)
    slot_of[ec] = np.arange(ec.size)
    slot_of[edc] = np.arange(edc.size)
    st = votes.make_stream(n_instances, N, seed=seed, byzantine=byzantine, pad=0, aux_lo=aux_lo, aux_hi=aux_hi, keys=(seeds, pubs))
    signer_k = st["signer"].astype(np.int64) - 1
    scheme = schemes[signer_k]
    key_slot = slot_of[signer_k]
    sig96 = sign_rows(scheme, st["msgs"], st["off"], key_slot, reg, rng)
    bad = np.flatnonzero(st["cls"] == votes.BAD_SIG)
    w = np.where(scheme[bad] == ED, 64, 2 * np.array([L.get(int(t), 32) for t in scheme[bad]], np.int64))
    b = (rng.random(bad.size) * 8 * w).astype(np.int64)
    sig96[bad, b >> 3] ^= (1 << (b & 7)).astype(np.uint8)
    st = dict(st, scheme=scheme, key_slot=key_slot, sig96=sig96)
    if pad:
        end = st["off"][-1]
        I = st["n_instances"]
        cat = np.concatenate
        st.update(off=cat([st["off"], np.full(pad, end, np.uint64)]), sig96=cat([sig96, np.zeros((pad, 96), np.uint8)]),
                  key_slot=cat([key_slot, np.full(pad, UNKNOWN, np.uint32)]), scheme=cat([scheme, np.full(pad, ED, np.uint8)]),
                  instance=cat([st["instance"], np.full(pad, max(I - 1, 0), np.uint32)]), sender=cat([st["sender"], np.ones(pad, np.uint16)]),
                  signer=cat([st["signer"], np.full(pad, 2, np.uint16)]), digest_match=cat([st["digest_match"], np.zeros(pad, np.uint8)]),
                  cls=cat([st["cls"], np.full(pad, votes.INERT, np.uint8)]))
    return st, reg


def expected_votes(st, reg, threshold, self_id="stream", ecdsa=None, ed_pub=None):
    """(ok, valid_count, reached): expected_ok for ok, oracle.ecdsa_ref.count_commit_votes_batch for the counts."""
    from oracle import ecdsa_ref
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    curve, xy = ecdsa if ecdsa is not None else (reg["ecdsa_curve"], reg["ecdsa_xy"])
    ok = expected_ok(st, curve, xy, reg["ed_pub"] if ed_pub is None else ed_pub)
    cnt, reached = ecdsa_ref.count_commit_votes_batch(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"], threshold,
                                                      sid)
    return ok, cnt, reached
