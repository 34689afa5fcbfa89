"""Seeded streams of Ed25519 commit votes for sbv_ed25519_verify_quorum (TEST / BENCH INFRASTRUCTURE).

make_stream(n_instances, n, seed) -> dict of the call's columns.  N consenters (ids 1..N) hold Ed25519 keys; registry
slot id - 1 holds consenter id's key, and a vote carries the slot of its claimed signer.  Per instance every consenter
except the instance's self id votes once, in a random order, over Msg = the instance's 32-byte proposal digest || aux
(the signed-bytes convention of INTEGRATION.md), signed by OpenSSL.  Up to f = (N - 1) // 3 votes of an instance are
Byzantine, each of one class: a bad signature, a wrong digest (digest_match = 0, signed over the wrong digest), a second
vote of a sender that already voted, or a signer other than the sender.  `pad` inert votes (signer != sender, slot
2^32 - 1, no message, zero signature) close the stream.  The expected outputs come from the oracles (`expected`), not
from the classes.
"""
from __future__ import annotations

import numpy as np

from . import pubkey, sign_batch, verify_batch

HONEST, BAD_SIG, WRONG_DIGEST, DOUBLE_VOTE, FOREIGN_SIGNER, INERT = range(6)
UNKNOWN_SLOT = 2**32 - 1


def consenter_keys(n: int, seed: int):
    """(seeds, pubs) of n consenters: n x 32 bytes each."""
    rng = np.random.default_rng(seed)
    seeds = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    pubs = np.frombuffer(b"".join(pubkey(bytes(s)) for s in seeds), np.uint8).reshape(n, 32)
    return seeds, pubs


def make_stream(n_instances: int, n: int = 16, seed: int = 0, byzantine: bool = True, pad: int = 0, aux_lo: int = 0, aux_hi: int = 64,
                keys=None):
    rng = np.random.default_rng(seed)
    f = (n - 1) // 3
    seeds, pubs = keys if keys is not None else consenter_keys(n, seed + 1)
    I, per = n_instances, n - 1
    self_id = (np.arange(I) % n + 1).astype(np.uint16)
    # the n - 1 foreign consenters of each instance in a random order
    order = rng.random((I, n))
    order[np.arange(I), self_id.astype(np.int64) - 1] = 2.0
    sender = (np.argsort(order, axis=1)[:, :per] + 1).astype(np.uint16)
    signer = sender.copy()
    cls = np.zeros((I, per), np.uint8)
    if byzantine and per > 1:
        nb = rng.integers(0, f + 1, I)
        for i in np.flatnonzero(nb):
            for pos in rng.choice(np.arange(1, per), int(nb[i]), replace=False):
                c = int(rng.integers(BAD_SIG, FOREIGN_SIGNER + 1))
                cls[i, pos] = c
                if c == DOUBLE_VOTE:
                    sender[i, pos] = signer[i, pos] = sender[i, int(rng.integers(pos))]
                elif c == FOREIGN_SIGNER:
                    signer[i, pos] = (int(sender[i, pos]) - 1 + int(rng.integers(1, n))) % n + 1
    instance = np.repeat(np.arange(I, dtype=np.uint32), per)
    sender, signer, cls = sender.reshape(-1), signer.reshape(-1), cls.reshape(-1)
    nv = I * per
    digests = rng.integers(0, 256, (I, 32), dtype=np.uint8)
    wrong = rng.integers(0, 256, (nv, 32), dtype=np.uint8)
    lens = 32 + rng.integers(aux_lo, aux_hi + 1, nv)
    first = int(rng.integers(1, 8))  # off[0] > 0: with the odd lengths the offsets are misaligned
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(first)
    msgs = rng.integers(0, 256, int(off[nv]) + 16, dtype=np.uint8)
    head = off[:-1].astype(np.int64)[:, None] + np.arange(32)
    dm = (cls != WRONG_DIGEST).astype(np.uint8)
    msgs[head] = np.where(dm[:, None] == 1, digests[instance], wrong)
    key_slot = signer.astype(np.uint32) - 1
    sig = sign_batch(seeds, key_slot, msgs, off) if nv else np.zeros((0, 64), np.uint8)
    bad = np.flatnonzero(cls == BAD_SIG)
    sig[bad, rng.integers(0, 64, bad.size)] ^= (1 << rng.integers(0, 8, bad.size)).astype(np.uint8)
    st = {"msgs": msgs, "off": off, "sig": sig, "key_slot": key_slot, "instance": instance, "sender": sender, "signer": signer,
          "digest_match": dm, "cls": cls, "self_id": self_id, "n_instances": I, "pub": pubs, "seeds": seeds, "n": n}
    return add_inert(st, pad) if pad else st


def add_inert(st, k: int):
    """k inert votes appended to the last instance: signer != sender, unknown slot, no message, zero signature."""
    end = st["off"][-1]
    out = dict(st)
    out["off"] = np.concatenate([st["off"], np.full(k, end, np.uint64)])
    out["sig"] = np.concatenate([st["sig"], np.zeros((k, 64), np.uint8)])
    out["key_slot"] = np.concatenate([st["key_slot"], np.full(k, UNKNOWN_SLOT, np.uint32)])
    out["instance"] = np.concatenate([st["instance"], np.full(k, max(st["n_instances"] - 1, 0), np.uint32)])
    out["sender"] = np.concatenate([st["sender"], np.full(k, 1, np.uint16)])
    out["signer"] = np.concatenate([st["signer"], np.full(k, 2, np.uint16)])
    out["digest_match"] = np.concatenate([st["digest_match"], np.zeros(k, np.uint8)])
    out["cls"] = np.concatenate([st["cls"], np.full(k, INERT, np.uint8)])
    return out


def expected_ok(st, registry=None) -> np.ndarray:
    """OpenSSL's verdict of every vote under the key registered in its slot (registry: n x 32 bytes, default the
    consenters' keys); a slot outside the registry rejects."""
    reg = st["pub"] if registry is None else np.asarray(registry, np.uint8).reshape(-1, 32)
    slot = st["key_slot"].astype(np.int64)
    known = slot < reg.shape[0]
    pub = np.zeros((slot.size, 32), np.uint8)
    pub[known] = reg[slot[known]]
    if slot.size == 0:
        return np.zeros(0, np.uint8)
    return verify_batch(st["msgs"], st["off"], st["sig"], pub) & known.astype(np.uint8)


def expected(st, threshold: int, self_id="stream", registry=None):
    """(ok, valid_count, reached) of the stream: OpenSSL for ok, oracle.ecdsa_ref.count_commit_votes_batch for the
    counts.  self_id: "stream" = the stream's self ids, None = no self filter, or an array."""
    from oracle import ecdsa_ref
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    ok = expected_ok(st, registry)
    cnt, reached = ecdsa_ref.count_commit_votes_batch(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"],
                                                      threshold, sid)
    return ok, cnt, reached
