"""Seeded streams of RSA commit votes for sbv_rsa_verify_quorum / sbv_rsa_pss_verify_quorum, shared by the CPU simulation
(tests/test_hostsim_rsa_quorum.py), the GPU tests (tests/test_gpu_rsa_quorum.py) and tools/rsa_quorum_bench.py.

consenters(sizes): consenter id c + 1 holds registry slot c, a key of sizes[c] bytes from tests/golden/rsa_keys.npz (five
keys per size; a key used again gets another public exponent, so every slot is a distinct key).

make_stream(cons, n_instances, seed): per instance every consenter except the instance's self id votes once, in a random
order, over the instance's proposal, drawn from a pool of a few messages so that each (consenter, message) pair is signed
once and its signature reused.  Up to f = (N - 1) // 3 votes of an instance are Byzantine, each of one class: a bad
signature, a wrong digest (digest_match = 0, signed over another message), a second vote of a sender that already voted,
or a signer other than the sender.  `pad` inert votes (signer != sender, unknown slot, no message, no signature) close the
stream.  The votes stay editable as lists (msg, sig) until pack(); expected() judges every vote with oracle_rsa.ref and
counts with oracle.ecdsa_ref.count_commit_votes_batch, independent of the classes."""
from __future__ import annotations

import functools
import hashlib
import math

import numpy as np

import rsa_edges
import rsa_registered as rr
from oracle import ecdsa_ref
from oracle_rsa import ref

HONEST, BAD_SIG, WRONG_DIGEST, DOUBLE_VOTE, FOREIGN_SIGNER, INERT = range(6)
UNKNOWN_SLOT = 2**32 - 1
SIZES = (256, 384, 512)
MIXED = (256,) * 10 + (384,) * 4 + (512,) * 2  # N = 16: ten 2048-bit, four 3072-bit and two 4096-bit consenters
ALL_2048 = (256,) * 16
EXPONENTS = (65537, 3, 5, 17, 257, 641)


@functools.lru_cache(maxsize=None)
def _golden(k: int, j: int):
    """The j-th key of size k: the golden keys in turn, each with the next public exponent it can sign with."""
    names = [f"std_{8 * k - d}" for d in (0, 1, 4, 7)] + [f"blum_{8 * k}"]
    K = rsa_edges.key(names[j % len(names)])
    es = [e for e in EXPONENTS if math.gcd(e, K.lam) == 1]
    return K, es[j // len(names)]


class Consenters:
    """keys[c] = (Key, k, e) of consenter c + 1 in slot c; reg = [(modulus bytes, e)] in slot order, extra slots appended."""

    def __init__(self, sizes):
        seen = {k: 0 for k in SIZES}
        self.keys = []
        for k in sizes:
            K, e = _golden(k, seen[k])
            seen[k] += 1
            self.keys.append((K, k, e))
        self.reg = [(K.mod_bytes(k), e) for K, k, e in self.keys]
        self._sig = {}

    @property
    def n(self):
        return len(self.keys)

    def arrays(self, reg=None):
        """(mod_bytes, modulus, exp) of sbv_rsa_set_keys for the registry reg (default: the consenters')."""
        reg = self.reg if reg is None else reg
        mb = np.array([len(m) for m, _ in reg], np.uint32)
        mods = np.frombuffer(b"".join(m for m, _ in reg) + b"\0", np.uint8)[:-1].copy()
        return mb, mods, np.array([e for _, e in reg], np.uint32)

    def sign(self, c: int, msg: bytes, hash: int, salt: bytes | None = None) -> bytes:
        """Consenter slot c's signature of msg: PKCS #1 v1.5, or PSS with the given salt; each one made once."""
        key = (c, msg, hash, salt)
        if key not in self._sig:
            K, k, e = self.keys[c]
            d = ref.HASHLIB[hash](msg).digest()
            self._sig[key] = K.sign(k, hash, d, e) if salt is None else K.sign_pss(k, hash, d, salt, e)
        return self._sig[key]


def make_stream(cons: Consenters, n_instances: int, seed: int = 0, hash: int = ref.SHA256, salt_bytes: int | None = None, byzantine: bool = True,
                pad: int = 0, pool: int = 4):
    """salt_bytes None: PKCS #1 v1.5 signatures; else PSS signatures with salts of that many bytes."""
    rng = np.random.default_rng(seed)
    n = cons.n
    f = (n - 1) // 3
    I, per = n_instances, n - 1
    self_id = (np.arange(I) % n + 1).astype(np.uint16)
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
    proposals = [rng.bytes(int(rng.integers(32, 97))) for _ in range(pool)]
    wrong = [rng.bytes(int(rng.integers(32, 97))) for _ in range(pool)]
    prop = rng.integers(0, pool, I)
    salts = [rng.bytes(salt_bytes) for _ in range(pool)] if salt_bytes is not None else [None] * pool
    msgs, sigs = [], []
    for v in range(I * per):
        c, p = int(signer[v]) - 1, int(prop[instance[v]])
        m = wrong[p] if cls[v] == WRONG_DIGEST else proposals[p]
        s = cons.sign(c, m, hash, salts[p])
        if cls[v] == BAD_SIG:
            b = bytearray(s)
            b[int(rng.integers(0, len(b)))] ^= 1 << int(rng.integers(0, 8))
            s = bytes(b)
        msgs.append(m)
        sigs.append(s)
    st = {"msgs_l": msgs, "sigs_l": sigs, "key_slot": signer.astype(np.uint32) - 1, "instance": instance, "sender": sender, "signer": signer,
          "digest_match": (cls != WRONG_DIGEST).astype(np.uint8), "cls": cls, "self_id": self_id, "n_instances": I, "hash": hash}
    return add_inert(st, pad) if pad else st


def add_inert(st, k: int):
    """k inert votes appended to the last instance: signer != sender, unknown slot, no message, no signature."""
    out = dict(st)
    out["msgs_l"] = st["msgs_l"] + [b""] * k
    out["sigs_l"] = st["sigs_l"] + [b""] * k
    out["key_slot"] = np.concatenate([st["key_slot"], np.full(k, UNKNOWN_SLOT, np.uint32)])
    out["instance"] = np.concatenate([st["instance"], np.full(k, max(st["n_instances"] - 1, 0), np.uint32)])
    out["sender"] = np.concatenate([st["sender"], np.full(k, 1, np.uint16)])
    out["signer"] = np.concatenate([st["signer"], np.full(k, 2, np.uint16)])
    out["digest_match"] = np.concatenate([st["digest_match"], np.zeros(k, np.uint8)])
    out["cls"] = np.concatenate([st["cls"], np.full(k, INERT, np.uint8)])
    return out


def blob(parts, first: int = 0):
    """(bytes as uint8, offsets as uint64) of the concatenation, starting at offset `first`."""
    lens = np.array([len(p) for p in parts], np.uint64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(first)
    data = np.frombuffer(bytes(first) + b"".join(parts) + bytes(16), np.uint8).copy()
    return data, off


def pack(st):
    """The columns of the call: msgs / off and sig / sig_off (both starting past offset 0, so that offsets are misaligned)."""
    out = dict(st)
    out["msgs"], out["off"] = blob(st["msgs_l"], 3)
    out["sig"], out["sig_off"] = blob(st["sigs_l"], 5)
    return out


def verdicts(reg, st, salt_len: int | None = None):
    """ok of every vote by oracle_rsa.ref: the slot's key at the signature's length, PKCS #1 v1.5 (salt_len None) or PSS."""
    hash = st["hash"]
    cache = {}
    ok = np.zeros(len(st["sigs_l"]), np.uint8)
    for v, (m, s) in enumerate(zip(st["msgs_l"], st["sigs_l"])):
        slot = int(st["key_slot"][v])
        key = (slot, m, s)
        if key not in cache:
            L = len(s)
            good = False
            if L in SIZES and slot < len(reg) and len(reg[slot][0]) == L:
                mod, e = reg[slot]
                d = ref.HASHLIB[hash](m).digest()
                good = ref.verify(L, hash, d, s, mod, e) if salt_len is None else ref.pss_verify(L, hash, d, s, mod, e, salt_len)
            cache[key] = int(good)
        ok[v] = cache[key]
    return ok


def expected(reg, st, thr, self_id="stream", salt_len=None):
    """(ok, valid_count, reached) from the oracles."""
    ok = verdicts(reg, st, salt_len)
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    cnt, reached = ecdsa_ref.count_commit_votes_batch(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"], thr, sid)
    return ok, cnt, reached


def append_vote(st, msg, sig, slot, sender):
    """One more vote, in the last instance, by a sender that has not voted there (ids past the consenters')."""
    out = dict(st)
    out["msgs_l"] = st["msgs_l"] + [msg]
    out["sigs_l"] = st["sigs_l"] + [sig]
    for name, v, dt in (("key_slot", slot, np.uint32), ("instance", st["n_instances"] - 1, np.uint32), ("sender", sender, np.uint16),
                        ("signer", sender, np.uint16), ("digest_match", 1, np.uint8), ("cls", HONEST, np.uint8)):
        out[name] = np.concatenate([st[name], np.array([v], dt)])
    return out


def edge_stream(cons, salt=None):
    """Two instances of the 16 consenters, then votes of the edge classes in the last instance, each one counted only by the
    verdict it gets (a fresh sender each): lengths k - 1, k + 1 and 0 of a valid signature, a size trap (PKCS #1 v1.5), a
    key the rule refuses, unknown slots, S = N and S = N + 1, and a rejected vote followed by a valid one of its sender.
    salt: PSS signatures with a salt of that many zero bytes.  Returns (registry, stream)."""
    hash = ref.SHA256
    st = make_stream(cons, 2, seed=5, hash=hash, salt_bytes=salt)
    reg = list(cons.reg)
    msg = b"edge votes"
    d = hashlib.sha256(msg).digest()
    sender = 100
    for c in (0, 10, 14):  # one consenter of each size
        s = cons.sign(c, msg, hash, None if salt is None else bytes(salt))
        for sig in (s[1:], s + b"\0", b"", s):
            st = append_vote(st, msg, sig, c, sender)
            sender += 1
        # the size trap: a slot of the next size whose bytes, read at this signature's size, accept it
        K, k, e = cons.keys[c]
        if salt is None:
            big = 384 if k == 256 else 512
            if k < 512:
                mod, sig = rr.size_trap(K.mod_bytes(k), s, big, seed=c)
                reg.append((mod, e))
                st = append_vote(st, msg, sig, len(reg) - 1, sender)
                sender += 1
    # a key the key rule refuses (e = 1) with S = EM, which e = 1 would accept
    K, k, e = cons.keys[1]
    reg.append((K.mod_bytes(k), 1))
    st = append_vote(st, msg, ref.encode(k, hash, d), len(reg) - 1, sender)
    sender += 1
    for slot in (len(reg), len(reg) + 7, UNKNOWN_SLOT):
        st = append_vote(st, msg, cons.sign(2, msg, hash, None if salt is None else bytes(salt)), slot, sender)
        sender += 1
    # S = N and S = N + 1 (k bytes each)
    for c in (3, 11):
        K, k, e = cons.keys[c]
        for s in (K.n, K.n + 1):
            st = append_vote(st, msg, s.to_bytes(k, "big"), c, sender)
            sender += 1
    # a rejected vote burns its sender's slot: the sender's later valid vote is verified but not counted
    good = cons.sign(4, msg, hash, None if salt is None else bytes(salt))
    st = append_vote(st, msg, good[:-1] + bytes([good[-1] ^ 1]), 4, sender)
    st = append_vote(st, msg, good, 4, sender)
    return reg, st


def take(st, n):
    """The first n votes of a stream."""
    out = dict(st)
    for name in ("key_slot", "instance", "sender", "signer", "digest_match", "cls"):
        out[name] = st[name][:n]
    out["msgs_l"], out["sigs_l"] = st["msgs_l"][:n], st["sigs_l"][:n]
    return out


def only(st, sizes):
    """The stream with the votes whose signature length is not in sizes made inert (no signature, unknown slot)."""
    out = dict(st)
    out["sigs_l"] = [s if len(s) in sizes else b"" for s in st["sigs_l"]]
    return out
