"""The RSA PKCS #1 v1.5 corpus shared by the CPU simulation, oracle and GPU tests: seeded keys (cached per session) and, per
modulus size and hash, items of every class of the accept set in include/sbv.h, each labelled and judged by oracle_rsa.ref.

Classes (per size k in 256 / 384 / 512 bytes and per hash):
  valid        e = 65537, e = 3, e = 2^31 - 1, and (k = 256) a 2047-bit modulus, whose top bit is clear
  msglen       valid signatures over messages of the lengths around every SHA-2 block boundary, the empty one included;
               the messages sit back to back, so most start at unaligned offsets
  corrupt      a wrong message, a flipped bit in the signature, a flipped bit in the modulus
  sigval       S in {0, 1, N - 1, N, N + 1, 2^(8k) - 1}, and S + N for a valid S chosen so that it fits in k bytes
  crafted      an arbitrary EM signed with d, so that S^e recovers exactly those bytes: block type 02, a first byte of 01,
               no 00 separator, a non-FF byte in the run, the DigestInfo of another hash, a DigestInfo without the NULL
               parameters, the right prefix with a wrong digest, and (e = 3) the digest followed by garbage with a shorter run
  badkey       items that only the key rule rejects: e = 1 with S = EM, e = 2^31 + 1 (or the next odd exponent the key
               can sign with) and e = 2^32 - 1 with signatures made under them, a key one byte short (its modulus has
               a leading zero byte in k bytes) signing the k-byte encoding; also e = 0, e = 2^31 and an even N
"""
from __future__ import annotations

import functools
import math
import random

import numpy as np

from oracle_rsa import ref

SIZES = (256, 384, 512)
HASHES = (ref.SHA256, ref.SHA384, ref.SHA512)
# around the 64- and 128-byte blocks of SHA-256 and SHA-512 / SHA-384 (the padding needs 9 and 17 bytes)
MSG_LENS = (0, 1, 55, 56, 63, 64, 65, 111, 112, 119, 120, 127, 128, 129, 183, 184, 239, 240, 256)


@functools.lru_cache(maxsize=None)
def key(bits: int, seed: int = 1) -> ref.Key:
    return ref.Key(bits, seed)


class _Builder:
    def __init__(self, k, hash, seed):
        self.k, self.hash, self.rng = k, hash, random.Random(f"cases-{k}-{hash}-{seed}")
        self.msgs, self.sig, self.mod, self.exp, self.cls = [], [], [], [], []

    def digest(self, m):
        return ref.HASHLIB[self.hash](m).digest()

    def add(self, cls, msg, sig, mod, e):
        assert len(sig) == self.k and len(mod) == self.k
        self.msgs.append(bytes(msg)); self.sig.append(bytes(sig)); self.mod.append(bytes(mod)); self.exp.append(e); self.cls.append(cls)

    def msg(self, n=None):
        return self.rng.randbytes(self.rng.randrange(1, 300) if n is None else n)

    def done(self):
        k, hl = self.k, ref.HLEN[self.hash]
        n = len(self.msgs)
        off = np.concatenate([[0], np.cumsum([len(m) for m in self.msgs])]).astype(np.uint64)
        digest = np.frombuffer(b"".join(self.digest(m) for m in self.msgs), np.uint8).reshape(n, hl).copy()
        out = dict(k=k, hash=self.hash, n=n, msgs=np.frombuffer(b"".join(self.msgs) + b"\0", np.uint8)[:-1].copy(), off=off, digest=digest,
                   sig=np.frombuffer(b"".join(self.sig), np.uint8).reshape(n, k).copy(),
                   mod=np.frombuffer(b"".join(self.mod), np.uint8).reshape(n, k).copy(),
                   exp=np.array(self.exp, np.uint32), cls=list(self.cls))
        out["want"] = ref.verify_batch(k, self.hash, digest, out["sig"], out["mod"], out["exp"])
        return out


def make_cases(k: int, hash: int, seed: int = 0, short: bool = False) -> dict:
    """Every class for modulus size k and the hash tag; short: one item per class (the CPU simulation's budget)."""
    b = _Builder(k, hash, seed)
    K = key(8 * k)
    N, mod = K.n, K.mod_bytes(k)
    sign = lambda m, e=65537: K.sign(k, hash, b.digest(m), e)  # noqa: E731
    # valid
    for e in ((65537, 3, ref.E_MAX) if short else (65537, 65537, 65537, 3, ref.E_MAX)):
        m = b.msg()
        b.add(f"valid_e{e}", m, sign(m, e), mod, e)
    if k == 256:
        K7 = key(8 * k - 1)
        m = b.msg()
        b.add("valid_2047bit", m, K7.sign(k, hash, b.digest(m)), K7.mod_bytes(k), 65537)
    # msglen
    for ln in (MSG_LENS[::6] if short else MSG_LENS):
        m = b.msg(ln)
        b.add(f"msglen_{ln}", m, sign(m), mod, 65537)
    # corrupt
    m = b.msg()
    b.add("corrupt_message", b.msg(), sign(m), mod, 65537)
    s = bytearray(sign(m)); s[b.rng.randrange(k)] ^= 1 << b.rng.randrange(8)
    b.add("corrupt_sig_bit", m, s, mod, 65537)
    md = bytearray(mod); md[b.rng.randrange(1, k - 1)] ^= 1 << b.rng.randrange(8)
    b.add("corrupt_mod_bit", m, sign(m), md, 65537)
    # sigval
    m = b.msg()
    for name, v in (("0", 0), ("1", 1), ("n-1", N - 1), ("n", N), ("n+1", N + 1), ("max", 2 ** (8 * k) - 1)):
        b.add(f"sigval_{name}", m, v.to_bytes(k, "big"), mod, 65537)
    for _ in range(64):  # a valid S whose twin S + N fits in k bytes
        sv = int.from_bytes(sign(m), "big")
        if sv + N < 2 ** (8 * k):
            b.add("sigval_s+n", m, (sv + N).to_bytes(k, "big"), mod, 65537)
            break
        m = b.msg()
    # crafted: EM signed with d
    other = (hash + 1) % 3
    m = b.msg()
    h = b.digest(m)
    good = ref.encode(k, hash, h)
    t = ref.DIGEST_INFO[hash] + h
    nonull = ref.DIGEST_INFO[hash][:15] + ref.DIGEST_INFO[hash][17:]  # without 05 00, lengths fixed below
    nonull = bytes([0x30, nonull[1] - 2, 0x30, 0x0b]) + nonull[4:]
    crafted = {
        "crafted_bt02": b"\x00\x02" + good[2:],
        "crafted_first01": b"\x01" + good[1:],
        "crafted_no_sep": good[:len(good) - len(t) - 1] + b"\xff" + t,
        "crafted_run_byte": good[:5] + b"\xfe" + good[6:],
        "crafted_other_di": b"\x00\x01" + b"\xff" * (k - len(ref.DIGEST_INFO[other]) - len(h) - 3) + b"\x00" + ref.DIGEST_INFO[other] + h,
        "crafted_di_no_null": b"\x00\x01" + b"\xff" * (k - len(nonull) - len(h) - 3) + b"\x00" + nonull + h,
        "crafted_wrong_digest": good[:-1] + bytes([good[-1] ^ 0x80]),
        "crafted_good": good,
    }
    for name, em in crafted.items():
        assert len(em) == k, name
        b.add(name, m, K.sign_em(em, 65537, k), mod, 65537)
    garbage = b"\x00\x01" + b"\xff" * 8 + b"\x00" + t
    garbage += b.rng.randbytes(k - len(garbage))
    b.add("crafted_e3_garbage", m, K.sign_em(garbage, 3, k), mod, 3)
    # badkey: each item is one the arithmetic alone would accept (S^e mod N is the right encoding), so only the key rule
    # of step 1 rejects it
    b.add("badkey_e0", m, sign(m), mod, 0)  # S^0 = 1: no S recovers an encoding, any S will do
    b.add("badkey_e1", m, good, mod, 1)  # S = EM
    b.add("badkey_e2147483648", m, sign(m), mod, 2**31)  # even: never invertible mod lcm(p-1, q-1)
    e_big = 2**31 + 1  # the smallest odd exponent above Go's bound that the key can sign with
    while math.gcd(e_big, K.lam) != 1:
        e_big += 2
    b.add("badkey_e_above_max", m, K.sign_em(good, e_big, k), mod, e_big)
    b.add("badkey_e4294967295", m, K.sign_em(good, 2**32 - 1, k), mod, 2**32 - 1)  # invertible: see ref._prime
    b.add("badkey_even_n", m, sign(m), (N ^ 1).to_bytes(k, "big"), 65537)
    K8 = key(8 * k - 8)  # a key one byte short: its modulus has a leading zero byte in k bytes
    b.add("badkey_lead0", m, K8.sign_em(good, 65537, k), K8.mod_bytes(k), 65537)
    for i in range(len(b.cls)):  # the arithmetic accepts these: only step 1 can reject them
        if b.cls[i] in ("badkey_e1", "badkey_e_above_max", "badkey_e4294967295", "badkey_lead0"):
            assert pow(int.from_bytes(b.sig[i], "big"), b.exp[i], int.from_bytes(b.mod[i], "big")).to_bytes(k, "big") == good, b.cls[i]
    return b.done()
