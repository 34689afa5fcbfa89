"""The RSA-PSS corpus shared by the CPU simulation, oracle and GPU tests: per modulus size and hash, items of every class of
the PSS accept set in include/sbv.h, each labelled; verdicts come from oracle_rsa.ref.pss_verify for whichever salt_len a
call uses (the salt length is an argument of the call, not of the item).

Keys: the committed keys of tests/golden/rsa_keys.npz (std_<b> for b = 8k, 8k - 1, 8k - 4, 8k - 7; see rsa_edges.py), and
for badkey_lead0 the 8k - 8 bit key of rsa_cases.py.  The main key is std_<8k>.

Classes (per size k in 256 / 384 / 512 bytes and per hash):
  valid     salts of 0, hLen, a middle length and the longest, emLen - hLen - 2 bytes (e = 65537); salt hLen with e = 3
            and e = 2^31 - 1; salt hLen and the longest on the keys of 8k - 1, 8k - 4 and 8k - 7 bits (emLen = k - 1)
  msglen    valid signatures (salt hLen) over messages of the lengths around every SHA-2 block boundary
  corrupt   a wrong message, a flipped bit in the signature, a flipped bit in the modulus
  sigval    S in {0, 1, N - 1, N, N + 1, 2^(8k) - 1}, and S + N for a valid S chosen so that it fits in k bytes
  crafted   an EM built piece by piece and signed with d, salt hLen unless named: the intact build; trailer BD, 00, 01; each
            forbidden top bit of maskedDB set where EM < N allows it (keys of 8k, 8k - 1 and 8k - 4 bits); a nonzero
            leading byte with emLen = k - 1; a nonzero PS byte first, in the middle and last; the separator 00 or 02; an
            all-zero DB; an H_em that is not Hash(M') (DB masked with it, so only the compare rejects); MGF1 with the
            counter off by one, little-endian, or over another hash; M' with 7 or 9 zero bytes; M' over the digest of
            another hash
  cross     a PKCS #1 v1.5 signature of the same digest
  badkey    items that only the key rule rejects (as in rsa_cases.py, with PSS encodings): e = 1 with S = EM, e = 2^31 + 1
            (or the next odd exponent the key can sign with) and e = 2^32 - 1 with signatures made under them, a key one
            byte short signing its own PSS encoding; also e = 0, e = 2^31 and an even N
"""
from __future__ import annotations

import math
import random

import numpy as np

import rsa_cases
import rsa_edges
from oracle_rsa import ref

SIZES = (256, 384, 512)
HASHES = (ref.SHA256, ref.SHA384, ref.SHA512)
MSG_LENS = rsa_cases.MSG_LENS
E = 65537


def key(bits: int) -> ref.Key:
    return rsa_edges.key(f"std_{bits}")


def em_geometry(K: ref.Key, k: int):
    """(emBits, emLen) of a key."""
    em_bits = K.bits - 1
    return em_bits, (em_bits + 7) // 8


def salts(k: int, hash: int, em_len: int | None = None) -> dict:
    """The valid salt lengths of a size and hash: none, hLen, a middle one and the longest."""
    hl = ref.HLEN[hash]
    longest = (k if em_len is None else em_len) - hl - 2
    return {"0": 0, "hlen": hl, "mid": longest // 2 + 1, "max": longest}


def mgf(seed: bytes, length: int, hash: int, counter=lambda c: c.to_bytes(4, "big")) -> bytes:
    """MGF1 with a choice of counter encoding (the crafted masks), independent of ref.mgf1."""
    out, c = b"", 0
    while len(out) < length:
        out += ref.HASHLIB[hash](seed + counter(c)).digest()
        c += 1
    return out[:length]


def build_em(em_bits: int, hash: int, db: bytes, h: bytes, mask_hash=None, counter=None, trailer=0xBC) -> bytes:
    """maskedDB || H_em || trailer, the mask MGF1(H_em) (over mask_hash, with the counter encoding given)."""
    em_len = (em_bits + 7) // 8
    assert len(db) == em_len - len(h) - 1
    m = mgf(h, len(db), hash if mask_hash is None else mask_hash, *(() if counter is None else (counter,)))
    masked = bytearray(x ^ y for x, y in zip(db, m))
    masked[0] &= 0xFF >> (8 * em_len - em_bits)
    return bytes(masked) + h + bytes([trailer])


def mprime_hash(hash: int, digest: bytes, salt: bytes, zeros: int = 8) -> bytes:
    return ref.HASHLIB[hash](bytes(zeros) + digest + salt).digest()


def db_of(em_len: int, hash: int, salt: bytes, ps_patch=None, sep=0x01) -> bytes:
    ps = bytearray(em_len - len(salt) - ref.HLEN[hash] - 2)
    if ps_patch:
        ps[ps_patch[0]] = ps_patch[1]
    return bytes(ps) + bytes([sep]) + salt


class _Builder(rsa_cases._Builder):
    def __init__(self, k, hash, seed):
        super().__init__(k, hash, seed)
        self.rng = random.Random(f"pss-cases-{k}-{hash}-{seed}")

    def done(self):  # no verdicts here: they depend on the call's salt_len (want below)
        k, hl = self.k, ref.HLEN[self.hash]
        n = len(self.msgs)
        off = np.concatenate([[0], np.cumsum([len(m) for m in self.msgs])]).astype(np.uint64)
        digest = np.frombuffer(b"".join(self.digest(m) for m in self.msgs), np.uint8).reshape(n, hl).copy()
        return dict(k=k, hash=self.hash, n=n, msgs=np.frombuffer(b"".join(self.msgs) + b"\0", np.uint8)[:-1].copy(), off=off, digest=digest,
                    sig=np.frombuffer(b"".join(self.sig), np.uint8).reshape(n, k).copy(),
                    mod=np.frombuffer(b"".join(self.mod), np.uint8).reshape(n, k).copy(),
                    exp=np.array(self.exp, np.uint32), cls=list(self.cls))


def want(c: dict, salt_len: int) -> np.ndarray:
    """ref's verdicts on the corpus c under salt_len."""
    return ref.pss_verify_batch(c["k"], c["hash"], c["digest"], c["sig"], c["mod"], c["exp"], salt_len)


def salt_lens(c: dict) -> list:
    """The salt_len values a corpus is run under: auto, equals-hash, and every valid salt length present with the lengths
    one shorter and one longer (an explicit 0 is auto, so it is left out), and 2^31 - 1."""
    hl = ref.HLEN[c["hash"]]
    explicit = set()
    for L in c["salts"]:
        explicit |= {L - 1, L, L + 1}
    explicit.discard(0)
    explicit.discard(-1)
    return [ref.SALT_AUTO, ref.SALT_EQUALS_HASH] + sorted(explicit | {hl}) + [2**31 - 1]


def make_cases(k: int, hash: int, seed: int = 0, short: bool = False) -> dict:
    """Every class for modulus size k and the hash tag; short: fewer message lengths and valid repeats (the CPU
    simulation's budget).  c["salts"] lists the salt lengths of the valid items."""
    b = _Builder(k, hash, seed)
    hl = ref.HLEN[hash]
    K = key(8 * k)
    N, mod = K.n, K.mod_bytes(k)
    em_bits, em_len = em_geometry(K, k)
    S = salts(k, hash)
    used = set()

    def salt(n):
        used.add(n)
        return b.rng.randbytes(n)

    def sign(m, s_len=hl, e=E, KK=K):
        return KK.sign_pss(k, hash, b.digest(m), salt(s_len), e)

    # valid
    for name, L in S.items():
        m = b.msg()
        b.add(f"valid_salt_{name}", m, sign(m, L), mod, E)
    for e in (3, ref.E_MAX):
        m = b.msg()
        b.add(f"valid_e{e}", m, sign(m, hl, e), mod, e)
    for bits in (8 * k - 1, 8 * k - 4, 8 * k - 7):
        Kb = key(bits)
        _, el = em_geometry(Kb, k)
        for name in (("hlen",) if short else ("hlen", "max")):
            L = salts(k, hash, el)[name]
            m = b.msg()
            b.add(f"valid_bitlen{bits}_salt_{name}", m, sign(m, L, E, Kb), Kb.mod_bytes(k), E)
    # msglen
    for ln in (MSG_LENS[::6] if short else MSG_LENS):
        m = b.msg(ln)
        b.add(f"msglen_{ln}", m, sign(m), mod, E)
    # corrupt
    m = b.msg()
    b.add("corrupt_message", b.msg(), sign(m), mod, E)
    s = bytearray(sign(m)); s[b.rng.randrange(k)] ^= 1 << b.rng.randrange(8)
    b.add("corrupt_sig_bit", m, s, mod, E)
    md = bytearray(mod); md[b.rng.randrange(1, k - 1)] ^= 1 << b.rng.randrange(8)
    b.add("corrupt_mod_bit", m, sign(m), md, E)
    # sigval
    m = b.msg()
    for name, v in (("0", 0), ("1", 1), ("n-1", N - 1), ("n", N), ("n+1", N + 1), ("max", 2 ** (8 * k) - 1)):
        b.add(f"sigval_{name}", m, v.to_bytes(k, "big"), mod, E)
    for _ in range(64):
        sv = int.from_bytes(sign(m), "big")
        if sv + N < 2 ** (8 * k):
            b.add("sigval_s+n", m, (sv + N).to_bytes(k, "big"), mod, E)
            break
        m = b.msg()
    # crafted: EMs built piece by piece, signed with d
    other = (hash + 1) % 3
    m = b.msg()
    h = b.digest(m)
    sl = salt(hl)
    H = mprime_hash(hash, h, sl)
    db = db_of(em_len, hash, sl)

    def crafted(name, em, KK=K):
        em = em.rjust(k, b"\0")
        assert len(em) == k and int.from_bytes(em, "big") < KK.n, name
        b.add(name, m, KK.sign_em(em, E, k), KK.mod_bytes(k), E)

    good = build_em(em_bits, hash, db, H)
    assert good == ref.pss_encode(em_bits, hash, h, sl)
    crafted("crafted_good", good)
    for t in (0xBD, 0x00, 0x01):
        crafted(f"crafted_trailer_{t:02x}", good[:-1] + bytes([t]))
    ps_len = em_len - hl - hl - 2
    for name, pos, v in (("first", 0, 0xFF), ("middle", ps_len // 2, 0x02), ("last", ps_len - 1, 0x01)):
        crafted(f"crafted_ps_{name}", build_em(em_bits, hash, db_of(em_len, hash, sl, (pos, v)), H))
    for sep in (0x00, 0x02):
        crafted(f"crafted_separator_{sep:02x}", build_em(em_bits, hash, db_of(em_len, hash, sl, sep=sep), H))
    crafted("crafted_db_all_zero", build_em(em_bits, hash, bytes(len(db)), H))
    Hx = H[:-1] + bytes([H[-1] ^ 1])
    crafted("crafted_hem_mismatch", build_em(em_bits, hash, db, Hx))
    crafted("crafted_mgf_counter_plus1", build_em(em_bits, hash, db, H, counter=lambda c: (c + 1).to_bytes(4, "big")))
    crafted("crafted_mgf_counter_le", build_em(em_bits, hash, db, H, counter=lambda c: c.to_bytes(4, "little")))
    crafted("crafted_mgf_other_hash", build_em(em_bits, hash, db, H, mask_hash=other))
    for z in (7, 9):
        crafted(f"crafted_mprime_zeros{z}", build_em(em_bits, hash, db, mprime_hash(hash, h, sl, z)))
    crafted("crafted_other_digest", build_em(em_bits, hash, db, mprime_hash(hash, ref.HASHLIB[other](m).digest(), sl)))
    # forbidden top bits of maskedDB[0], set where EM < N still holds (only the lowest, bit emBits, ever can)
    for bits in (8 * k, 8 * k - 1, 8 * k - 4):
        Kb = key(bits)
        eb, el = em_geometry(Kb, k)
        zb = 8 * el - eb
        for bit in range(8 - zb, 8):
            for _ in range(64):
                s2 = salt(hl)
                em = bytearray(build_em(eb, hash, db_of(el, hash, s2), mprime_hash(hash, h, s2)))
                em[0] |= 1 << bit
                if int.from_bytes(em, "big") < Kb.n:
                    crafted(f"crafted_bitlen{bits}_top_bit{bit}", bytes(em), Kb)
                    break
    # emLen = k - 1: a nonzero leading byte over a valid EM'
    K7 = key(8 * k - 7)
    eb7, el7 = em_geometry(K7, k)
    for _ in range(64):
        s2 = salt(hl)
        em = b"\x01" + ref.pss_encode(eb7, hash, h, s2)
        if int.from_bytes(em, "big") < K7.n:
            crafted("crafted_bitlen_k-7_lead_byte", em, K7)
            break
    # cross: a PKCS #1 v1.5 signature of the same digest
    b.add("cross_pkcs1", m, K.sign(k, hash, h), mod, E)
    # badkey: the arithmetic alone would accept each of these (S^e mod N is a valid encoding)
    b.add("badkey_e0", m, sign(m), mod, 0)
    b.add("badkey_e1", m, good.rjust(k, b"\0"), mod, 1)
    b.add("badkey_e2147483648", m, sign(m), mod, 2**31)
    e_big = 2**31 + 1
    while math.gcd(e_big, K.lam) != 1:
        e_big += 2
    b.add("badkey_e_above_max", m, K.sign_em(good.rjust(k, b"\0"), e_big, k), mod, e_big)
    b.add("badkey_e4294967295", m, K.sign_em(good.rjust(k, b"\0"), 2**32 - 1, k), mod, 2**32 - 1)
    b.add("badkey_even_n", m, sign(m), (N ^ 1).to_bytes(k, "big"), E)
    K8 = rsa_cases.key(8 * k - 8)
    b.add("badkey_lead0", m, K8.sign_pss(k, hash, h, salt(hl)), K8.mod_bytes(k), E)
    out = b.done()
    out["salts"] = sorted(used)
    return out
