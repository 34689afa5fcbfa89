"""Message layouts past 32 bits for the hashing calls, and their references (TEST INFRASTRUCTURE; no engine, no GPU).

The kernels and the staging code carry offsets, lengths and bit counts in 64 bits.  These helpers build what exercises
that: a probe set of lengths at the SHA-256 and SHA-512 block boundaries placed at every start residue mod 4 (and, for the
mixed calls, at every destination residue mod 16 inside the item's family region), each probe with a twin that must
reject; sparse buffers that put the probes past 2^32 without backing the 4 GiB in front of them; and messages long enough
that the bit length needs its high word.

A layout is a list of items in call order: a length, a family tag (the scheme tags of the mixed calls) and a kind.
Spacers are ordinary items inserted only to move the next probe to the residues it wants; like fillers they carry valid
signatures.  Twins copy their probe's bytes with the last byte flipped; an empty twin keeps the empty message and gets a
flipped signature byte instead.
"""
from __future__ import annotations

import hashlib

import numpy as np

P256, P384, ED = 0, 1, 2
FILLER, SPACER, PROBE, TWIN = 0, 1, 2, 3

# message lengths at the SHA-256 block boundaries (the 0x80 byte and the 8-byte length in one block or spilling into the next)
SHA_LENS = (0, 1, 3, 4, 5, 55, 56, 57, 63, 64, 65, 119, 120, 121, 127, 128, 129)
# Ed25519 message lengths at the SHA-512 block boundaries, counting the 64-byte R || A prefix (16-byte length field)
ED_LENS = (0, 1, 46, 47, 48, 49, 63, 64, 65, 175, 176, 177, 191, 192, 193)

FAR = 2**32 + 4096  # where the probes start in a sparse buffer: past 2^32, 16-byte aligned

# SHA-256: 2^29 - 1 bytes has bit length 2^32 - 8 (w[14] = 0, w[15] = 2^32 - 8); 2^29 + 56 bytes has high word 1 and its
# length in a block of its own
HUGE_SHA = (2**29 - 1, 2**29 + 56)
# Ed25519: 64 + M bytes are hashed, so M = 2^29 - 63 gives a bit length of 2^32 + 8
HUGE_ED = 2**29 - 63


class Layout:
    """lens, tag, kind, twin_of (the probe a twin copies, -1 otherwise), as numpy arrays in item order."""

    def __init__(self, lens, tag, kind, twin_of):
        self.lens = np.asarray(lens, np.int64)
        self.tag = np.asarray(tag, np.uint8)
        self.kind = np.asarray(kind, np.uint8)
        self.twin_of = np.asarray(twin_of, np.int64)

    @property
    def n(self):
        return self.lens.size

    @property
    def bytes(self):
        return int(self.lens.sum())

    def offsets(self, start):
        return (np.concatenate([[0], np.cumsum(self.lens)]) + start).astype(np.uint64)


def probe_layout(filler_lens=()):
    """Fillers (P-256) first, then every probe length at start residues 0..3 mod 4, each followed by its twin.  SHA lengths
    go to P-256 and P-384 in turn, Ed25519 lengths to Ed25519; the k-th probe or twin of a family lands at destination
    residue k mod 16 of its family region.  Residues are relative to the first item's offset and to the family's region
    start, so place the layout 16-byte aligned."""
    lens, tag, kind, twin_of = [], [], [], []
    total, fam = 0, [0, 0, 0]
    count = [0, 0, 0]

    def add(ln, f, k, tw=-1):
        nonlocal total
        lens.append(ln); tag.append(f); kind.append(k); twin_of.append(tw)
        total += ln
        fam[f] += ln

    for ln in filler_lens:
        add(int(ln), P256, FILLER)
    want = [(ln, (i + r) % 2, r) for i, ln in enumerate(SHA_LENS) for r in range(4)] + [(ln, ED, r) for ln in ED_LENS for r in range(4)]
    for ln, f, r in want:
        probe = -1
        for k in (PROBE, TWIN):
            x = (count[f] - fam[f]) % 16  # a spacer of the family moves the destination residue
            if x:
                add(x, f, SPACER)
            y = (r - total) % 4           # a spacer of another family moves only the source residue
            if y:
                add(y, (f + 1) % 3, SPACER)
            if k == PROBE:
                probe = len(lens)
            add(ln, f, k, probe if k == TWIN else -1)
            count[f] += 1
    return Layout(lens, tag, kind, twin_of)


def fill(buf, start, lay, seed):
    """Writes the items of lay (fillers excluded: the caller writes them) into buf from offset start; returns the offsets."""
    off = lay.offsets(start)
    rng = np.random.default_rng(seed)
    for i in range(lay.n):
        a, b = int(off[i]), int(off[i + 1])
        if lay.kind[i] == FILLER or a == b:
            continue
        if lay.kind[i] == TWIN:
            p = int(lay.twin_of[i])
            buf[a:b] = buf[int(off[p]):int(off[p + 1])]
            buf[b - 1] ^= 0x01
        else:
            buf[a:b] = rng.integers(0, 256, b - a, dtype=np.uint8)
    return off


def empty_twins(lay):
    """The twins whose message is empty: their signatures get a flipped byte instead."""
    return np.flatnonzero((lay.kind == TWIN) & (lay.lens == 0))


def sparse(nbytes):
    """A zero buffer of nbytes: the pages nobody writes stay unbacked, so 4 GiB in front of the probes cost nothing."""
    return np.zeros(nbytes, np.uint8)


def pattern(nbytes, seed):
    """nbytes of a cheap non-repeating-looking pattern (a random block of odd length tiled), for the huge messages."""
    block = np.random.default_rng(seed).integers(0, 256, 65537, dtype=np.uint8)
    return np.resize(block, nbytes)


def sha256_ref(buf, off):
    return [hashlib.sha256(memoryview(buf[int(off[i]):int(off[i + 1])])).digest() for i in range(off.size - 1)]


def sha512_ref(buf, off, sig, pub):
    """SHA-512(R || A || M) of every item (R: the first 32 bytes of its signature row, A: its key)."""
    out = []
    for i in range(off.size - 1):
        h = hashlib.sha512(bytes(sig[i, :32]) + bytes(pub[i]))
        h.update(memoryview(buf[int(off[i]):int(off[i + 1])]))
        out.append(h.digest())
    return out


def expected_kinds(lay):
    """What every item's verdict must be: probes, spacers and fillers accept, twins reject."""
    return (lay.kind != TWIN).astype(np.uint8)


def sign_items(reg, msgs, off, lay, seed):
    """Signatures of every item under each scheme's key in slot 0 of its registry (tests/mixed_cases.registries with one
    P-256, one P-384 and one Ed25519 key): {P256: (r, s), P384: (r, s), ED: sig}.  A twin carries its probe's signatures,
    an empty twin with a byte flipped in each.  Also returns the SHA-256 digests.  msgs / off may be a multi-GiB blob:
    nothing is copied."""
    import oracle
    import oracle_ed25519 as oe
    rng = np.random.default_rng(seed)
    n = off.size - 1
    dig = oracle.sha256_batch(msgs, off)
    out = {}
    for c, L in ((P256, 32), (P384, 48)):
        slot = int(np.flatnonzero(reg["ecdsa_curve"] == c)[0])
        nonces = rng.integers(0, 256, (n, L), dtype=np.uint8)
        nonces[:, 0] &= 0x7F
        nonces[:, -1] |= 1
        r, s = oracle.sign_batch(c, np.ascontiguousarray(reg["ecdsa_priv"][slot:slot + 1, 48 - L:]), np.zeros(n, np.uint32), dig, nonces)
        out[c] = (r, s)
    out[ED] = oe.sign_batch(reg["ed_seeds"][:1], np.zeros(n, np.uint32), msgs, off)
    twins = np.flatnonzero(lay.kind == TWIN)  # a twin carries its probe's signatures
    for c in (P256, P384):
        out[c][0][twins], out[c][1][twins] = out[c][0][lay.twin_of[twins]], out[c][1][lay.twin_of[twins]]
    out[ED][twins] = out[ED][lay.twin_of[twins]]
    for i in empty_twins(lay):
        out[P256][1][i, 7] ^= 0x10
        out[P384][1][i, 7] ^= 0x10
        out[ED][i, 40] ^= 0x10
    return out, dig


def expected_ok(reg, msgs, off, sigs, dig):
    """The oracles' verdicts of every item under each scheme: {P256, P384, ED: verdict bytes}."""
    import oracle
    import oracle_ed25519 as oe
    n = off.size - 1
    out = {}
    for c, L in ((P256, 32), (P384, 48)):
        xy = reg["ecdsa_xy"][int(np.flatnonzero(reg["ecdsa_curve"] == c)[0])]
        qx, qy = np.tile(xy[48 - L:48], (n, 1)), np.tile(xy[96 - L:], (n, 1))
        out[c] = oracle.verify_batch(c, sigs[c][0], sigs[c][1], qx, qy, dig)
    out[ED] = oe.verify_batch(msgs, off, sigs[ED], np.tile(reg["ed_pub"][0], (n, 1)))
    return out
