"""Edge operands of the Ed25519 arithmetic, shared by the CPU simulation and the GPU tests (tests/test_hostsim_ed25519.py,
tests/test_gpu_ed25519.py): a runner takes (op, in_slots) and returns out_slots, 24 little-endian words per slot as in
consensus_b200/csrc/ed25519_debug.cuh."""
import hashlib

import numpy as np

from oracle_ed25519 import corpus, ref

p, L = ref.p, ref.L
WORDS = 24
MUL, SQR, ADD, SUB, CANON, INV, SQRT, DECODE, REDUCE = range(9)


def slots(rows):
    """rows: lists of ints, each placed as 8-limb (or 16-limb for a single wide value) fields."""
    out = np.zeros((len(rows), WORDS), np.uint32)
    for i, vals in enumerate(rows):
        pos = 0
        for v, width in vals:
            for k in range(width):
                out[i, pos + k] = (v >> (32 * k)) & 0xFFFFFFFF
            pos += width
    return out


def val(row, lo, width=8):
    return sum(int(row[lo + k]) << (32 * k) for k in range(width))


def field_operands(rng, n=300):
    """Values across [0, 2^256): edges around 0, p and 2^256, and random ones, including [p, 2^256)."""
    e = [0, 1, 2, 19, 37, 38, 39, p - 1, p, p + 1, p + 18, p + 19, 2 * p - 1, 2 * p, 2**255 - 1, 2**255, 2**256 - 39, 2**256 - 38,
         2**256 - 1, 2**128, 2**224 - 1]
    r = [int.from_bytes(rng.bytes(32), "little") for _ in range(n)]
    r += [p + int(rng.integers(0, 2**62)) for _ in range(20)]
    return e + r


def check_field(run, rng):
    xs = field_operands(rng)
    ys = list(reversed(xs))
    pairs = list(zip(xs, ys)) + [(x, x) for x in xs[:21]] + [(a, b) for a in xs[:21] for b in xs[:21]]
    inp = slots([[(a, 8), (b, 8)] for a, b in pairs])
    for op, f in ((MUL, lambda a, b: a * b), (SQR, lambda a, b: a * a), (ADD, lambda a, b: a + b), (SUB, lambda a, b: a - b),
                  (CANON, lambda a, b: a)):
        out = run(op, inp)
        for (a, b), row in zip(pairs, out):
            got = val(row, 0)
            assert got % p == f(a, b) % p, (op, hex(a), hex(b), hex(got))
            if op == CANON:
                assert got < p
    out = run(INV, inp)
    for (a, _), row in zip(pairs, out):
        want = pow(a % p, p - 2, p)
        assert val(row, 0) == want, (hex(a),)
    return len(pairs)


def check_sqrt_ratio(run, rng):
    rows = []
    for _ in range(200):
        u = int.from_bytes(rng.bytes(32), "little") % 2**256
        v = int.from_bytes(rng.bytes(32), "little") % 2**256
        rows.append((u, v))
    rows += [(0, 1), (1, 1), (p - 1, 1), (p, 1), (4, 1), (ref.SQRT_M1, 1), (2, 1), (9, 4 + p)]
    out = run(SQRT, slots([[(u, 8), (v, 8)] for u, v in rows]))
    squares = 0
    for (u, v), row in zip(rows, out):
        r, was = val(row, 0), int(row[8])
        uu, vv = u % p, v % p
        q = uu * pow(vv, p - 2, p) % p if vv else None
        if vv == 0:
            continue
        is_sq = q == 0 or pow(q, (p - 1) // 2, p) == 1
        assert was == int(is_sq), (hex(u), hex(v))
        assert r < p and r % 2 == 0
        if is_sq:
            squares += 1
            assert r * r % p == q
        else:
            assert r * r % p == q * ref.SQRT_M1 % p
    assert squares > 50


def edge_keys(rng):
    keys = corpus.small_order_encodings() + corpus.big_y_encodings() + corpus.off_curve_encodings(rng, 16)
    keys += [ref.encode(ref.mul(int(rng.integers(1, 2**62)) ** 3, ref.B)) for _ in range(16)]
    keys += [(y | (s << 255)).to_bytes(32, "little") for y in (0, 1, 2, p - 1, 2**255 - 1) for s in (0, 1)]
    return keys


def check_decode(run, rng):
    keys = edge_keys(rng)
    out = run(DECODE, slots([[(int.from_bytes(k, "little"), 8)] for k in keys]))
    accepted = 0
    for k, row in zip(keys, out):
        P = ref.decode(k)
        assert int(row[16]) == int(P is not None), k.hex()
        if P is not None:
            accepted += 1
            assert (val(row, 0), val(row, 8)) == ref.affine(P), k.hex()
    assert accepted and accepted < len(keys)


def reduce_operands():
    vals = [0, 1, L - 1, L, L + 1, 2 * L - 1, 2 * L, 2**512 - 1, 2**256, 2**252, 2**511]
    for k in (2, 3, 8, 2**100 + 7, (2**512 - 1) // L, (2**512 - 1) // L - 1):
        vals += [k * L - 1, k * L, k * L + 1]
    return [v for v in vals if 0 <= v < 2**512]


def check_reduce(run, rng):
    vals = reduce_operands() + [int.from_bytes(rng.bytes(64), "little") for _ in range(200)]
    out = run(REDUCE, slots([[(v, 16)] for v in vals]))
    for v, row in zip(vals, out):
        assert val(row, 0) == v % L, hex(v)


def ragged_batch(rng):
    """Every message length from 0 to 320 — the one / two / three / four block boundaries of SHA-512 with the 64-byte
    prefix are 47 / 48, 175 / 176 and 303 / 304 — and 10 KiB, shuffled, from a misaligned off[0] on, with random R and A."""
    lens = np.array(list(range(321)) + corpus.EDGE_LENGTHS, np.int64)
    rng.shuffle(lens)
    off = (np.concatenate([[0], np.cumsum(lens)]) + int(rng.integers(1, 8))).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    n = lens.size
    sig = rng.integers(0, 256, (n, 64), dtype=np.uint8)
    pub = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    return msgs, off, sig, pub


def expected_digests(msgs, off, sig, pub):
    n = off.size - 1
    out = []
    for i in range(n):
        M = bytes(msgs[int(off[i]): int(off[i + 1])])
        out.append(hashlib.sha512(bytes(sig[i, :32]) + bytes(pub[i]) + M).digest())
    return out
