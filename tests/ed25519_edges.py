"""Crafted Ed25519 inputs for the edges of k_ed_verify (consensus_b200/csrc/ed25519_verify.cuh), shared by the CPU
simulation and the GPU tests (tests/test_hostsim_ed25519_edges.py, tests/test_gpu_ed25519_edges.py).

A Python model of the kernel's schedule comes with them, so that each set asserts that the case it is named for really
occurs instead of hoping a random input reaches it:
- ed_digit4 / ed_digit8, the signed-digit recodings exactly as the kernel computes them;
- the k loop: windows 63 down to 0, four doublings then one addition of the digit's multiple of A (d > 0 subtracts dA, so
  the accumulator is [h](-A));
- the B loop: windows 0 to 31, one affine addition of +-entry from the table of B, which the model builds on its own by
  walking each column with affine additions of 256^w B.

Each set is a `Rows` of (A, M, R || S, k or None, expected verdict, tag).  Rows with k = None go through
sbv_ed25519_verify_batch (k = SHA-512(R || A || M) mod L); rows with a k go through the test hook that runs k_ed_verify
with that k.  The expected verdict is the one the construction implies; the tests compare it with the device, the CPU
simulation, OpenSSL (production rows) and oracle_ed25519.ref on a sample.
"""
import functools
import hashlib

import numpy as np

from oracle_ed25519 import corpus, ref

p, L, d = ref.p, ref.L, ref.d
O = ref.IDENTITY
ENC_O = corpus._enc_y(1)


# ---- the kernel's recodings ----
def digit4(k, win):
    """ed_digit4: Booth digit `win` of k in [-8, 8] (nibble `win` as a signed value plus the top bit of the one below)."""
    w = (k >> (4 * win)) & 15
    prev = (k >> (4 * win - 1)) & 1 if win else 0
    return (w & 7) - (w & 8) + prev


def digit8(s, win):
    """ed_digit8: Booth digit `win` of the 32-byte little-endian scalar s in [-128, 128]."""
    v = s[win]
    prev = s[win - 1] >> 7 if win else 0
    return (v & 127) - (v & 128) + prev


def digits8(S):
    b = S.to_bytes(32, "little")
    return [digit8(b, w) for w in range(32)]


def k_loop(k):
    """The k loop on scalars: returns (h, additions, additions to O) with the accumulator [h](-A) after window 0.
    An addition is (window, digit); `to_O` lists the windows whose addition meets an accumulator that is still O."""
    h, adds, to_O = 0, [], []
    for win in range(63, -1, -1):
        h *= 16 if win != 63 else 1
        dg = digit4(k, win)
        if dg:
            adds.append((win, dg))
            if h == 0:
                to_O.append(win)
            h += dg
    return h, adds, to_O


# ---- points (extended tuples of oracle_ed25519.ref) ----
def same(P, Q):
    return (P[0] * Q[2] - Q[0] * P[2]) % p == 0 and (P[1] * Q[2] - Q[1] * P[2]) % p == 0


def is_O(P):
    return P[0] % p == 0 and (P[1] - P[2]) % p == 0


def encode_many(points):
    """ref.encode of every point with one inversion (Montgomery's trick)."""
    pref, acc = [], 1
    for P in points:
        pref.append(acc)
        acc = acc * P[2] % p
    inv = pow(acc, p - 2, p)
    out = [None] * len(points)
    for i in range(len(points) - 1, -1, -1):
        X, Y, Z, _ = points[i]
        zi = inv * pref[i] % p
        inv = inv * Z % p
        x, y = X * zi % p, Y * zi % p
        out[i] = (y | ((x & 1) << 255)).to_bytes(32, "little")
    return out


def _aff_add(P1, P2):
    (x1, y1), (x2, y2) = P1, P2
    t = d * x1 * x2 * y1 * y2 % p
    return (x1 * y2 + y1 * x2) * pow(1 + t, p - 2, p) % p, (y1 * y2 + x1 * x2) * pow(1 - t, p - 2, p) % p


@functools.lru_cache(None)
def btab():
    """The table of B: btab()[w][j - 1] = affine j * 256^w * B, each column walked by affine additions of its base."""
    base, tab = ref.affine(ref.B), []
    for _ in range(32):
        col, cur = [], base
        for _ in range(128):
            col.append(cur)
            cur = _aff_add(cur, base)
        tab.append(col)
        base = _aff_add(col[127], col[127])
    return tab


@functools.lru_cache(None)
def btab_words():
    """The table as k_ed_btab_init lays it out: (32, 128, 24) words, y + x, y - x, 2dxy, canonical, little-endian."""
    blob = b"".join(v.to_bytes(32, "little") for col in btab() for x, y in col
                    for v in ((y + x) % p, (y - x) % p, 2 * d * x * y % p))
    return np.frombuffer(blob, "<u4").reshape(32, 128, 24)


EQ, NEG, FROM_O = "P=Q", "P=-Q", "from O"


def b_loop(S, acc=O, events=None):
    """The B loop: acc + [S]B added window by window from the table.  events (a list) receives (window, EQ) when the
    accumulator equals the entry it is about to add, (window, NEG) when it equals its negative (the sum is O) and
    (window, FROM_O) when the accumulator is O."""
    s, tab = S.to_bytes(32, "little"), btab()
    for w in range(32):
        dg = digit8(s, w)
        if dg == 0:
            continue
        x, y = tab[w][abs(dg) - 1]
        Q = ref.point_from_affine(x if dg > 0 else (p - x) % p, y)
        if events is not None:
            if is_O(acc):
                events.append((w, FROM_O))
            elif same(acc, Q):
                events.append((w, EQ))
            elif same(acc, ref.neg(Q)):
                events.append((w, NEG))
        acc = ref.add(acc, Q)
    return acc


def bmul(c):
    return b_loop(c % L)


class KeyModel:
    """[k]A for any k < 2^256 from the unsigned nibbles of k (16^w A times 1..15): an order of operations unlike the
    kernel's signed windows."""

    def __init__(self, A):
        self.P = ref.decode(A)
        self.tab = None
        self.small = None
        if self.P is not None and order(A) is not None:  # order divides 8: [k]A = [k mod 8]A
            self.small = [O]
            for _ in range(7):
                self.small.append(ref.add(self.small[-1], self.P))

    def mul(self, k):
        if self.P is None:
            raise ValueError("A does not decode")
        if self.small is not None:
            return self.small[k % 8]
        if self.tab is None:
            self.tab, base = [], self.P
            for _ in range(64):
                row = [O, base]
                for _ in range(14):
                    row.append(ref.add(row[-1], base))
                self.tab.append(row)
                base = ref.add(row[8], row[8])
        acc = O
        for w in range(64):
            v = (k >> (4 * w)) & 15
            if v:
                acc = ref.add(acc, self.tab[w][v])
        return acc


@functools.lru_cache(None)
def key_model(A):
    return KeyModel(A)


def order(A):
    """Order of the decoded point A when it divides 8, else None."""
    P = ref.decode(A)
    Q = P
    for e in (1, 2, 4, 8):
        if is_O(Q):
            return e
        Q = ref.add(Q, Q)
    return None


def challenge(R, A, M):
    return int.from_bytes(hashlib.sha512(R + A + M).digest(), "little") % L


def noncanonical(x, y):
    """The encodings other than the canonical one that decode to (x, y): y + p when y < 19, sign bit set when x = 0."""
    out = []
    for yy in (y, y + p):
        for s in sorted({x & 1, 1}):
            if yy < 2**255 and (yy, s) != (y, x & 1) and (s == x & 1 or x == 0):
                out.append(corpus._enc_y(yy, s))
    return out


class Rows:
    def __init__(self):
        self.A, self.M, self.sig, self.k, self.want, self.tag = [], [], [], [], [], []

    def add(self, A, M, sig, want, tag, k=None):
        self.A.append(A)
        self.M.append(M)
        self.sig.append(sig)
        self.k.append(k)
        self.want.append(bool(want))
        self.tag.append(tag)

    def __len__(self):
        return len(self.A)

    def extend(self, other):
        for f in ("A", "M", "sig", "k", "want", "tag"):
            getattr(self, f).extend(getattr(other, f))
        return self

    def arrays(self, first=3):
        """msgs (from off[0] = first, so that odd lengths misalign what follows; padded by 16), off, sig, pub, k, want."""
        lens = np.array([len(m) for m in self.M], np.int64)
        off = (np.concatenate([[0], np.cumsum(lens)]) + first).astype(np.uint64)
        msgs = np.frombuffer(bytes(first) + b"".join(self.M) + bytes(16), np.uint8).copy()
        sig = np.frombuffer(b"".join(self.sig), np.uint8).reshape(-1, 64).copy()
        pub = np.frombuffer(b"".join(self.A), np.uint8).reshape(-1, 32).copy()
        k = None
        if self.k and self.k[0] is not None:
            k = np.frombuffer(b"".join(kk.to_bytes(32, "little") for kk in self.k), "<u4").reshape(-1, 8).copy()
        return {"msgs": msgs, "off": off, "sig": sig, "pub": pub, "k": k, "want": np.array(self.want, np.uint8)}


def _sig(R, S):
    return R + S.to_bytes(32, "little")


def _flip(R, bit):
    b = bytearray(R)
    b[bit // 8] ^= 1 << (bit % 8)
    return bytes(b)


def _grind(A, R, M0, pred):
    """The first M = M0 || i (i = 0, 1, ...) whose k = SHA-512(R || A || M) mod L satisfies pred."""
    i = 0
    while True:
        M = M0 + i.to_bytes(4, "little")
        k = challenge(R, A, M)
        if pred(k):
            return M, k
        i += 1


def _variants(rows, A, M, R, S, Rp, k, tag, bit):
    """The rejecting variants of an accepting row with R' = Rp: R with bit `bit` flipped (its verdict recomputed, as a new
    R changes k on the production path) and S + 1 where that stays below L."""
    R2 = _flip(R, bit)
    if k is None:
        k2 = challenge(R2, A, M)
        Rp2 = ref.add(ref.add(Rp, key_model(A).mul(challenge(R, A, M))), ref.neg(key_model(A).mul(k2)))
        rows.add(A, M, _sig(R2, S), ref.encode(Rp2) == R2, tag + "/R bit %d" % bit)
    else:
        rows.add(A, M, _sig(R2, S), False, tag + "/R bit %d" % bit, k)
    if S + 1 < L:
        rows.add(A, M, _sig(R, S + 1), False, tag + "/S+1", k)


# ---- the S boundary (production path) ----
IDENTITY_KEYS = [corpus._enc_y(1), corpus._enc_y(1 + p), corpus._enc_y(1, 1)]  # canonical, y = 1 + p, "-0"


@functools.lru_cache(None)
def s_boundary():
    rows, rng = Rows(), np.random.default_rng(101)
    for A in IDENTITY_KEYS:
        for S in (0, 1, L - 2, L - 1):
            Rp = bmul(S)
            R = ref.encode(Rp)
            rows.add(A, b"boundary", _sig(R, S), True, "S=%d" % S if S < 2 else "S=L-%d" % (L - S))
            _variants(rows, A, b"boundary", R, S, Rp, None, "S boundary", 255 if S < 2 else 0)
        s = int(rng.integers(1, 2**62)) ** 5 % L
        mmax = (2**256 - 1 - s) // L
        for S in [L, L + 1, 2 * L - 1, 2**256 - 1] + [s + m * L for m in range(1, mmax + 1)]:
            rows.add(A, b"boundary", _sig(ref.encode(bmul(S % L)), S), False, "S>=L")
    assert mmax == (2**256 - 1) // L - (s > (2**256 - 1) % L) and mmax >= 15
    ss = [int.from_bytes(sg[32:], "little") for sg, w in zip(rows.sig, rows.want) if w]
    assert max(ss) == L - 1 and min(ss) == 0
    bad = [int.from_bytes(sg[32:], "little") for sg, t in zip(rows.sig, rows.tag) if t == "S>=L"]
    assert min(bad) == L and max(bad) == 2**256 - 1
    return rows


# ---- every B-loop digit (production path) ----
def reachable8():
    """Every (window, nonzero digit) that ed_digit8 yields for some S < L: the least S with byte v at the window and
    bit 8w - 1 = prev is v * 256^w + prev * 2^(8w - 1)."""
    out = {}
    for w in range(32):
        for v in range(256):
            for prev in ((0, 1) if w else (0,)):
                S = v * 256**w + (prev << (8 * w - 1) if prev else 0)
                dg = (v & 127) - (v & 128) + prev
                if S < L and dg and (w, dg) not in out:
                    out[(w, dg)] = S
    return out


def _order_keys():
    """The small-order encodings of order 2, 4 or 8 (not the identity's)."""
    return [A for A in corpus.small_order_encodings() if order(A) in (2, 4, 8)]


@functools.lru_cache(None)
def digit_sweep():
    """One S per reachable (window, digit), plus all bytes 0x80, all bytes 0x7f and 2^248 - 1 (31 bytes each: S < L),
    R = enc([S]B) from the table model.  A = identity for most rows; every 8th row takes a key of order 2, 4 or 8 with M
    ground until [k]A = O, so that R' = [S]B still.  Each accepting row has its rejecting variants."""
    reach = reachable8()
    Ss = list(reach.values()) + [sum(b * 256**i for i in range(31)) for b in (0x80, 0x7F)] + [2**248 - 1]
    Rps = [bmul(S) for S in Ss]
    Rs = encode_many(Rps)
    small = _order_keys()
    rows, seen = Rows(), set()
    for i, (S, Rp, R) in enumerate(zip(Ss, Rps, Rs)):
        seen.update((w, dg) for w, dg in enumerate(digits8(S)) if dg)
        M0 = bytes([i % 251]) * (i % 200)
        if i % 8 == 7:
            A = small[(i // 8) % len(small)]
            e = order(A)
            M, _ = _grind(A, R, M0, lambda k: k % e == 0)
        else:
            A, M = IDENTITY_KEYS[i % 3], M0
        rows.add(A, M, _sig(R, S), True, "digit sweep")
        _variants(rows, A, M, R, S, Rp, None, "digit sweep", (i * 97 + 255) % 256)
    assert set(reach) <= seen and len(reach) == 31 * 256 - 1 + 16, len(reach)
    assert {(0, -128), (31, 16), (31, 1), (30, 128), (1, 128)} <= seen
    assert digits8(Ss[-3]) == [-128] + [-127] * 30 + [1] and digits8(Ss[-2]) == [127] * 31 + [0]
    return rows


# ---- small-order R' (production path) ----
@functools.lru_cache(None)
def small_order_r():
    """S = 0 and A of order 2, 4 or 8 in every encoding: R' = -[k]A, M ground until R' is the chosen target of <A>.  The
    canonical R of the target accepts; each of its non-canonical encodings rejects.  Then R' = O under a full-order key
    ([a]B, S = k a) and under mixed-order keys ([a]B + T, S = k a: accepts iff [k]T = O)."""
    rows, rng = Rows(), np.random.default_rng(102)
    hit_canon, hit_non = set(), set()
    for n, A in enumerate(_order_keys()):
        P, e = ref.decode(A), order(A)
        mults = [O]
        for _ in range(e - 1):
            mults.append(ref.add(mults[-1], P))
        for j in range(e):
            x, y = ref.affine(mults[j])
            canon = ref.encode(mults[j])
            for R, want in [(canon, True)] + [(R, False) for R in noncanonical(x, y)]:
                M, k = _grind(A, R, b"small order %d %d " % (n, j), lambda k: (-k) % e == j)
                assert same(ref.neg(key_model(A).mul(k)), mults[j])
                rows.add(A, M, _sig(R, 0), want, "R'=small order")
                (hit_canon if want else hit_non).add(R)
                if want:
                    _variants(rows, A, M, R, 0, mults[j], None, "R'=small order", 255 - 8 * j)
    every = {ref.encode(ref.point_from_affine(*pt)) for pt in ref.small_order_points()}
    every_non = {R for pt in ref.small_order_points() for R in noncanonical(*pt)}
    assert hit_canon == every and hit_non == every_non and len(every_non) == 6
    # R' = O under a full-order key
    a = int(rng.integers(1, 2**62)) ** 5 % L
    A = ref.encode(bmul(a))
    for R in [ENC_O] + noncanonical(0, 1):
        k = challenge(R, A, b"full")
        S = k * a % L
        rows.add(A, b"full", _sig(R, S), R == ENC_O, "R'=O full order")
        if R == ENC_O:
            rows.add(A, b"full", _sig(R, (S + 1) % L), False, "R'=O full order/S+1")
    # mixed order: [a]B + T for T of order 2, 4 and 8; accept iff [k]T = O
    seen = set()
    for T in [pt for pt in ref.small_order_points() if pt != (0, 1)]:
        Tp = ref.point_from_affine(*T)
        e = order(ref.encode(Tp))
        a = int(rng.integers(1, 2**62)) ** 5 % L
        A = ref.encode(ref.add(bmul(a), Tp))
        for want in (True, False):
            M, k = _grind(A, ENC_O, b"mixed %d " % e, lambda k: (k % e == 0) == want)
            rows.add(A, M, _sig(ENC_O, k * a % L), want, "R'=O mixed order")
            seen.add((e, want))
    assert seen == {(e, w) for e in (2, 4, 8) for w in (True, False)}
    return rows


# ---- crafted k (test hook) ----
def crafted_ks():
    ks = [0, 1, 2, L - 2, L - 1, sum(8 << (4 * i) for i in range(63)), sum(7 << (4 * i) for i in range(63))]
    ks += [v << (4 * w) for w in range(63) for v in range(1, 16)]
    ks += [0x78 << (4 * (w - 1)) for w in range(1, 63)]  # digit +8 at window w (nibble 7 above a nibble 8)
    return ks


def reachable4():
    """Every (window, nonzero digit) that ed_digit4 yields for some k < L (least k: nibble * 16^w + prev * 2^(4w-1))."""
    out = set()
    for w in range(64):
        for v in range(16):
            for prev in ((0, 1) if w else (0,)):
                if v * 16**w + (prev << (4 * w - 1) if prev else 0) < L:
                    dg = (v & 7) - (v & 8) + prev
                    if dg:
                        out.add((w, dg))
    return out


def crafted_k_keys():
    rng = np.random.default_rng(103)
    a = [int(rng.integers(1, 2**62)) ** 5 % L for _ in range(2)]
    full = [ref.encode(bmul(x)) for x in a]
    T8 = ref.point_from_affine(*[pt for pt in ref.small_order_points() if pt[0] and pt[1]][0])
    T4 = ref.point_from_affine(ref.SQRT_M1, 0)
    mixed = [ref.encode(ref.add(bmul(a[0]), T8)), ref.encode(ref.add(bmul(a[1]), T4))]
    big_y = [A for A in corpus.big_y_encodings() if ref.decode(A) is not None]
    minus0 = [corpus._enc_y(1, 1), corpus._enc_y(p - 1, 1), corpus._enc_y(1 + p, 1)]
    keys = []
    for A in full + corpus.small_order_encodings() + mixed + big_y + minus0:
        if A not in keys:
            keys.append(A)
    return keys


@functools.lru_cache(None)
def crafted_k():
    """Every crafted k with every key: R = enc([S]B - [k]A), S from a pool of random scalars.  Every fourth accepting row
    is followed by a rejecting variant, R with a bit flipped and S + 1 in turn."""
    rng = np.random.default_rng(104)
    ks, keys = crafted_ks(), crafted_k_keys()
    pool = [int.from_bytes(rng.bytes(32), "little") % L for _ in range(61)]
    pool_pts = [bmul(S) for S in pool]
    seen = set()
    for k in ks:
        h, adds, to_O = k_loop(k)
        assert h == k and k < L
        seen.update(adds)
    assert seen == reachable4()
    assert k_loop(0)[1] == [] and k_loop(1)[1] == [(0, 1)] and k_loop(1)[2] == [0]
    assert [dg for _, dg in k_loop(ks[5])[1]] == [1] + [-7] * 62 + [-8] and [dg for _, dg in k_loop(ks[6])[1]] == [7] * 63
    items = []
    for A in keys:
        km = key_model(A)
        for k in ks:
            j = len(items) % len(pool)
            items.append((A, k, pool[j], ref.add(pool_pts[j], ref.neg(km.mul(k)))))
    Rs = encode_many([it[3] for it in items])
    rows = Rows()
    for i, ((A, k, S, _), R) in enumerate(zip(items, Rs)):
        rows.add(A, b"", _sig(R, S), True, "crafted k", k)
        if i % 4:
            continue
        if i % 8 or S + 1 >= L:
            rows.add(A, b"", _sig(_flip(R, (i * 89 + 255) % 256), S), False, "crafted k/R flip", k)
        else:
            rows.add(A, b"", _sig(R, S + 1), False, "crafted k/S+1", k)
    return rows


# ---- B-loop collisions (test hook) ----
def _with_digit(S, w, dg):
    """S with ed_digit8 window w = dg: byte w set for the carry-in bit below it, which is flipped when dg needs it."""
    b = bytearray(S.to_bytes(32, "little"))
    prev = b[w - 1] >> 7 if w else 0
    if not -128 <= dg - prev <= 127:
        b[w - 1] ^= 0x80
        prev ^= 1
    b[w] = (dg - prev) & 0xFF
    return int.from_bytes(b, "little")


@functools.lru_cache(None)
def collisions():
    """A = [a]B with a solved so that the accumulator of the B loop, just before the addition of window w, is +entry
    (the affine addition doubles), -entry (the sum is O and later additions start from O) or -entry with every digit
    above w zero (R' = O at the end, R = 01 00..00)."""
    rng = np.random.default_rng(105)
    rows, hits = Rows(), {EQ: set(), NEG: set(), "final O": set(), "restart": set()}
    for w in range(32):
        for kind in (EQ, NEG, "final O"):
            if w == 31:
                dgs = [1, 15, int(rng.integers(2, 15))]
            elif kind == "final O":
                dgs = [1, 127 if w == 0 else 128, int(rng.integers(2, 127))]
            else:
                dgs = [1, -128, 127 if w == 0 else 128, int(rng.integers(-127, 127)) or 5]
            for dg in dgs:
                S = int.from_bytes(rng.bytes(31), "little")
                S = _with_digit(S, w, dg)
                if kind == "final O":
                    S %= 256 ** (w + 1)
                ds = digits8(S)
                assert S < L and ds[w] == dg
                low = sum(x * 256**i for i, x in enumerate(ds[:w]))
                k = int.from_bytes(rng.bytes(32), "little") % L
                eps = 1 if kind == EQ else -1
                a = (low - eps * dg * 256**w) * pow(k, -1, L) % L
                A = ref.encode(bmul(a))
                ev = []
                Rp = b_loop(S, bmul(-k * a), ev)
                assert (w, EQ if kind == EQ else NEG) in ev, (w, kind, dg, ev)
                hits[EQ if kind == EQ else NEG].add(w)
                if kind == NEG and any(ds[w + 1:]):
                    nxt = min(i for i in range(w + 1, 32) if ds[i])
                    assert (nxt, FROM_O) in ev
                    hits["restart"].add(w)
                if kind == "final O":
                    assert is_O(Rp) and not any(ds[w + 1:])
                    hits["final O"].add(w)
                R = ref.encode(Rp)
                tag = "collision %s w=%d" % (kind, w)
                rows.add(A, b"", _sig(R, S), True, tag, k)
                _variants(rows, A, b"", R, S, Rp, k, tag, (w * 8 + 255) % 256)
    for kind, ws in hits.items():  # "restart": O partway, the next addition starts from O (windows 0 to 30)
        assert ({0, 30} if kind == "restart" else {0, 31}) <= ws and len(ws) >= 31, (kind, sorted(ws))
    return rows


def ref_verdict(A, M, sig, k=None):
    """oracle_ed25519.ref.verify, with k given instead of hashed when k is not None."""
    if k is None:
        return ref.verify(A, M, sig)
    S = int.from_bytes(sig[32:], "little")
    P = ref.decode(A)
    if S >= L or P is None:
        return False
    return ref.encode(ref.add(ref.mul(S, ref.B), ref.neg(ref.mul(k, P)))) == sig[:32]


def ref_sample(rows, n, seed):
    """Indices of a seeded sample of n rows whose ref verdict must equal the expected one."""
    rng = np.random.default_rng(seed)
    idx = rng.choice(len(rows), min(n, len(rows)), replace=False)
    return sorted(int(i) for i in idx)


def mixed_length_batch(n=4096, seed=106):
    """n items signed by four keys, messages of 0 to 300 bytes with six of 70 KB and 1 MiB among them (block counts
    past the 1023 at which the length sort clamps its bin), a third of the signatures corrupted (two long ones too)."""
    from oracle_ed25519 import pubkey, sign_batch
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 301, n)
    long_idx = sorted(int(i) for i in rng.choice(n, 6, replace=False))
    for j, i in enumerate(long_idx):
        lens[i] = 70000 if j % 2 else 1 << 20
    off = (np.concatenate([[0], np.cumsum(lens)]) + 5).astype(np.uint64)
    msgs = rng.integers(0, 256, int(off[-1]) + 16, dtype=np.uint8)
    seeds = rng.integers(0, 256, (4, 32), dtype=np.uint8)
    pubs = np.frombuffer(b"".join(pubkey(bytes(s)) for s in seeds), np.uint8).reshape(4, 32)
    kidx = (np.arange(n) % 4).astype(np.uint32)
    sig = sign_batch(seeds, kidx, msgs, off)
    bad = rng.random(n) < 0.3
    bad[long_idx[:2]], bad[long_idx[2:]] = True, False
    sig[bad, 40] ^= np.uint8(1)
    return {"msgs": msgs, "off": off, "sig": sig, "pub": pubs[kidx].copy(), "long": long_idx}


def _subset(rows, idx):
    out = Rows()
    for i in idx:
        out.add(rows.A[i], rows.M[i], rows.sig[i], rows.want[i], rows.tag[i], rows.k[i])
    return out


def _mismatch(rows, got, want):
    bad = np.flatnonzero(np.asarray(got) != np.asarray(want))
    return [(int(i), rows.tag[i], int(want[i])) for i in bad[:10]], bad.size


def check(rows, verify=None, verify_k=None, sort_pass=False, ref_n=150, seed=0):
    """Runs a set and compares every verdict with the one the construction implies.
    verify(arrays) -> verdicts runs the production path, in calls of at most 2047 items (no length sort) and, with
    sort_pass, once more with the rows repeated past 2048 items (length sort on); those rows are also checked against
    OpenSSL.  verify_k(arrays) runs the hook with the rows' k.  A seeded sample of ref_n rows is checked against
    oracle_ed25519.ref."""
    want = np.array(rows.want, np.uint8)
    n = len(rows)
    if verify_k is not None:
        got = verify_k(rows.arrays())
    else:
        got = np.zeros(n, np.uint8)
        for lo in range(0, n, 2047):
            got[lo: lo + 2047] = verify(_subset(rows, range(lo, min(n, lo + 2047))).arrays())
        a = rows.arrays()
        from oracle_ed25519 import verify_batch
        ossl = verify_batch(a["msgs"], a["off"], a["sig"], a["pub"])
        assert np.array_equal(ossl, want), _mismatch(rows, ossl, want)
        if sort_pass:
            reps = 2049 // n + 1
            big = _subset(rows, list(range(n)) * reps)
            got2 = verify(big.arrays())
            assert np.array_equal(got2, np.tile(want, reps)), _mismatch(big, got2, np.tile(want, reps))
    assert np.array_equal(got, want), _mismatch(rows, got, want)
    for i in ref_sample(rows, ref_n, seed):
        assert ref_verdict(rows.A[i], rows.M[i], rows.sig[i], rows.k[i]) == rows.want[i], (i, rows.tag[i])
    return int(want.sum()), n
