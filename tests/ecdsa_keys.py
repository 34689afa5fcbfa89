"""Per-key tables of the ECDSA paths and the inputs that reach every part of them, shared by the CPU simulation tests
(test_hostsim_key_tables.py) and the GPU tests (test_gpu_key_tables.py):

  - models of the tables with Python integers: the window tables (KeyTab: registered keys with W = 8, P-384 keys grouped
    in a launch with W = 5) and the P-256 comb (CombTab), laid out as the device stores them;
  - the digit readers of the verification kernels (booth_digit_u2, comb_mask_u2) restated on integers;
  - digit sweeps: signatures whose u2 makes every reachable (window, digit) pair of a window table, or every (block,
    column, mask) triple of the comb, appear in some row;
  - key encodings at the range edges: (x + p, y) and (x, y + p) for valid points with a small coordinate, x = p, y = p,
    (0, 0), all-ones coordinates, P-256 keys with nonzero high bytes in 48-byte slots;
  - keys that agree with a valid key in every word the key-grouping hash once read (x's even words, y's odd words).

Every helper checks with Python integers that its rows reach the edge it names."""
import numpy as np

import oracle
from oracle import ecdsa_ref as ref


def _be(v, L):
    return np.frombuffer(int(v).to_bytes(L, "big"), np.uint8)


def limbs(P, L):
    """an affine point (x, y) in Montgomery form as the device stores it: x*R mod p then y*R mod p, L/4 little-endian
    32-bit limbs each"""
    return np.frombuffer(P[0].to_bytes(L, "little") + P[1].to_bytes(L, "little"), np.uint32)


def _batch_add(c, Ps, Qs):
    """[P_i + Q_i] in affine coordinates with one inversion (Montgomery's trick); no P_i = +-Q_i, none at infinity,
    except P_i == Q_i (a doubling)"""
    p = c.p
    dens = [(2 * P[1] if P == Q else Q[0] - P[0]) % p for P, Q in zip(Ps, Qs)]
    pref, acc = [], 1
    for d in dens:
        pref.append(acc)
        acc = acc * d % p
    assert acc
    inv = pow(acc, -1, p)
    out = [None] * len(Ps)
    for i in range(len(Ps) - 1, -1, -1):
        di = inv * pref[i] % p
        inv = inv * dens[i] % p
        (x1, y1), (x2, y2) = Ps[i], Qs[i]
        lam = (3 * x1 * x1 - 3) * di % p if Ps[i] == Qs[i] else (y2 - y1) * di % p
        x3 = (lam * lam - x1 - x2) % p
        out[i] = (x3, (lam * (x1 - x3) - y1) % p)
    return out


def windows(curve, W):
    """number of W-bit Booth windows of a scalar of the curve's size (Windows<BITS, W>::COUNT)"""
    bits = 8 * ref.CURVES[curve].size
    return (bits + 1 + W - 1) // W


def window_table(curve, W, Q):
    """KeyTab<BITS, W> of Q: entry win * 2^(W-1) + e - 1 = e * 2^(W win) * Q, e = 1..2^(W-1), as limbs (uint32 array of
    NWIN * 2^(W-1) * 2N words).  The windows walk e in step, one batched inversion per step."""
    c = ref.CURVES[curve]
    L, Rm = c.size, (1 << (8 * c.size)) % c.p
    nwin, ent = windows(curve, W), 1 << (W - 1)
    bases = [Q]
    for _ in range(nwin - 1):
        B = bases[-1]
        for _ in range(W):
            B = ref._add(c, B, B)
        bases.append(B)
    cols = [[B] for B in bases]
    cur = list(bases)
    for _ in range(2, ent + 1):
        cur = _batch_add(c, cur, bases)
        for col, P in zip(cols, cur):
            col.append(P)
    mont = lambda P: (P[0] * Rm % c.p, P[1] * Rm % c.p)
    return np.concatenate([limbs(mont(P), L) for col in cols for P in col])


SPACING = 16  # P-256 comb: 16 rows of 16 bits


def comb_slot(b, m):
    """CombTab::slot: chain (b, m >> 4), position = inverse Gray code of m & 15"""
    g = m & 15
    return (b * 16 + (m >> 4)) * 16 + (g ^ (g >> 1) ^ (g >> 2) ^ (g >> 3))


def comb_table(Q, curve=oracle.P256):
    """CombTab<P256> of Q in slot order: T_b[m] = sum of 2^(16 (8b + t)) * Q over the set bits t of m, m = 1..255, at
    comb_slot(b, m); the slot of m = 0 is zeros.  Limbs as window_table."""
    c = ref.CURVES[curve]
    L, Rm = c.size, (1 << (8 * c.size)) % c.p
    bases = [Q]
    for _ in range(15):
        B = bases[-1]
        for _ in range(SPACING):
            B = ref._add(c, B, B)
        bases.append(B)
    out = np.zeros((2 * 16 * 16, L // 2), np.uint32)
    for b in range(2):
        T = {0: None}
        for m in range(1, 256):
            low = m & -m
            T[m] = ref._add(c, T[m ^ low], bases[8 * b + low.bit_length() - 1])
            P = T[m]
            out[comb_slot(b, m)] = limbs((P[0] * Rm % c.p, P[1] * Rm % c.p), L)
    slots = {comb_slot(b, m) for b in range(2) for m in range(256)}
    assert slots == set(range(512))                                        # the slots are a permutation
    return out.reshape(-1)


# ---------------------------------------------------------------- digit readers of the kernels
def booth_digit(u, W, win):
    """booth_digit_u2<C, W>: the bits [W win - 1, W win + W - 1] of u (bit -1 is zero) as a signed digit in
    [-2^(W-1), 2^(W-1)]; sum d_i 2^(W i) = u"""
    pos = W * win - 1
    b = (u << 1) & ((2 << W) - 1) if pos < 0 else (u >> pos) & ((2 << W) - 1)
    sign = b >> W
    d = ((2 << W) - 1) - b if sign else b
    d = (d + 1) >> 1
    return -d if sign else d


def comb_mask(u, b, j):
    """comb_mask_u2<P256>: bit t = bit 16 (8b + t) + j of u"""
    return sum(((u >> (SPACING * (8 * b + t) + j)) & 1) << t for t in range(8))


def reachable_digits(curve, W):
    """{(window, digit)} over every u2 in [1, n): the field of window i (bits [W i - 1, W i + W - 1]) holds pattern f for
    some u < n iff its smallest such u, f at that position and every other bit zero, is < n"""
    n, out = ref.CURVES[curve].n, set()
    for win in range(windows(curve, W)):
        pos = W * win - 1
        for f in range(2 << W):
            if pos < 0 and f & 1:
                continue                                                     # bit -1 is zero
            u = f >> 1 if pos < 0 else f << pos
            if u < n:
                out.add((win, booth_digit(u, W, win)))
    return out


# ---------------------------------------------------------------- scalars and signatures
def _rand(rng, c):
    return int.from_bytes(rng.bytes(c.size + 8), "big") % (c.n - 1) + 1


def window_sweep_u2(curve, W, seed):
    """u2 values in [1, n) whose Booth digits, over all of them, take every reachable (window, digit) pair: row by row,
    window by window from the bottom, each window takes a digit it has not had yet that its carry-in bit allows (the
    top bit of the window below is the bit -1 of its field); rounds alternate the preferred sign of the chosen digit so
    that both carries reach every window.  Asserts the coverage with booth_digit."""
    c = ref.CURVES[curve]
    bits, nwin, half = 8 * c.size, windows(curve, W), 1 << (W - 1)
    rng = np.random.default_rng(seed)
    want = reachable_digits(curve, W)
    seen, out = set(), []
    for rnd in range(8 * half + 16):
        if want <= seen:
            break
        u, cin = 0, 0
        for win in range(nwin):
            free = [k for k in range(W) if W * win + k < bits]
            cands = []
            for v in range(1 << len(free)):
                vv = sum(((v >> i) & 1) << k for i, k in enumerate(free))
                top = (vv >> (W - 1)) & 1
                cands.append((cin + vv - (top << W), vv, top))
            new = [x for x in cands if (win, x[0]) not in seen]
            pool = new or cands
            pref = [x for x in pool if x[2] == (rnd & 1)]
            pick = (pref or pool)[int(rng.integers(len(pref or pool)))]
            u |= pick[1] << (W * win)
            cin = pick[2]
        if not 0 < u < c.n:
            continue
        out.append(u)
        seen |= {(w, booth_digit(u, W, w)) for w in range(nwin)}
    assert seen == want, sorted(want - seen)[:8]
    return out


def comb_sweep_u2(seed):
    """P-256 u2 values in [1, n) whose comb masks, over all of them, take every (block, column, mask) triple, mask =
    1..255: row r gives column j of block b the mask (r + 37 j + 101 b) mod 255 + 1.  Asserts the coverage with
    comb_mask."""
    n = ref.CURVES[oracle.P256].n
    out = []
    for r in range(255):
        u = 0
        for b in range(2):
            for j in range(SPACING):
                m = (r + 37 * j + 101 * b) % 255 + 1
                for t in range(8):
                    u |= ((m >> t) & 1) << (SPACING * (8 * b + t) + j)
        assert 0 < u < n, r
        out.append(u)
    seen = {(b, j, comb_mask(u, b, j)) for u in out for b in range(2) for j in range(SPACING)}
    assert seen == {(b, j, m) for b in range(2) for j in range(SPACING) for m in range(1, 256)}
    return out


def _point(curve, k):
    c = ref.CURVES[curve]
    x, y = oracle.pubkey(curve, (k % c.n).to_bytes(c.size, "big"))
    return int.from_bytes(x, "big"), int.from_bytes(y, "big")


def _lincomb(curve, u1, u2, Q):
    """u1*G + u2*Q (None: infinity), by the C oracle"""
    c = ref.CURVES[curve]
    L = c.size
    if u1 % c.n == 0:
        return ref.scalar_mult(c, u2 % c.n, Q)
    R = oracle.lincomb(curve, (u1 % c.n).to_bytes(L, "big"), (u2 % c.n).to_bytes(L, "big"), Q[0].to_bytes(L, "big"), Q[1].to_bytes(L, "big"))
    return None if R is None else tuple(int.from_bytes(v, "big") for v in R)


def signature_for(curve, Q, u1, u2):
    """(r, s, e) whose verification under the valid key Q computes u1*G + u2*Q (s = r/u2, e = u1*s): it accepts unless
    that point is infinity or has x = 0 mod n (asserted not to happen)"""
    c = ref.CURVES[curve]
    R = _lincomb(curve, u1, u2, Q)
    assert R is not None and R[0] % c.n
    r = R[0] % c.n
    s = r * pow(u2, -1, c.n) % c.n
    return r, s, u1 * s % c.n


def rows_to_batch(curve, rows):
    """[(r, s, qx, qy, e)] -> the batch dict of the verify calls (e: the digest, L bytes)"""
    L = ref.CURVES[curve].size
    f = lambda j: np.stack([_be(row[j], L) for row in rows])
    return {"r": f(0), "s": f(1), "qx": f(2), "qy": f(3), "digest": f(4)}


def sweep_batch(curve, u2s, seed, keys=4):
    """One signature per u2 (random u1, the key one of `keys` random keys; accepts), then every row again with r + 1
    (u1 unchanged, another u2 and another R: rejects).  Returns the batch dict and the verdicts by construction."""
    c = ref.CURVES[curve]
    rng = np.random.default_rng(seed)
    Qs = [_point(curve, _rand(rng, c)) for _ in range(keys)]
    rows = []
    for i, u2 in enumerate(u2s):
        Q = Qs[i % keys]
        r, s, e = signature_for(curve, Q, _rand(rng, c), u2)
        rows.append((r, s, Q[0], Q[1], e))
    rows += [(r + 1, s, qx, qy, e) for r, s, qx, qy, e in rows]
    want = np.array([1] * len(u2s) + [0] * len(u2s), np.uint8)
    return rows_to_batch(curve, rows), want


# ---------------------------------------------------------------- the shuffle tree of k_verify_kt_warp
TREE = (16, 8, 4, 2, 1)


def warp_lane_sums(curve, u1, u2, GW=16):
    """The partial sum of each lane of k_verify_kt_warp before the tree, as (g_L, q_L) with S_L = g_L*G + q_L*Q mod n:
    lane L adds the key windows w = L, L + 32 (8-bit Booth digits of u2, d_w * 2^(8w) * Q) and the G windows w = L, L + 32,
    ... below 8L / GW (GW-bit comb digits of u1, b_w * 2^(GW w) * G).  GW = 16 as libsbv builds the table of G (the CPU
    simulation builds P-384's with GW = 8)."""
    c = ref.CURVES[curve]
    g, q = [0] * 32, [0] * 32
    for w in range(windows(curve, 8)):
        q[w % 32] += booth_digit(u2, 8, w) << (8 * w)
    for w in range(8 * c.size // GW):
        g[w % 32] += ((u1 >> (GW * w)) & ((1 << GW) - 1)) << (GW * w)
    return [v % c.n for v in g], [v % c.n for v in q]


def warp_tree_operands(curve, u1, u2, k, GW=16):
    """{(off, L): (A, B)}: the two partial sums (as multiples of G, for Q = k*G) that lane L adds at level off of the
    tree (L < off: the lanes whose result reaches lane 0); asserts that the last one sums to u1 + u2*k"""
    n = ref.CURVES[curve].n
    g, q = warp_lane_sums(curve, u1, u2, GW)
    cur = [(a + b * k) % n for a, b in zip(g, q)]
    out = {}
    for off in TREE:
        for L in range(off):
            out[(off, L)] = (cur[L], cur[L + off])
        cur = [(cur[L] + cur[L + off]) % n for L in range(off)]
    assert cur[0] == (u1 + u2 * k) % n
    return out


def warp_tree_event(A, B, n):
    return "infinity operand" if A == 0 or B == 0 else "equal" if A == B else "opposite" if (A + B) % n == 0 else None


def warp_tree_cases(curve, seed, GW=16):
    """(u1, u2, k, (off, L, event)) for Q = k*G: for every level off of the tree, lanes L = 0 and off - 1, the two
    partial sums lane L adds are equal (the general addition doubles) or opposite (its sum is infinity, which the
    levels above carry: as the shuffled operand when L >= off / 2, with the mp_is_zero(z2) flag).  The group
    coefficients of both sums are linear in k, so k solves one linear equation mod n.  At off = 1 the opposite case is
    R = infinity (the row must reject).  Asserts with warp_tree_operands that each row meets its event there, and
    only there among the operands that reach lane 0 (besides the infinity it leaves above itself)."""
    c = ref.CURVES[curve]
    n = c.n
    rng = np.random.default_rng(seed)
    cases = []
    for off in TREE:
        for L in sorted({0, off - 1}):
            for event in ("equal", "opposite"):
                while True:
                    u1, u2 = _rand(rng, c), _rand(rng, c)
                    g, q = warp_lane_sums(curve, u1, u2, GW)
                    grp = lambda v, j: sum(v[i] for i in range(32) if i % (2 * off) == j) % n
                    aG, aQ, bG, bQ = grp(g, L), grp(q, L), grp(g, L + off), grp(q, L + off)
                    num, den = ((bG - aG), (aQ - bQ)) if event == "equal" else (-(aG + bG), (aQ + bQ))
                    if den % n == 0:
                        continue
                    k = num * pow(den, -1, n) % n
                    if k == 0:
                        continue
                    ops = warp_tree_operands(curve, u1, u2, k, GW)
                    assert warp_tree_event(*ops[(off, L)], n) == event
                    others = {key: warp_tree_event(*v, n) for key, v in ops.items() if key != (off, L)}
                    if any(e in ("equal", "opposite") for e in others.values()):
                        continue
                    if event == "equal" and any(others.values()):
                        continue
                    cases.append((u1, u2, k, (off, L, event)))
                    break
    return cases


def warp_tree_batch(curve, seed, GW=16):
    """The rows of warp_tree_cases plus two rows with R = u1*G + u2*Q = infinity reached by random scalars (u1 =
    -u2*k): a signature per row (r = R.x mod n, s = r / u2, e = u1 * s; r = 1 when R is infinity, which must reject),
    then every accepting row again with r + 1 (rejects).  Returns the batch dict, the verdicts by construction and the
    events."""
    c = ref.CURVES[curve]
    n = c.n
    rng = np.random.default_rng(seed + 1)
    cases = warp_tree_cases(curve, seed, GW)
    for _ in range(2):
        u2, k = _rand(rng, c), _rand(rng, c)
        cases.append(((n - u2 * k % n) % n, u2, k, (1, 0, "R = infinity")))
    rows, want, events = [], [], []
    for u1, u2, k, ev in cases:
        Q = _point(curve, k)
        R = _lincomb(curve, u1, u2, Q)
        assert (R is None) == (ev[2] in ("opposite", "R = infinity") and ev[0] == 1), ev
        r = 1 if R is None else R[0] % n
        assert r
        s = r * pow(u2, -1, n) % n
        rows.append((r, s, Q[0], Q[1], u1 * s % n))
        want.append(0 if R is None else 1)
        events.append(ev)
    rows += [(r + 1, s, qx, qy, e) for (r, s, qx, qy, e), w in zip(list(rows), want) if w]
    events += [ev + ("r + 1",) for ev, w in zip(list(events), want) if w]
    want += [0] * sum(want)
    return rows_to_batch(curve, rows), np.array(want, np.uint8), events


# ---------------------------------------------------------------- key encodings
def _sqrt(a, p):
    assert p % 4 == 3
    x = pow(a, (p + 1) // 4, p)
    return x if x * x % p == a % p else None


def small_x_point(curve):
    """the valid point with the smallest x >= 1 (y the smaller root)"""
    c = ref.CURVES[curve]
    x = 1
    while True:
        y = _sqrt((x ** 3 - 3 * x + c.b) % c.p, c.p)
        if y is not None:
            return x, min(y, c.p - y)
        x += 1


def _pmulmod(a, b, f, p):
    """a*b mod (f, p) for polynomials as coefficient lists, low degree first, f monic of degree 3"""
    prod = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            prod[i + j] = (prod[i + j] + x * y) % p
    for k in range(len(prod) - 1, 2, -1):                                  # reduce by x^3 = -(f0 + f1 x + f2 x^2)
        t = prod[k]
        if t:
            for i in range(3):
                prod[k - 3 + i] = (prod[k - 3 + i] - t * f[i]) % p
        prod[k] = 0
    return (prod + [0, 0, 0])[:3]


def _pgcd(a, b, p):
    trim = lambda v: v[: max([i + 1 for i, x in enumerate(v) if x % p] or [0])]
    a, b = trim(a), trim(b)
    while b:
        inv = pow(b[-1], -1, p)
        while len(a) >= len(b):
            t = a[-1] * inv % p
            sh = len(a) - len(b)
            a = trim([(x - (t * b[i - sh] if i >= sh else 0)) % p for i, x in enumerate(a)])
            if not a:
                break
        a, b = b, a
    return a


def small_y_point(curve):
    """the valid point with the smallest y >= 1: x a root of x^3 - 3x + b - y^2 mod p, taken from gcd(x^p - x, f) when
    that gcd is linear (exactly one root)"""
    c = ref.CURVES[curve]
    p = c.p
    y = 1
    while True:
        f = [(c.b - y * y) % p, p - 3, 0, 1]                                # x^3 - 3x + (b - y^2)
        r, base, e = [1, 0, 0], [0, 1, 0], p                                # x^p mod f
        while e:
            if e & 1:
                r = _pmulmod(r, base, f, p)
            base = _pmulmod(base, base, f, p)
            e >>= 1
        r[1] = (r[1] - 1) % p
        g = _pgcd(f, r, p)
        if len(g) == 2:
            x = -g[0] * pow(g[1], -1, p) % p
            assert ref.on_curve(c, x, y)
            return x, y
        y += 1


def low_x_point(curve, seed):
    """a valid point whose x + p still fits the curve's L bytes: x drawn at random from the middle half of
    [0, 2^(8L) - p) (2^(8L) - p is about 2^224 for P-256, 2^128 for P-384), then the first x from there with
    x^3 - 3x + b a square (its discrete log is unknown, as for any key a client sends)"""
    c = ref.CURVES[curve]
    bound = (1 << (8 * c.size)) - c.p
    x = int.from_bytes(np.random.default_rng(seed).bytes(c.size), "big") % (bound // 2) + bound // 4
    while True:
        y = _sqrt((x ** 3 - 3 * x + c.b) % c.p, c.p)
        if y is not None:
            assert x + c.p < (1 << (8 * c.size))
            return x, y
        x += 1


def encoding_cases(curve, seed):
    """[(label, qx, qy, Q)]: key encodings that every path must reject, each with the valid point Q whose signature it
    carries (its canonical twin accepts).  qx, qy are integers below 2^(8L)."""
    c = ref.CURVES[curve]
    L, p = c.size, c.p
    top = (1 << (8 * L)) - 1
    X, Y = small_x_point(curve), small_y_point(curve)
    assert X[0] + p <= top and Y[1] + p <= top and X[0] < 2 ** 16 and Y[1] < 2 ** 16
    R = low_x_point(curve, seed)
    out = [("x + p", X[0] + p, X[1], X), ("y + p", Y[0], Y[1] + p, Y), ("x + p of a key with a large x", R[0] + p, R[1], R),
           ("x = p", p, X[1], X), ("y = p", X[0], p, X), ("(0, 0)", 0, 0, X), ("all ones", top, top, X),
           ("x all ones", top, X[1], X), ("y all ones", X[0], top, X)]
    y0 = _sqrt(c.b, p)                                                       # (0, y0) on the curve: (p, y0) encodes it
    if y0 is not None:
        out.append(("x = p, (0, y) valid", p, y0, (0, y0)))
    for label, qx, qy, Q in out:
        assert ref.on_curve(c, *Q) and not ref.on_curve(c, qx, qy), label
        assert (qx % p, qy % p) == Q or label in ("(0, 0)", "all ones", "x all ones", "y all ones", "y = p", "x = p"), label
    return out


def encoding_batch(curve, seed, u1_zero=False):
    """Per encoding case: a signature that accepts under the canonical key (twin row) and the same signature under the
    edge encoding (rejects).  u1_zero: e = 0 (u1 = 0), so that the digest fits 32 bytes on every curve.  Returns the
    batch dict (digest: L bytes, or 32 with u1_zero), the verdicts by construction and the labels."""
    c = ref.CURVES[curve]
    rng = np.random.default_rng(seed)
    rows, want, labels = [], [], []
    for label, qx, qy, Q in encoding_cases(curve, seed):
        r, s, e = signature_for(curve, Q, 0 if u1_zero else _rand(rng, c), _rand(rng, c))
        rows += [(r, s, Q[0], Q[1], e), (r, s, qx, qy, e)]
        want += [1, 0]
        labels += ["canonical twin of " + label, label]
    b = rows_to_batch(curve, rows)
    if u1_zero:
        b["digest"] = np.zeros((len(rows), 32), np.uint8)
    return b, np.array(want, np.uint8), labels


# ---------------------------------------------------------------- keys that collide in the old grouping hash
def colliding_keys(curve, Q, count):
    """`count` distinct keys equal to the valid key Q in x's even 32-bit words and y's odd words (word k = bytes
    [4k, 4k + 4) of the big-endian coordinate: what kg_hash read before it mixed every word) and different in x's odd
    words; none is on the curve.  Returns (qx, qy) as (count, L) byte arrays."""
    c = ref.CURVES[curve]
    L = c.size
    qx = np.tile(_be(Q[0], L), (count, 1))
    qy = np.tile(_be(Q[1], L), (count, 1))
    for i in range(count):
        v = i + 1
        for w in range(1, L // 4, 2):                                       # odd words of x
            qx[i, 4 * w:4 * w + 4] ^= np.frombuffer(((v * (w + 0x9E37)) & 0xFFFFFFFF or 1).to_bytes(4, "big"), np.uint8)
    keys = {(bytes(a), bytes(b)) for a, b in zip(qx, qy)}
    assert len(keys) == count and (bytes(_be(Q[0], L)), bytes(_be(Q[1], L))) not in keys
    for a, b in zip(qx[:64], qy[:64]):
        assert not ref.on_curve(c, int.from_bytes(a.tobytes(), "big"), int.from_bytes(b.tobytes(), "big"))
    wx = lambda a: a.reshape(-1, L // 4, 4)
    assert (wx(qx)[:, 0::2] == wx(np.tile(_be(Q[0], L), (1, 1)))[:, 0::2]).all()
    assert (wx(qy)[:, 1::2] == wx(np.tile(_be(Q[1], L), (1, 1)))[:, 1::2]).all()
    return qx, qy
