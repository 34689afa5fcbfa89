"""The Ed25519 field, scalar and point arithmetic of consensus_b200/csrc/ed25519.cuh at its carry boundaries, shared by the
CPU simulation (tests/test_hostsim_ed25519_arith.py) and the GPU tests (tests/test_gpu_ed25519_arith.py).

Each model below restates a device routine limb for limb and returns its value together with the branch it took: the
carries of fe_fold, the carry and wrap of fe_add / fe_sub, fe_canon's bit 255 and its t >= p select, and the quotient
error of sc_reduce512's Barrett reduction.  Every operand construction asserts with the model that it reaches the branch it
was built for, so the boundaries are reached by construction rather than by the luck of a seed.  A runner takes (op, slots)
and returns the output slots: ED_DEBUG_WORDS-word slots for the field and scalar ops (ed25519_cases), ED_POINT_WORDS-word
slots for the point ops (ed25519_debug.cuh)."""
from collections import Counter
from fractions import Fraction

import numpy as np

from oracle_ed25519 import ref

import ed25519_cases as cases

p, L, d = ref.p, ref.L, ref.d
M256 = 1 << 256
MASK255 = (1 << 255) - 1
D2 = 2 * d % p

# point ops of ed25519_debug.cuh (ed_point_dispatch): low byte the operation, flags above it
PT_DOUBLE, PT_ADD, PT_CACHED, PT_ENCODE = range(4)
PT_NO_T, PT_AFFINE, PT_NEG = 0x100, 0x200, 0x400
PT_WORDS = 64


# ---- models of the field routines (values in [0, 2^256), as the limbs hold them) ----
def fold(T):
    """fe_fold of a 512-bit T: (r, c1, c2).  c1 in [0, 38] is the carry limb of T_lo + 38 T_hi, c2 whether adding
    38 c1 carries out of 2^256 again (then the result is the low half plus 38)."""
    assert 0 <= T < M256 * M256
    s = (T % M256) + 38 * (T >> 256)
    c1, r1 = s >> 256, s % M256
    s2 = r1 + 38 * c1
    c2, r = s2 >> 256, s2 % M256
    r += 38 * c2
    assert r < M256 and (c2 == 0 or r < 38 * 38)
    return r, c1, c2


def fe_mul(a, b):
    return fold(a * b)[0]


def fe_sqr(a):
    return fold(a * a)[0]


def add_model(a, b):
    """fe_add: (r, carry, wrap)."""
    s = a + b
    c, r = s >> 256, s % M256
    s2 = r + 38 * c
    w, r = s2 >> 256, s2 % M256
    return r + 38 * w, c, w


def sub_model(a, b):
    """fe_sub: (r, borrow, wrap)."""
    s = a - b
    bw, r = int(s < 0), s % M256
    s2 = r - 38 * bw
    w, r = int(s2 < 0), s2 % M256
    return r - 38 * w, bw, w


def fe_add(a, b):
    return add_model(a, b)[0]


def fe_sub(a, b):
    return sub_model(a, b)[0]


def canon_model(a):
    """fe_canon: (r, bit 255, t >= p) with t = (a mod 2^255) + 19 * bit 255."""
    bit = a >> 255
    t = (a & MASK255) + 19 * bit
    ge = int(t + 19 >= 1 << 255)
    r = (t + 19) & MASK255 if ge else t
    assert r == a % p
    return r, bit, ge


MU = (1 << 512) // L


def reduce_model(x):
    """sc_reduce512: (x mod L, quotient error q - q3, final subtractions taken).  q3 = floor(floor(x / b^7) mu / b^9),
    t = (x - q3 L) mod b^9, then t -= L while t >= L (the device takes at most two passes)."""
    assert 0 <= x < 1 << 512
    q3 = ((x >> 224) * MU) >> 288
    t = (x - q3 * L) % (1 << 288)
    subs = 0
    while t >= L:
        t -= L
        subs += 1
    assert subs <= 2 and t == x % L
    return t, x // L - q3, subs


def barrett_bound():
    """An exact bound B with x / L - q3 < B for every x < 2^512.  With x = (q1 + f1) 2^224 (q1 < 2^288, 0 <= f1 < 1) and
    mu = 2^512 / L - f2 (0 <= f2 < 1): x / L - q3 = (q1 mu / 2^288 - q3) + (q1 f2 + f1 (mu + f2)) / 2^288, where the first
    term is a fractional part, at most 1 - 2^-288, and the second is below ((2^288 - 1) f2 + 2^512 / L) / 2^288.  q3 <= x / L
    since mu <= 2^512 / L, so q - q3 is an integer in [0, B) and t = x - q3 L < B L."""
    f2 = Fraction(1 << 512, L) - MU
    assert 0 <= f2 < 1
    return Fraction((1 << 288) - 1, 1 << 288) + ((2**288 - 1) * f2 + Fraction(1 << 512, L)) / (1 << 288)


def sqrt_ratio_model(u, v):
    """fe_sqrt_ratio (Go's SqrtRatio): (r, was square).  r is the even root in [0, p) of u/v when that is a square, else
    of i u/v; (0, u == 0) when v = 0 mod p."""
    uu, vv = u % p, v % p
    if vv == 0:
        return 0, int(uu == 0)
    q = uu * pow(vv, p - 2, p) % p
    sq = q == 0 or pow(q, (p - 1) // 2, p) == 1
    w = q if sq else q * ref.SQRT_M1 % p
    r = pow(w, (p + 3) // 8, p)
    if r * r % p != w:
        r = r * ref.SQRT_M1 % p
    assert r * r % p == w
    return (p - r if r & 1 else r), int(sq)


# ---- models of the point routines (the same sequence of field ops as the device) ----
def double_model(P, with_t=True):
    X, Y, Z, T = P
    A, B, C = fe_sqr(X), fe_sqr(Y), fe_sqr(Z)
    C = fe_add(C, C)
    H = fe_add(A, B)
    E = fe_sqr(fe_add(X, Y))
    E = fe_sub(H, E)
    G = fe_sub(A, B)
    F = fe_add(C, G)
    return fe_mul(E, F), fe_mul(G, H), fe_mul(F, G), (fe_mul(E, H) if with_t else T)


def cached_model(Q):
    X, Y, Z, T = Q
    return fe_add(Y, X), fe_sub(Y, X), fe_add(Z, Z), fe_mul(T, D2)


def add_point_model(P, Q, with_t=True, affine=False, neg=False):
    """ed_add<with_t, affine>(P, ed_to_cached(Q), neg)."""
    X, Y, Z, T = P
    ypx, ymx, z2, t2d = cached_model(Q)
    A = fe_mul(fe_sub(Y, X), ypx if neg else ymx)
    B = fe_mul(fe_add(Y, X), ymx if neg else ypx)
    C = fe_mul(T, t2d)
    D = fe_add(Z, Z) if affine else fe_mul(Z, z2)
    E, H, s, G = fe_sub(B, A), fe_add(B, A), fe_sub(D, C), fe_add(D, C)
    F, G = (G, s) if neg else (s, G)
    return fe_mul(E, F), fe_mul(G, H), fe_mul(F, G), (fe_mul(E, H) if with_t else T)


# ---- operand constructions ----
def _roots_mod_2p(R):
    """The a in [0, 2^256) with a^2 = R mod 2p (2^256 - 38 = 2p)."""
    r = ref._sqrt(R)
    if r is None:
        return []
    out = set()
    for s in {r % p, (p - r) % p}:
        for a in (s, s + p, s + 2 * p):
            if a < M256 and a * a % (2 * p) == R % (2 * p):
                out.add(a)
    return sorted(out)


def _mul_solve(S):
    """Operand pairs (a, b), a = 2^256 - u, with T_lo + 38 T_hi = S exactly for T = a b.  For u b = m 2^256 + n with
    0 < n < 2^256: T_hi = b - m - 1, T_lo = 2^256 - n, so S = (m + 1)(2^256 - 38) + (38 - u) b, linear in b for fixed m."""
    out = []
    for u in list(range(1, 38)) + list(range(39, 120)):
        for m in range(u):
            num = S - (m + 1) * (M256 - 38)
            if num % (38 - u):
                continue
            b = num // (38 - u)
            if 0 < b < M256 and (u * b) >> 256 == m and (u * b) % M256:
                out.append((M256 - u, b))
                break
        if len(out) >= 2:
            break
    return out


def fold_sets():
    """(mul pairs, sqr operands), each reaching its fold branch by construction.  For every c1 = 0..38 a product can reach,
    results just past 0 after the first fold, just below 2^256 after the second (the +38 c1 does not carry) and at or just
    past 2^256 (it carries: the result is the low half + 38), from operands mostly in [p, 2^256)."""
    mul = []
    for c in range(39):
        targets = [0, 1, 2 * p % M256 + c, M256 - 38 * c - 1, M256 - 38 * c - 2]  # c2 = 0 (2p + c: a mid value)
        if 1 <= c <= 37:
            targets += [M256 - 38 * c, M256 - 38 * c + 1, M256 - 1]               # c2 = 1
        for r1 in targets:
            if r1 < 0 or r1 >= M256:
                continue
            S = c * M256 + r1
            if c == 0:
                sols = [(1, S), (S, 1)] + ([(2, S // 2)] if S % 2 == 0 else [(3, S // 3)] if S % 3 == 0 else [])
            elif c == 38:
                sols = []
            else:
                sols = _mul_solve(S)
                sols += [(b, a) for a, b in sols]
            for a, b in sols:
                s = (a * b) % M256 + 38 * ((a * b) >> 256)
                assert s == S, (c, hex(r1))
                mul.append((a, b))
    # c1 = 38: (2^256 - u)(2^256 - v) with u v < 2^256 gives S = 38 2^256 + u v - 38 (u + v); it never carries again
    for u, v in ((76, 76), (76, 77), (77, 76), (100, 100), (2**20, 39), (2**128 - 1, 2**128 - 3), (2**127, 2**128 + 76)):
        mul.append((M256 - u, M256 - v))
    # squares: a^2 = R mod 2p for small R, so that S = R + j (2^256 - 38) sits just below (R < 38) or just past
    # (38 <= R < 38 j) the second carry, or just past 0 (R >= 38 j), for whatever j the magnitude of a gives
    sqr, per = [], Counter()
    for R in range(0, 1600):
        for a in _roots_mod_2p(R):
            key = fold_branch(a * a)
            if per[key] < 6:
                per[key] += 1
                sqr.append(a)
    sqr += [M256 - u for u in (1, 2, 19, 31, 32, 37, 38, 39, 75, 76, 77, 100)]
    sqr += [0, 1, p - 1, p, p + 1, 2**255, 2**128, 2**128 - 1]
    return mul, sqr


def fold_branch(T):
    _, c1, c2 = fold(T)
    return c1, c2


def reachable_folds():
    """The (c1, c2) pairs some product of two values below 2^256 reaches: c2 = 1 needs c1 >= 1 (the first fold's low half
    is below 2^256), and c1 = 38 never carries again.  For the latter: c2 = 1 at c1 = 38 needs T_lo + 38 T_hi >= 39 2^256
    - 38^2, so T_hi = 2^256 - k with k <= 37 and T_lo >= 2^256 - 1444 + 38 k.  Writing a = 2^256 - u, b = 2^256 - v and
    w = floor(u v / 2^256), T_hi = 2^256 - (u + v) + w, so u + v = k + w; w = 0 leaves u v <= 18 * 19 < T_lo; w >= 1 needs
    (k + w)^2 >= (u + v)^2 >= 4 u v >= 4 w 2^256, which the convex (k + w)^2 - 4 w 2^256 refuses at both ends of
    w in [1, 2^256): so nowhere between."""
    for k in range(2, 38):
        for w in (1, M256 - 1):
            assert (k + w) ** 2 < 4 * w * M256
    return {(c, 0) for c in range(39)} | {(c, 1) for c in range(1, 38)}


ADDSUB_VALUES = [0, 1, 2, 19, 37, 38, 39, p - 1, p, p + 1, 2**255 - 1, 2**255, 2 * p] + [M256 - k for k in range(1, 40)]


def addsub_pairs():
    vs = ADDSUB_VALUES
    return [(a, b) for a in vs for b in vs]


def canon_values():
    """a mod 2^255 at both ends of each (bit 255, t >= p) case, with and without bit 255."""
    lows = [0, 1, 2, 18, 19, p - 21, p - 20, p - 19, p - 18, p - 2, p - 1, p, p + 1, p + 17, p + 18, 2**254]
    return [m | (bit << 255) for m in lows for bit in (0, 1)]


def reduce_values():
    """x with quotient error 0 and 1: x = kL - 1, kL, kL + 1 at the extremes, the largest x of each k whose q3 still falls
    short (t up to ~1.225 L) and the next x, whose q3 is exact, and 2^512 - 1."""
    top = ((1 << 512) - 1) // L
    vals = set(cases.reduce_operands()) | {(1 << 512) - 1, (1 << 512) - 2, (1 << 512) - L}
    for k in (1, 2, 3, 2**8, 2**64 + 1, 2**200, 2**259, 2**259 + 12345, top // 3, top // 2, top - 2, top - 1, top):
        vals |= {k * L - 1, k * L, k * L + 1, k * L + L - 1}
        # q3 < k exactly while q1 = floor(x / 2^224) < ceil(k 2^288 / mu)
        q1 = -(-(k << 288) // MU)
        for x in (q1 * (1 << 224) - 1, q1 * (1 << 224), q1 * (1 << 224) - 2, q1 * (1 << 224) + 1):
            vals.add(x)
    return sorted(v for v in vals if 0 <= v < 1 << 512)


def inv_values():
    return [0, 1, 2, 19, 38, p - 1, p, p + 1, 2 * p, 2 * p + 1, 2**255, M256 - 1, M256 - 2, M256 - 37, 2**128 + 7]


def sqrt_rows():
    """(u, v) for fe_sqrt_ratio: u = 0, v = 0, u/v a square, i u/v a square, non-canonical u and v, and the roots 0 and
    p - 1 (u = v gives the even root p - 1 of 1; u = -i v gives it for i u/v = 1)."""
    i = ref.SQRT_M1
    rows = [(0, 1), (0, 0), (0, p), (1, 0), (5, p), (0, 7), (0, 2 * p), (M256 - 1, 2 * p + 1)]
    for v in (1, 2, 7, p - 1, 2**254 + 3):
        rows += [(v, v), ((p - i) * v % p, v), (v + p, v), (v, v + p) if v + p < M256 else (v, v)]
        for x in (1, 2, 3, p - 1, 2**200 + 1):
            sq = x * x * v % p
            rows += [(sq, v), (sq * i % p, v), (sq + p, v + p) if max(sq, v) + p < M256 else (sq, v)]
    rows += [(4, 1), (2, 1), (p - 1, 1), (i, 1), (M256 - 1, M256 - 2), (M256 - 1, 1), (M256 - 38, 1), (1, M256 - 38)]
    return rows


# ---- runs ----
def _run_pairs(run, op, pairs):
    out = run(op, cases.slots([[(a, 8), (b, 8)] for a, b in pairs]))
    return [cases.val(row, 0) for row in out], out


def check_fold(run):
    """MUL and SQR on fold_sets: limbs equal to the model's, every reachable (c1, c2) reached at least 3 times.  Returns
    the branch counts {op: Counter((c1, c2))}."""
    mul, sqr = fold_sets()
    counts = {}
    for op, pairs in ((cases.MUL, mul), (cases.SQR, [(a, 0) for a in sqr])):
        got, _ = _run_pairs(run, op, pairs)
        cnt = Counter()
        for (a, b), g in zip(pairs, got):
            T = a * b if op == cases.MUL else a * a
            r, c1, c2 = fold(T)
            cnt[(c1, c2)] += 1
            assert r % p == T % p
            assert g == r, (op, hex(a), hex(b), hex(g), hex(r), c1, c2)
        counts[op] = cnt
    reach = reachable_folds()
    assert set(counts[cases.MUL]) == reach
    for key in reach:
        assert counts[cases.MUL][key] >= 3, ("mul", key)
    # a square cannot be aimed at a c1 as a product can; the small residues of fold_sets reach all but (1, 1)
    assert set(counts[cases.SQR]) <= reach
    for key in reach - {(1, 1)}:
        assert counts[cases.SQR][key] >= 3, ("sqr", key)
    return counts


def check_addsub(run):
    """ADD and SUB over ADDSUB_VALUES squared: limbs equal to the model's; counts of {no carry, carry, carry and wrap}."""
    pairs = addsub_pairs()
    counts = {}
    for op, model in ((cases.ADD, add_model), (cases.SUB, sub_model)):
        got, _ = _run_pairs(run, op, pairs)
        cnt = Counter()
        for (a, b), g in zip(pairs, got):
            r, c, w = model(a, b)
            assert r % p == (a + b if op == cases.ADD else a - b) % p and r < M256
            assert g == r, (op, hex(a), hex(b), hex(g), hex(r))
            cnt[(c, w)] += 1
        assert set(cnt) == {(0, 0), (1, 0), (1, 1)}
        assert min(cnt.values()) >= 3, (op, cnt)
        counts[op] = cnt
    return counts


def check_canon(run):
    vals = canon_values() + [v for v in ADDSUB_VALUES]
    got, _ = _run_pairs(run, cases.CANON, [(a, 0) for a in vals])
    cnt = Counter()
    for a, g in zip(vals, got):
        r, bit, ge = canon_model(a)
        assert g == r, (hex(a), hex(g))
        cnt[(bit, ge)] += 1
    assert set(cnt) == {(0, 0), (0, 1), (1, 0), (1, 1)} and min(cnt.values()) >= 3, cnt
    return cnt


def check_inv(run):
    vals = inv_values()
    got, _ = _run_pairs(run, cases.INV, [(a, 0) for a in vals])
    for a, g in zip(vals, got):
        assert g == pow(a % p, p - 2, p), hex(a)


def check_reduce(run):
    vals = reduce_values()
    out = run(cases.REDUCE, cases.slots([[(x, 16)] for x in vals]))
    cnt = Counter()
    tmax = 0
    for x, row in zip(vals, out):
        r, err, subs = reduce_model(x)
        assert cases.val(row, 0) == r, hex(x)
        assert all(int(w) == 0 for w in row[8:]), hex(x)
        assert subs == err  # t >= L exactly when q3 fell short
        cnt[err] += 1
        tmax = max(tmax, r + err * L)  # t before the final subtraction
    assert cnt[0] >= 3 and cnt[1] >= 3 and set(cnt) == {0, 1}, cnt
    assert Fraction(tmax, L) > Fraction(1224, 1000)  # the top of the bound, 1.2249 L, is reached
    return cnt, Fraction(tmax, L)


def check_sqrt(run):
    rows = sqrt_rows()
    out = run(cases.SQRT, cases.slots([[(u, 8), (v, 8)] for u, v in rows]))
    seen = Counter()
    for (u, v), row in zip(rows, out):
        r, ok = sqrt_ratio_model(u, v)
        assert (cases.val(row, 0), int(row[8])) == (r, ok), (hex(u), hex(v))
        seen["v=0" if v % p == 0 else "u=0" if u % p == 0 else "square" if ok else "non-square"] += 1
        seen["root p-1"] += r == p - 1
        seen["non-canonical"] += u >= p or v >= p
    assert min(seen.values()) >= 3, seen
    return seen


# ---- points ----
def _ext(x, y):
    return (x, y, 1, x * y % p)


def base_points():
    """(name, extended point with canonical coordinates): the identity, the eight small-order points, B, a mixed-order point
    and P, -P, 2P for a random P."""
    pts = [("identity", ref.IDENTITY)]
    pts += [(f"small{i}", _ext(x, y)) for i, (x, y) in enumerate(ref.small_order_points())]
    pts += [("B", ref.B)]
    x8, y8 = [pt for pt in ref.small_order_points() if pt[0] not in (0, ref.SQRT_M1, p - ref.SQRT_M1)][0]
    pts += [("B+T8", _ext(*ref.affine(ref.add(ref.B, _ext(x8, y8)))))]
    P = ref.mul(0x1d2c3b4a5968778695a4b3c2d1e0f, ref.B)
    for name, Q in (("P", P), ("-P", ref.neg(P)), ("2P", ref.add(P, P))):
        pts.append((name, _ext(*ref.affine(Q))))
    return pts


def _forms(P, lam):
    """Representatives of P: canonical, Z scaled by lam, and coordinates as v + p (every limb >= p where v + p < 2^256)."""
    scaled = tuple(c * lam % p for c in P)
    return [P, scaled, tuple(c + p for c in P), tuple(c + p for c in scaled)]


def point_set():
    lams = [2, p - 1, 0x5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5a5, 2**255 - 20]
    out = []
    for i, (name, P) in enumerate(base_points()):
        for j, f in enumerate(_forms(P, lams[i % len(lams)])):
            out.append((f"{name}/{j}", f))
    return out


def _same_point(got, want_affine):
    X, Y, Z, _ = (c % p for c in got)
    x, y = want_affine
    return Z != 0 and X == x * Z % p and Y == y * Z % p


def point_slots(rows):
    """rows: tuples of 4 (one point) or 8 (two points) coordinates, as ED_POINT_WORDS-word slots."""
    out = np.zeros((len(rows), PT_WORDS), np.uint32)
    for i, coords in enumerate(rows):
        for k, v in enumerate(coords):
            assert 0 <= v < M256
            for w in range(8):
                out[i, 8 * k + w] = (v >> (32 * w)) & 0xFFFFFFFF
    return out


def point_of(row, at=0):
    return tuple(cases.val(row, at + 8 * k) for k in range(4))


def _check_result(got, want, P, ref_affine, with_t):
    assert all(c < M256 for c in got)
    assert got == want, "limbs differ from the model"
    assert _same_point(got, ref_affine)
    if with_t:
        X, Y, Z, T = (c % p for c in got)
        assert T * Z % p == X * Y % p
    else:
        assert got[3] == P[3]  # T is not written


def check_double(run):
    pts = point_set()
    n = 0
    for flags, with_t in ((0, True), (PT_NO_T, False)):
        out = run(PT_DOUBLE | flags, point_slots([P for _, P in pts]))
        for (name, P), row in zip(pts, out):
            got = point_of(row)
            want_aff = ref.affine(ref.add(_reduce(P), _reduce(P)))
            _check_result(got, double_model(P, with_t), P, want_aff, with_t)
            assert all(int(w) == 0 for w in row[32:]), name
            n += 1
    return n


def _reduce(P):
    return tuple(c % p for c in P)


def _affine_form(Q):
    """Q with Z = 1 (as an affine table entry holds it), in the same representative class as Q's coordinates: canonical, or
    each coordinate + p when Q's are non-canonical."""
    x, y = ref.affine(_reduce(Q))
    t = x * y % p
    shift = p if Q[0] >= p else 0
    return (x + shift, y + shift, 1, t + shift)


def add_cases():
    pts = point_set()
    rows = []
    for i, (na, P) in enumerate(pts):
        for j, (nb, Q) in enumerate(pts):
            if (i * 7 + j * 3) % 4 and not (na.endswith("/0") or nb.endswith("/0")):
                continue  # every pair with a canonical point in it, and a quarter of the others
            rows.append((na, nb, P, Q))
    return rows


def check_add(run):
    rows = add_cases()
    n = 0
    for with_t in (True, False):
        for affine in (False, True):
            for neg in (False, True):
                op = PT_ADD | (0 if with_t else PT_NO_T) | (PT_AFFINE if affine else 0) | (PT_NEG if neg else 0)
                qs = [(_affine_form(Q) if affine else Q) for _, _, _, Q in rows]
                out = run(op, point_slots([P + Q for (_, _, P, _), Q in zip(rows, qs)]))
                for (na, nb, P, _), Q, row in zip(rows, qs, out):
                    Qr = _reduce(Q)
                    want_aff = ref.affine(ref.add(_reduce(P), ref.neg(Qr) if neg else Qr))
                    try:
                        _check_result(point_of(row), add_point_model(P, Q, with_t, affine, neg), P, want_aff, with_t)
                    except AssertionError as ex:
                        raise AssertionError(f"{na} {'-' if neg else '+'} {nb} with_t={with_t} affine={affine}: {ex}")
                    assert all(int(w) == 0 for w in row[32:])
                    n += 1
    return n


def check_cached(run):
    pts = point_set()
    out = run(PT_CACHED, point_slots([P for _, P in pts]))
    for (name, P), row in zip(pts, out):
        assert point_of(row) == cached_model(P), name
        ypx, ymx, z2, t2d = (c % p for c in point_of(row))
        X, Y, Z, T = _reduce(P)
        assert (ypx, ymx, z2, t2d) == ((Y + X) % p, (Y - X) % p, 2 * Z % p, T * D2 % p), name


def encode_points():
    """Points with x = 0, both parities of x, and X, Y or Z limbs >= p (alone or together), Z scaled."""
    out = []
    for name, P in base_points():
        x, y = ref.affine(P)
        for lam in (1, 3, p - 1, 2**255 - 20):
            X, Y, Z, T = (c * lam % p for c in P)
            for k in range(8):
                Q = [X, Y, Z, T]
                for c in range(3):
                    if k >> c & 1:
                        Q[c] += p
                out.append((f"{name}*{lam:x}/{k}", tuple(Q), x, y))
    return out


def check_encode(run):
    pts = encode_points()
    out = run(PT_ENCODE, point_slots([P for _, P, _, _ in pts]))
    seen = Counter()
    for (name, P, x, y), row in zip(pts, out):
        want = y | ((x & 1) << 255)
        assert cases.val(row, 0) == want, name
        assert all(int(w) == 0 for w in row[8:]), name
        seen["x=0" if x == 0 else f"x parity {x & 1}"] += 1
        seen["limb >= p"] += any(c >= p for c in P[:3])
    assert min(seen.values()) >= 3 and len(seen) == 4, seen
    return seen
