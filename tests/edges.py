"""Crafted inputs for the edge-case tests, shared by the CPU simulation tests (test_hostsim*.py) and the GPU tests
(test_gpu_arith.py, test_gpu_edges.py): operands that put a Montgomery reduction on its final conditional subtraction,
signatures whose R has x >= n, digests whose leftmost bytes are >= n or longer than the field, and scalars chosen for
the order of operations of the fixed-base kernels.  Every helper checks that its inputs reach the edge it names, with
Python integers, so a test that uses one proves what it covers.  Random corpora hit none of these edges: their
probabilities are between 2^-32 and 2^-256 per item."""
import numpy as np

import oracle
from oracle import ecdsa_ref as ref


def _be(v, L):
    return np.frombuffer(int(v).to_bytes(L, "big"), np.uint8)


def _rows(rows, L):
    """rows of (r, s, qx, qy, digest) -> the batch dict of the verify calls (digest: an int of L bytes or bytes)"""
    f = lambda j: np.stack([_be(row[j], L) for row in rows])
    dig = np.stack([np.frombuffer(row[4], np.uint8) if isinstance(row[4], bytes) else _be(row[4], L) for row in rows])
    return {"r": f(0), "s": f(1), "qx": f(2), "qy": f(3), "digest": dig}


def edge_values(m, rng, count):
    """Residues mod m that stress carry chains: small values, m - 1, limbs of all ones or all zeros, and `count` random
    residues plus count / 4 values built limb by limb from 0, 1, 2^32 - 1, 2^32 - 2, 2^31 and a random limb."""
    F = (1 << 32) - 1
    vals = [0, 1, 2, m - 1, m - 2, (m - 1) // 2, F, 1 << 32, (1 << 64) - 1, 1 << 96, (1 << 224) % m, m >> 1,
            0xFFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000 % m, ((1 << 96) - 1), (m - (1 << 96)) % m,
            (m - (1 << 192)) % m, ((1 << 256) - 1) % m, ((1 << 255) + 12345) % m]
    vals += [int.from_bytes(rng.bytes(48), "big") % m for _ in range(count)]
    for _ in range(count // 4):
        v = 0
        for k in range(12):
            v |= int(rng.choice([0, F, 1, F - 1, 0x80000000, int(rng.integers(0, F))])) << (32 * k)
        vals.append(v % m)
    return vals


def _sqrt(a, m):
    """a square root of a mod m, or None (m prime, m = 3 mod 4)"""
    assert m % 4 == 3
    x = pow(a, (m + 1) // 4, m)
    return x if x * x % m == a % m else None


def mod_inv_model(a, m, N, check=True):
    """mod_inv of curve.cuh on the plain residue a (binary extended GCD, batched trailing-zero strips), limb for limb:
    returns (x1 = a^-1 mod m, passes of the main loop).  check: assert at every strip that the cofactor is below m, so
    the conditional subtraction after the shift never fires."""
    mask = (1 << (32 * N)) - 1
    minv = -pow(m, -1, 1 << 32) % (1 << 32)

    def strip(t, x):
        while t & 1 == 0:
            low = t & 0xFFFFFFFF
            tz = (low & -low).bit_length() - 1 if low else 31
            t >>= tz
            k = ((x & 0xFFFFFFFF) * minv) & ((1 << tz) - 1)
            x = ((x + k * m) >> tz) & mask
            assert not check or x < m
            if x >= m:
                x -= m
        return t, x

    u, v, x1, x2 = a, m, 1, 0
    if u & 1 == 0:
        u, x1 = strip(u, x1)
    passes = 0
    while u != v:
        passes += 1
        lt = u < v
        d = v - u if lt else u - v
        xd = (x1 - x2) % m
        if lt:
            xd = m - xd
        d, xd = strip(d, xd)
        if lt:
            v, x2 = d, xd
        else:
            u, x1 = d, xd
    return x1, passes


def longest_inverse_inputs(m, N):
    """Residues whose mod_inv takes the most passes, 32N - 1 (the bound, tests/test_mutant_proofs.py): a = -m mod 2^k.
    Then v = m shrinks one bit per pass, (v - a) / 2 with exactly one trailing zero, while u = a stays, for k - 1 passes;
    the tail of the run takes the rest.  Random residues need ~0.8 * 32N."""
    W = 32 * N
    return [(-m) % (1 << k) for k in range(W - 8, W) if mod_inv_model((-m) % (1 << k), m, N)[1] == W - 1]


def mp_mul_row_carries(a, b, N):
    """mp_mul of mp.cuh, limb for limb: the carry out of each row's E and O chains, {(accumulator, row): carry}"""
    B = 1 << 32
    A = [(a >> (32 * i)) % B for i in range(N)]
    Bv = [(b >> (32 * i)) % B for i in range(N)]
    E, O, out = [0] * (2 * N), [0] * (2 * N), {}

    def chain(acc, cells, i0, j):
        c = 0
        for i in range(i0, N, 2):
            lo, hi = cells(i)
            t = acc[lo] + A[i] * Bv[j] + c + (acc[hi] << 32)
            acc[lo], acc[hi], c = t % B, (t >> 32) % B, t >> 64
        return c

    for j in range(N):
        if j % 2 == 0:
            out[("E", j)] = c = chain(E, lambda i: (i + j, i + j + 1), 0, j)
            E[j + N] = (E[j + N] + c) % B
            out[("O", j)] = c = chain(O, lambda i: (i + j - 1, i + j), 1, j)
            O[j + N] = (O[j + N] + c) % B
        else:
            out[("E", j)] = c = chain(E, lambda i: (i + j, i + j + 1), 1, j)
            if j + N + 1 < 2 * N:
                E[j + N + 1] = (E[j + N + 1] + c) % B
            out[("O", j)] = c = chain(O, lambda i: (i + j - 1, i + j), 0, j)
            O[j + N - 1] = (O[j + N - 1] + c) % B
    assert sum(E[k] << (32 * k) for k in range(2 * N)) + sum(O[k] << (32 * (k + 1)) for k in range(2 * N)) == a * b
    return out


def reduction_value(x, y, m, R):
    """U = (x*y + M*m) / R with M = -x*y/m mod R: the value a Montgomery reduction holds before its final conditional
    subtraction (whatever the algorithm, M is the unique multiplier in [0, R) that clears the low half)."""
    M = (-x * y * pow(m, -1, R)) % R
    return (x * y + M * m) // R


def reduction_targets(m, R):
    """U = m - 1 (no subtraction, the largest such value), U in [m, R) (the subtraction without a carry out of the top
    limb: m + 1, m + 2^32, R - 1), U >= R (with the carry: R, R + 1).  U = m needs x*y = 0 mod m, so it cannot occur."""
    return [m - 1, m + 1, m + (1 << 32), R - 1, R, R + 1]


def reduction_boundary_operands(m, R, targets, rng, per_target=8, square=False):
    """Pairs (x, y), x, y < m, whose Montgomery product x*y/R mod m has the pre-subtraction value U equal to each
    target: y = u*R/x mod m, M = (u*R - x*y)/m, kept if 0 <= M < R.  square: x == y, x = +-sqrt(u*R) mod m, for the
    targets whose u*R is a square.  Returns [(x, y, u)]; asserts U == u under the model of reduction_value."""
    out = []
    for u in targets:
        got = 0
        if square:
            x0 = _sqrt(u * R % m, m)
            cands = [] if x0 is None else [(x0, x0), (m - x0, m - x0)]
        else:
            cands = []
            while len(cands) < 4 * per_target:
                x = int.from_bytes(rng.bytes(56), "big") % m
                if x:
                    cands.append((x, u * R * pow(x, -1, m) % m))
        for x, y in cands:
            M, rem = divmod(u * R - x * y, m)
            if rem == 0 and 0 <= M < R:
                assert reduction_value(x, y, m, R) == u
                out.append((x, y, u))
                got += 1
                if got == per_target:
                    break
        assert square or got == per_target, (hex(m), hex(u))
    return out


def unreduced_operands(m, R, rng, count):
    """Pairs (a, y) with a in [m, R) and y < m: the inputs k_prep (e >= n in nmul(e, w)) and load_key pass unreduced.
    a*y < m*R, so the product is still a valid Montgomery input; the result must come out canonical."""
    As = [m, m + 1, R - 1, R - 2, R - (1 << 32), m + (1 << 32) - 1]
    As += [m + int.from_bytes(rng.bytes(56), "big") % (R - m) for _ in range(count)]
    Ys = [m - 1, 1, R % m, (R * R) % m] + [int.from_bytes(rng.bytes(56), "big") % m for _ in range(len(As) - 4)]
    return list(zip(As, Ys))


# sbv_debug_op / hs_debug_op: operations (low byte) and flags (csrc/debug_ops.cuh)
FMUL, FADD, FSUB, NMUL, DBL, ADD, MADD, FSQR = 0, 1, 2, 3, 5, 6, 7, 9
INL, NEG, SKIP = 0x100, 0x200, 0x400


def montgomery_cases(curve, rng, count):
    """[(label, op, xs, ys, want)] for the Montgomery products and the field additions: fmul, fsqr, fadd, fsub mod p and
    nmul mod n on edge values; fmul / nmul / fsqr on operands that put the reduction on each side of its final
    subtraction (reduction_boundary_operands); fmul / nmul with one operand in [m, R) (unreduced_operands)."""
    c = ref.CURVES[curve]
    R = 1 << (8 * c.size)
    out = []
    for m, mulop in ((c.p, FMUL), (c.n, NMUL)):
        Rinv = pow(R, -1, m)
        mont = lambda xs, ys: [x * y * Rinv % m for x, y in zip(xs, ys)]
        xs = edge_values(m, rng, count)
        ys = list(reversed(edge_values(m, rng, count)))
        out.append(("edge values", mulop, xs, ys, mont(xs, ys)))
        if m == c.p:
            out.append(("edge values", FSQR, xs, xs, mont(xs, xs)))
            out.append(("edge values", FADD, xs, ys, [(x + y) % m for x, y in zip(xs, ys)]))
            out.append(("edge values", FSUB, xs, ys, [(x - y) % m for x, y in zip(xs, ys)]))
        bx, by, _ = zip(*reduction_boundary_operands(m, R, reduction_targets(m, R), rng))
        out.append(("reduction boundary", mulop, list(bx), list(by), mont(bx, by)))
        if m == c.p:
            sq = [x for x, _, _ in reduction_boundary_operands(m, R, reduction_targets(m, R), rng, square=True)]
            assert len(sq) >= 4 and any(reduction_value(x, x, m, R) >= R for x in sq)
            out.append(("reduction boundary", FSQR, sq, sq, mont(sq, sq)))
        ua, uy = zip(*unreduced_operands(m, R, rng, count // 10))
        out.append(("unreduced", mulop, list(ua), list(uy), mont(ua, uy)))
        out.append(("unreduced", mulop, list(uy), list(ua), mont(ua, uy)))
    return out


def group_cases(curve, ks):
    """[(op, a, b, want)] for the group-law ops on the points k*G: doubling, mixed addition (Z2 = 1) and general
    addition (2P + 3-scaled Q), each with neg / skip as the verification loops pass them, and with an accumulator at
    infinity.  P == Q, P == -Q (infinity: (0, 0)) occur among the pairs."""
    c = ref.CURVES[curve]
    pts = [ref.scalar_mult(c, k, (c.gx, c.gy)) for k in ks]
    acc = pts + [None]                                           # None: the accumulator at infinity, passed as (0, 0)
    z = lambda P: P or (0, 0)
    dbl = lambda P: ref._add(c, P, P)
    ng = lambda P: (P[0], (c.p - P[1]) % c.p)
    pairs = [(P, Q) for P in acc for Q in pts]
    A, B = [z(P) for P, _ in pairs], [Q for _, Q in pairs]
    cases = [(DBL, [z(P) for P in acc], [z(P) for P in acc], [z(dbl(P)) for P in acc])]
    for first, op in ((lambda P: P, MADD), (dbl, ADD)):
        cases.append((op, A, B, [z(ref._add(c, first(P), Q)) for P, Q in pairs]))
        cases.append((op | NEG, A, B, [z(ref._add(c, first(P), ng(Q))) for P, Q in pairs]))
        cases.append((op | SKIP, A, B, [z(first(P)) for P, _ in pairs]))
        cases.append((op | NEG | SKIP, A, B, [z(first(P)) for P, _ in pairs]))
    return cases


# ---------------------------------------------------------------- signatures
def crafted(curve, cases):
    """(u1, u2, k) -> a signature on Q = k*G whose verification computes exactly u1*G + u2*Q (s = r/u2, e = u1*s): places
    exceptional points (doubling, P + (-P), infinity in the middle or at the end) inside the scalar multiplication.
    When R is infinity, r = 1 (such a row must reject).  Cases with u2 = 0 mod n or R.x = 0 mod n are dropped."""
    c = ref.CURVES[curve]
    rows = []
    for u1, u2, k in cases:
        if u2 % c.n == 0:
            continue
        Q = ref.scalar_mult(c, k % c.n, (c.gx, c.gy))
        R = ref._add(c, ref.scalar_mult(c, u1 % c.n, (c.gx, c.gy)), ref.scalar_mult(c, u2 % c.n, Q))
        r = 1 if R is None else R[0] % c.n
        if r == 0:
            continue
        s = r * pow(u2, -1, c.n) % c.n
        rows.append((r, s, Q[0], Q[1], u1 * s % c.n))
    return _rows(rows, c.size)


def big_x_points(curve, count):
    """The first `count` points R = (x, y) with x in (n, p): x = n+1, n+2, ... where x^3 - 3x + b is a square mod p."""
    c = ref.CURVES[curve]
    pts, x = [], c.n + 1
    while len(pts) < count:
        y = _sqrt((x * x * x - 3 * x + c.b) % c.p, c.p)
        if y is not None:
            pts.append((x, y))
        x += 1
    assert all(c.n < x < c.p for x, _ in pts)
    return pts


def small_x_points(curve, count):
    """The first `count` points R = (x, y) with x = 1, 2, ... (x^3 - 3x + b a square mod p): x < 2n - p, so r = x + p - n
    is a scalar in range."""
    c = ref.CURVES[curve]
    pts, x = [], 1
    while len(pts) < count:
        y = _sqrt((x * x * x - 3 * x + c.b) % c.p, c.p)
        if y is not None:
            pts.append((x, y))
        x += 1
    assert all(x + c.p - c.n < c.n for x, _ in pts)
    return pts


def big_x_signatures(curve, count, seed, digests=None):
    """Signatures whose R = u1*G + u2*Q has x in [n, p), so a correct verifier accepts r = R.x - n (Go: R.x mod n == r).
    Random u1, u2; Q = (R - u1*G)/u2, s = r/u2, e = u1*s.  Four rows per R: r = R.x - n (accept), r = R.x (>= n: reject),
    r = R.x - n + 1 (reject), and, on a second point R' with a small x, r = R'.x + p - n (reject: R'.x mod n != r, but
    r + n = R'.x + p is R'.x mod p, so a verifier that compares (r + n) * Z^2 without checking r < p - n accepts it).
    digests: one per R, taken as given (u1 = e*u2/r instead of random), for the hashing entry points; the fourth row uses
    the same digest.  Returns the batch dict plus "rx" (the x of the row's R) and "want" (the verdicts by construction)."""
    c = ref.CURVES[curve]
    L, n = c.size, c.n
    rng = np.random.default_rng(seed)
    rnd = lambda: int.from_bytes(rng.bytes(L + 8), "big") % (n - 1) + 1
    rows, rx, want = [], [], []

    def signature(x, y, r, dig):
        """(s, qx, qy, e) with R = u1*G + u2*Q = (x, y) for the row's r"""
        u2 = rnd()
        u1 = rnd() if dig is None else ref.hash_to_int(c, dig) * u2 * pow(r, -1, n) % n
        iu2 = pow(u2, -1, n)
        Q = oracle.lincomb(curve, ((n - u1) * iu2 % n).to_bytes(L, "big"), iu2.to_bytes(L, "big"), x.to_bytes(L, "big"), y.to_bytes(L, "big"))
        qx, qy = (int.from_bytes(v, "big") for v in Q)
        s = r * iu2 % n
        return s, qx, qy, (u1 * s % n if dig is None else dig)

    for i, ((x, y), (x2, y2)) in enumerate(zip(big_x_points(curve, count), small_x_points(curve, count))):
        dig = None if digests is None else bytes(np.asarray(digests[i], np.uint8))
        r = x - n
        s, qx, qy, e = signature(x, y, r, dig)
        for rr, ok in ((r, 1), (x, 0), (r + 1, 0)):
            rows.append((rr, s, qx, qy, e))
            rx.append(x)
            want.append(ok)
        r2 = x2 + c.p - n
        rows.append((r2, *signature(x2, y2, r2, dig)))
        rx.append(x2)
        want.append(0)
    b = _rows(rows, L)
    b["rx"], b["want"] = rx, np.array(want, np.uint8)
    return b


def sparse_s_signatures(curve, count, seed):
    """Valid signatures whose s has only its top 32-bit limb set (s = t * 2^(32(N-1))): a zero test that reads fewer limbs
    takes s for 0 and rejects.  R = k*G, r = R.x mod n, e = s*k - r*d; per signature the row (accept) and the row with
    e + 1 (reject).  Returns the batch dict plus "want"."""
    c = ref.CURVES[curve]
    L, n, N = c.size, c.n, c.size // 4
    rng = np.random.default_rng(seed)
    rnd = lambda m: int.from_bytes(rng.bytes(L + 8), "big") % (m - 1) + 1
    rows, want = [], []
    for _ in range(count):
        d, k = rnd(n), rnd(n)
        qx, qy = ref.pubkey(curve, d)
        r = ref.scalar_mult(c, k, (c.gx, c.gy))[0] % n
        s = rnd(n >> (32 * (N - 1))) << (32 * (N - 1))
        assert 0 < s < n and s % (1 << (32 * (N - 1))) == 0
        e = (s * k - r * d) % n
        rows += [(r, s, qx, qy, e), (r, s, qx, qy, (e + 1) % n)]
        want += [1, 0]
    b = _rows(rows, L)
    b["want"] = np.array(want, np.uint8)
    return b


def s_plus_n_signatures(curve, count, seed):
    """Signatures (r, 1), valid for e = k - r*d, and the same signature with s = n + 1 (>= n: reject).  k_prep computes
    with s = 1 for an item whose s is out of range, so a kernel that ignores k_prep's range flag accepts the second row.
    Returns the batch dict plus "want"."""
    c = ref.CURVES[curve]
    L, n = c.size, c.n
    rng = np.random.default_rng(seed)
    rnd = lambda: int.from_bytes(rng.bytes(L + 8), "big") % (n - 1) + 1
    rows, want = [], []
    for _ in range(count):
        d, k = rnd(), rnd()
        qx, qy = ref.pubkey(curve, d)
        r = ref.scalar_mult(c, k, (c.gx, c.gy))[0] % n
        e = (k - r * d) % n
        rows += [(r, 1, qx, qy, e), (r, n + 1, qx, qy, e)]
        want += [1, 0]
    b = _rows(rows, L)
    b["want"] = np.array(want, np.uint8)
    return b


def wide_digest_signatures(curve, dlen, count, seed):
    """Signatures over digests of `dlen` bytes (the verifier takes the leftmost min(dlen, BYTES) bytes, crypto/ecdsa
    hashToNat).  Per digest: the signature (accept); when dlen >= BYTES, the leftmost BYTES bytes are >= n for every
    other digest, and a row with the same e mod n written below n (accept); when dlen > BYTES, a bit flipped beyond the
    first BYTES bytes (accept: a verifier that reads them rejects); a bit flipped inside the first min(dlen, BYTES)
    bytes (reject).  Returns the batch dict plus "e" (the integer of the leftmost bytes of every row) and "want"."""
    c = ref.CURVES[curve]
    L, n = c.size, c.n
    rng = np.random.default_rng(seed)
    keys = [int.from_bytes(rng.bytes(L + 8), "big") % (n - 1) + 1 for _ in range(2)]
    pubs = [ref.pubkey(curve, d) for d in keys]
    rows, es, want = [], [], []

    def add(i, dig, sig, ok):
        rows.append((sig[0], sig[1], pubs[i % 2][0], pubs[i % 2][1], dig))
        es.append(ref.hash_to_int(c, dig))
        want.append(ok)

    for i in range(count):
        dig = bytearray(rng.bytes(dlen))
        if dlen >= L and i % 2 == 0:                       # leftmost BYTES bytes in [n, 2^(8L))
            hi = n + int.from_bytes(rng.bytes(L), "big") % ((1 << (8 * L)) - n)
            dig[:L] = hi.to_bytes(L, "big")
        dig = bytes(dig)
        sig = ref.sign(curve, keys[i % 2], dig, int.from_bytes(rng.bytes(L + 8), "big") % (n - 1) + 1)
        add(i, dig, sig, 1)
        if dlen >= L:
            add(i, (ref.hash_to_int(c, dig) % n).to_bytes(L, "big") + dig[L:], sig, 1)
        if dlen > L:
            t = bytearray(dig); t[L + i % (dlen - L)] ^= 1 << (i % 8)
            add(i, bytes(t), sig, 1)
        t = bytearray(dig); t[i % min(dlen, L)] ^= 1 << (i % 8)
        add(i, bytes(t), sig, 0)
    b = _rows(rows, L)
    b["e"], b["want"] = es, np.array(want, np.uint8)
    return b


# ---------------------------------------------------------------- scalars for the fixed-base kernels
def comb_cases(curve):
    """(u1, u2, k) for Q = k*G, chosen for the comb's order: u2*Q column by column from the top, then u1*G (k_gpart's
    point in one closing addition)."""
    c = ref.CURVES[curve]
    n, L = c.n, c.size
    sp = 8 * L // 16
    ones_col = lambda j: sum(1 << (sp * r + j) for r in range(16))          # column j all ones: both masks 255
    cases = []
    for k in (1, 3, 2**70 + 9):
        kinv = pow(k, -1, n)
        for d in (5, 0xFFFF, 2**15 + 3):
            cases.append((d, d * kinv % n, k))                               # u2*Q = u1*G = the first G entry: the closing addition doubles
            cases.append((d, (n - d) * kinv % n, k))                         # ... its negative: infinity: reject
            cases.append((d + (7 << 16), (n - d) * kinv % n, k))             # u1*G = -u2*Q + a second G entry
        for v in (7, 2**200 + 11, n - 5):
            cases.append((v * k % n, v, k))                                  # u1*G = u2*Q: the closing addition doubles
            cases.append(((n - v * k % n) % n, v, k))                        # u1*G = -u2*Q: R = infinity, reject
        for u2 in ((1 << (sp * 8)) - 1,                                      # block 0 masks all ones, block 1 all zero
                   ((1 << (8 * L)) - 1) ^ ((1 << (sp * 8)) - 1),             # the other way round (mod n)
                   n - 1, ones_col(0), ones_col(sp - 1), ones_col(0) | ones_col(sp - 1), (1 << sp) - 1, 1 << (8 * L - 1)):
            cases.append((12345, u2 % n, k))
            cases.append((u2 * k % n, u2 % n, k))
    return cases


def fixed_base_cases(curve):
    """(u1, u2, k) that make the running sum of a fixed-base verification meet the next table entry (doubling inside a
    mixed addition), its negative (infinity in the middle), or end at infinity (must reject)."""
    n = ref.CURVES[curve].n
    ks = [1, 2, 3, n - 1, 5, 2**8 + 1] if curve == 0 else [1, 3, n - 2]
    cases = []
    for k in ks:
        for u1, u2 in [(1, 1), (k, 1), (n - k, 1), (k, n - 1), (2, n - 1), (1, 2), (7, 3), (2**255, 2**255), (n - 1, n - 1), (k * 5 % n, 5),
                       (n - (k * 5 % n), 5), (k * 16 % n, 16), (n - (k * 16 % n), 16), (k * 33 % n, 33), (2**64, 2**64), (16, 1), (1, 16),
                       (0, 1), (0, 77), ((k << 5) % n, 32), (n - ((k << 5) % n), 32)]:
            cases.append((u1, u2, k))
    return cases


def u1_digit_cases(curve, seed):
    """(u1, u2, k) whose u1 has the same 16-bit comb digit of G in every column — 0x0000 (u1 = 0: the G part is
    infinity), 0x0001, 0x8000, 0xFFFF (the top column 0xFFFE, to stay below n) — or digits mixed from those four."""
    c = ref.CURVES[curve]
    n, cols = c.n, 8 * c.size // 16
    rng = np.random.default_rng(seed)
    rep = lambda d: sum(d << (16 * i) for i in range(cols))
    u1s = [0, rep(1), rep(0x8000), rep(0xFFFF) - (1 << (16 * (cols - 1))), n - 1]
    for _ in range(6):
        v = sum(int(rng.choice([0, 1, 0x8000, 0xFFFF])) << (16 * i) for i in range(cols))
        u1s.append(v if v < n else v & ((1 << (16 * (cols - 1))) - 1) | (0x8000 << (16 * (cols - 1))))
    assert all(0 <= u < n for u in u1s)
    cases = []
    for j, u1 in enumerate(u1s):
        for k in (1, 2**90 + 7):
            cases.append((u1, int.from_bytes(rng.bytes(c.size + 8), "big") % (n - 1) + 1, k + j))
    return cases


def with_bumped_r(b):
    """The batch followed by a copy with r + 1: u2 = r/s changes and u1 = e/s does not, so the copy keeps u1's digits
    and has another R, which does not have x = r + 1 mod n."""
    L = b["r"].shape[1]
    out = {k: np.concatenate([b[k], b[k]]) for k in ("r", "s", "qx", "qy", "digest")}
    m = len(b["r"])
    out["r"][m:] = np.stack([_be(int.from_bytes(v.tobytes(), "big") + 1, L) for v in b["r"]])
    return out
