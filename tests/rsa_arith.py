"""The RSA arithmetic of consensus_b200/csrc/rsa.cuh at its boundaries, shared by the CPU simulation
(tests/test_hostsim_rsa.py, through hs_rsa_debug) and the GPU tests (tests/test_gpu_rsa_arith.py, through sbv_debug_rsa): the
Montgomery product, R^2 mod N with n0', S - N with its borrow, the carry resolution that ends a product, and S^e mod N by
the production primitives, all bit for bit against Python integers.

The models below restate what the device computes lane by lane (16 lanes of W = 32 * NL bits), so that every set can
assert in Python which branch each case takes: the three outcomes of a product's final subtraction, the generate and
propagate bits of the borrow and carry ballots in every lane, the doubling count of rsa_r2.  The boundaries are reached
by construction, not by the luck of a seed.  A runner (see `runner`) takes (k, op, a, b, n[, e]) and returns the output
values and the aux words of rsa_debug.cuh."""
import random

import numpy as np

import rsa_cases as rc
import rsa_edges

SIZES = rc.SIZES
MONT, R2, SUB, RESOLVE, POW = range(5)  # the ops of rsa_debug.cuh
M32 = 2**32

# the exponents of op 4: both ends of the accept set, powers of two (a last step that squares), long runs of set and clear
# bits; a random one of every bit length from 2 to 31 is added per size
EXPONENTS = [2, 3, 4, 5, 17, 65537, 2**16, 2**30, 2**30 + 1, 2**31 - 2, 2**31 - 1, 0x55555555, 0x2AAAAAAA]


def shape(k):
    """(K limbs, NL limbs per lane, W bits per lane) of a k-byte modulus."""
    K = k // 4
    return K, K // 16, 32 * (K // 16)


def ninv(N):
    return (-pow(N, -1, M32)) % M32


def runner(call, shift=0):
    """A runner over call(mod_bytes, op, n, a, b, mod, exp, out, aux) -> status (the C signature of sbv_debug_rsa without
    the engine).  shift = 1 puts one dummy item (op on 0 mod the first modulus) in front of every batch, so that each case
    also runs in the other half of its warp.  For op 3, b holds the 16 lazy words of each item."""
    def run(k, op, a, b, n, e=None):
        e = list(e) if e is not None else [0] * len(n)
        if shift:
            a, n, e = [0] + list(a), [n[0]] + list(n), [3] + e
            b = [[0] * 16 if op == RESOLVE else 0] + list(b)
        cnt = len(n)
        rows = lambda vals: np.frombuffer(b"".join(v.to_bytes(k, "big") for v in vals), np.uint8).reshape(cnt, k).copy()  # noqa: E731
        A, N = rows(a), rows(n)
        if op == RESOLVE:
            B = np.zeros((cnt, k // 4), np.uint32)
            B[:, :16] = np.array(b, np.uint32)
            B = B.view(np.uint8)
        else:
            B = rows(b)
        E = np.array(e, np.uint32)
        out, aux = np.zeros((cnt, k), np.uint8), np.full(cnt, 0xDEADBEEF, np.uint32)
        assert call(k, op, cnt, A, B, N, E, out, aux) == 0
        vals = [int.from_bytes(r.tobytes(), "big") for r in out]
        return vals[shift:], [int(x) for x in aux][shift:]
    return run


def moduli(k, full=True):
    """Odd moduli of every shape for size k, as (name, N): every bit length 8k - j (j = 0..7, every leading byte shape
    from 0xff to 0x01), an all-ones top limb and top lane, 2^(8k-8) + 1, n0' = 2^32 - 1 and n0' = 1, a lane of all-zero
    or all-one limbs at every lane, random moduli and the real keys of the edge sets.  full=False: a subset that keeps one
    of each kind (the CPU simulation's budget)."""
    _, _, W = shape(k)
    bits = 8 * k
    rng = random.Random(f"rsa-arith-moduli-{k}")

    def rnd(b=bits):
        return rng.getrandbits(b) | 1 | (1 << (b - 1))

    lane = lambda l: ((1 << W) - 1) << (W * l)  # noqa: E731
    out = [(f"b={bits - j}", rnd(bits - j)) for j in range(8)]
    out += [("top limb ones", rnd() | ((M32 - 1) << (bits - 32))), ("top lane ones", rnd() | lane(15)), ("2^(8k-8)+1", 2 ** (bits - 8) + 1),
            ("n0'=2^32-1", (rnd() >> 32 << 32) | 1), ("n0'=1", rnd() | (M32 - 1))]
    for l in range(16):
        out.append((f"lane {l} ones", rnd() | lane(l)))
        if 0 < l < 15:
            out.append((f"lane {l} zero", rnd() & ~lane(l)))
    out += [("random", rnd()), ("random", rnd())]
    out += [(f"key {b}", rsa_edges.key(f"std_{b}").n) for b in (bits, bits - 1, bits - 4, bits - 7)]
    for name, N in out:
        assert N % 2 == 1 and bits - 7 <= N.bit_length() <= bits, name
    if not full:
        keep = {"b=%d" % (bits - 7), "top lane ones", "2^(8k-8)+1", "n0'=2^32-1", "n0'=1", "lane 7 zero", f"key {bits}"}
        out = [m for m in out if m[0] in keep]
    return out


# ---- the Montgomery product: the value u before the final subtraction ------------------------------------------------
def mont_u(a, b, N, k):
    """u = (a*b + m*N) / R, m = -a*b*N^-1 mod R: what the K rows of rsa_mont accumulate before rsa_resolve's subtraction
    (the row form's quotient digits q_i = t_0 * n0' make up exactly this m)."""
    R = 2 ** (8 * k)
    m = (-a * b * pow(N, -1, R)) % R
    u, rem = divmod(a * b + m * N, R)
    assert rem == 0 and u < 2 * N
    return u


def mont_branch(u, N, k):
    return "top" if u >= 2 ** (8 * k) else "sub" if u >= N else "none"


def check_products(run, k, full=True):
    """Products of 0, 1, N - 1, values near R and random operands on every modulus shape, and for every size at least one
    product through each outcome of the final subtraction: u >= R (the top path), N <= u < R, u < N."""
    R = 2 ** (8 * k)
    rng = random.Random(f"rsa-arith-products-{k}")
    a, b, n = [], [], []
    for _, N in moduli(k, full):
        near_r = [N - 1, N - 2, (R - 1) % N, (R - M32) % N]
        pairs = [(0, rng.randrange(N)), (1, 1), (N - 1, N - 1), (N - 1, 1), (near_r[2], near_r[2]), (near_r[3], near_r[0]),
                 (rng.randrange(N), rng.randrange(N))]
        want = {"top", "sub", "none"} if full or N > R // 2 else {"sub", "none"}
        for _ in range(300):  # one search per outcome the modulus can reach (u >= R needs N > R / 2)
            x, y = rng.randrange(N // 2, N), rng.randrange(N)
            br = mont_branch(mont_u(x, y, N, k), N, k)
            if br in want:
                want.discard(br)
                pairs.append((x, y))
            if not want:
                break
        for x, y in pairs:
            a.append(x); b.append(y); n.append(N)
    got, aux = run(k, MONT, a, b, n)
    rinv = {N: pow(R, -1, N) for N in set(n)}
    seen = set()
    for i, (x, y, N) in enumerate(zip(a, b, n)):
        assert got[i] == x * y * rinv[N] % N, (i, hex(N)[:12])
        assert aux[i] == ninv(N)
        seen.add(mont_branch(mont_u(x, y, N, k), N, k))
    assert seen == {"top", "sub", "none"}, seen
    return len(a)


def check_r2_ninv(run, k, full=True):
    """R^2 mod N and n0' on every modulus shape, which takes rsa_r2 through all 8 doubling counts 33K - b + 1 of a size
    (b = N's bit length, 8k - 7 to 8k), and n0' through 2^32 - 1 and 1."""
    K, _, _ = shape(k)
    ns = [N for _, N in moduli(k, full)]
    got, aux = run(k, R2, [0] * len(ns), [0] * len(ns), ns)
    for N, r2, ni in zip(ns, got, aux):
        assert r2 == 2 ** (16 * k) % N, hex(N)[:12]
        assert ni == ninv(N)
    if full:
        assert {33 * K - N.bit_length() + 1 for N in ns} == set(range(K + 1, K + 9))
    assert {M32 - 1, 1} <= set(aux)


# ---- S - N: the borrow ballot of rsa_sub ------------------------------------------------------------------------------
def sub_model(x, N, k):
    """rsa_sub's ballot for x - N: (generate lanes, lanes a borrow passes through, borrow out of the top)."""
    _, _, W = shape(k)
    mask = (1 << W) - 1
    gen, prop = 0, 0
    for l in range(16):
        xl, nl = (x >> (W * l)) & mask, (N >> (W * l)) & mask
        gen |= (xl < nl) << l
        prop |= (xl == nl) << l
    bin_ = ((gen << 1) + prop) ^ prop
    through = {l for l in range(16) if (prop >> l) & 1 and (bin_ >> l) & 1}
    return {l for l in range(16) if (gen >> l) & 1}, through, (bin_ >> 16) & 1


def check_sub(run, k):
    """S - N and its borrow: generated in every lane l (S = N with one limb of lane l one smaller; the limb rotates within
    the lane), carried through every lane above it (those lanes equal N's) and out of the top; S = N; a difference that
    stops in a lane above; values on both sides of N."""
    _, NL, _ = shape(k)
    R = 2 ** (8 * k)
    a, n = [], []
    gens, throughs, outs = set(), set(), set()
    for name, N in moduli(k):
        if name not in (f"key {8 * k}", "lane 7 zero", "n0'=1"):
            continue
        xs = [0, 1, N - 1, N, N + 1, R - 1, N - (1 << 300), (N >> 64) << 64]
        for l in range(16):
            for j in range(NL):
                limb = l * NL + (l + j) % NL
                if (N >> (32 * limb)) % M32:
                    break
            xs.append(N - (1 << (32 * limb)))   # generate in lane l, propagate through l+1..15 and out of the top
            if N + (1 << (32 * limb)) < R:
                xs.append(N + (1 << (32 * limb)))  # a difference in lane l and no borrow
        for x in xs:
            g, t, o = sub_model(x, N, k)
            gens |= g; throughs |= t; outs.add(o)
            a.append(x); n.append(N)
    assert gens == set(range(16)) and throughs == set(range(1, 16)) and outs == {0, 1}
    got, aux = run(k, SUB, a, [0] * len(a), n)
    for x, N, d, bo in zip(a, n, got, aux):
        assert d == (x - N) % R and bo == (1 if x < N else 0), (hex(x)[:20], hex(N)[:12])
    return len(a)


# ---- the carry resolution that ends a product (rsa_resolve) -----------------------------------------------------------
def resolve_model(t, cz, k):
    """rsa_resolve's ballot on the limbs t and lazy words cz (lane l's word lands on lane l + 1; lane 15's on the top):
    (generate lanes, all-ones lanes, lanes a carry passes through, carry out of the top lane)."""
    _, _, W = shape(k)
    mask = (1 << W) - 1
    gen, prop = 0, 0
    for l in range(16):
        s = ((t >> (W * l)) & mask) + (cz[l - 1] if l else 0)
        gen |= (s >> W) << l
        prop |= ((s & mask) == mask) << l
    cin = ((gen << 1) + prop) ^ prop
    through = {l for l in range(16) if (prop >> l) & 1 and (cin >> l) & 1}
    return {l for l in range(16) if (gen >> l) & 1}, {l for l in range(16) if (prop >> l) & 1}, through, (cin >> 16) & 1


def resolve_forms(k):
    """Redundant forms (t, cz, value) built to reach every branch of rsa_resolve's ballot in every lane: lane l (l >= 1)
    overflowing on the lazy word of the lane below (generate), the carry stopping in the next lane or passing through
    every all-ones lane above it and out of the top, all-ones lanes with nothing to carry (lane 0 included), and values on
    both sides of N.  A value is t plus cz_l * 2^(W(l+1)) for cz_l <= 3, below 2N (N's top 40 bits are all ones, so that
    values up to about 2R fit); the result must be that value mod N.  Lane 0 adds no lazy word, so it never generates and
    no carry enters lanes 0 or 1."""
    _, _, W = shape(k)
    R = 2 ** (8 * k)
    ones = (1 << W) - 1
    rng = random.Random(f"rsa-arith-resolve-{k}")
    N = R - 1 - 2 * rng.getrandbits(8 * k - 40)
    forms = []

    def add(t, cz):
        v = t + sum(c << (W * (l + 1)) for l, c in enumerate(cz))
        if 0 <= t < R and v < 2 * N:
            forms.append((t, cz, v))

    add(R - 4, [0] * 16)                           # no lazy words: lanes 1..15 all ones, nothing moves
    add(R - 3, [2] + [0] * 15)                     # lane 1 overflows; lanes 2..15 propagate; the carry leaves the top
    add(R - 1 - (3 << W), [3] + [0] * 15)          # lane 1 becomes all ones: it propagates, nothing to propagate
    add(R - (3 << W), [3] + [0] * 15)              # value R: lane 1 overflows and the carry leaves the top
    add(R - (1 << (W * 15)), [0] * 14 + [1, 0])    # lane 15 overflows on its lazy word alone
    add(N - 1, [0] * 16)
    add(N, [0] * 16)
    add(N - (2 << (W * 3)), [0, 0, 2] + [0] * 13)
    for l in range(1, 16):
        for stop in range(l + 1, 17):  # lanes l+1 .. stop-1 all ones: the carry stops in lane `stop` (16: out of the top)
            cz = [rng.randrange(4) if rng.random() < 0.5 else 0 for _ in range(15)] + [0]
            cz[l - 1] = 3                       # lands on lane l
            for m in range(l + 1, min(stop, 15) + 1):
                cz[m - 1] = 0                   # nothing lands on lanes l+1 .. stop
            t = 0
            for m in range(16):
                if m == l:
                    lv = ones - rng.randrange(3)             # overflows on 3
                elif l < m < stop:
                    lv = ones                                # propagates
                elif m == stop:
                    lv = ones - 1 - rng.randrange(2 ** 20)   # absorbs the carry
                else:
                    lv = rng.getrandbits(W)
                t |= lv << (W * m)
            add(t, cz)
    add(ones + (rng.getrandbits(8 * k - W - 8) << W), [0] * 16)  # lane 0 all ones
    for _ in range(40):
        cz = [rng.randrange(4) if rng.random() < 0.7 else 0 for _ in range(15)] + [rng.randrange(2)]
        t = 0
        for l in range(16):  # limbs mostly all ones, so that carries meet propagating lanes
            t |= (ones - (rng.randrange(4) if rng.random() < 0.3 else 0)) << (W * l)
        add(t - rng.randrange(2 ** 20), cz)
        add(rng.randrange(2 * N) - sum(c << (W * (l + 1)) for l, c in enumerate(cz)), cz)
    return N, forms


def check_resolve(run, k):
    """The forms of resolve_forms, with every reachable branch of the ballot asserted as reached."""
    N, forms = resolve_forms(k)
    gens, props, throughs, outs, sides = set(), set(), set(), set(), set()
    for t, cz, v in forms:
        g, p, th, o = resolve_model(t, cz, k)
        gens |= g; props |= p; throughs |= th; outs.add(o); sides.add(v >= N)
        for l in g | th:  # a carry out of lane l: into lane l + 1, or out of the top
            outs.add(("lane", l))
    assert gens == set(range(1, 16)), sorted(set(range(1, 16)) - gens)
    assert props == set(range(16)), sorted(set(range(16)) - props)
    assert throughs == set(range(2, 16)), sorted(set(range(2, 16)) - throughs)
    assert outs >= {0, 1} | {("lane", l) for l in range(1, 16)}
    assert sides == {False, True}
    got, aux = run(k, RESOLVE, [f[0] for f in forms], [f[1] for f in forms], [N] * len(forms))
    for (t, cz, v), o in zip(forms, got):
        assert o == v % N, (hex(t)[:20], cz)
    return len(forms)


# ---- S^e mod N ------------------------------------------------------------------------------------------------------
def exponents(k):
    rng = random.Random(f"rsa-arith-exponents-{k}")
    return EXPONENTS + [rng.randrange(2 ** (j - 1), 2**j) for j in range(2, 32)]


def pow_items(k, full=True):
    """(S, e, N) for S in {0, 1, 2, N - 1, N - 2, random}, every exponent and every modulus shape; neighbouring items differ
    in exponent and modulus (a diagonal walk of exponent x modulus per S).  full=False: one item per exponent class on
    the subset of moduli."""
    rng = random.Random(f"rsa-arith-pow-{k}")
    ns = [N for _, N in moduli(k, full)]
    if not full:
        items = []
        for i, e in enumerate([2, 5, 2**16, 65537]):
            N = ns[3 * i % len(ns)]
            items.append(([N - 1, rng.randrange(N), 2, N - 2][i], e, N))
        return items
    es = exponents(k)
    items = []
    for si in range(6):
        for d in range(len(ns)):
            for ei, e in enumerate(es):
                N = ns[(ei + d + si) % len(ns)]
                items.append(([0, 1, 2, N - 1, N - 2, rng.randrange(N)][si], e, N))
    for x, y in zip(items, items[1:]):
        assert x[1] != y[1] and x[2] != y[2]
    return items


def check_pow(run, k, full=True):
    items = pow_items(k, full)
    got, aux = run(k, POW, [s for s, _, _ in items], [0] * len(items), [N for _, _, N in items], [e for _, e, _ in items])
    for (S, e, N), g, ni in zip(items, got, aux):
        assert g == pow(S, e, N), (hex(S)[:12], e, hex(N)[:12])
        assert ni == ninv(N)
    return len(items)


def check_refused(call):
    """The hook refuses, with nothing written, a modulus size outside 256 / 384 / 512, an op outside 0-4, a null buffer and
    n >= 2^31 (call as for `runner`, buffers passed as arrays or None)."""
    k, n = 256, 2
    bufs = [np.ones((n, k), np.uint8), np.ones((n, k), np.uint8), np.full((n, k), 0xff, np.uint8), np.full(n, 3, np.uint32)]
    out, aux = np.full((n, k), 0x5A, np.uint8), np.full(n, 0x5A5A5A5A, np.uint32)
    args = bufs + [out, aux]
    bad = [(mb, MONT, n, args) for mb in (0, 128, 255, 257, 300, 1024)] + [(k, op, n, args) for op in (-1, 5, 255)]
    bad += [(k, MONT, n, args[:i] + [None] + args[i + 1:]) for i in range(6)]
    bad += [(k, MONT, 1 << 31, args), (k, POW, (1 << 64) - 1, args)]
    for mb, op, cnt, a in bad:
        assert call(mb, op, cnt, *a) != 0, (mb, op, cnt, [x is None for x in a])
        assert (out == 0x5A).all() and (aux == 0x5A5A5A5A).all(), (mb, op, cnt)
    assert call(k, MONT, 0, *args) == 0
    assert (out == 0x5A).all() and (aux == 0x5A5A5A5A).all()
