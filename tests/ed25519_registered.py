"""Registered-key Ed25519 sets for k_ed_verify_keyed (consensus_b200/csrc/ed25519_keyed.cuh), shared by the CPU
simulation and the GPU tests (tests/test_hostsim_ed25519_registered.py, tests/test_gpu_ed25519_registered.py).

Builds on tests/ed25519_edges.py, whose rows carry their keys; here the distinct keys of a set become a registry and
each row refers to its key by slot.  The schedule model is extended with the registered kernel's loop: the key loop,
windows 0 to 31 of k (ed_digit8w, the 8-bit recoding ed_digit8 applies to S), one affine addition of -d * 256^w * A
from the key's table each, then the B loop of k_ed_verify on that accumulator.  The model table of any key generalises
edges.btab_words().
"""
import functools

import numpy as np

import ed25519_edges as edges
from oracle_ed25519 import corpus, ref

p, L, d = ref.p, ref.L, ref.d
O = ref.IDENTITY
DELTA = L - 2**252
EQ, NEG, FROM_O = edges.EQ, edges.NEG, edges.FROM_O


# ---- the key's table ----
@functools.lru_cache(None)
def ktab(A):
    """ktab(A)[w][j - 1] = affine j * 256^w * A, each column walked by affine additions of its base (as edges.btab)."""
    P = ref.decode(A)
    if P is None:
        raise ValueError("A does not decode")
    base, tab = ref.affine(P), []
    for _ in range(32):
        col, cur = [], base
        for _ in range(128):
            col.append(cur)
            cur = edges._aff_add(cur, base)
        tab.append(col)
        base = edges._aff_add(col[127], col[127])
    return tab


def ktab_words(A):
    """The table of A as k_ed_ktab_build lays it out: (32, 128, 24) words, y + x, y - x, 2dxy, canonical."""
    blob = b"".join(v.to_bytes(32, "little") for col in ktab(A) for x, y in col
                    for v in ((y + x) % p, (y - x) % p, 2 * d * x * y % p))
    return np.frombuffer(blob, "<u4").reshape(32, 128, 24)


# ---- the registered kernel's loop ----
def digitsk(k):
    """ed_digit8w of every window of k < L (the word-major reader gives ed_digit8 of k's little-endian bytes)."""
    return edges.digits8(k)


def key_loop(k, P, acc=O, events=None):
    """acc - [k]P added window by window as the key loop does (d > 0 subtracts d * 256^w * P).  events receives
    ("key", w, EQ / NEG / FROM_O) as edges.b_loop records them."""
    base = P
    for w, dg in enumerate(digitsk(k)):
        if w:
            for _ in range(8):
                base = ref.add(base, base)
        if dg == 0:
            continue
        Q = ref.mul(abs(dg), base)
        if dg > 0:
            Q = ref.neg(Q)
        if events is not None:
            if edges.is_O(acc):
                events.append(("key", w, FROM_O))
            elif edges.same(acc, Q):
                events.append(("key", w, EQ))
            elif edges.same(acc, ref.neg(Q)):
                events.append(("key", w, NEG))
        acc = ref.add(acc, Q)
    return acc


def reg_loop(k, S, A, events=None):
    """R' of k_ed_verify_keyed: the key loop from O, then the B loop.  events gets ("key", ...) and ("B", w, kind)."""
    acc = key_loop(k, ref.decode(A), O, events)
    ev = [] if events is not None else None
    Rp = edges.b_loop(S, acc, ev)
    if events is not None:
        events.extend(("B", w, kind) for w, kind in ev)
    return Rp


# ---- registries ----
def registry(keys):
    """(pub (n, 32) uint8, slot of each row): the distinct keys in order of first use."""
    order, slot = {}, []
    for A in keys:
        slot.append(order.setdefault(A, len(order)))
    pub = np.frombuffer(b"".join(order), np.uint8).reshape(-1, 32).copy()
    return pub, np.array(slot, np.uint32)


def corpus_registry(c):
    """The distinct keys of an oracle_ed25519.corpus batch and each item's slot."""
    pub, inv = np.unique(c["pub"], axis=0, return_inverse=True)
    return np.ascontiguousarray(pub), inv.reshape(-1).astype(np.uint32)


def merge(c, rows):
    """Corpus c followed by the rows of an edges.Rows set (msgs, off, sig, pub, cls; the rows' class is EDGE)."""
    a = rows.arrays()
    o0 = int(c["off"][-1])
    msgs = np.concatenate([c["msgs"][:o0], a["msgs"][int(a["off"][0]):]])
    off = np.concatenate([c["off"], a["off"][1:] - a["off"][0] + np.uint64(o0)]).astype(np.uint64)
    return {"msgs": msgs, "off": off, "sig": np.concatenate([c["sig"], a["sig"]]), "pub": np.concatenate([c["pub"], a["pub"]]),
            "cls": np.concatenate([c["cls"], np.full(len(rows), EDGE, np.uint8)])}


EDGE = 255


def key_class(A):
    """'y>=p', '-0' (sign bit set on x = 0), 'off-curve', 'small order', 'mixed order' or 'full order' for a 32-byte key."""
    y, sign = int.from_bytes(A, "little") & (2**255 - 1), A[31] >> 7
    P = ref.decode(A)
    if P is None:
        return "off-curve"
    if y >= p:
        return "y>=p"
    if sign and ref.affine(P)[0] == 0:
        return "-0"
    if edges.order(A) is not None:
        return "small order"
    return "full order" if edges.is_O(ref.mul(L, P)) else "mixed order"


def class_rows():
    """Production rows with accepting and rejecting items for keys with y >= p, "-0" keys, small-order and mixed-order
    keys and non-canonical R (edges.s_boundary and edges.small_order_r)."""
    return edges.Rows().extend(edges.s_boundary()).extend(edges.small_order_r())


# ---- the key loop's digits (test hook) ----
def k_sweep_ks():
    """One k per reachable (window, 8-bit digit) of k < L (edges.reachable8, the S sweep's set), plus all bytes 0x80, all
    bytes 0x7f, 2^248 - 1, L - 1, L - 2 delta (the key loop's P = Q at window 31) and 0."""
    reach = edges.reachable8()
    ks = list(reach.values()) + [sum(b * 256**i for i in range(31)) for b in (0x80, 0x7F)]
    ks += [2**248 - 1, L - 1, L - 2 * DELTA, 0]
    seen = set()
    for k in ks:
        assert k < L
        seen.update((w, dg) for w, dg in enumerate(digitsk(k)) if dg)
    assert set(reach) <= seen and len(reach) == 7951
    return ks


@functools.lru_cache(None)
def k_sweep():
    """Every k of k_sweep_ks with a key from edges.crafted_k_keys() in turn (full, small, mixed order, y >= p, "-0"):
    R = enc([S]B - [k]A), S from a pool.  Every fourth accepting row is followed by a rejecting variant."""
    rng = np.random.default_rng(201)
    ks, keys = k_sweep_ks(), edges.crafted_k_keys()
    pool = [int.from_bytes(rng.bytes(32), "little") % L for _ in range(61)]
    pool_pts = [edges.bmul(S) for S in pool]
    items = []
    for i, k in enumerate(ks):
        A = keys[i % len(keys)]
        j = i % len(pool)
        items.append((A, k, pool[j], ref.add(pool_pts[j], ref.neg(edges.key_model(A).mul(k)))))
    Rs = edges.encode_many([it[3] for it in items])
    rows = edges.Rows()
    for i, ((A, k, S, _), R) in enumerate(zip(items, Rs)):
        rows.add(A, b"", edges._sig(R, S), True, "k sweep", k)
        if i % 4:
            continue
        if i % 8 or S + 1 >= L:
            rows.add(A, b"", edges._sig(edges._flip(R, (i * 89 + 255) % 256), S), False, "k sweep/R flip", k)
        else:
            rows.add(A, b"", edges._sig(R, S + 1), False, "k sweep/S+1", k)
    return rows


def slot0_rows(n=64):
    """(A0, rows): n accepting k-sweep rows of its first key A0 (full order) with their k, for runs by slot.  Registered in
    slot 0 they accept; by an unknown slot the kernel itself must reject them, since with k given no gather is involved."""
    rows, A0 = k_sweep(), edges.crafted_k_keys()[0]
    assert key_class(A0) == "full order"
    idx = [i for i, (A, w) in enumerate(zip(rows.A, rows.want)) if A == A0 and w][:n]
    assert len(idx) == n
    return A0, edges._subset(rows, idx)


# ---- collisions of the registered loop (test hook) ----
@functools.lru_cache(None)
def collisions():
    """edges.collisions() (A = [a]B solved so that the B loop, entered with -[k]A as the key loop leaves it, meets +entry,
    -entry, or ends at R' = O at windows 0 to 31) and the key loop's own P = Q: k = L - 2 delta makes the accumulator
    [delta]A before window 31, whose addend -16 * 2^248 * A = -[L - delta]A is [delta]A too.  The model of the
    registered loop asserts each event."""
    rng = np.random.default_rng(202)
    rows = edges.Rows().extend(edges.collisions())
    hits = {EQ: set(), NEG: set(), "final O": set()}
    for A, sig, k, want, tag in zip(rows.A, rows.sig, rows.k, rows.want, rows.tag):
        if not want or "/" in tag:
            continue
        ev = []
        S = int.from_bytes(sig[32:], "little")
        Rp = reg_loop(k, S, A, ev)
        assert ref.encode(Rp) == sig[:32], tag
        kind, w = tag.split()[1], int(tag.split("w=")[1])
        if kind == "final":
            assert edges.is_O(Rp)
            hits["final O"].add(w)
        else:
            assert ("B", w, kind) in ev, (tag, ev)
            hits[kind].add(w)
    for kind, ws in hits.items():
        assert {0, 31} <= ws and len(ws) >= 31, (kind, sorted(ws))
    k = L - 2 * DELTA
    assert digitsk(k)[31] == 16
    for _ in range(4):
        a = int(rng.integers(1, 2**62)) ** 5 % L
        A = ref.encode(edges.bmul(a))
        S = int.from_bytes(rng.bytes(32), "little") % L
        ev = []
        Rp = reg_loop(k, S, A, ev)
        assert ("key", 31, EQ) in ev, ev
        R = ref.encode(Rp)
        rows.add(A, b"", edges._sig(R, S), True, "key loop P=Q w=31", k)
        edges._variants(rows, A, b"", R, S, Rp, k, "key loop P=Q w=31", 77)
    return rows


# ---- runners ----
def check(rows, set_keys, verify=None, verify_k=None, ref_n=100, seed=0):
    """Registers the distinct keys of a set, runs it by slot and compares every verdict with the construction's.
    verify(arrays, slot) runs the production path in calls of at most 2047 items (rows with k = None; also checked against
    OpenSSL); verify_k(arrays, slot) runs the hook with the rows' k.  A seeded sample is checked against ref."""
    pub, slot = registry(rows.A)
    set_keys(pub)
    want = np.array(rows.want, np.uint8)
    n = len(rows)
    a = rows.arrays()
    if verify_k is not None:
        got = verify_k(a, slot)
    else:
        got = np.zeros(n, np.uint8)
        for lo in range(0, n, 2047):
            sub = edges._subset(rows, range(lo, min(n, lo + 2047))).arrays()
            got[lo: lo + 2047] = verify(sub, slot[lo: lo + 2047])
        from oracle_ed25519 import verify_batch
        ossl = verify_batch(a["msgs"], a["off"], a["sig"], a["pub"])
        assert np.array_equal(ossl, want), edges._mismatch(rows, ossl, want)
    assert np.array_equal(got, want), edges._mismatch(rows, got, want)
    for i in edges.ref_sample(rows, ref_n, seed):
        assert edges.ref_verdict(rows.A[i], rows.M[i], rows.sig[i], rows.k[i]) == rows.want[i], (i, rows.tag[i])
    return int(want.sum()), n


def table_keys():
    """Keys whose tables are compared entry by entry: a random full-order key, a small-order key (order 8), a y >= p key
    (y = p: order 4) and a mixed-order key."""
    rng = np.random.default_rng(203)
    a = int(rng.integers(1, 2**62)) ** 5 % L
    full = ref.encode(edges.bmul(a))
    small = [A for A in corpus.small_order_encodings() if edges.order(A) == 8][0]
    big_y = corpus._enc_y(p, 0)
    T = ref.point_from_affine(*[pt for pt in ref.small_order_points() if pt[0] and pt[1]][0])
    mixed = ref.encode(ref.add(edges.bmul(a + 1), T))
    keys = [full, small, big_y, mixed]
    assert [key_class(A) for A in keys] == ["full order", "small order", "y>=p", "mixed order"]
    return keys
