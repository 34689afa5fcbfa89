"""Cases for Ed25519 keys grouped inside a keys-per-item launch (comb tables, k_ed_verify_comb), shared by
tests/test_hostsim_ed25519_grouped.py (CPU simulation) and tests/test_gpu_ed25519_grouped.py (device)."""
import functools

import numpy as np

import ed25519_edges as edges
import ed25519_registered as reg
from oracle_ed25519 import corpus, ref

L, p, d = ref.L, ref.p, ref.d
TAB_WORDS = 510 * 24


def comb_words(A):
    """The comb table of A as k_edc_final leaves it: (510, 24) words, y + x, y - x, 2dxy, canonical; None if A does not
    decode."""
    tab = ref.comb_table(A)
    if tab is None:
        return None
    blob = b"".join(v.to_bytes(32, "little") for x, y in tab for v in ((y + x) % p, (y - x) % p, 2 * d * x * y % p))
    return np.frombuffer(blob, "<u4").reshape(510, 24)


def table_keys():
    """Random keys and B; the identity encodings; small-order, mixed-order and y >= p keys; one off-curve key."""
    rng = np.random.default_rng(404)
    full = [ref.encode(edges.bmul(int.from_bytes(rng.bytes(32), "little") % L)) for _ in range(2)]
    small = [A for A in corpus.small_order_encodings() if edges.order(A) in (4, 8)][:2]
    keys = full + [ref.encode(ref.B)] + list(edges.IDENTITY_KEYS) + small + reg.table_keys()[1:]
    keys += [A for A in corpus.big_y_encodings() if ref.decode(A) is not None][:2]
    keys += list(corpus.off_curve_encodings(rng, 1))
    out = []
    for A in keys:
        if A not in out:
            out.append(A)
    return out


def comb_ks():
    """Scalars aimed at the comb: 0, 1, L - 1, 2^252; every column's mask 0xFF in either block (where k < L allows it)
    and both blocks' masks zero in turn; a single set bit at every comb position below 2^253."""
    ks = [0, 1, 2, L - 1, L - 2, 2**252, 2**128 - 1, (L - 1) >> 128 << 128, 2**252 - 1]
    for b in range(2):
        for j in range(16):
            k = sum(1 << (16 * (8 * b + t) + j) for t in range(8))
            if k < L:
                ks.append(k)
    ks += [1 << pos for pos in range(253)]
    assert all(0 <= k < L for k in ks)
    return ks


@functools.lru_cache(None)
def comb_rows():
    """Every comb_ks scalar under every kind of key: R = enc([S]B - [k]A) accepts; every third row is followed by a
    rejecting variant with one bit of R flipped."""
    rng = np.random.default_rng(405)
    keys = [A for A in table_keys() if ref.decode(A) is not None]
    keys = keys[:1] + [A for A in keys if reg.key_class(A) != "full order"][:6]
    rows = edges.Rows()
    i = 0
    for A in keys:
        km = edges.key_model(A)
        for k in comb_ks():
            S = int.from_bytes(rng.bytes(32), "little") % L
            R = ref.encode(ref.add(edges.bmul(S), ref.neg(km.mul(k))))
            rows.add(A, b"", edges._sig(R, S), True, "comb k", k)
            if i % 3 == 0:
                rows.add(A, b"", edges._sig(edges._flip(R, (i * 37 + 255) % 256), S), False, "comb k/R flip", k)
            i += 1
    return rows


def repeat_rows(rows, times):
    """The rows of a set repeated, so that every key occurs at least `times` times."""
    return edges._subset(rows, [i for i in range(len(rows)) for _ in range(times)])


def mixed_corpus(n, seed, n_keys):
    """A corpus with every corruption class plus the edge rows of the registered-key tests (y >= p, "-0", small- and
    mixed-order keys), with the edge keys repeated."""
    c = corpus.make_corpus(n, seed=seed, n_keys=n_keys, crafted_max=64)
    return reg.merge(c, repeat_rows(reg.class_rows(), 3))
