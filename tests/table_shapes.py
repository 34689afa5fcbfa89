"""Key sets and cached models for the per-key table builds at the key counts where their grids turn over, shared by
tests/test_hostsim_table_shapes.py (CPU simulation) and tests/test_gpu_table_shapes.py (device).

Each build spreads one key's work over a grid (a thread per key, per (key, chain) or per (key, window); 32 or 64 keys
per block; at most 1,024 keys per k_ed_ktab_build launch), finds its key with t % nkeys, and lays its scratch out
[...][cap] with the key innermost.  A fault in that arithmetic damages only the keys past a block or a chunk, or only a
launch whose capacity differs from its key count, so the tests here read back every entry of every table at those
shapes and compare it with the Python models: ed25519_grouped.comb_words (Ed25519 comb tables of keys grouped in a
launch), ecdsa_keys.window_table (registered ECDSA keys, 8-bit windows) and ed25519_registered.ktab_words (registered
Ed25519 keys).  The models are cached per key, so the shapes share them."""
import functools

import numpy as np

import ecdsa_keys as ek
import ed25519_grouped as grp
import ed25519_registered as reg
import oracle
import oracle_ed25519 as oe
from oracle import ecdsa_ref as eref
from oracle_ed25519 import corpus, ref

P256, P384 = oracle.P256, oracle.P384

# Ed25519 comb tables of keys grouped in a launch: K distinct keys, each repeated R times (interleaved), so that the
# launch has R * K table slots at threshold 1 and the [...][cap] strides differ from the key count when R = 2
COMB_KEYS = (1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129)
COMB_REPEATS = (1, 2)
# registered ECDSA keys of one curve, around k_kt_bases4's 32 keys per block and the fill's 64-thread blocks
ECDSA_KEYS = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129)


# ---------------------------------------------------------------- Ed25519 keys
def ed_seed(i):
    return int(i).to_bytes(4, "little") + b"table shapes" + bytes(16)


@functools.lru_cache(None)
def ed_pool(count):
    """count distinct full-order keys (OpenSSL key generation from fixed seeds), with their seeds."""
    seeds = [ed_seed(i) for i in range(count)]
    return seeds, [oe.pubkey(s) for s in seeds]


UNDECODABLE = corpus.off_curve_encodings(np.random.default_rng(907), 1)[0]
assert ref.decode(UNDECODABLE) is None


@functools.lru_cache(None)
def comb_model(A):
    return grp.comb_words(A)


@functools.lru_cache(None)
def ktab_model(A):
    return reg.ktab_words(A)


def niels(P):
    """An extended point as the tables store it: y + x, y - x, 2dxy (canonical), 24 words."""
    x, y = ref.affine(P)
    p, d = ref.p, ref.d
    return np.frombuffer(b"".join(v.to_bytes(32, "little") for v in ((y + x) % p, (y - x) % p, 2 * d * x * y % p)), "<u4")


def ktab_entry(A, win, j):
    """Entry (win, j - 1) of A's registered table, computed directly as j * 256^win * A."""
    return niels(ref.mul(j * 256**win, ref.decode(A)))


def comb_launch(K, R):
    """The keys of a grouped launch of K distinct keys (the last one does not decode when K > 1) and the R * K items
    that carry them, interleaved: item i carries keys[i % K]."""
    keys = list(ed_pool(K)[1])
    if K > 1:
        keys[-1] = UNDECODABLE
    idx = np.tile(np.arange(K), R)
    return keys, np.frombuffer(b"".join(keys[i] for i in idx), np.uint8).copy()


def check_comb_tables(keys, items_key, status, out):
    """Every queried item: status 2 for the key that does not decode, else status 0 and every entry of its table equal
    to the model of the item's own key."""
    for q, A in enumerate(items_key):
        if A == UNDECODABLE:
            assert status[q] == 2, (len(keys), q, status[q])
            continue
        assert status[q] == 0, (len(keys), q, status[q])
        bad = np.nonzero((out[q] != comb_model(A)).any(axis=1))[0]
        assert bad.size == 0, f"{len(keys)} keys, item {q} (key {keys.index(A)}): {bad.size} entries differ, first {bad[:8].tolist()}"


def ed_chunk_order(n_good, bad_at):
    """A registry of the first n_good keys of the pool with an undecodable slot inserted before each local index in
    bad_at (a local index may repeat; n_good: after the last key): (pub (n, 32), slot of each local index, seed of
    every slot)."""
    seeds, keys = ed_pool(n_good)
    order, slot_of, slot_seed = [], [], []
    for i in range(n_good + 1):
        for _ in range(list(bad_at).count(i)):
            order.append(UNDECODABLE)
            slot_seed.append(seeds[0])
        if i == n_good:
            break
        slot_of.append(len(order))
        order.append(keys[i])
        slot_seed.append(seeds[i])
    return np.frombuffer(b"".join(order), np.uint8).reshape(-1, 32).copy(), slot_of, slot_seed


# ---------------------------------------------------------------- ECDSA keys
@functools.lru_cache(None)
def ecdsa_pool(curve, count):
    """count (d, Q) pairs of the curve (OpenSSL key generation from fixed scalars)."""
    c = eref.CURVES[curve]
    L = c.size
    out = []
    for i in range(count):
        d = (0x7AB1E + 0x10001 * i + 977 * curve) % c.n
        qx, qy = oracle.pubkey(curve, d.to_bytes(L, "big"))
        out.append((d, (int.from_bytes(qx, "big"), int.from_bytes(qy, "big"))))
    return out


@functools.lru_cache(None)
def window_model(curve, Q):
    return ek.window_table(curve, 8, Q)


def ecdsa_registry(curve, K):
    """A registry whose keys of `curve` are the first K of the pool, interleaved with keys of the other curve and with
    P-256 slots that sbv_keys_build leaves unmapped (a nonzero byte above the low 32 of x: a value >= 2^256), so that a
    key's local index differs from its slot.  Returns the curve tags, the 96-byte slots (x then y, 48 bytes each,
    big-endian), and per slot (tag, d, Q, mapped)."""
    other = 1 - curve
    mine, theirs = ecdsa_pool(curve, K), ecdsa_pool(other, (K + 2) // 3)
    slots = []
    for i, (d, Q) in enumerate(mine):
        if i % 3 == 1:
            slots.append((other,) + theirs[i // 3] + (True,))
        if i % 4 == 2 or i == K - 1:
            d0, Q0 = ecdsa_pool(P256, 1)[0]
            slots.append((P256, d0, Q0, False))
        slots.append((curve, d, Q, True))
    tags = np.array([s[0] for s in slots], np.uint8)
    xy = np.zeros((len(slots), 2, 48), np.uint8)
    for i, (tag, _, Q, mapped) in enumerate(slots):
        L = eref.CURVES[tag].size
        xy[i, 0, 48 - L:], xy[i, 1, 48 - L:] = ek._be(Q[0], L), ek._be(Q[1], L)
        if not mapped:
            xy[i, 0, 48 - L - 1 - i % (48 - L)] = 1 + i % 255
    return tags, xy.reshape(-1, 96), slots
