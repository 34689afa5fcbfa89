"""The per-key table builds on the device at the key counts where their grids turn over, every entry against the models
of tests/table_shapes.py:

  - Ed25519 comb tables of keys grouped in a launch (sbv_debug_ed25519_comb_tab) for K keys around the 64-thread
    blocks of k_edc_*, each key once or twice (launch capacity = the key count or twice it), and 1,024 keys;
  - registered ECDSA tables (sbv_set_keys, sbv_debug_key_table) of K keys of one curve in a registry that interleaves
    keys of the other curve and slots sbv_keys_build leaves unmapped, so that a key's local index is not its slot;
  - registered Ed25519 tables (sbv_ed25519_set_keys, sbv_debug_ed25519_ktab) around the 1,024-key launches of
    k_ed_ktab_build, with undecodable slots next to a chunk boundary.

Each registry is also run through its verification call, one row per slot, against OpenSSL: the slot-to-table map and
the tables agree.  tests/test_hostsim_table_shapes.py runs the same shapes, at sizes a CPU affords, on the CPU
simulation."""
import ctypes as C

import numpy as np
import pytest

import ecdsa_keys as ek
import oracle
import oracle_ed25519 as oe
import table_shapes as ts
from oracle import ecdsa_ref as eref
from oracle_ed25519 import ref
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu

ERR_ARG = -1


@pytest.fixture(scope="module")
def eng():
    e = _engine(SBV_GROUP_THRESHOLD=1)
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------- Ed25519 comb tables of keys grouped in a launch
def _comb_tab(eng, pub, items):
    items = np.ascontiguousarray(items, np.uint32)
    status = np.full(items.size, -1, np.int32)
    out = np.zeros((items.size, 510, 24), np.uint32)
    assert eng._lib.sbv_debug_ed25519_comb_tab(eng._h, C.c_size_t(pub.size // 32), _p(pub), C.c_size_t(items.size), _p(items), _p(status),
                                               _p(out)) == 0
    return status, out


@pytest.mark.parametrize("R", ts.COMB_REPEATS)
@pytest.mark.parametrize("K", ts.COMB_KEYS)
def test_every_entry_of_grouped_ed25519_comb_tables(eng, K, R):
    """K keys, R items each (interleaved) at threshold 1: every item's table equals the model of its own key (key ids
    come from k_kg_assign's atomics, so tables are matched by item); the last key does not decode (status 2)."""
    keys, pub = ts.comb_launch(K, R)
    n = K * R
    status, out = _comb_tab(eng, pub, np.arange(n))
    ts.check_comb_tables(keys, [keys[i % K] for i in range(n)], status, out)


def test_grouped_ed25519_comb_tables_of_1024_keys(eng):
    """1,024 keys, 2 items each: every key's status, entry (block 0, mask 1) = A itself for every key, and every entry of
    32 sampled keys."""
    K = 1024
    keys, pub = ts.comb_launch(K, 2)
    status, out = _comb_tab(eng, pub, K + np.arange(K))                        # the second item of every key
    assert status.tolist() == [0] * (K - 1) + [2]
    for k in range(K - 1):
        assert np.array_equal(out[k, 0], ts.niels(ref.decode(keys[k]))), k
    sample = np.sort(np.random.default_rng(11).choice(K - 1, 32, replace=False))
    ts.check_comb_tables(keys, [keys[k] for k in sample], status[sample], out[sample])


# ---------------------------------------------------------------- registered ECDSA tables
def _key_table(eng, curve, slot, count):
    N = eref.CURVES[curve].size // 4
    out = np.zeros(max(count, 1) * 2 * N, np.uint32)
    rc = eng._lib.sbv_debug_key_table(eng._h, C.c_uint8(curve), C.c_uint32(slot), C.c_size_t(0), C.c_size_t(count), _p(out))
    return rc, out


def _ecdsa_rows(curve, slots, rng):
    """One row per slot for verification under `curve`, then the same rows with one byte of the digest flipped: signed
    by the slot's key when it is a mapped key of the curve, else by a key of the curve (those rows must reject)."""
    c = eref.CURVES[curve]
    L, n = c.size, len(slots)
    d0 = ts.ecdsa_pool(curve, 1)[0][0]
    d = np.stack([ek._be(s[1] if s[0] == curve and s[3] else d0, L) for s in slots])
    dig = np.frombuffer(rng.bytes(n * L), np.uint8).reshape(n, L)
    k = np.stack([ek._be(1 + int.from_bytes(rng.bytes(L), "big") % (c.n - 1), L) for _ in range(n)])
    r, s = oracle.sign_batch(curve, d, np.arange(n, dtype=np.uint32), dig, k)
    flipped = dig.copy()
    flipped[np.arange(n), np.arange(n) % L] ^= 0x20
    return np.concatenate([r, r]), np.concatenate([s, s]), np.concatenate([dig, flipped])


@pytest.mark.parametrize("curve", [ts.P256, ts.P384])
def test_every_entry_of_registered_ecdsa_tables(eng, curve):
    """For each K, one registry of K keys of the curve interleaved with keys of the other curve and unmapped slots:
    every entry of every key's table equals the model, the other slots return SBV_ERR_ARG, and sbv_verify_registered
    with one row per slot (accepting, and with one byte flipped) gives OpenSSL's verdicts under both curves."""
    rng = np.random.default_rng(60 + curve)
    entries = ek.windows(curve, 8) * 128
    for K in ts.ECDSA_KEYS:
        tags, xy, slots = ts.ecdsa_registry(curve, K)
        eng.set_keys(tags, xy)
        for slot, (tag, _, Q, mapped) in enumerate(slots):
            rc, got = _key_table(eng, curve, slot, entries)
            if tag != curve or not mapped:
                assert rc == ERR_ARG, (K, slot)
                continue
            assert rc == 0, (K, slot)
            bad = np.nonzero(got != ts.window_model(curve, Q))[0]
            assert bad.size == 0, f"K={K}, slot {slot}: {bad.size} words differ, first {bad[:8].tolist()}"
        for c in (ts.P256, ts.P384):
            L = eref.CURVES[c].size
            r, s, dig = _ecdsa_rows(c, slots, rng)
            slot = np.tile(np.arange(len(slots), dtype=np.uint32), 2)
            qx, qy = xy[slot, 48 - L:48], xy[slot, 96 - L:]
            want = oracle.verify_batch(c, r, s, np.ascontiguousarray(qx), np.ascontiguousarray(qy), dig)
            mine = np.array([tags[i] == c and slots[i][3] for i in slot])
            want[~mine] = 0
            assert want[:len(slots)][mine[:len(slots)]].all() and not want[len(slots):].any()
            got = eng.verify_registered(c, slot, r, s, dig)
            assert np.array_equal(got, want), (K, c, np.nonzero(got != want)[0][:10].tolist())


# ---------------------------------------------------------------- registered Ed25519 tables
# (decodable keys, undecodable slots before these local indices): around the 1,024-key launches of k_ed_ktab_build,
# and 1,025 keys with undecodable slots before local 1,023, between it and 1,024 (where the second launch starts), and
# after 1,024, the last
ED_REGISTRIES = [(1023, ()), (1024, ()), (1025, ()), (2049, ()), (1025, (0, 517, 1023, 1024, 1024, 1025))]
FULL = (0, 1023, 1024, 2047, 2048)


@pytest.mark.parametrize("n_good,bad_at", ED_REGISTRIES)
def test_every_registered_ed25519_table(n_good, bad_at):
    """Every entry of the tables at local indices 0, 1,023, 1,024, 2,047, 2,048 and the last; for every key entry
    (win 0, j = 1) and one pseudo-random (win, j), computed directly as j * 256^win * A; undecodable slots have no
    table; sbv_ed25519_verify_registered with one row per slot (every third one with its message altered) gives
    OpenSSL's verdicts."""
    import consensus_b200 as sbv
    pub, slot_of, slot_seed = ts.ed_chunk_order(n_good, bad_at)
    keys = ts.ed_pool(n_good)[1]
    rng = np.random.default_rng(n_good + len(bad_at))
    with sbv.Engine(devices=[0]) as e:
        e.ed25519_set_keys(pub)
        one = np.zeros((1, 24), np.uint32)

        def entry(slot, first):
            assert e._lib.sbv_debug_ed25519_ktab(e._h, C.c_uint32(slot), C.c_size_t(first), C.c_size_t(1), _p(one)) == 0, (slot, first)
            return one[0]
        for local, slot in enumerate(slot_of):
            A = keys[local]
            if local in FULL or local == n_good - 1:
                got = np.zeros((32 * 128, 24), np.uint32)
                assert e._lib.sbv_debug_ed25519_ktab(e._h, C.c_uint32(slot), C.c_size_t(0), C.c_size_t(32 * 128), _p(got)) == 0
                bad = np.nonzero((got.reshape(32, 128, 24) != ts.ktab_model(A)).any(axis=2))
                assert bad[0].size == 0, f"{n_good} keys, local {local}: {bad[0].size} entries differ, first (win, j - 1) " \
                                         f"{list(zip(bad[0][:4].tolist(), bad[1][:4].tolist()))}"
            assert np.array_equal(entry(slot, 0), ts.niels(ref.decode(A))), (n_good, local)
            win, j = int(rng.integers(32)), int(rng.integers(1, 129))
            assert np.array_equal(entry(slot, win * 128 + j - 1), ts.ktab_entry(A, win, j)), (n_good, local, win, j)
        for slot in set(range(pub.shape[0] + 1)) - set(slot_of):
            assert e._lib.sbv_debug_ed25519_ktab(e._h, C.c_uint32(slot), C.c_size_t(0), C.c_size_t(1), _p(one)) == ERR_ARG, slot
        # one row per slot, signed with the slot's seed (an undecodable slot: with another key's), every third altered
        n = pub.shape[0]
        lens = rng.integers(0, 40, n)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        msgs = np.frombuffer(rng.bytes(int(off[-1]) + 1), np.uint8).copy()
        seeds = np.frombuffer(b"".join(slot_seed), np.uint8).reshape(n, 32)
        sig = oe.sign_batch(seeds, np.arange(n, dtype=np.uint32), msgs, off)
        for i in range(0, n, 3):
            if lens[i]:
                msgs[off[i]] ^= 1
            else:
                sig[i, 40] ^= 1
        want = oe.verify_batch(msgs, off, sig, pub)
        assert 0 < want.sum() < n - len(bad_at)
        got = e.ed25519_verify_registered(msgs, off, np.arange(n, dtype=np.uint32), sig)
        assert np.array_equal(got, want), np.nonzero(got != want)[0][:10].tolist()
