"""The key cache kernels (k_kc_lookup / k_kc_insert, consensus_b200/csrc/key_cache.cuh) compiled into the CPU simulation,
against a Python dict model: lookup, the renumbering of the launch's keys (misses first), the hit copy and the insert, for
hits, misses and a mix, forced probe collisions, a full pool, two launches inserting overlapping keys, a slot caught
BUSY, and invalid keys, on all three families.  The tables are stand-ins (a hash of the key bytes): the cache moves
tables and never looks inside them."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
EMPTY, BUSY, READY = 0, 1, 2
FAMS = {0: (32, 16), 1: (48, 24), 2: (32, 8)}  # family: (bytes per coordinate / encoding, key words)
TW4 = 40  # 16-byte words per stand-in table: more than a warp copies in one step


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    lib = C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))
    lib.hs_kc_slot.restype = C.c_uint32
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def table_of(key: bytes) -> np.ndarray:
    return np.frombuffer(hashlib.shake_256(b"table" + key).digest(TW4 * 16), np.uint32)


def make_keys(fam, count, seed):
    L, _ = FAMS[fam]
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (2 if fam < 2 else 1) * L, dtype=np.uint8).tobytes() for _ in range(count)]


class Cache:
    """One family's cache as the arrays the device holds, with the dict model beside it."""

    def __init__(self, hs, fam, cap, slots=None, seed=0x5EED):
        self.hs, self.fam, self.cap, self.seed = hs, fam, cap, seed
        slots = slots or max(2, 1 << (2 * cap - 1).bit_length())
        assert slots & (slots - 1) == 0
        self.smask = slots - 1
        self.kw = FAMS[fam][1]
        self.state = np.zeros(slots, np.uint32)
        self.keys = np.zeros(slots * self.kw, np.uint32)
        self.pidx = np.zeros(slots, np.uint32)
        self.pool = np.zeros(max(cap, 1) * TW4 * 4, np.uint32)
        self.stats = np.zeros(4, np.uint64)
        self.model = {}  # key bytes -> True (resident)
        self.hits = self.misses = 0

    def args(self):
        return (_p(self.state), _p(self.keys), _p(self.pidx), _p(self.pool), _p(self.stats), C.c_uint32(self.smask), C.c_uint32(self.cap),
                C.c_uint32(self.seed))

    def slot_of(self, key, fp=False):
        """The first probe slot of key, or with fp its fingerprint (the state word's upper 30 bits)."""
        a, b = Launch.arrays(self.fam, [key])
        return self.hs.hs_kc_slot(self.fam, _p(a), _p(b), C.c_uint32(1), C.c_uint32(self.seed), C.c_uint32(self.smask), C.c_int(int(fp)))

    def check_map(self):
        """READY slots hold exactly the model's keys, each once, with its table in its pool entry."""
        ready = np.flatnonzero((self.state & 3) == READY)
        got = [self.keys[s * self.kw:(s + 1) * self.kw].tobytes() for s in ready]
        assert sorted(got) == sorted(self.model), "resident keys differ from the model"
        assert len(set(got)) == len(got)
        assert len(set(self.pidx[ready].tolist())) == len(ready)
        for s, k in zip(ready, got):
            e = int(self.pidx[s])
            assert e < self.cap
            assert np.array_equal(self.pool[e * TW4 * 4:(e + 1) * TW4 * 4], table_of(k))
        assert int(self.stats[1]) == len(self.model)
        assert int(self.stats[2]) == self.hits and int(self.stats[3]) == self.misses


class Launch:
    """One simulated keys-per-item launch of the grouped keys `keys` (key k at item 2k + 1), of which `invalid` fail the
    build's validity check."""

    @staticmethod
    def arrays(fam, keys):
        L, _ = FAMS[fam]
        n = 2 * len(keys) + 1
        w = 2 * L if fam < 2 else L
        rows = np.zeros((n, w), np.uint8)
        for k, key in enumerate(keys):
            rows[2 * k + 1] = np.frombuffer(key, np.uint8)
        if fam == 2:
            return np.ascontiguousarray(rows), np.ascontiguousarray(rows)
        return np.ascontiguousarray(rows[:, :L]), np.ascontiguousarray(rows[:, L:])

    def __init__(self, cache, keys, invalid=(), kcap=None, nkeys=None):
        self.c, self.keys, self.invalid = cache, list(keys), set(invalid)
        self.kcap = kcap if kcap is not None else len(keys)
        self.nkeys = np.array([nkeys if nkeys is not None else len(keys)], np.uint32)
        self.a, self.b = self.arrays(cache.fam, self.keys)
        self.n = 2 * len(self.keys) + 1
        self.keylist = np.array([2 * k + 1 for k in range(len(self.keys))] or [0], np.uint32)
        self.keyid = np.full(self.n, -7, np.int32)
        self.lk = np.full(2 + self.kcap, 0xDEAD, np.uint32)
        self.keyflags = np.zeros(max(self.kcap, 1), np.uint8)
        self.ktab = np.zeros(max(self.kcap, 1) * TW4 * 4, np.uint32)

    def key_of_item(self, item):
        return self.keys[(item - 1) // 2]

    def lookup(self):
        c = self.c
        resident = dict(c.model)
        assert c.hs.hs_kc_lookup(c.fam, _p(self.a), _p(self.b), _p(self.nkeys), C.c_uint32(self.kcap), _p(self.keylist), *c.args(), C.c_uint32(TW4),
                                 _p(self.keyid), _p(self.lk), _p(self.keyflags), _p(self.ktab)) == 0
        K = min(int(self.nkeys[0]), self.kcap)
        m, h = int(self.lk[0]), int(self.lk[1])
        assert m + h == K
        ids = self.lk[2:2 + K]
        assert sorted(ids.tolist()) == sorted(self.keylist[:K].tolist()), "the renumbering is not a permutation of the grouped keys"
        for kid, item in enumerate(ids.tolist()):
            key = self.key_of_item(item)
            assert self.keyid[item] == kid
            assert (key in resident) == (kid >= m), (kid, m)
            if kid >= m:
                assert self.keyflags[kid] == 1
                assert np.array_equal(self.ktab[kid * TW4 * 4:(kid + 1) * TW4 * 4], table_of(key))
        for k in range(K, len(self.keys)):
            assert self.keyid[2 * k + 1] == -7, "a key past the launch's table slots was renumbered"
        c.hits += h
        self.m = m
        return m, h

    def build_and_insert(self):
        """The build of the misses ktab[0, m), then k_kc_insert; the model inserts the valid misses in id order while
        there is room, and skips keys already resident."""
        c = self.c
        for kid in range(self.m):
            key = self.key_of_item(int(self.lk[2 + kid]))
            ok = key not in self.invalid
            self.keyflags[kid] = ok
            self.ktab[kid * TW4 * 4:(kid + 1) * TW4 * 4] = table_of(key) if ok else 0
            if ok:
                c.misses += 1
                if key not in c.model and len(c.model) < c.cap:
                    c.model[key] = True
        assert c.hs.hs_kc_insert(c.fam, _p(self.a), _p(self.b), C.c_uint32(self.kcap), _p(self.lk), *c.args(), C.c_uint32(TW4), _p(self.keyflags),
                                 _p(self.ktab)) == 0
        c.check_map()

    def run(self):
        r = self.lookup()
        self.build_and_insert()
        return r


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_cold_warm_and_mixed(hs, fam):
    c = Cache(hs, fam, cap=16)
    keys = make_keys(fam, 10, seed=fam)
    assert Launch(c, keys).run() == (10, 0)
    assert Launch(c, keys).run() == (0, 10)
    more = make_keys(fam, 5, seed=100 + fam)
    mix = [keys[3], more[0], keys[7], more[1], more[2], keys[0]]
    assert Launch(c, mix).run() == (3, 3)
    assert int(c.stats[1]) == 13 and int(c.stats[2]) == 13 and int(c.stats[3]) == 13


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_forced_collisions(hs, fam):
    """A map of 8 slots for 4 tables and a seed under which several keys start on one slot."""
    keys = make_keys(fam, 4, seed=7 + fam)
    for seed in range(1, 1000):
        c = Cache(hs, fam, cap=4, slots=8, seed=seed)
        starts = [c.slot_of(k) for k in keys]
        if len(set(starts)) <= 2:
            break
    else:
        pytest.fail("no colliding seed")
    assert Launch(c, keys).run() == (4, 0)
    assert Launch(c, keys[::-1]).run() == (0, 4)
    # keys that are not resident probe past the occupied slots and miss
    other = make_keys(fam, 3, seed=50 + fam)
    assert Launch(c, other + keys[:2]).run() == (3, 2)


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_full_pool(hs, fam):
    c = Cache(hs, fam, cap=3)
    keys = make_keys(fam, 8, seed=20 + fam)
    assert Launch(c, keys).run() == (8, 0)
    assert int(c.stats[1]) == 3
    resident = set(c.model)
    m, h = Launch(c, keys).run()
    assert (m, h) == (5, 3)
    assert set(c.model) == resident and int(c.stats[1]) == 3
    assert ((c.state & 3) == BUSY).sum() == 0


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_two_launches_insert_overlapping_keys(hs, fam):
    """Both launches look up before either inserts, so both miss the shared keys; exactly one insert per key lands."""
    c = Cache(hs, fam, cap=32)
    keys = make_keys(fam, 12, seed=30 + fam)
    a, b = Launch(c, keys[:8]), Launch(c, keys[4:])
    assert a.lookup() == (8, 0)
    assert b.lookup() == (8, 0)
    a.build_and_insert()
    b.build_and_insert()
    assert int(c.stats[1]) == 12 and int(c.stats[3]) == 16
    assert Launch(c, keys).run() == (0, 12)


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_busy_slot_is_a_miss_and_blocks_a_second_insert(hs, fam):
    """A slot caught between its claim and its publication: a lookup misses it and an insert of the same key gives up,
    so the key never gets a second slot; published, it hits."""
    c = Cache(hs, fam, cap=8)
    keys = make_keys(fam, 3, seed=40 + fam)
    Launch(c, keys).run()
    ready = np.flatnonzero((c.state & 3) == READY)
    mine = next(s for s in ready if c.keys[s * c.kw:(s + 1) * c.kw].tobytes() == keys[1])
    c.state[mine] = (c.state[mine] & ~np.uint32(3)) | BUSY  # the key's own fingerprint stays
    del c.model[keys[1]]
    before = c.state.copy()
    L = Launch(c, [keys[1], keys[0]])
    assert L.lookup() == (1, 1)
    L.keyflags[0] = 1  # the launch builds keys[1] again, valid
    L.ktab[:TW4 * 4] = table_of(keys[1])
    c.model[keys[1]] = True  # the key stays resident through its one slot, still BUSY
    c.misses += 1
    assert c.hs.hs_kc_insert(c.fam, _p(L.a), _p(L.b), C.c_uint32(L.kcap), _p(L.lk), *c.args(), C.c_uint32(TW4), _p(L.keyflags), _p(L.ktab)) == 0
    assert np.array_equal(c.state, before), "an insert claimed a second slot for a key whose slot is BUSY"
    c.state[mine] = (c.state[mine] & ~np.uint32(3)) | READY
    assert Launch(c, [keys[1]]).lookup() == (0, 1)


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_busy_slot_of_another_key_is_passed(hs, fam):
    """A BUSY slot whose fingerprint is not the key's holds another key being inserted: the insert probes past it."""
    c = Cache(hs, fam, cap=8)
    key = make_keys(fam, 1, seed=45 + fam)[0]
    start = c.slot_of(key)
    c.state[start] = (0x2BCDE << 2) | BUSY
    assert Launch(c, [key]).run() == (1, 0)
    assert int(c.stats[1]) == 1 and (c.state[(start + 1) & c.smask] & 3) == READY
    assert Launch(c, [key]).lookup() == (0, 1)


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_invalid_keys_are_never_inserted(hs, fam):
    c = Cache(hs, fam, cap=16)
    keys = make_keys(fam, 6, seed=60 + fam)
    bad = {keys[1], keys[4]}
    for _ in range(3):
        m, h = Launch(c, keys, invalid=bad).run()
    assert (m, h) == (2, 4)
    assert int(c.stats[1]) == 4 and int(c.stats[3]) == 4


@pytest.mark.parametrize("fam", [0, 2])
def test_key_count_clamped_to_table_slots(hs, fam):
    """The grouping's key count may exceed the launch's table slots: only the first kcap keys take part."""
    c = Cache(hs, fam, cap=16)
    keys = make_keys(fam, 6, seed=70 + fam)
    Launch(c, keys[:2]).run()
    assert Launch(c, keys, kcap=4, nkeys=9).run() == (2, 2)


def test_keys_differing_in_one_byte_are_distinct(hs):
    """Keyed by the exact bytes: Ed25519 encodings that differ only in the sign bit, or by y >= p, are keys of their own."""
    c = Cache(hs, 2, cap=8)
    base = bytearray(make_keys(2, 1, seed=80)[0])
    variants = []
    for flip in (None, (31, 0x80), (0, 0x01), (17, 0x10)):
        v = bytearray(base)
        if flip:
            v[flip[0]] ^= flip[1]
        variants.append(bytes(v))
    assert Launch(c, variants[:1]).run() == (1, 0)
    assert Launch(c, variants).run() == (3, 1)
    assert int(c.stats[1]) == 4


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_a_fingerprint_collision_compares_every_key_word(hs, fam):
    """A READY slot with the key's start slot and fingerprint but bytes that differ in the last byte only (a forged
    collision of both hashes): the lookup compares every key word and misses, and the insert probes past it."""
    c = Cache(hs, fam, cap=4, slots=8)
    key = make_keys(fam, 1, seed=90 + fam)[0]
    twin = key[:-1] + bytes([key[-1] ^ 0x80])
    start = c.slot_of(key)
    c.state[start] = c.slot_of(key, fp=True) | READY
    c.keys[start * c.kw:(start + 1) * c.kw] = np.frombuffer(twin, np.uint32)
    c.pidx[start] = 3
    c.pool[3 * TW4 * 4:4 * TW4 * 4] = table_of(twin)
    c.stats[1] = 1
    c.model[twin] = True
    assert Launch(c, [key]).run() == (1, 0)
    assert Launch(c, [key]).lookup() == (0, 1)
