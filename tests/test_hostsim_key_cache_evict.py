"""The evicting key cache kernels (k_kca_lookup / k_kca_insert, consensus_b200/csrc/key_cache_assoc.cuh) compiled into the
CPU simulation, against a Python model of the map that predicts every way: its state word (fingerprint, pins, EMPTY /
BUSY / READY), its stamp, its key and its table, and all six counters.  Cold, warm and mixed launches; a pinned way is
never evicted; a BUSY way is a miss and, with the key's fingerprint, blocks the insert; a READY way with the key's
fingerprint over other key words (the ABA case) is a miss and its pin is released; the victim is the least recently
stamped way and never one the launch has used; a set with no way to take gives up and counts it; invalid keys; keys one
byte apart; the key count clamped to kcap; and exactly sum(min(c_b, 16)) keys admitted from per-set counts c_b.  The
simulation runs one warp at a time, in warp order, which is the order the model replays.  The tables are stand-ins (a hash
of the key bytes): the cache moves tables and never looks inside them."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
EMPTY, BUSY, READY = 0, 1, 2
WAYS = 16  # KCA_WAYS
PIN = 4
FAMS = {0: (32, 16), 1: (48, 24), 2: (32, 8)}  # family: (bytes per coordinate / encoding, key words)
TW4 = 40  # 16-byte words per stand-in table: more than a warp copies in one step


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    lib = C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))
    lib.hs_kca_set.restype = C.c_uint32
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def table_of(key: bytes) -> np.ndarray:
    return np.frombuffer(hashlib.shake_256(b"table" + key).digest(TW4 * 16), np.uint32)


def make_keys(fam, count, seed):
    L, _ = FAMS[fam]
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (2 if fam < 2 else 1) * L, dtype=np.uint8).tobytes() for _ in range(count)]


def arrays(fam, keys):
    """Item arrays of a launch over `keys`: key k at item 2k + 1."""
    L, _ = FAMS[fam]
    n = 2 * len(keys) + 1
    rows = np.zeros((n, 2 * L if fam < 2 else L), np.uint8)
    for k, key in enumerate(keys):
        rows[2 * k + 1] = np.frombuffer(key, np.uint8)
    if fam == 2:
        return np.ascontiguousarray(rows), np.ascontiguousarray(rows)
    return np.ascontiguousarray(rows[:, :L]), np.ascontiguousarray(rows[:, L:])


class Way:
    def __init__(self):
        self.key, self.fp, self.stamp, self.pins, self.busy = None, 0, 0, 0, False

    def word(self):
        if self.key is None and not self.busy:
            return 0
        return self.fp | self.pins * PIN | (BUSY if self.busy else READY)


class Cache:
    """One family's evicting cache as the arrays the device holds, with the model beside it."""

    def __init__(self, hs, fam, sets, seed=0x5EED):
        self.hs, self.fam, self.sets, self.seed = hs, fam, sets, seed
        self.kw = FAMS[fam][1]
        n = sets * WAYS
        self.state = np.zeros(n, np.uint64)
        self.stamp = np.zeros(n, np.uint64)
        self.keys = np.zeros(n * self.kw, np.uint32)
        self.pool = np.zeros(n * TW4 * 4, np.uint32)
        self.stats = np.zeros(6, np.uint64)
        self.ways = [Way() for _ in range(n)]
        self.want = [0] * 6  # unused, resident, hits, misses, evictions, given up
        self.now = 0

    def args(self):
        return (_p(self.state), _p(self.stamp), _p(self.keys), _p(self.pool), _p(self.stats), C.c_uint32(self.sets), C.c_uint32(self.seed))

    def where(self, key):
        """(set, fingerprint as the state word holds it) of key."""
        a, b = arrays(self.fam, [key])
        fp = C.c_uint64()
        s = self.hs.hs_kca_set(self.fam, _p(a), _p(b), C.c_uint32(1), C.c_uint32(self.seed), C.c_uint32(self.sets), C.byref(fp))
        return int(s), int(fp.value)

    def set_ways(self, key):
        s, _ = self.where(key)
        return range(s * WAYS, (s + 1) * WAYS)

    def resident(self):
        return {w.key for w in self.ways if w.key is not None and not w.busy}

    def force(self, i, **kw):
        """Set way i's model fields and write them to the device arrays (a test driving a state the kernels reach only
        under concurrency)."""
        w = self.ways[i]
        for k, v in kw.items():
            setattr(w, k, v)
        self.state[i] = w.word()
        self.stamp[i] = w.stamp
        if w.key is not None:
            self.keys[i * self.kw:(i + 1) * self.kw] = np.frombuffer(w.key, np.uint32)
            self.pool[i * TW4 * 4:(i + 1) * TW4 * 4] = table_of(w.key)

    def check(self):
        for i, w in enumerate(self.ways):
            assert int(self.state[i]) == w.word(), (i, hex(int(self.state[i])), hex(w.word()))
            assert int(self.stamp[i]) == w.stamp, (i, int(self.stamp[i]), w.stamp)
            if w.key is not None:
                assert self.keys[i * self.kw:(i + 1) * self.kw].tobytes() == w.key, i
                assert np.array_equal(self.pool[i * TW4 * 4:(i + 1) * TW4 * 4], table_of(w.key)), i
        assert [int(v) for v in self.stats[1:]] == self.want[1:], (self.stats.tolist(), self.want)
        assert self.want[1] <= len(self.ways)

    # ---- the model: the rules of key_cache_assoc.cuh, one warp at a time ----
    def model_hit(self, key, now):
        _, fp = self.where(key)
        for i in self.set_ways(key):
            w = self.ways[i]
            if not w.busy and w.key == key and w.fp == fp:
                w.stamp = max(w.stamp, now)
                return True
        return False

    def model_insert(self, key, now):
        _, fp = self.where(key)
        self.want[3] += 1
        ws = [self.ways[i] for i in self.set_ways(key)]
        if any(w.fp == fp and (w.busy or w.key == key) for w in ws if w.key is not None or w.busy):
            return
        empty = [w for w in ws if w.key is None and not w.busy]
        if empty:
            v = empty[0]
            self.want[1] += 1
        else:
            old = [w for w in ws if not w.busy and w.pins == 0 and w.stamp < now]
            if not old:
                self.want[5] += 1
                return
            v = min(old, key=lambda w: w.stamp)  # the first of equal stamps
            self.want[4] += 1
        v.key, v.fp, v.stamp, v.pins, v.busy = key, fp, now, 0, False


class Launch:
    """One simulated keys-per-item launch of the grouped keys `keys`, of which `invalid` fail the build's validity check."""

    def __init__(self, cache, keys, invalid=(), kcap=None, nkeys=None):
        cache.now += 1
        self.c, self.keys, self.invalid, self.now = cache, list(keys), set(invalid), cache.now
        self.kcap = kcap if kcap is not None else len(keys)
        self.nkeys = np.array([nkeys if nkeys is not None else len(keys)], np.uint32)
        self.a, self.b = arrays(cache.fam, self.keys)
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
        K = min(int(self.nkeys[0]), self.kcap)
        hit = {self.keys[k]: c.model_hit(self.keys[k], self.now) for k in range(K)}
        c.want[2] += sum(hit.values())
        assert c.hs.hs_kca_lookup(c.fam, _p(self.a), _p(self.b), _p(self.nkeys), C.c_uint32(self.kcap), _p(self.keylist), *c.args(),
                                  C.c_uint64(self.now), C.c_uint32(TW4), _p(self.keyid), _p(self.lk), _p(self.keyflags), _p(self.ktab)) == 0
        m, h = int(self.lk[0]), int(self.lk[1])
        assert m + h == K
        ids = self.lk[2:2 + K]
        assert sorted(ids.tolist()) == sorted(self.keylist[:K].tolist()), "the renumbering is not a permutation of the grouped keys"
        for kid, item in enumerate(ids.tolist()):
            key = self.key_of_item(item)
            assert self.keyid[item] == kid
            assert hit[key] == (kid >= m), (kid, m)
            if kid >= m:
                assert self.keyflags[kid] == 1
                assert np.array_equal(self.ktab[kid * TW4 * 4:(kid + 1) * TW4 * 4], table_of(key))
        for k in range(K, len(self.keys)):
            assert self.keyid[2 * k + 1] == -7, "a key past the launch's table slots was renumbered"
        c.check()
        self.m = m
        return m, h

    def build_and_insert(self):
        """The build of the misses ktab[0, m), then k_kca_insert; the model inserts the valid misses in id order."""
        c = self.c
        for kid in range(self.m):
            key = self.key_of_item(int(self.lk[2 + kid]))
            ok = key not in self.invalid
            self.keyflags[kid] = ok
            self.ktab[kid * TW4 * 4:(kid + 1) * TW4 * 4] = table_of(key) if ok else 0
            if ok:
                c.model_insert(key, self.now)
        assert c.hs.hs_kca_insert(c.fam, _p(self.a), _p(self.b), C.c_uint32(self.kcap), _p(self.lk), *c.args(), C.c_uint64(self.now),
                                  C.c_uint32(TW4), _p(self.keyflags), _p(self.ktab)) == 0
        c.check()

    def run(self):
        r = self.lookup()
        self.build_and_insert()
        return r


def keys_in_set(c, count, seed, where=None):
    """count keys of c's family that share one set (that of the first key drawn, or `where`)."""
    out, s = [], where
    for key in make_keys(c.fam, 200 * count, seed):
        ks, _ = c.where(key)
        if s is None:
            s = ks
        if ks == s:
            out.append(key)
            if len(out) == count:
                return out
    pytest.fail("not enough keys in one set")


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_cold_warm_and_mixed(hs, fam):
    c = Cache(hs, fam, sets=4)
    keys = make_keys(fam, 10, seed=fam)
    assert Launch(c, keys).run() == (10, 0)
    assert Launch(c, keys).run() == (0, 10)
    more = make_keys(fam, 5, seed=100 + fam)
    mix = [keys[3], more[0], keys[7], more[1], more[2], keys[0]]
    assert Launch(c, mix).run() == (3, 3)
    assert c.stats.tolist() == [0, 13, 13, 13, 0, 0]


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_lru_victim_and_the_launch_own_ways(hs, fam):
    """A full set whose ways were inserted by launches 1..16: the victim is the least recently stamped way, a hit
    refreshes a way's stamp, and ways the current launch has hit or inserted are never victims."""
    c = Cache(hs, fam, sets=2)
    keys = keys_in_set(c, 20, seed=10 + fam)
    for k in keys[:16]:
        Launch(c, [k]).run()
    assert [c.ways[i].stamp for i in c.set_ways(keys[0])] == list(range(1, 17))
    L = Launch(c, [keys[0], keys[16]])  # keys[0] (stamp 1) is hit, so keys[1] (stamp 2) is the victim
    assert L.run() == (1, 1)
    assert keys[1] not in c.resident() and {keys[0], keys[16]} <= c.resident()
    assert int(c.stats[4]) == 1
    # every way of the set used by this launch: the extra keys give up, counted
    res = sorted(c.resident())
    assert Launch(c, res + keys[17:19]).run() == (2, 16)
    assert int(c.stats[5]) == 2 and c.resident() == set(res)


@pytest.mark.parametrize("fam", [0, 2])
def test_pinned_way_is_never_evicted(hs, fam):
    c = Cache(hs, fam, sets=1)
    keys = keys_in_set(c, 19, seed=20 + fam)
    assert Launch(c, keys[:16]).run() == (16, 0)  # one launch: equal stamps, ties take the first way
    c.force(0, pins=1)  # a lookup of another launch is copying way 0 out
    c.force(1, pins=3)
    assert Launch(c, [keys[16]]).run() == (1, 0)
    assert c.ways[0].key == keys[0] and c.ways[1].key == keys[1] and c.ways[2].key == keys[16]
    # every way pinned or used by the launch: given up
    for i in range(3, 16):
        c.force(i, pins=1)
    assert Launch(c, [keys[2], keys[16], keys[17]]).run() == (2, 1)  # keys[2] was the victim above
    assert int(c.stats[5]) == 2 and int(c.stats[4]) == 1
    # pins released: the oldest unpinned way goes
    for i in range(16):
        c.force(i, pins=0)
    assert Launch(c, [keys[18]]).run() == (1, 0)
    assert c.ways[0].key == keys[18]


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_busy_way_is_a_miss_and_blocks_an_insert_of_its_fingerprint(hs, fam):
    c = Cache(hs, fam, sets=2)
    keys = keys_in_set(c, 3, seed=30 + fam)
    Launch(c, keys).run()
    mine = next(i for i in c.set_ways(keys[1]) if c.ways[i].key == keys[1])
    c.force(mine, busy=True)  # caught between a claim (by keys[1] again) and its publication
    before = c.state.copy()
    L = Launch(c, [keys[1], keys[0]])
    assert L.run() == (1, 1)
    assert np.array_equal(c.state, before), "an insert took a second way beside a BUSY way of the key's fingerprint"
    assert c.stats[5] == 0
    c.force(mine, busy=False)
    assert Launch(c, [keys[1]]).lookup() == (0, 1)


@pytest.mark.parametrize("fam", [0, 2])
def test_busy_way_of_another_key_is_passed_or_given_up(hs, fam):
    c = Cache(hs, fam, sets=1)
    keys = keys_in_set(c, 17, seed=35 + fam)
    c.force(0, busy=True, fp=0x2BCDE << 32)
    assert Launch(c, keys[:1]).run() == (1, 0)
    assert c.ways[1].key == keys[0]
    for i in range(2, 16):
        c.force(i, busy=True, fp=(0x100 + i) << 32)
    assert Launch(c, keys[1:2]).run() == (1, 0)  # way 1 is the launch before's: it is replaced
    assert c.ways[1].key == keys[1] and int(c.stats[4]) == 1
    assert Launch(c, [keys[1], keys[2]]).run() == (1, 1)  # way 1 used by this launch, the rest BUSY: given up
    assert int(c.stats[5]) == 1


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_aba_fingerprint_over_other_key_words_is_a_miss(hs, fam):
    """A READY way with the key's fingerprint but another key's words (evicted and refilled between a lookup's read and
    its pin, or a fingerprint collision): the lookup pins it, compares, misses and unpins; the insert takes another way."""
    c = Cache(hs, fam, sets=2)
    key = make_keys(fam, 1, seed=40 + fam)[0]
    twin = key[:-1] + bytes([key[-1] ^ 0x80])
    _, fp = c.where(key)
    w0 = c.set_ways(key)[0]
    c.force(w0, key=twin, fp=fp, stamp=0)
    c.want[1] = c.stats[1] = 1
    assert Launch(c, [key]).run() == (1, 0)
    assert c.ways[w0].key == twin and c.ways[w0].pins == 0, "the pin of a mismatched way was not released"
    assert c.ways[w0 + 1].key == key
    assert Launch(c, [key]).lookup() == (0, 1)


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_invalid_keys_are_never_inserted(hs, fam):
    c = Cache(hs, fam, sets=2)
    keys = make_keys(fam, 6, seed=60 + fam)
    bad = {keys[1], keys[4]}
    for _ in range(3):
        m, h = Launch(c, keys, invalid=bad).run()
    assert (m, h) == (2, 4)
    assert c.stats.tolist() == [0, 4, 8, 4, 0, 0]
    assert not bad & c.resident()


def test_keys_differing_in_one_byte_are_distinct(hs):
    c = Cache(hs, 2, sets=2)
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


@pytest.mark.parametrize("fam", [0, 2])
def test_key_count_clamped_to_table_slots(hs, fam):
    c = Cache(hs, fam, sets=2)
    keys = make_keys(fam, 6, seed=70 + fam)
    Launch(c, keys[:2]).run()
    assert Launch(c, keys, kcap=4, nkeys=9).run() == (2, 2)
    assert c.resident() == set(keys[:4])


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_admission_is_sum_of_min_count_and_ways(hs, fam):
    """One launch of c_b keys per set b admits exactly sum(min(c_b, 16)); over a cache full of other keys, the next launch
    of the same keys hits exactly that many, and a fresh set of keys evicts only what the launch does not use."""
    c = Cache(hs, fam, sets=4)
    a = make_keys(fam, 64, seed=90 + fam)
    cnt = np.bincount([c.where(k)[0] for k in a], minlength=4)
    assert cnt.max() > WAYS > cnt.min()  # some sets overflow, some do not
    adm = int(np.minimum(cnt, WAYS).sum())
    assert Launch(c, a).run() == (64, 0)
    assert int(c.stats[1]) == adm and int(c.stats[5]) == 64 - adm
    b = make_keys(fam, 70, seed=190 + fam)
    cb = np.bincount([c.where(k)[0] for k in b], minlength=4)
    want = int(np.minimum(cb, WAYS).sum())
    assert Launch(c, b).run() == (70, 0)
    assert Launch(c, b).run() == (70 - want, want)
    assert len(c.resident() & set(b)) == want


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_python_set_function_matches_the_kernel(hs, fam):
    """tests/kca_sets.py, which the GPU tests use to predict per-set counts, agrees with kca_base."""
    import kca_sets
    for sets in (1, 3, 16, 1000):
        c = Cache(hs, fam, sets=1, seed=0x1234567 + fam)
        c.sets = sets
        for key in make_keys(fam, 40, seed=300 + fam):
            assert kca_sets.kca_set(key, c.seed, sets) == c.where(key)[0]


@pytest.mark.parametrize("fam", [0, 1, 2])
def test_two_launches_insert_overlapping_keys(hs, fam):
    """Both launches look up before either inserts, so both miss the shared keys; the second insert finds them READY and
    takes no second way (uncounted), then every key hits once."""
    c = Cache(hs, fam, sets=4)
    keys = make_keys(fam, 12, seed=130 + fam)
    a, b = Launch(c, keys[:8]), Launch(c, keys[4:])
    assert a.lookup() == (8, 0)
    assert b.lookup() == (8, 0)
    a.build_and_insert()
    b.build_and_insert()
    assert c.stats.tolist() == [0, 12, 0, 16, 0, 0]
    assert Launch(c, keys).run() == (0, 12)
