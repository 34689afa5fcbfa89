"""The host-side shard arithmetic of a multi-device engine (consensus_b200/csrc/shards.h, compiled into the CPU
simulation) against consensus_b200/sharding.py: the contiguous split of a batch, the split of commit votes by instance,
the words per device slot and the unpack of the gathered words.  On a machine with fewer than two GPUs this is the only
check these functions get."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from consensus_b200 import sharding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _shards(hs, votes, n, instance, n_instances, G):
    ranges = np.zeros((G, 4), np.uint64)
    words = np.zeros(2, np.uint64)
    inst = _p(instance, C.c_uint32) if instance is not None else None
    assert hs.hs_shards(C.c_int(votes), C.c_size_t(n), inst, C.c_size_t(n_instances), C.c_int(G), _p(ranges, C.c_size_t), _p(words, C.c_size_t)) == 0
    return ranges.astype(np.int64), int(words[0]), int(words[1])


def _unpack(hs, votes, n, instance, n_instances, G, gathered, ok_len):
    ok = np.full(ok_len, 7, np.uint8)
    reached = np.full(max(n_instances, 1), 7, np.uint8)
    inst = _p(instance, C.c_uint32) if instance is not None else None
    assert hs.hs_unpack_shards(C.c_int(votes), C.c_size_t(n), inst, C.c_size_t(n_instances), C.c_int(G), _p(gathered, C.c_uint32),
                               _p(ok, C.c_uint8), _p(reached, C.c_uint8)) == 0
    return ok, reached[:n_instances]


def _gathered(parts, wv, wi):
    """the all-gathered buffer: device g's slot is its verdict bits in wv words, then its reached bits in wi words
    (k_pack_bits layout, which test_hostsim.py checks against sharding.pack_bits)"""
    slots = []
    for ok_bits, rch_bits in parts:
        slots.append(sharding.pack_bits(ok_bits, wv))
        if wi:
            slots.append(sharding.pack_bits(rch_bits, wi))
    return np.ascontiguousarray(np.concatenate(slots).astype(np.uint32))


@pytest.mark.parametrize("G", range(1, 9))
def test_batch_shards(hs, G):
    rng = np.random.default_rng(G)
    for n in [1, 2, 3, 5, 7, 8, 31, 32, 33, 255, 1003, 4097, 65537]:
        ranges, wv, wi = _shards(hs, 0, n, None, 0, G)
        for g in range(G):
            lo, hi = sharding.shard_range(n, g, G)
            assert list(ranges[g]) == [lo, hi - lo, 0, 0], (n, g)
        assert wv == sharding.words_per_shard(n, G) and wi == 0, n
        ok = (rng.random(n) < 0.6).astype(np.uint8)
        gathered = _gathered([(ok[lo:lo + cnt], None) for lo, cnt, _, _ in ranges], wv, 0)
        got, _ = _unpack(hs, 0, n, None, 0, G, gathered, n)
        assert np.array_equal(got, ok), n
        for g, (lo, cnt, _, _) in enumerate(ranges):  # each slot as sharding.unpack_bits reads it
            assert np.array_equal(sharding.unpack_bits(gathered[wv * g: wv * (g + 1)], cnt), ok[lo:lo + cnt])


def _vote_streams(rng, G):
    """(instance ids, n_instances): uneven instances, instances (and whole devices) without votes, fewer instances than
    devices, no votes at all, and trailing ids out of range"""
    out = []
    for n_instances in sorted({1, max(G - 1, 1), G, G + 1, 3 * G + 2, 100, 257}):
        per = rng.integers(0, 70, n_instances)
        per[rng.random(n_instances) < 0.3] = 0
        out.append((np.repeat(np.arange(n_instances), per).astype(np.uint32), n_instances))
        # the first devices' instances hold no votes at all
        late = per.copy()
        late[: n_instances // 2 + 1] = 0
        out.append((np.repeat(np.arange(n_instances), late).astype(np.uint32), n_instances))
        # trailing padding votes with ids >= n_instances
        pad = np.concatenate([np.repeat(np.arange(n_instances), per), np.full(5, n_instances), np.full(3, n_instances + 40)])
        out.append((pad.astype(np.uint32), n_instances))
    out.append((np.zeros(0, np.uint32), 5))
    return out


@pytest.mark.parametrize("G", range(1, 9))
def test_quorum_shards(hs, G):
    rng = np.random.default_rng(100 + G)
    for inst, n_instances in _vote_streams(rng, G):
        n = inst.size
        ranges, wv, wi = _shards(hs, 1, n, inst, n_instances, G)
        for g in range(G):
            vlo, vhi, ilo, ihi, _ = sharding.shard_votes(inst, n_instances, g, G)
            assert list(ranges[g]) == [vlo, vhi - vlo, ilo, ihi - ilo], (n, n_instances, g)
        assert ranges[:, 1].sum() == n  # every vote has one device
        assert wv == max((int(c) + 31) // 32 for c in ranges[:, 1])
        assert wi == max((int(c) + 31) // 32 for c in ranges[:, 3])
        ok = (rng.random(n) < 0.6).astype(np.uint8)
        reached = (rng.random(n_instances) < 0.5).astype(np.uint8)
        parts = [(ok[vlo:vlo + nv], reached[ilo:ilo + ni]) for vlo, nv, ilo, ni in ranges]
        got_ok, got_rch = _unpack(hs, 1, n, inst, n_instances, G, _gathered(parts, wv, wi), max(n, 1))
        assert np.array_equal(got_ok[:n], ok) and np.array_equal(got_rch, reached), (n, n_instances)
