"""RSA commit votes in the CPU simulation (tools/hostsim): hs_rsa_quorum_shard runs the device part of one shard of
sbv_rsa_verify_quorum -- each vote's family from its signature's length (rsa_shard.h: rsa_family), k_mix_count, k_mix_scan,
k_rsa_split, k_mix_compact, rsa_launch_shard per key size over a registry built by k_rsa_kprep, and k_mix_ok -- and hs_quorum
counts its verdicts as k_quorum_count / k_quorum_reached do.

- every verdict against oracle_rsa.ref, all three key sizes in one shard, for both paddings: votes of the lengths k - 1,
  k + 1 and 0, a signature whose length is not its slot's size but which the slot, read at the signature's size, would
  accept (rsa_registered.size_trap), unknown slots and a slot whose key fails the key rule;
- shards where one family is empty and where only one is present, and vote counts at the edges of the split's tiles;
- the counts against oracle.ecdsa_ref.count_commit_votes_batch.
The GPU twin of this file is test_gpu_rsa_quorum.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rsa_quorum_cases as q
from oracle_rsa import ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
THR = 10


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def kprep(hs, cons, reg):
    mb, mods, exp = cons.arrays(reg)
    n = len(reg)
    rec = np.zeros(max(8 * n, 8), np.uint32)
    pool = np.zeros(max(int(mb.sum()) // 2, 1), np.uint32)
    if n:
        assert hs.hs_rsa_kprep(C.c_size_t(n), _p(mb), _p(mods), _p(exp), _p(rec), _p(pool)) == 0
    return n, rec, pool


def run(hs, cons, reg, st, salt_len=None, self_id="stream", thr=THR):
    """(ok, valid_count, reached) of one shard in the simulation."""
    st = q.pack(st)
    n = len(st["sigs_l"])
    hl = ref.HLEN[st["hash"]]
    digest = np.frombuffer(b"".join(ref.HASHLIB[st["hash"]](m).digest() for m in st["msgs_l"]) + b"\0", np.uint8)[:n * hl].copy()
    nslots, rec, pool = kprep(hs, cons, reg)
    ok = np.full(n, 7, np.uint8)
    rc = hs.hs_rsa_quorum_shard(C.c_uint8(st["hash"]), C.c_int(salt_len is not None), C.c_int32(salt_len or 0), C.c_size_t(n), _p(digest),
                                _p(st["key_slot"]), _p(st["sig"]), _p(st["sig_off"]), C.c_uint32(nslots), _p(rec), _p(pool), _p(ok))
    assert rc == 0
    I = st["n_instances"]
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    cnt = np.full(I, 9, np.uint32)
    reached = np.full(I, 9, np.uint8)
    assert hs.hs_quorum(C.c_size_t(n), _p(st["instance"]), _p(st["sender"]), _p(st["signer"]), _p(st["digest_match"]), _p(ok),
                        _p(None if sid is None else np.ascontiguousarray(sid, np.uint16)), C.c_uint32(0), C.c_size_t(I), C.c_uint32(thr), _p(cnt),
                        _p(reached)) == 0
    return ok, cnt, reached


def check(hs, cons, reg, st, salt_len=None, **kw):
    got = run(hs, cons, reg, st, salt_len, **kw)
    want = q.expected(reg, st, kw.get("thr", THR), kw.get("self_id", "stream"), salt_len)
    for g, w, name in zip(got, want, ("ok", "valid_count", "reached")):
        assert np.array_equal(g, w), (name, np.flatnonzero(g != w)[:20])
    return got


@pytest.fixture(scope="module")
def cons():
    return q.Consenters(q.MIXED)


def test_edges_mixed_sizes_pkcs1(hs, cons):
    reg, st = q.edge_stream(cons)
    ok, _, _ = check(hs, cons, reg, st)
    per = cons.n - 1
    tail = ok[2 * per:]
    # per size: k - 1, k + 1, 0 reject and the signature itself accepts; the size traps and the refused key reject
    assert tail[:4].tolist() == [0, 0, 0, 1] and tail[5:9].tolist() == [0, 0, 0, 1] and tail[10:14].tolist() == [0, 0, 0, 1]
    assert not tail[4] and not tail[9] and not tail[14:18].any()
    assert {len(s) for s in st["sigs_l"]} >= {0, 255, 256, 257, 383, 384, 385, 511, 512, 513}


def test_edges_mixed_sizes_pss(hs, cons):
    reg, st = q.edge_stream(cons, salt=32)
    ok, _, _ = check(hs, cons, reg, st, salt_len=ref.SALT_EQUALS_HASH)
    assert ok[:2 * (cons.n - 1)].sum() > 0
    check(hs, cons, reg, st, salt_len=ref.SALT_AUTO)
    check(hs, cons, reg, st, salt_len=31)


@pytest.mark.parametrize("n", [15, 16, 17, 33])
def test_vote_counts_at_tile_edges(hs, cons, n):
    st = q.make_stream(cons, 3, seed=10 + n)
    got = check(hs, cons, cons.reg, q.take(st, n))
    assert got[0].any()


@pytest.mark.parametrize("sizes", [(256,), (384,), (512,), (256, 512), (384, 512), (256, 384)])
def test_empty_and_lone_families(hs, cons, sizes):
    st = q.only(q.make_stream(cons, 2, seed=20), sizes)
    ok, _, _ = check(hs, cons, cons.reg, st)
    lens = np.array([len(s) for s in st["sigs_l"]])
    assert ok[lens > 0].any() and not ok[lens == 0].any()


def test_no_family_and_empty_registry(hs, cons):
    st = q.make_stream(cons, 1, seed=30)
    ok, cnt, _ = check(hs, cons, cons.reg, q.only(st, ()))
    assert not ok.any() and not cnt.any()
    ok, cnt, reached = check(hs, cons, [], st, thr=0)
    assert not ok.any() and not cnt.any() and reached.all()


def test_self_id_and_thresholds(hs, cons):
    st = q.make_stream(cons, 3, seed=40)
    check(hs, cons, cons.reg, st, self_id=None)
    for thr in (0, 14, 15):
        check(hs, cons, cons.reg, st, thr=thr)


def test_refused_calls(hs):
    z = np.zeros(1, np.uint64)
    assert hs.hs_rsa_quorum_shard(C.c_uint8(3), C.c_int(0), C.c_int32(0), C.c_size_t(0), None, None, None, _p(z), C.c_uint32(0), None, None, None) == -1
    assert hs.hs_rsa_quorum_shard(C.c_uint8(0), C.c_int(1), C.c_int32(-2), C.c_size_t(0), None, None, None, _p(z), C.c_uint32(0), None, None, None) == -1
