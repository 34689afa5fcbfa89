"""RSA commit votes verified and counted in one call on the H100: sbv_rsa_verify_quorum and sbv_rsa_pss_verify_quorum over
registered consenter keys of every modulus size, against oracle_rsa.ref (ok) and oracle.ecdsa_ref.count_commit_votes_batch
(valid_count, reached), and against the two-call form (sbv_rsa_hash_verify_registered per key size + sbv_quorum).  Streams
come from tests/rsa_quorum_cases.py; the CPU twin of this file is test_hostsim_rsa_quorum.py."""
import ctypes as C
import threading

import numpy as np
import pytest

import rsa_quorum_cases as q
from oracle_rsa import ref

pytestmark = pytest.mark.gpu

THR = 10  # N = 16, Q = 11


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


@pytest.fixture(scope="module")
def cons():
    return q.Consenters(q.MIXED)


def set_reg(eng, cons, reg):
    mb, mods, exp = cons.arrays(reg)
    eng.rsa_set_keys(mb, mods, exp)


def run(eng, st, thr=THR, self_id="stream", salt_len=None):
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    args = (st["msgs"], st["off"], st["key_slot"], st["sig"], st["sig_off"], st["instance"], st["sender"], st["signer"], st["digest_match"],
            st["n_instances"], thr)
    if salt_len is None:
        return eng.rsa_verify_quorum(st["hash"], *args, self_id=sid)
    return eng.rsa_pss_verify_quorum(st["hash"], salt_len, *args, self_id=sid)


def same(got, want):
    for g, w, name in zip(got, want, ("ok", "valid_count", "reached")):
        assert np.array_equal(g, w), (name, np.flatnonzero(g != w)[:20])


def two_calls(eng, st, thr=THR, salt_len=None):
    """Per key size, the votes of that signature length through the registered fused call, then sbv_quorum."""
    lens = np.diff(st["sig_off"].astype(np.int64))
    ok = np.zeros(lens.size, np.uint8)
    for k in q.SIZES:
        idx = np.flatnonzero(lens == k)
        if not idx.size:
            continue
        msgs, off = q.blob([st["msgs_l"][i] for i in idx])
        sig = np.frombuffer(b"".join(st["sigs_l"][i] for i in idx), np.uint8)
        if salt_len is None:
            ok[idx] = eng.rsa_hash_verify_registered(st["hash"], msgs, off, st["key_slot"][idx], sig)
        else:
            ok[idx] = eng.rsa_pss_hash_verify_registered(st["hash"], salt_len, msgs, off, st["key_slot"][idx], sig)
    cnt, reached = eng.quorum(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"], thr, self_id=st["self_id"])
    return ok, cnt, reached


def test_c4_shape(eng, cons):
    """N = 16 (ten 2048-bit, four 3072-bit, two 4096-bit keys), Q = 11: 17,476 instances x 15 votes + 4 inert votes = 262,144
    votes, SHA-256, PKCS #1 v1.5."""
    st = q.pack(q.make_stream(cons, 17476, seed=1, pad=4))
    assert st["instance"].size == 262144
    set_reg(eng, cons, cons.reg)
    got = run(eng, st)
    same(got, q.expected(cons.reg, st, THR))
    ok = got[0]
    for c in (q.BAD_SIG, q.INERT):
        assert not ok[st["cls"] == c].any()
    assert ok[st["cls"] == q.HONEST].all()
    same(got, two_calls(eng, st))


@pytest.mark.parametrize("hash", [ref.SHA256, ref.SHA384, ref.SHA512])
def test_pss_every_hash_and_salt_mode(eng, cons, hash):
    hl = ref.HLEN[hash]
    st = q.pack(q.make_stream(cons, 48, seed=2 + hash, hash=hash, salt_bytes=hl, pad=3))
    set_reg(eng, cons, cons.reg)
    for salt_len in (ref.SALT_EQUALS_HASH, ref.SALT_AUTO, hl, hl - 1):
        got = run(eng, st, salt_len=salt_len)
        same(got, q.expected(cons.reg, st, THR, salt_len=salt_len))
        assert got[0].any() == (salt_len != hl - 1)
        same(got, two_calls(eng, st, salt_len=salt_len))


@pytest.mark.parametrize("pss", [False, True])
def test_vote_classes(eng, cons, pss):
    reg, st = q.edge_stream(cons, salt=32 if pss else None)
    st = q.pack(st)
    salt_len = ref.SALT_AUTO if pss else None
    set_reg(eng, cons, reg)
    got = run(eng, st, salt_len=salt_len)
    same(got, q.expected(reg, st, THR, salt_len=salt_len))
    ok = got[0]
    assert ok[-1] and not ok[-2]  # the valid vote after its sender's rejected one: verified, not counted
    same(got, q.expected(reg, st, THR, salt_len=salt_len))
    # an empty registry: every vote rejects and every count is 0
    set_reg(eng, cons, [])
    ok, cnt, reached = run(eng, st, salt_len=salt_len)
    assert not ok.any() and not cnt.any() and not reached.any()
    ok, cnt, reached = run(eng, st, thr=0, salt_len=salt_len)
    assert reached.all()


@pytest.fixture(scope="module")
def small(cons):
    return q.pack(q.make_stream(cons, 160, seed=4, pad=3))


def test_self_id_and_thresholds(eng, cons, small):
    st = small
    set_reg(eng, cons, cons.reg)
    same(run(eng, st, self_id=None), q.expected(cons.reg, st, THR, self_id=None))
    sid = np.full(st["n_instances"], 3, np.uint16)
    same(run(eng, st, self_id=sid), q.expected(cons.reg, st, THR, self_id=sid))
    for thr in (0, 1, 9, 10, 11, 15, 16, 2**32 - 1):
        same(run(eng, st, thr=thr), q.expected(cons.reg, st, thr))


def test_instances_without_votes(eng, cons, small):
    st = dict(small)
    I = st["n_instances"]
    st["instance"] = st["instance"] * 3 + 1
    st["n_instances"] = 3 * I + 1
    sid = np.zeros(3 * I + 1, np.uint16)
    sid[np.arange(I) * 3 + 1] = small["self_id"]
    st["self_id"] = sid
    set_reg(eng, cons, cons.reg)
    got = run(eng, st)
    same(got, q.expected(cons.reg, st, THR))
    assert got[1][0] == 0 and got[1][-1] == 0


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_no_votes_and_no_instances(eng):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    cnt = np.full(3, 7, np.uint32)
    reached = np.full(3, 7, np.uint8)
    assert lib.sbv_rsa_verify_quorum(eng._h, C.c_uint8(0), C.c_size_t(0), *([None] * 9), C.c_size_t(3), None, C.c_uint32(1), None, _p(cnt),
                                     _p(reached)) == 0
    assert not cnt.any() and not reached.any()
    assert lib.sbv_rsa_pss_verify_quorum(eng._h, C.c_uint8(0), C.c_int32(0), C.c_size_t(4), *([None] * 9), C.c_size_t(0), None, C.c_uint32(0),
                                         None, None, None) == 0


@pytest.mark.parametrize("k", [1, 15, 16, 17, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049])
def test_vote_counts_around_block_sizes(eng, cons, k):
    src = _prefix_source(cons)
    sub = q.take(src, k)
    sub["n_instances"] = int(sub["instance"][k - 1]) + 1
    sub["self_id"] = src["self_id"][:sub["n_instances"]]
    sub = q.pack(sub)
    set_reg(eng, cons, cons.reg)
    same(run(eng, sub), q.expected(cons.reg, sub, THR))


_PREFIX = {}


def _prefix_source(cons):
    if not _PREFIX:
        _PREFIX.update(q.make_stream(cons, 140, seed=6))
    return _PREFIX


def _args(st, hash=0, salt=None):
    """The ctypes arguments after the engine and fresh sentinel-filled outputs (index 0: hash; PSS: 1 = salt_len)."""
    n, I = st["instance"].size, st["n_instances"]
    outs = (np.full(n, 0xAB, np.uint8), np.full(I, 0xABABABAB, np.uint32), np.full(I, 0xAB, np.uint8))
    a = [C.c_uint8(hash)] + ([] if salt is None else [C.c_int32(salt)])
    a += [C.c_size_t(n), _p(st["msgs"]), _p(st["off"]), _p(st["key_slot"]), _p(st["sig"]), _p(st["sig_off"]), _p(st["instance"]), _p(st["sender"]),
          _p(st["signer"]), _p(st["digest_match"]), C.c_size_t(I), _p(st["self_id"]), C.c_uint32(THR), _p(outs[0]), _p(outs[1]), _p(outs[2])]
    return a, outs


def test_bad_arguments_leave_outputs_untouched(eng, cons, small):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    st = small
    set_reg(eng, cons, cons.reg)
    bad_sig_off = st["sig_off"].copy()
    bad_sig_off[50] = bad_sig_off[49] - 1
    bad_off = st["off"].copy()
    bad_off[50] = bad_off[49] - 1
    bad_inst = st["instance"].copy()
    bad_inst[100], bad_inst[101] = bad_inst[101] + 1, bad_inst[100]
    cases = {"non-monotonic sig_off": (lib.sbv_rsa_verify_quorum, None, {6: _p(bad_sig_off)}),
             "null sig with signatures": (lib.sbv_rsa_verify_quorum, None, {5: None}),
             "null sig_off": (lib.sbv_rsa_verify_quorum, None, {6: None}),
             "non-monotonic msg_off": (lib.sbv_rsa_verify_quorum, None, {3: _p(bad_off)}),
             "null key_slot": (lib.sbv_rsa_verify_quorum, None, {4: None}),
             "unsorted instances": (lib.sbv_rsa_verify_quorum, None, {7: _p(bad_inst)}),
             "n_votes >= 2^31": (lib.sbv_rsa_verify_quorum, None, {1: C.c_size_t(2**31)}),
             "hash tag 3": (lib.sbv_rsa_verify_quorum, None, {0: C.c_uint8(3)}),
             "PSS hash tag 3": (lib.sbv_rsa_pss_verify_quorum, 0, {0: C.c_uint8(3)}),
             "salt_len -2": (lib.sbv_rsa_pss_verify_quorum, 0, {1: C.c_int32(-2)})}
    for name, (fn, salt, repl) in cases.items():
        a, outs = _args(st, salt=salt)
        for idx, v in repl.items():
            a[idx] = v
        assert fn(eng._h, *a) < 0, name
        assert lib.sbv_last_error(eng._h)
        for o in outs:
            assert (o.view(np.uint8) == 0xAB).all(), name
    a, outs = _args(st)
    assert lib.sbv_rsa_verify_quorum(eng._h, *a) == 0
    same(outs, q.expected(cons.reg, st, THR))


def test_pinned_and_pageable_input(eng, cons, small):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    st = small
    set_reg(eng, cons, cons.reg)
    want = q.expected(cons.reg, st, THR)
    cols = ("msgs", "off", "key_slot", "sig", "sig_off", "instance", "sender", "signer", "digest_match", "self_id")
    ptrs, pinned = [], {}
    try:
        for c in cols:
            a = np.ascontiguousarray(st[c])
            p = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
            assert p
            ptrs.append(p)
            view = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(p)).view(a.dtype).reshape(a.shape)
            view[...] = a
            pinned[c] = view
        for src in (pinned, {c: np.ascontiguousarray(st[c]) for c in cols}):
            n, I = st["instance"].size, st["n_instances"]
            ok, cnt, reached = np.zeros(n, np.uint8), np.zeros(I, np.uint32), np.zeros(I, np.uint8)
            eng.rsa_verify_quorum_ptr(st["hash"], n, *(src[c].ctypes.data for c in cols[:9]), I, src["self_id"].ctypes.data, THR, ok.ctypes.data,
                                      cnt.ctypes.data, reached.ctypes.data)
            same((ok, cnt, reached), want)
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_concurrent_callers_while_the_registry_changes(eng, cons, small):
    """Callers on four threads while a fifth swaps the registry between the consenters' keys and the same keys in reverse
    slot order: every outcome is the whole outcome of one of the two registries."""
    st = small
    rev = list(reversed(cons.reg))
    wants = [q.expected(cons.reg, st, THR), q.expected(rev, st, THR)]
    assert not np.array_equal(wants[0][0], wants[1][0])
    set_reg(eng, cons, cons.reg)
    stop = threading.Event()
    errors, seen = [], set()

    def caller():
        try:
            for _ in range(12):
                got = run(eng, st)
                hit = [i for i, w in enumerate(wants) if all(np.array_equal(g, x) for g, x in zip(got, w))]
                assert hit, "an outcome that mixes registries"
                seen.add(hit[0])
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def swapper():
        i = 0
        while not stop.is_set():
            i += 1
            set_reg(eng, cons, rev if i % 2 else cons.reg)

    ts = [threading.Thread(target=caller) for _ in range(4)]
    sw = threading.Thread(target=swapper)
    sw.start()
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    stop.set()
    sw.join()
    assert not errors, errors[0]


def test_two_devices_shard_by_instance(cons):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import consensus_b200 as sbv
    st = q.pack(q.make_stream(cons, 301, seed=8, pad=2))
    with sbv.Engine(devices=[0, 1]) as e2:
        set_reg(e2, cons, cons.reg)
        same(run(e2, st), q.expected(cons.reg, st, THR))
        same(run(e2, st, salt_len=None, self_id=None), q.expected(cons.reg, st, THR, self_id=None))
