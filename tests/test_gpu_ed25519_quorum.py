"""Ed25519 commit votes verified and counted in one call on the H100: sbv_ed25519_verify_quorum against OpenSSL (ok) and
oracle.ecdsa_ref.count_commit_votes_batch (valid_count, reached), and against the two-call form
(sbv_ed25519_verify_registered + sbv_quorum).  Streams come from oracle_ed25519.votes."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_ed25519 as oe
from oracle import ecdsa_ref
from oracle_ed25519 import corpus, ref, votes

pytestmark = pytest.mark.gpu

N, Q = 16, 11
THR = Q - 1


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


@pytest.fixture(scope="module")
def keys():
    return votes.consenter_keys(N, 901)


def _run(eng, st, thr=THR, self_id="stream"):
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    return eng.ed25519_verify_quorum(st["msgs"], st["off"], st["key_slot"], st["sig"], st["instance"], st["sender"], st["signer"],
                                     st["digest_match"], st["n_instances"], thr, self_id=sid)


def _same(got, want):
    for g, w, name in zip(got, want, ("ok", "valid_count", "reached")):
        assert np.array_equal(g, w), (name, np.flatnonzero(g != w)[:20])


def test_c4_shape(eng, keys):
    """N = 16, Q = 11: 17,476 instances x 15 votes + 4 inert votes = 262,144 votes."""
    st = votes.make_stream(17476, N, seed=1, pad=4, keys=keys)
    assert st["instance"].size == 262144
    eng.ed25519_set_keys(st["pub"])
    got = _run(eng, st)
    want = votes.expected(st, THR)
    _same(got, want)
    ok = got[0]
    for c in (votes.BAD_SIG, votes.INERT):
        assert not ok[st["cls"] == c].any()
    assert ok[st["cls"] == votes.HONEST].all()
    # the two-call form gives the same outputs
    ok2 = eng.ed25519_verify_registered(st["msgs"], st["off"], st["key_slot"], st["sig"])
    cnt2, reached2 = eng.quorum(st["instance"], st["sender"], st["signer"], st["digest_match"], ok2, st["n_instances"], THR, self_id=st["self_id"])
    _same(got, (ok2, cnt2, reached2))


def _resign(st, i, slot, seeds):
    st["key_slot"][i] = slot
    st["sig"][i] = oe.sign_batch(seeds, np.array([slot], np.uint32), st["msgs"], st["off"][i:i + 2])[0]


def test_ed25519_classes_inside_votes(eng, keys):
    st = votes.make_stream(40, N, seed=2, byzantine=False, keys=keys)
    seeds, pubs = keys
    small = corpus.small_order_encodings()[0]
    undecodable = corpus.off_curve_encodings(np.random.default_rng(3), 1)[0]
    identity = (1).to_bytes(32, "little")
    registry = np.concatenate([pubs, np.frombuffer(small + undecodable + identity, np.uint8).reshape(3, 32)])
    S_SMALL, S_BAD, S_ID = N, N + 1, N + 2
    per = N - 1
    at = lambda inst, pos: inst * per + pos  # noqa: E731
    # S >= L
    a = at(0, 0)
    s = int.from_bytes(bytes(st["sig"][a, 32:]), "little") + ref.L
    st["sig"][a, 32:] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
    # R' = O under the identity key: the canonical R accepts, the non-canonical encodings reject
    rs = [identity, (1 + ref.p).to_bytes(32, "little"), (1 | 1 << 255).to_bytes(32, "little")]
    for k, R in enumerate(rs):
        i = at(1, k)
        st["key_slot"][i] = S_ID
        st["sig"][i] = np.frombuffer(R + bytes(32), np.uint8)
    # a small-order key and a key that does not decode, registered for a consenter: the vote rejects but burns the
    # sender's slot, so a later valid vote of the same sender (under its real key) is verified yet not counted
    burnt = []
    for inst, bad_slot in ((2, S_SMALL), (3, S_BAD)):
        i, j = at(inst, 0), at(inst, 5)
        st["key_slot"][i] = bad_slot
        st["sender"][j] = st["signer"][j] = st["sender"][i]
        _resign(st, j, int(st["sender"][i]) - 1, seeds)
        burnt.append((inst, i, j))
    # unknown slots
    for k, slot in enumerate((registry.shape[0], registry.shape[0] + 7, 2**32 - 1)):
        st["key_slot"][at(4, k)] = slot
    eng.ed25519_set_keys(registry)
    got = _run(eng, st)
    want = votes.expected(st, THR, registry=registry)
    _same(got, want)
    ok, cnt, _ = got
    assert not ok[a] and ok[at(1, 0)] and not ok[at(1, 1)] and not ok[at(1, 2)]
    assert not ok[at(4, 0): at(4, 3)].any()
    full = per  # every vote of an untouched instance is valid
    assert cnt[5] == full and cnt[0] == full - 1 and cnt[1] == full - 2 and cnt[4] == full - 3
    for inst, i, j in burnt:
        assert not ok[i] and ok[j]
        assert cnt[inst] == full - 2  # the rejected vote and the vote its sender's burnt slot left out
    # an empty registry: every vote rejects and every count is 0
    eng.ed25519_set_keys(np.zeros(0, np.uint8))
    ok, cnt, reached = _run(eng, st)
    assert not ok.any() and not cnt.any() and not reached.any()
    ok, cnt, reached = _run(eng, st, thr=0)
    assert reached.all()


@pytest.fixture(scope="module")
def small_stream(keys):
    return votes.make_stream(160, N, seed=4, pad=3, keys=keys)


def test_self_id_and_thresholds(eng, small_stream):
    st = small_stream
    eng.ed25519_set_keys(st["pub"])
    _same(_run(eng, st, self_id=None), votes.expected(st, THR, self_id=None))
    sid = np.full(st["n_instances"], 3, np.uint16)
    _same(_run(eng, st, self_id=sid), votes.expected(st, THR, self_id=sid))
    prev = None
    for thr in (0, 1, 5, 9, 10, 11, 14, 15, 16, 2**32 - 1):
        got = _run(eng, st, thr=thr)
        _same(got, votes.expected(st, thr))
        if prev is not None:
            assert np.array_equal(got[1], prev[1]) and (got[2] <= prev[2]).all()
        prev = got
    assert prev[2].sum() == 0


def test_instances_without_votes(eng, small_stream):
    st = dict(small_stream)
    I = st["n_instances"]
    st["instance"] = st["instance"] * 3 + 1  # instances 0, 2, 3, 5, ... and the last one, 3I, hold no votes
    st["n_instances"] = 3 * I + 1
    sid = np.zeros(3 * I + 1, np.uint16)
    sid[np.arange(I) * 3 + 1] = small_stream["self_id"]
    st["self_id"] = sid
    eng.ed25519_set_keys(st["pub"])
    got = _run(eng, st)
    _same(got, votes.expected(st, THR))
    assert got[1][0] == 0 and got[1][-1] == 0 and got[2][0] == 0


def test_no_votes_and_no_instances(eng):
    import consensus_b200 as sbv
    e0 = np.zeros(0)
    for thr in (0, 3):
        ok, cnt, reached = eng.ed25519_verify_quorum(e0, np.zeros(1, np.uint64), e0, e0, e0, e0, e0, e0, 5, thr)
        assert ok.size == 0 and not cnt.any() and np.array_equal(reached, np.full(5, thr == 0, np.uint8))
    ok, cnt, reached = eng.ed25519_verify_quorum(e0, np.zeros(1, np.uint64), e0, e0, e0, e0, e0, e0, 0, 0)
    assert ok.size == cnt.size == reached.size == 0
    # n_instances = 0 touches nothing, not even NULL outputs; n_votes = 0 needs no vote buffers
    lib = sbv.load_library()
    assert lib.sbv_ed25519_verify_quorum(eng._h, C.c_size_t(4), *([None] * 8), C.c_size_t(0), None, C.c_uint32(0), None, None, None) == 0
    cnt = np.full(3, 7, np.uint32)
    reached = np.full(3, 7, np.uint8)
    assert lib.sbv_ed25519_verify_quorum(eng._h, C.c_size_t(0), *([None] * 8), C.c_size_t(3), None, C.c_uint32(1), None, _p(cnt), _p(reached)) == 0
    assert not cnt.any() and not reached.any()


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_empty_messages_with_null_msgs(eng, keys):
    seeds, pubs = keys
    I, per = 6, N - 1
    inst = np.repeat(np.arange(I, dtype=np.uint32), per)
    sender = np.tile(np.arange(2, N + 1, dtype=np.uint16), I)
    off = np.zeros(I * per + 1, np.uint64)
    slot = sender.astype(np.uint32) - 1
    sig = oe.sign_batch(seeds, slot, np.zeros(1, np.uint8), off)
    sig[3, 40] ^= 1
    dm = np.ones(I * per, np.uint8)
    st = {"msgs": np.zeros(0, np.uint8), "off": off, "sig": sig, "key_slot": slot, "instance": inst, "sender": sender, "signer": sender.copy(),
          "digest_match": dm, "self_id": np.ones(I, np.uint16), "n_instances": I, "pub": pubs}
    eng.ed25519_set_keys(pubs)
    want = votes.expected(st, THR)
    n = I * per
    ok, cnt, reached = np.zeros(n, np.uint8), np.zeros(I, np.uint32), np.zeros(I, np.uint8)
    eng.ed25519_verify_quorum_ptr(n, None, off.ctypes.data, slot.ctypes.data, sig.ctypes.data, inst.ctypes.data, sender.ctypes.data,
                                  sender.ctypes.data, dm.ctypes.data, I, st["self_id"].ctypes.data, THR, ok.ctypes.data, cnt.ctypes.data,
                                  reached.ctypes.data)
    _same((ok, cnt, reached), want)
    assert want[0].sum() == n - 1


def test_10KiB_messages(eng, keys):
    st = votes.make_stream(12, N, seed=5, aux_lo=10240 - 32, aux_hi=10240, keys=keys)
    eng.ed25519_set_keys(st["pub"])
    _same(_run(eng, st), votes.expected(st, THR))


@pytest.mark.parametrize("k", [1, 2, 127, 128, 129, 2047, 2048, 2049])
def test_vote_counts_around_block_sizes(eng, keys, k):
    st = _prefix_source(keys)
    sub = {key: st[key][:k] for key in ("key_slot", "sig", "instance", "sender", "signer", "digest_match")}
    sub.update(msgs=st["msgs"], off=st["off"][:k + 1], n_instances=int(st["instance"][k - 1]) + 1, self_id=st["self_id"], pub=st["pub"])
    sub["self_id"] = st["self_id"][: sub["n_instances"]]
    assert st["off"][0] % 8 != 0  # misaligned offsets
    eng.ed25519_set_keys(st["pub"])
    _same(_run(eng, sub), votes.expected(sub, THR))


_PREFIX = {}


def _prefix_source(keys):
    if not _PREFIX:
        _PREFIX.update(votes.make_stream(140, N, seed=6, keys=keys))
    return _PREFIX


def _args(st, self_id=True):
    """The 16 ctypes arguments after the engine (pointers of st's arrays) and fresh sentinel-filled outputs."""
    n, I = st["instance"].size, st["n_instances"]
    outs = (np.full(n, 0xAB, np.uint8), np.full(I, 0xABABABAB, np.uint32), np.full(I, 0xAB, np.uint8))
    a = [C.c_size_t(n), _p(st["msgs"]), _p(st["off"]), _p(st["key_slot"]), _p(st["sig"]), _p(st["instance"]), _p(st["sender"]),
         _p(st["signer"]), _p(st["digest_match"]), C.c_size_t(I), _p(st["self_id"]) if self_id else None, C.c_uint32(THR),
         _p(outs[0]), _p(outs[1]), _p(outs[2])]
    return a, outs


def test_bad_arguments_leave_outputs_untouched(eng, small_stream):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    st = small_stream
    eng.ed25519_set_keys(st["pub"])
    cases = {f"null {name}": {idx: None} for idx, name in [(1, "msgs"), (2, "msg_off"), (3, "key_slot"), (4, "sig"), (5, "instance"),
                                                          (6, "sender"), (7, "signer"), (8, "digest_match"), (12, "ok"),
                                                          (13, "valid_count"), (14, "reached")]}
    cases["n_votes >= 2^31"] = {0: C.c_size_t(2**31)}
    cases["n_instances >= 2^31"] = {9: C.c_size_t(2**31)}
    bad_off = st["off"].copy()
    bad_off[50] = bad_off[49] - 1
    cases["non-monotonic msg_off"] = {2: _p(bad_off)}
    bad_inst = st["instance"].copy()
    bad_inst[100], bad_inst[101] = bad_inst[101] + 1, bad_inst[100]
    cases["unsorted instances"] = {5: _p(bad_inst)}
    for name, repl in cases.items():
        a, outs = _args(st)
        for idx, v in repl.items():
            a[idx] = v
        assert lib.sbv_ed25519_verify_quorum(eng._h, *a) < 0, name
        assert lib.sbv_last_error(eng._h)
        for o in outs:
            assert (o.view(np.uint8) == 0xAB).all(), name
    a, outs = _args(st)  # the same buffers are accepted as they are
    assert lib.sbv_ed25519_verify_quorum(eng._h, *a) == 0
    _same(outs, votes.expected(st, THR))


def test_pinned_and_pageable_input(eng, small_stream):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    st = small_stream
    eng.ed25519_set_keys(st["pub"])
    want = votes.expected(st, THR)
    cols = ("msgs", "off", "key_slot", "sig", "instance", "sender", "signer", "digest_match", "self_id")
    ptrs = []
    pinned = {}
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
            eng.ed25519_verify_quorum_ptr(n, *(src[c].ctypes.data for c in cols[:8]), I, src["self_id"].ctypes.data, THR, ok.ctypes.data,
                                          cnt.ctypes.data, reached.ctypes.data)
            _same((ok, cnt, reached), want)
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_concurrent_callers_see_one_registry(eng, small_stream):
    """Callers on several threads while another thread alternates the registry between two key sets: every call's
    outputs are the whole outcome of one of them."""
    st = small_stream
    keys_a = st["pub"]
    keys_b = np.concatenate([keys_a[1:], keys_a[:1]])  # every slot holds another consenter's key: every vote rejects
    want_a, want_b = votes.expected(st, THR, registry=keys_a), votes.expected(st, THR, registry=keys_b)
    assert not np.array_equal(want_a[1], want_b[1])
    eng.ed25519_set_keys(keys_a)
    stop, errs, seen = threading.Event(), [], {"a": 0, "b": 0}

    def swapper():
        k = 0
        while not stop.is_set():
            k += 1
            eng.ed25519_set_keys(keys_b if k % 2 else keys_a)

    def caller():
        try:
            for _ in range(12):
                got = _run(eng, st)
                if all(np.array_equal(g, w) for g, w in zip(got, want_a)):
                    seen["a"] += 1
                elif all(np.array_equal(g, w) for g, w in zip(got, want_b)):
                    seen["b"] += 1
                else:
                    errs.append("mixed outcome")
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    sw = threading.Thread(target=swapper)
    callers = [threading.Thread(target=caller) for _ in range(4)]
    sw.start()
    for t in callers:
        t.start()
    for t in callers:
        t.join()
    stop.set()
    sw.join()
    assert not errs, errs[:5]
    assert seen["a"] + seen["b"] == 48


def test_two_device_engine_shards_by_instance(small_stream, keys):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import consensus_b200 as sbv
    big = votes.make_stream(901, N, seed=7, pad=2, keys=keys)
    I = small_stream["n_instances"]
    # votes only in the first half of the instances (device 1 holds none), then only in the second (device 0 holds none)
    lo_half = dict(small_stream, n_instances=2 * I, self_id=np.concatenate([small_stream["self_id"], np.ones(I, np.uint16)]))
    hi_half = dict(lo_half, instance=small_stream["instance"] + np.uint32(I), self_id=np.concatenate([np.ones(I, np.uint16), small_stream["self_id"]]))
    streams = [big, lo_half, hi_half]
    with sbv.Engine(devices=[0]) as e1:
        e1.ed25519_set_keys(keys[1])
        single = [_run(e1, s) for s in streams]
    with sbv.Engine(n_devices=2) as e2:
        e2.ed25519_set_keys(keys[1])
        for _ in range(2):
            for s, want in zip(streams, single):
                _same(_run(e2, s), want)
    _same(single[0], votes.expected(big, THR))
    _same(single[1], votes.expected(lo_half, THR))
    assert not single[1][1][I:].any() and not single[2][1][:I].any()


def test_count_rule_matches_the_python_restatement(small_stream):
    """The oracle's count is the one the tests above compare with: spot-check it against a direct VoteSet restatement."""
    st = small_stream
    ok = np.ones(st["instance"].size, np.uint8)
    cnt, _ = ecdsa_ref.count_commit_votes_batch(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"], THR,
                                                st["self_id"])
    for i in range(5):
        m = st["instance"] == i
        seen, valid = set(), 0
        for s, g, d in zip(st["sender"][m], st["signer"][m], st["digest_match"][m]):
            if s == st["self_id"][i] or s != g or s in seen:
                continue
            seen.add(s)
            valid += int(d)
        assert cnt[i] == valid
