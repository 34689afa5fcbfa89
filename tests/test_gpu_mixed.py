"""Mixed ECDSA / Ed25519 registered-key batches and commit votes on the H100: sbv_mixed_verify_registered and
sbv_mixed_verify_quorum against OpenSSL (oracle/, oracle_ed25519/), the single-scheme calls and
oracle.ecdsa_ref.count_commit_votes_batch.  Corpora and vote streams come from tests/mixed_cases.py."""
import ctypes as C
import threading

import numpy as np
import pytest

import mixed_cases as mc
from oracle_ed25519 import votes

pytestmark = pytest.mark.gpu

N, Q = 16, 11
THR = Q - 1
C4_SCHEMES = [mc.P256] * 7 + [mc.P384] * 2 + [mc.ED] * 7


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


@pytest.fixture(scope="module")
def reg():
    return mc.registries(n256=3, n384=2, n_ed=4, seed=21)


def _set(eng, reg, ed_pub=None, ecdsa=None):
    curve, xy = ecdsa if ecdsa is not None else (reg["ecdsa_curve"], reg["ecdsa_xy"])
    eng.set_keys(curve, xy)
    eng.ed25519_set_keys(reg["ed_pub"] if ed_pub is None else ed_pub)


def _mixed(eng, cp):
    return eng.mixed_verify_registered(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"])


def _single(eng, cp):
    """The single-scheme calls, item by item family: what the mixed call must return byte for byte."""
    ok = np.zeros(cp["scheme"].size, np.uint8)
    for c in (mc.P256, mc.P384, mc.ED):
        idx = np.flatnonzero(cp["scheme"] == c)
        if idx.size == 0:
            continue
        m, o = mc.gather(cp["msgs"], cp["off"], idx)
        if c == mc.ED:
            ok[idx] = eng.ed25519_verify_registered(m, o, cp["key_slot"][idx], cp["sig96"][idx, :64])
        else:
            Lc = mc.L[c]
            ok[idx] = eng.hash_verify_registered(c, m, o, cp["key_slot"][idx], cp["sig96"][idx, :Lc], cp["sig96"][idx, Lc:2 * Lc])
    return ok


def _check(eng, cp, reg, ed_pub=None, ecdsa=None):
    curve, xy = ecdsa if ecdsa is not None else (reg["ecdsa_curve"], reg["ecdsa_xy"])
    got = _mixed(eng, cp)
    want = mc.expected_ok(cp, curve, xy, reg["ed_pub"] if ed_pub is None else ed_pub)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    assert np.array_equal(got, _single(eng, cp))
    return got


@pytest.mark.parametrize("kind", ["p256", "p384", "ed", "alternating", "random", "runs"])
def test_tag_patterns_and_corruption_classes(eng, reg, kind):
    _set(eng, reg)
    cp = mc.make_corpus(mc.tag_pattern(kind, 1500, np.random.default_rng(1)), reg, seed=2)
    got = _check(eng, cp, reg)
    assert 0 < got.sum() < got.size


def test_ed25519_classes_and_bad_registered_keys(eng, reg):
    ed_pub = reg["ed_pub"].copy()
    ed_pub[2], ed_pub[3] = mc.small_order_key(), mc.y_ge_p_key()
    _set(eng, reg, ed_pub=ed_pub)
    cp = mc.make_corpus(mc.tag_pattern("random", 2000, np.random.default_rng(3)), reg, seed=4)
    for c in (mc.S_PLUS_L, mc.NONCANON_R):
        assert (cp["cls"] == c).any()
    _check(eng, cp, reg, ed_pub=ed_pub)


def test_block_boundary_and_10KiB_messages(eng, reg):
    _set(eng, reg)
    lens = np.array([0, 1, 55, 56, 63, 64, 111, 112, 119, 120, 127, 128, 183, 184, 239, 240, 10240, 10239] * 9)
    tag = mc.tag_pattern("alternating", lens.size, None)
    _check(eng, mc.make_corpus(tag, reg, seed=5, lens=lens), reg)


@pytest.mark.parametrize("size", [1, 2, 2047, 2048, 2049])
def test_family_sizes_around_thresholds(eng, reg, size):
    _set(eng, reg)
    rng = np.random.default_rng(size)
    for big in (mc.P256, mc.P384, mc.ED):
        others = np.array([t for t in (mc.P256, mc.P384, mc.ED) if t != big], np.uint8)
        tag = np.concatenate([np.full(size, big, np.uint8), rng.choice(others, 40)])  # the big family holds exactly `size` items
        rng.shuffle(tag)
        assert int((tag == big).sum()) == size
        _check(eng, mc.make_corpus(tag, reg, seed=6 + big, hi=80), reg)


def test_one_large_batch(eng, reg):
    _set(eng, reg)
    tag = mc.tag_pattern("random", 262144, np.random.default_rng(7))
    cp = mc.make_corpus(tag, reg, seed=8, hi=64)
    got = _mixed(eng, cp)
    assert np.array_equal(got, mc.expected_ok(cp, reg["ecdsa_curve"], reg["ecdsa_xy"], reg["ed_pub"]))


def test_junk_in_ignored_row_bytes(eng, reg):
    _set(eng, reg)
    tag = mc.tag_pattern("random", 600, np.random.default_rng(9))
    clean = mc.make_corpus(tag, reg, seed=10)
    junk = dict(clean, sig96=clean["sig96"].copy())
    rng = np.random.default_rng(11)
    for c, lo in ((mc.P256, 64), (mc.ED, 64)):
        idx = np.flatnonzero(tag == c)
        junk["sig96"][idx, lo:] = rng.integers(0, 256, (idx.size, 96 - lo), dtype=np.uint8)
    assert np.array_equal(_mixed(eng, junk), _mixed(eng, clean))


def test_slot_cases(eng, reg):
    _set(eng, reg)
    tag = mc.tag_pattern("alternating", 300, None)
    cp = mc.make_corpus(tag, reg, seed=12, corrupt=False)
    k_ecdsa, k_ed = reg["ecdsa_curve"].size, reg["ed_pub"].shape[0]
    other = {mc.P256: int(np.flatnonzero(reg["ecdsa_curve"] == mc.P384)[0]), mc.P384: int(np.flatnonzero(reg["ecdsa_curve"] == mc.P256)[0])}
    for j, i in enumerate(range(0, 300, 7)):
        t = int(tag[i])
        n_reg = k_ed if t == mc.ED else k_ecdsa
        cp["key_slot"][i] = [n_reg, 2**32 - 1, other.get(t, n_reg + 5)][j % 3]
    got = _check(eng, cp, reg)
    assert not got[::7].any()
    # the same slot number holds different keys in the two registries: each item reads its own scheme's registry
    same = mc.make_corpus(tag, reg, seed=13, corrupt=False)
    same["key_slot"][:] = 1
    # ECDSA slot 1 holds a P-256 key and Ed25519 slot 1 an Ed25519 key; every item is signed under slot 1 of its registry
    r2 = dict(reg, ecdsa_curve=np.array([reg["ecdsa_curve"][1], mc.P256], np.uint8))
    r2["ecdsa_xy"] = np.stack([reg["ecdsa_xy"][1], reg["ecdsa_xy"][0]])
    r2["ecdsa_priv"] = np.stack([reg["ecdsa_priv"][1], reg["ecdsa_priv"][0]])
    same["scheme"] = np.where(tag == mc.P384, mc.P256, tag).astype(np.uint8)
    same["sig96"] = mc.sign_rows(same["scheme"], same["msgs"], same["off"], same["key_slot"], r2, np.random.default_rng(14))
    _set(eng, r2)
    got = _check(eng, same, r2)
    assert got.all()
    # either registry empty
    for ecdsa, edp in (((np.zeros(0, np.uint8), np.zeros((0, 96), np.uint8)), r2["ed_pub"]),
                       ((r2["ecdsa_curve"], r2["ecdsa_xy"]), np.zeros((0, 32), np.uint8))):
        eng.set_keys(*ecdsa)
        eng.ed25519_set_keys(edp)
        got = _mixed(eng, same)
        assert np.array_equal(got, mc.expected_ok(same, ecdsa[0], ecdsa[1], edp))
        assert np.array_equal(got, _single(eng, same))


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_bad_arguments_leave_outputs_untouched(eng, reg):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    _set(eng, reg)
    cp = mc.make_corpus(mc.tag_pattern("random", 200, np.random.default_rng(15)), reg, seed=16)
    n = 200

    def batch_args():
        out = np.full(n, 0xAB, np.uint8)
        return [C.c_size_t(n), _vp(cp["scheme"]), _vp(cp["msgs"]), _vp(cp["off"]), _vp(cp["key_slot"]), _vp(cp["sig96"]), _vp(out)], out

    cases = {f"null {nm}": {k: None} for k, nm in [(1, "scheme"), (3, "msg_off"), (4, "key_slot"), (5, "sig96"), (6, "ok")]}
    cases["null msgs"] = {2: None}
    cases["n = 2^31, NULL msgs, 4 offsets"] = {0: C.c_size_t(2**31), 2: None, 3: _vp(np.zeros(4, np.uint64))}
    bad_off = cp["off"].copy()
    bad_off[50] = bad_off[49] - 1
    cases["non-monotonic msg_off"] = {3: _vp(bad_off)}
    for at in (0, 97, n - 1):
        bad = cp["scheme"].copy()
        bad[at] = 3
        cases[f"tag 3 at {at}"] = {1: _vp(bad)}
    for name, repl in cases.items():
        a, out = batch_args()
        for k, v in repl.items():
            a[k] = v
        before = eng.kernel_launches
        assert lib.sbv_mixed_verify_registered(eng._h, *a) < 0, name
        assert eng.kernel_launches == before, name
        assert (out == 0xAB).all(), name
        if name.startswith("tag"):
            assert lib.sbv_last_error(eng._h).decode().endswith(f"at {name.split()[-1]}")
    a, out = batch_args()
    assert lib.sbv_mixed_verify_registered(eng._h, *a) == 0
    assert np.array_equal(out, mc.expected_ok(cp, reg["ecdsa_curve"], reg["ecdsa_xy"], reg["ed_pub"]))


@pytest.fixture(scope="module")
def stream():
    return mc.make_votes(160, C4_SCHEMES, seed=30, pad=3)


def _q(eng, st, thr=THR, self_id="stream"):
    sid = st["self_id"] if isinstance(self_id, str) else self_id
    return eng.mixed_verify_quorum(st["scheme"], st["msgs"], st["off"], st["key_slot"], st["sig96"], st["instance"], st["sender"], st["signer"],
                                   st["digest_match"], st["n_instances"], thr, self_id=sid)


def _same(got, want):
    for g, w, name in zip(got, want, ("ok", "valid_count", "reached")):
        assert np.array_equal(g, w), (name, np.flatnonzero(g != w)[:20])


def test_c4_mixed_stream(eng):
    st, r = mc.make_votes(17476, C4_SCHEMES, seed=31, pad=4)
    assert st["instance"].size == 262144
    _set(eng, r)
    got = _q(eng, st)
    _same(got, mc.expected_votes(st, r, THR))
    ok = got[0]
    for c in (votes.BAD_SIG, votes.INERT):
        assert not ok[st["cls"] == c].any()
    assert ok[st["cls"] == votes.HONEST].all()
    # the composition: the family calls, a host scatter and sbv_quorum
    ok2 = _single(eng, st)
    cnt2, reached2 = eng.quorum(st["instance"], st["sender"], st["signer"], st["digest_match"], ok2, st["n_instances"], THR, self_id=st["self_id"])
    _same(got, (ok2, cnt2, reached2))


def test_votes_self_id_and_thresholds(eng, stream):
    st, r = stream
    _set(eng, r)
    _same(_q(eng, st, self_id=None), mc.expected_votes(st, r, THR, self_id=None))
    for thr in (0, 1, 10, 15, 2**32 - 1):
        _same(_q(eng, st, thr=thr), mc.expected_votes(st, r, thr))


def test_votes_instances_without_votes_and_empty_calls(eng, stream):
    st, r = stream
    _set(eng, r)
    I = st["n_instances"]
    sp = dict(st, instance=st["instance"] * 3 + 1, n_instances=3 * I + 1)
    sid = np.zeros(3 * I + 1, np.uint16)
    sid[np.arange(I) * 3 + 1] = st["self_id"]
    sp["self_id"] = sid
    got = _q(eng, sp)
    _same(got, mc.expected_votes(sp, r, THR))
    e0 = np.zeros(0)
    ok, cnt, reached = eng.mixed_verify_quorum(e0, e0, np.zeros(1, np.uint64), e0, e0, e0, e0, e0, e0, 5, 0)
    assert ok.size == 0 and not cnt.any() and reached.all()
    ok, cnt, reached = eng.mixed_verify_quorum(e0, e0, np.zeros(1, np.uint64), e0, e0, e0, e0, e0, e0, 0, 0)
    assert ok.size == cnt.size == reached.size == 0
    import consensus_b200 as sbv
    lib = sbv.load_library()
    assert lib.sbv_mixed_verify_quorum(eng._h, C.c_size_t(4), *([None] * 9), C.c_size_t(0), None, C.c_uint32(0), None, None, None) == 0
    assert lib.sbv_mixed_verify_registered(eng._h, C.c_size_t(0), *([None] * 6)) == 0


def test_votes_bad_arguments(eng, stream):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    st, r = stream
    _set(eng, r)
    n, I = st["instance"].size, st["n_instances"]

    def args():
        outs = (np.full(n, 0xAB, np.uint8), np.full(I, 0xABABABAB, np.uint32), np.full(I, 0xAB, np.uint8))
        a = [C.c_size_t(n), _vp(st["scheme"]), _vp(st["msgs"]), _vp(st["off"]), _vp(st["key_slot"]), _vp(st["sig96"]), _vp(st["instance"]),
             _vp(st["sender"]), _vp(st["signer"]), _vp(st["digest_match"]), C.c_size_t(I), _vp(st["self_id"]), C.c_uint32(THR), _vp(outs[0]),
             _vp(outs[1]), _vp(outs[2])]
        return a, outs

    cases = {f"null {k}": {k: None} for k in (1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 14, 15)}
    cases["n = 2^31"] = {0: C.c_size_t(2**31), 2: None, 3: _vp(np.zeros(4, np.uint64))}
    bad_inst = st["instance"].copy()
    bad_inst[100], bad_inst[101] = bad_inst[101] + 1, bad_inst[100]
    cases["unsorted instances"] = {6: _vp(bad_inst)}
    bad_off = st["off"].copy()
    bad_off[30] = bad_off[29] - 1
    cases["non-monotonic msg_off"] = {3: _vp(bad_off)}
    for at in (0, n // 2, n - 1):
        bad = st["scheme"].copy()
        bad[at] = 7
        cases[f"tag at {at}"] = {1: _vp(bad)}
    for name, repl in cases.items():
        a, outs = args()
        for k, v in repl.items():
            a[k] = v
        before = eng.kernel_launches
        assert lib.sbv_mixed_verify_quorum(eng._h, *a) < 0, name
        assert eng.kernel_launches == before, name
        for o in outs:
            assert (o.view(np.uint8) == 0xAB).all(), name
    a, outs = args()
    assert lib.sbv_mixed_verify_quorum(eng._h, *a) == 0
    _same(outs, mc.expected_votes(st, r, THR))


@pytest.mark.parametrize("schemes", [[mc.ED] * N, [mc.P256] * N, [mc.P384] * N])
def test_single_scheme_consenter_sets(eng, schemes):
    st, r = mc.make_votes(60, schemes, seed=32, pad=2)
    _set(eng, r)
    got = _q(eng, st)
    _same(got, mc.expected_votes(st, r, THR))
    if schemes[0] == mc.ED:
        want = eng.ed25519_verify_quorum(st["msgs"], st["off"], st["key_slot"], st["sig96"][:, :64], st["instance"], st["sender"], st["signer"],
                                         st["digest_match"], st["n_instances"], THR, self_id=st["self_id"])
    else:
        c, Lc = schemes[0], mc.L[schemes[0]]
        ok = eng.hash_verify_registered(c, st["msgs"], st["off"], st["key_slot"], st["sig96"][:, :Lc], st["sig96"][:, Lc:2 * Lc])
        want = (ok, *eng.quorum(st["instance"], st["sender"], st["signer"], st["digest_match"], ok, st["n_instances"], THR, self_id=st["self_id"]))
    _same(got, want)


def test_pinned_and_pageable_input(eng, stream):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    st, r = stream
    _set(eng, r)
    want = mc.expected_votes(st, r, THR)
    cols = ("scheme", "msgs", "off", "key_slot", "sig96", "instance", "sender", "signer", "digest_match", "self_id")
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
            eng.mixed_verify_quorum_ptr(n, *(src[c].ctypes.data for c in cols[:9]), I, src["self_id"].ctypes.data, THR, ok.ctypes.data,
                                        cnt.ctypes.data, reached.ctypes.data)
            _same((ok, cnt, reached), want)
            ok2 = np.zeros(n, np.uint8)
            eng.mixed_verify_registered_ptr(n, *(src[c].ctypes.data for c in cols[:5]), ok2.ctypes.data)
            assert np.array_equal(ok2, want[0])
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_concurrent_callers_see_one_ed25519_registry(eng, stream):
    st, r = stream
    keys_a = r["ed_pub"]
    keys_b = np.concatenate([keys_a[1:], keys_a[:1]])
    want_a = mc.expected_ok(st, r["ecdsa_curve"], r["ecdsa_xy"], keys_a)
    want_b = mc.expected_ok(st, r["ecdsa_curve"], r["ecdsa_xy"], keys_b)
    ed = st["scheme"] == mc.ED
    assert not np.array_equal(want_a[ed], want_b[ed])
    _set(eng, r)
    stop, errs, seen = threading.Event(), [], [0]

    def swapper():
        k = 0
        while not stop.is_set():
            k += 1
            eng.ed25519_set_keys(keys_b if k % 2 else keys_a)

    def caller():
        try:
            for _ in range(10):
                for got in (_q(eng, st)[0], eng.mixed_verify_registered(st["scheme"], st["msgs"], st["off"], st["key_slot"], st["sig96"])):
                    if not (np.array_equal(got, want_a) or np.array_equal(got, want_b)):
                        errs.append("mixed outcome")
                    seen[0] += 1
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
    assert seen[0] == 80


def test_two_device_engine(stream, reg):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import consensus_b200 as sbv
    st, r = stream
    cp = mc.make_corpus(mc.tag_pattern("runs", 5000, np.random.default_rng(33)), reg, seed=34)
    with sbv.Engine(n_devices=2) as e2:
        _set(e2, r)
        _same(_q(e2, st), mc.expected_votes(st, r, THR))
        _set(e2, reg)
        assert np.array_equal(_mixed(e2, cp), mc.expected_ok(cp, reg["ecdsa_curve"], reg["ecdsa_xy"], reg["ed_pub"]))


def test_existing_calls_reject_the_ed25519_tag(eng, reg):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    z = np.zeros(4 * 96, np.uint8)
    off = np.zeros(5, np.uint64)
    slot = np.zeros(4, np.uint32)
    ok = np.full(4, 0xAB, np.uint8)
    tags = np.full(4, sbv.ED25519, np.uint8)
    n, ed = C.c_size_t(4), C.c_uint8(sbv.ED25519)
    calls = {
        "sbv_verify_batch": (ed, n, _vp(z), _vp(z), _vp(z), _vp(z), _vp(z), C.c_uint8(32), _vp(ok)),
        "sbv_verify_batch_der": (ed, n, _vp(z), _vp(np.zeros(5, np.uint32)), _vp(z), _vp(z), C.c_uint8(32), _vp(ok)),
        "sbv_hash_verify_batch": (ed, n, _vp(z), _vp(off), _vp(z), _vp(z), _vp(z), _vp(z), None, _vp(ok)),
        "sbv_verify_mixed": (n, _vp(tags), _vp(z), _vp(z), _vp(z), _vp(z), _vp(z), _vp(ok)),
        "sbv_set_keys": (C.c_uint64(0), n, _vp(np.zeros(4, np.uint64)), _vp(tags), _vp(z)),
        "sbv_verify_registered": (ed, n, _vp(slot), _vp(z), _vp(z), _vp(z), C.c_uint8(32), _vp(ok)),
        "sbv_hash_verify_registered": (ed, n, _vp(z), _vp(off), _vp(slot), _vp(z), _vp(z), _vp(ok)),
        "sbv_verify_quorum": (ed, n, _vp(z), _vp(z), _vp(z), _vp(z), _vp(z), C.c_uint8(32), _vp(slot), _vp(np.ones(4, np.uint16)),
                              _vp(np.ones(4, np.uint16)), _vp(z), C.c_size_t(1), None, C.c_uint32(1), _vp(ok), _vp(np.zeros(1, np.uint32)),
                              _vp(np.zeros(1, np.uint8))),
        "sbv_verify_batch_device": (C.c_int(0), ed, n, _vp(z), _vp(z), _vp(z), _vp(z), _vp(z), C.c_uint8(32), _vp(ok), None),
        "sbv_verify_registered_device": (C.c_int(0), ed, n, _vp(slot), _vp(z), _vp(z), _vp(z), C.c_uint8(32), _vp(ok), None),
    }
    before = eng.kernel_launches
    for name, a in calls.items():
        assert getattr(lib, name)(eng._h, *a) == -1, name
    assert eng.kernel_launches == before and (ok == 0xAB).all()
