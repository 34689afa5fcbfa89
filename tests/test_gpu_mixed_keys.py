"""Mixed ECDSA / Ed25519 batches with the key of each item on the H100: sbv_mixed_verify_batch against OpenSSL
(oracle/, oracle_ed25519/) and against the single-scheme keys-per-item calls (sbv_hash_verify_batch per curve,
sbv_ed25519_verify_batch) run on each family's items.  Corpora come from tests/mixed_keys_cases.py."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import launch_counts as lc
import mixed_keys_cases as mk

pytestmark = pytest.mark.gpu

SBV_ERR_ARG = -1
THRESHOLD = 16  # SBV_GROUP_THRESHOLD's default


def _engine(env=None):
    """An engine on device 0, created with the SBV_GROUP_* settings of env (read once, by sbv_create)."""
    import consensus_b200 as sbv
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        os.environ.update({k: str(v) for k, v in (env or {}).items()})
        return sbv.Engine(devices=[0])
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


@pytest.fixture(scope="module")
def pools():
    return mk.key_pools(k256=24, k384=24, k_ed=24, seed=51)


def _mixed(eng, cp):
    return eng.mixed_verify_batch(cp["scheme"], cp["msgs"], cp["off"], cp["sig96"], cp["key96"])


def _single(eng, cp):
    """The single-scheme keys-per-item calls on each family's items: what the mixed call must return byte for byte."""
    ok = np.zeros(cp["scheme"].size, np.uint8)
    for c in (mk.P256, mk.P384, mk.ED):
        idx, m, o, sig, key = mk.family_arrays(cp, c)
        if idx.size == 0:
            continue
        ok[idx] = eng.ed25519_verify_batch(m, o, sig[0], key[0]) if c == mk.ED else eng.hash_verify_batch(c, m, o, sig[0], sig[1], key[0], key[1])
    return ok


def _check(eng, cp):
    got = _mixed(eng, cp)
    want = mk.expected_ok(cp)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    assert np.array_equal(got, _single(eng, cp))
    return got


@pytest.mark.parametrize("kind", ["p256", "p384", "ed", "alternating", "random", "runs"])
def test_tag_patterns_and_corruption_classes(eng, pools, kind):
    cp = mk.make_corpus(mk.tag_pattern(kind, 1500, np.random.default_rng(1)), pools, seed=2, corrupt=0.3, junk=True)
    got = _check(eng, cp)
    assert 0 < got.sum() < got.size


@pytest.mark.parametrize("classes", ["keys", "signatures"])
def test_every_class(eng, pools, classes):
    cl = mk.BAD_KEY_CLASSES if classes == "keys" else sorted(set(mk.EC_CLASSES + mk.ED_CLASSES) - set(mk.BAD_KEY_CLASSES))
    cp = mk.make_corpus(mk.tag_pattern("random", 3000, np.random.default_rng(3)), pools, seed=4, corrupt=0.5, classes=cl)
    assert set(cp["cls"][cp["cls"] >= 0].tolist()) == set(cl)
    got = _check(eng, cp)
    if classes == "keys":
        assert not got[cp["cls"] >= 0].any() and got[cp["cls"] < 0].all()


def _repeats(tag, counts, rng):
    """key_idx: in every family, key k is used counts[k] times, the remaining items each get a key of their own (from
    len(counts) on, modulo the pool)."""
    key_idx = np.zeros(tag.size, np.int64)
    for c in (mk.P256, mk.P384, mk.ED):
        idx = rng.permutation(np.flatnonzero(tag == c))
        rep = np.repeat(np.arange(len(counts)), counts)
        assert idx.size >= rep.size
        key_idx[idx[:rep.size]] = rep
        key_idx[idx[rep.size:]] = len(counts) + np.arange(idx.size - rep.size)
    return key_idx


def test_keys_repeating_around_the_threshold(eng):
    pools = mk.key_pools(k256=200, k384=200, k_ed=200, seed=52)
    rng = np.random.default_rng(5)
    tag = mk.tag_pattern("random", 450, rng)
    counts = [THRESHOLD - 1, THRESHOLD, THRESHOLD + 1, 3 * THRESHOLD]
    key_idx = _repeats(tag, counts, rng) % 200
    cp = mk.make_corpus(tag, pools, seed=6, hi=100, corrupt=0.2, key_idx=key_idx)
    _check(eng, cp)


def _launches(e, fn, cp):
    """fn(e, cp), and the kernels it launched."""
    before = e.kernel_launches
    got = fn(e, cp)
    return got, e.kernel_launches - before


@pytest.mark.parametrize("env", [{"SBV_GROUP_THRESHOLD": 0}, {"SBV_GROUP_MAX_KEYS": 3}, {"SBV_GROUP_THRESHOLD": 2, "SBV_GROUP_MAX_KEYS": 5},
                                 {"SBV_CHUNK_ITEMS": 256}, {"SBV_GROUP_THRESHOLD": 0, "SBV_CHUNK_ITEMS": 256}],
                         ids=["no-grouping", "max-keys-3", "threshold-2-max-keys-5", "chunked", "no-grouping-chunked"])
def test_other_grouping_settings_give_identical_verdicts(eng, pools, env):
    rng = np.random.default_rng(7)
    tag = mk.tag_pattern("runs", 2400, rng)
    key_idx = _repeats(tag, [40] * 10, rng) % 24  # ten keys repeated in every family: more than the tables of max-keys-3 / -5
    cp = mk.make_corpus(tag, pools, seed=8, hi=80, corrupt=0.3, key_idx=key_idx)
    want = _check(eng, cp)
    n = [int((tag == c).sum()) for c in (mk.P256, mk.P384, mk.ED)]
    e2 = _engine(env)
    try:
        got, k = _launches(e2, _mixed, cp)
        assert np.array_equal(got, want)
        assert k == lc.mixed(n, env) + 1  # + k_ed_btab_init: the engine's first Ed25519 call
        got, k = _launches(e2, _single, cp)
        assert np.array_equal(got, want)
        assert k == lc.ecdsa(mk.P256, n[0], env=env) + lc.ecdsa(mk.P384, n[1], env=env) + lc.ed25519(n[2], env)
    finally:
        e2.close()


@pytest.mark.parametrize("size", [63, 64, 65])
def test_family_sizes_around_the_minimum_batch(pools, size):
    e2 = _engine({"SBV_GROUP_MIN_BATCH": 64})
    try:
        rng = np.random.default_rng(size)
        for big in (mk.P256, mk.P384, mk.ED):
            others = np.array([t for t in (mk.P256, mk.P384, mk.ED) if t != big], np.uint8)
            tag = np.concatenate([np.full(size, big, np.uint8), rng.choice(others, 30)])
            rng.shuffle(tag)
            key_idx = np.where(tag == big, np.arange(tag.size) % 3, rng.integers(0, 24, tag.size))  # three keys, >= 21 items each
            cp = mk.make_corpus(tag, pools, seed=9 + big, hi=60, corrupt=0.2, key_idx=key_idx)
            _check(e2, cp)
    finally:
        e2.close()


def test_equal_bytes_as_ed25519_key_and_p256_x_are_not_one_group(eng, pools):
    tag = np.array([mk.ED, mk.P256] * 60, np.uint8)
    cp = mk.make_corpus(tag, pools, seed=10, hi=60, corrupt=0, key_idx=np.zeros(tag.size, np.int64))
    p256 = np.flatnonzero(tag == mk.P256)
    ed_key = cp["key96"][0, :32].copy()
    cp["key96"][p256[::2], :32] = ed_key  # 30 P-256 items whose X is the 32 bytes of the Ed25519 key of every Ed25519 item
    got = _check(eng, cp)
    assert got[tag == mk.ED].all() and not got[p256[::2]].any() and got[p256[1::2]].all()


def test_every_message_empty_with_null_msgs(eng, pools):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    tag = mk.tag_pattern("alternating", 300, None)
    cp = mk.make_corpus(tag, pools, seed=11, lens=np.zeros(300, np.int64), corrupt=0.3)
    ok = np.full(300, 0xAB, np.uint8)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.sbv_mixed_verify_batch(eng._h, C.c_size_t(300), vp(cp["scheme"]), None, vp(cp["off"]), vp(cp["sig96"]), vp(cp["key96"]), vp(ok)) == 0
    assert np.array_equal(ok, mk.expected_ok(cp))
    assert np.array_equal(ok, _single(eng, cp))


def test_block_boundaries_and_10KiB_messages(eng, pools):
    # SHA-256 pads at 55 / 56 and 119 / 120 bytes; SHA-512 hashes R || A || M, so 64 more: 47 / 48, 175 / 176, 303 / 304
    lens = np.array([0, 1, 47, 48, 55, 56, 63, 64, 111, 112, 119, 120, 127, 128, 175, 176, 239, 240, 303, 304, 10239, 10240] * 8)
    tag = mk.tag_pattern("alternating", lens.size, None)
    _check(eng, mk.make_corpus(tag, pools, seed=12, lens=lens, corrupt=0.3))


def test_one_batch_of_300K_items(eng):
    pools = mk.key_pools(k256=1024, k384=256, k_ed=1024, seed=53)
    tag = mk.tag_pattern("random", 30_000, np.random.default_rng(13))
    cp = mk.tile(mk.make_corpus(tag, pools, seed=14, hi=64, corrupt=0.05), 10, seed=15)
    assert cp["scheme"].size == 300_000
    got = _mixed(eng, cp)
    want = mk.expected_ok(cp)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    assert np.array_equal(got, _single(eng, cp))


def test_pinned_and_pageable_input(eng, pools):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    lib.sbv_host_alloc.restype = C.c_void_p
    cp = mk.make_corpus(mk.tag_pattern("random", 4000, np.random.default_rng(15)), pools, seed=16, corrupt=0.3)
    want = mk.expected_ok(cp)
    cols = ("scheme", "msgs", "off", "sig96", "key96")
    ptrs, pinned = [], {}
    try:
        for c in cols:
            a = np.ascontiguousarray(cp[c])
            p = lib.sbv_host_alloc(C.c_size_t(a.nbytes))
            assert p
            ptrs.append(p)
            view = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(p)).view(a.dtype).reshape(a.shape)
            view[...] = a
            pinned[c] = view
        ok_pin = lib.sbv_host_alloc(C.c_size_t(4000))
        ptrs.append(ok_pin)
        for src, out in ((pinned, ok_pin), ({c: np.ascontiguousarray(cp[c]) for c in cols}, None)):
            ok = np.zeros(4000, np.uint8)
            eng.mixed_verify_batch_ptr(4000, *(src[c].ctypes.data for c in cols), out or ok.ctypes.data)
            if out:
                ok = np.ctypeslib.as_array((C.c_uint8 * 4000).from_address(out)).copy()
            assert np.array_equal(ok, want)
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_six_threads_with_distinct_batches(eng, pools):
    corpora = [mk.make_corpus(mk.tag_pattern(k, 1200 + 300 * t, np.random.default_rng(20 + t)), pools, seed=30 + t, corrupt=0.3)
               for t, k in enumerate(["p256", "p384", "ed", "alternating", "random", "runs"])]
    wants = [mk.expected_ok(cp) for cp in corpora]
    errs = []

    def caller(t):
        try:
            for _ in range(8):
                if not np.array_equal(_mixed(eng, corpora[t]), wants[t]):
                    errs.append(f"thread {t}: wrong verdicts")
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=caller, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs[:5]


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_bad_arguments_leave_ok_untouched(eng, pools):
    import consensus_b200 as sbv
    lib = sbv.load_library()
    n = 200
    cp = mk.make_corpus(mk.tag_pattern("random", n, np.random.default_rng(17)), pools, seed=18, corrupt=0.3)

    def batch_args():
        out = np.full(n, 0xAB, np.uint8)
        return [C.c_size_t(n), _vp(cp["scheme"]), _vp(cp["msgs"]), _vp(cp["off"]), _vp(cp["sig96"]), _vp(cp["key96"]), _vp(out)], out

    cases = {f"null {nm}": {k: None} for k, nm in [(1, "scheme"), (2, "msgs"), (3, "msg_off"), (4, "sig96"), (5, "key96"), (6, "ok")]}
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
        assert lib.sbv_mixed_verify_batch(eng._h, *a) == SBV_ERR_ARG, name
        assert eng.kernel_launches == before, name
        assert (out == 0xAB).all(), name
        if name.startswith("tag"):
            assert lib.sbv_last_error(eng._h).decode().endswith(f"at {name.split()[-1]}")
    assert lib.sbv_mixed_verify_batch(eng._h, C.c_size_t(0), *([None] * 6)) == 0
    a, out = batch_args()
    assert lib.sbv_mixed_verify_batch(eng._h, *a) == 0
    assert np.array_equal(out, mk.expected_ok(cp))


def test_registries_are_not_read(eng, pools):
    """Keys per item: the ECDSA and Ed25519 registries, empty or not, change nothing."""
    cp = mk.make_corpus(mk.tag_pattern("random", 600, np.random.default_rng(19)), pools, seed=20, corrupt=0.3)
    want = mk.expected_ok(cp)
    eng.set_keys(np.zeros(0, np.uint8), np.zeros((0, 96), np.uint8))
    eng.ed25519_set_keys(np.zeros((0, 32), np.uint8))
    assert np.array_equal(_mixed(eng, cp), want)
    eng.ed25519_set_keys(pools[mk.ED][1])
    assert np.array_equal(_mixed(eng, cp), want)


def test_two_device_engine(pools):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import consensus_b200 as sbv
    cp = mk.make_corpus(mk.tag_pattern("runs", 5000, np.random.default_rng(33)), pools, seed=34, corrupt=0.3)
    with sbv.Engine(n_devices=2) as e2:
        got = _mixed(e2, cp)
        assert np.array_equal(got, mk.expected_ok(cp))
        assert np.array_equal(got, _single(e2, cp))
