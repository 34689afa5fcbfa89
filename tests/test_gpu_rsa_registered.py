"""Registered RSA keys on the device: sbv_rsa_set_keys and the four registered verify calls (the CPU twin of the kernels is
test_hostsim_rsa_registered.py).

Every class of tests/rsa_cases.py and tests/rsa_pss_cases.py, for every size, hash and salt mode, through all four calls
against one registry that holds the keys of all three sizes: bit-exact against oracle_rsa.ref and against the keys-per-item
call on the same items, digests against hashlib.  Then the registry itself (records against Python integers, replace,
empty, slots that reject, duplicates, a refused sbv_rsa_set_keys), every argument fault, item counts off the group and
block sizes, launch counts, pinned and pageable buffers, six concurrent callers, sbv_rsa_set_keys racing registered
calls, and two devices."""
import ctypes as C
import threading

import numpy as np
import pytest

import rsa_cases
import rsa_pss_cases as pc
import rsa_registered as rr
from oracle_rsa import ref

pytestmark = pytest.mark.gpu

P8, P32, P64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
PAIRS = [(k, h) for k in rr.SIZES for h in (ref.SHA256, ref.SHA384, ref.SHA512)]


def _engine(n_devices=1):
    import consensus_b200 as sbv
    return sbv.Engine(n_devices=n_devices)


@pytest.fixture(scope="module")
def corpora():
    """Both case modules for every size and hash, and one registry of all their keys (each item's slots in c["slot"])."""
    cs = {}
    for k, h in PAIRS:
        cs[("pkcs1", k, h)] = rsa_cases.make_cases(k, h)
        cs[("pss", k, h)] = pc.make_cases(k, h)
    reg, slots = rr.corpus_registry(*cs.values())
    for c, s in zip(cs.values(), slots):
        c["slot"] = s
    return reg, cs


@pytest.fixture(scope="module")
def eng(corpora):
    reg, _ = corpora
    with _engine() as e:
        e.rsa_set_keys(*reg.arrays())
        yield e


def test_one_registry_holds_every_size(corpora):
    reg, _ = corpora
    assert sorted(set(reg.arrays()[0].tolist())) == [256, 384, 512]


@pytest.mark.parametrize("k,hash", PAIRS)
def test_pkcs1_every_class_all_calls(eng, corpora, k, hash):
    c = corpora[1][("pkcs1", k, hash)]
    per_item = eng.rsa_verify_batch(hash, c["digest"], c["sig"], c["mod"], c["exp"])
    got = eng.rsa_verify_registered(hash, c["slot"], c["digest"], c["sig"])
    bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, c["want"]) if g != w]
    assert not bad, bad
    assert np.array_equal(got, per_item)
    fused, dig = eng.rsa_hash_verify_registered(hash, c["msgs"], c["off"], c["slot"], c["sig"], want_digest=True)
    assert np.array_equal(fused, got) and np.array_equal(dig, c["digest"])
    assert np.array_equal(eng.rsa_hash_verify_registered(hash, c["msgs"], c["off"], c["slot"], c["sig"]), got)
    assert 0 < int(got.sum()) < c["n"]


@pytest.mark.parametrize("k,hash", PAIRS)
def test_pss_every_class_every_salt_mode_all_calls(eng, corpora, k, hash):
    c = corpora[1][("pss", k, hash)]
    for i, sl in enumerate(pc.salt_lens(c)):
        want = pc.want(c, sl)
        got = eng.rsa_pss_verify_registered(hash, sl, c["slot"], c["digest"], c["sig"])
        bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, want) if g != w]
        assert not bad, (sl, bad)
        assert np.array_equal(got, eng.rsa_pss_verify_batch(hash, sl, c["digest"], c["sig"], c["mod"], c["exp"])), sl
        if i == 0:
            fused, dig = eng.rsa_pss_hash_verify_registered(hash, sl, c["msgs"], c["off"], c["slot"], c["sig"], want_digest=True)
            assert np.array_equal(dig, c["digest"])
        else:
            fused = eng.rsa_pss_hash_verify_registered(hash, sl, c["msgs"], c["off"], c["slot"], c["sig"])
        assert np.array_equal(fused, got), sl
        if sl in (ref.SALT_AUTO, ref.SALT_EQUALS_HASH):
            assert 0 < int(want.sum()) < c["n"]


def _debug_record(e, slot):
    out = np.zeros(8 + 256, np.uint32)
    rc = e._lib.sbv_debug_rsa_key(e._h, C.c_uint32(slot), out.ctypes.data_as(P32))
    return rc, out


def test_debug_records_against_python_integers():
    keys = rr.record_keys()
    reg = rr.Registry()
    for _, mod, e in keys:
        reg.slot(mod, e)
    offs = reg.offsets()
    with _engine() as e:
        e.rsa_set_keys(*reg.arrays())
        for i, (name, mod, ex) in enumerate(keys):
            rc, out = _debug_record(e, i)
            want = rr.record(mod, ex, int(offs[i]))
            assert rc == 0 and out[:want.size].tolist() == want.tolist(), name
        assert _debug_record(e, reg.n)[0] == -1


def _tiled(c, n):
    idx = np.arange(n) % c["n"]
    parts = [c["msgs"][int(c["off"][i]):int(c["off"][i + 1])] for i in idx]
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)
    msgs = np.concatenate(parts) if off[-1] else np.zeros(0, np.uint8)
    return dict(n=n, msgs=msgs, off=off, digest=c["digest"][idx].copy(), sig=c["sig"][idx].copy(), mod=c["mod"][idx].copy(), exp=c["exp"][idx].copy(),
                slot=c["slot"][idx].copy(), idx=idx)


@pytest.mark.parametrize("n", [1, 2, 17, 4097])
def test_item_counts_off_the_group_and_block(eng, corpora, n):
    c1, c2 = corpora[1][("pkcs1", 256, ref.SHA256)], corpora[1][("pss", 256, ref.SHA256)]
    t1, t2 = _tiled(c1, n), _tiled(c2, n)
    w1, w2 = c1["want"][t1["idx"]], pc.want(c2, ref.SALT_AUTO)[t2["idx"]]
    assert np.array_equal(eng.rsa_verify_registered(0, t1["slot"], t1["digest"], t1["sig"]), w1)
    assert np.array_equal(eng.rsa_hash_verify_registered(0, t1["msgs"], t1["off"], t1["slot"], t1["sig"]), w1)
    assert np.array_equal(eng.rsa_pss_verify_registered(0, ref.SALT_AUTO, t2["slot"], t2["digest"], t2["sig"]), w2)
    assert np.array_equal(eng.rsa_pss_hash_verify_registered(0, ref.SALT_AUTO, t2["msgs"], t2["off"], t2["slot"], t2["sig"]), w2)


def test_launch_counts_equal_the_keys_per_item_calls(eng, corpora):
    c = _tiled(corpora[1][("pss", 384, ref.SHA384)], 3000)  # above the 2048 items where the hash launches sort by length

    def delta(f):
        before = eng.kernel_launches
        f()
        return eng.kernel_launches - before

    h, sl = ref.SHA384, ref.SALT_EQUALS_HASH
    pairs = [
        (lambda: eng.rsa_verify_batch(h, c["digest"], c["sig"], c["mod"], c["exp"]), lambda: eng.rsa_verify_registered(h, c["slot"], c["digest"], c["sig"])),
        (lambda: eng.rsa_hash_verify_batch(h, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]),
         lambda: eng.rsa_hash_verify_registered(h, c["msgs"], c["off"], c["slot"], c["sig"])),
        (lambda: eng.rsa_pss_verify_batch(h, sl, c["digest"], c["sig"], c["mod"], c["exp"]),
         lambda: eng.rsa_pss_verify_registered(h, sl, c["slot"], c["digest"], c["sig"])),
        (lambda: eng.rsa_pss_hash_verify_batch(h, sl, c["msgs"], c["off"], c["sig"], c["mod"], c["exp"]),
         lambda: eng.rsa_pss_hash_verify_registered(h, sl, c["msgs"], c["off"], c["slot"], c["sig"])),
    ]
    got = [(delta(a), delta(b)) for a, b in pairs]
    assert all(a == b for a, b in got) and [a for a, _ in got][::2] == [1, 2], got


def _one_item(pad, k=256, hash=ref.SHA256):
    c = (rsa_cases if pad == "pkcs1" else pc).make_cases(k, hash, short=True)
    i = c["cls"].index("valid_e65537" if pad == "pkcs1" else "valid_salt_hlen")
    return c, i


def _call(e, pad, slots, sig, dig):
    if pad == "pkcs1":
        return e.rsa_verify_registered(ref.SHA256, slots, dig, sig)
    return e.rsa_pss_verify_registered(ref.SHA256, ref.SALT_AUTO, slots, dig, sig)


@pytest.mark.parametrize("pad", ["pkcs1", "pss"])
def test_registry_semantics(pad):
    """Replace, empty, slots past the registry, a key of another size (one whose bytes, read at the call's size, would
    accept), an invalid key, duplicates, and a refused sbv_rsa_set_keys that leaves the old registry working."""
    c, i = _one_item(pad)
    mod, e_ = c["mod"][i], int(c["exp"][i])
    trap_mod, trap_sig = rr.size_trap(mod.tobytes(), c["sig"][i].tobytes(), 384)  # read as a 2048-bit key, it would accept
    reg = rr.Registry()
    s_big = reg.slot(trap_mod, e_)
    s_bad = reg.slot(mod.tobytes(), 1)  # the key rule refuses e = 1
    s_good = reg.slot(mod.tobytes(), e_)
    mb, mods, exp = reg.arrays()
    # the same key again in a fourth slot: a duplicate behaves as the first
    mb2, mods2, exp2 = np.append(mb, 256).astype(np.uint32), np.concatenate([mods, mod]), np.append(exp, e_).astype(np.uint32)
    slots = np.array([s_good, 3, 4, 2**32 - 1, s_big, s_bad, s_good], np.uint32)
    sig, dig = np.repeat(c["sig"][i:i + 1], 7, 0), np.repeat(c["digest"][i:i + 1], 7, 0)
    sig[4] = np.frombuffer(trap_sig, np.uint8)
    with _engine() as e:
        assert not _call(e, pad, slots, sig, dig).any(), "an engine starts with an empty registry"
        e.rsa_set_keys(mb, mods, exp)
        assert _call(e, pad, slots, sig, dig).tolist() == [1, 0, 0, 0, 0, 0, 1]
        e.rsa_set_keys(mb2, mods2, exp2)
        assert _call(e, pad, slots, sig, dig).tolist() == [1, 1, 0, 0, 0, 0, 1]
        # replace: the valid key alone in slot 0 (slot 0 held the 3072-bit key)
        e.rsa_set_keys([256], mod, [e_])
        assert _call(e, pad, np.array([0, 1, 2], np.uint32), sig[:3], dig[:3]).tolist() == [1, 0, 0]
        # a refused call names the bad size and leaves that registry in place
        lib = e._lib
        bad_mb = np.array([256, 384, 300], np.uint32)
        bad_mods = np.zeros(int(bad_mb.sum()), np.uint8)
        bad_exp = np.full(3, 65537, np.uint32)
        assert lib.sbv_rsa_set_keys(e._h, C.c_size_t(3), bad_mb.ctypes.data_as(P32), bad_mods.ctypes.data_as(P8), bad_exp.ctypes.data_as(P32)) == -1
        assert "mod_bytes[2]" in lib.sbv_last_error(e._h).decode()
        for args in ((3, None, bad_mods.ctypes.data_as(P8), bad_exp.ctypes.data_as(P32)), (3, bad_mb.ctypes.data_as(P32), None, bad_exp.ctypes.data_as(P32)),
                     (3, bad_mb.ctypes.data_as(P32), bad_mods.ctypes.data_as(P8), None), (1 << 31, bad_mb.ctypes.data_as(P32), bad_mods.ctypes.data_as(P8),
                                                                                       bad_exp.ctypes.data_as(P32))):
            assert lib.sbv_rsa_set_keys(e._h, C.c_size_t(args[0]), *args[1:]) == -1
        assert _call(e, pad, np.array([0, 1], np.uint32), sig[:2], dig[:2]).tolist() == [1, 0]
        # n = 0 empties
        e.rsa_set_keys(np.zeros(0, np.uint32), np.zeros(0, np.uint8), np.zeros(0, np.uint32))
        assert not _call(e, pad, slots, sig, dig).any()
        assert _debug_record(e, 0)[0] == -1


VERIFY_FAULTS = ["mod_bytes", "hash", "null_slot", "null_sig", "null_ok", "null_digest", "salt_-2", "decreasing", "null_off", "null_msgs"]
CALLS = {
    "sbv_rsa_verify_registered": ("digest", False),
    "sbv_rsa_hash_verify_registered": ("msgs", False),
    "sbv_rsa_pss_verify_registered": ("digest", True),
    "sbv_rsa_pss_hash_verify_registered": ("msgs", True),
}


def _faults(name):
    src, pss = CALLS[name]
    out = []
    for f in VERIFY_FAULTS:
        if f.startswith("salt") and not pss:
            continue
        if f == "null_digest" and src != "digest":
            continue
        if f in ("decreasing", "null_off", "null_msgs") and src != "msgs":
            continue
        out.append(f)
    return out


@pytest.mark.parametrize("name,fault", [(n, f) for n in CALLS for f in _faults(n)])
def test_argument_faults(eng, name, fault):
    """SBV_ERR_ARG before anything is written or launched, with ok (and the digests) untouched; then the same call with
    n >= 2^31."""
    n, k = 4, 256
    msgs = np.arange(64, dtype=np.uint8)
    off = np.array([0, 5, 3, 9, 20] if fault == "decreasing" else [0, 5, 9, 9, 20], np.uint64)
    sig, dig, slot = np.ones(k * n, np.uint8), np.ones(64 * n, np.uint8), np.zeros(n, np.uint32)
    ok, out = np.full(n, 0x5A, np.uint8), np.full(64 * n, 0x5A, np.uint8)
    nul = lambda f, a, t=P8: None if fault == f else a.ctypes.data_as(t)  # noqa: E731
    mb = C.c_uint32(300 if fault == "mod_bytes" else k)
    hs = C.c_uint8(3 if fault == "hash" else 0)
    sl = C.c_int32(-2 if fault == "salt_-2" else 0)
    _, pss = CALLS[name]
    head = (mb, hs, sl) if pss else (mb, hs)
    if CALLS[name][0] == "digest":
        args = head + (C.c_size_t(n), nul("null_slot", slot, P32), nul("null_digest", dig), nul("null_sig", sig), nul("null_ok", ok))
    else:
        args = head + (C.c_size_t(n), nul("null_msgs", msgs), nul("null_off", off, P64), nul("null_slot", slot, P32), nul("null_sig", sig),
                       out.ctypes.data_as(P8), nul("null_ok", ok))
    before = eng.kernel_launches
    assert getattr(eng._lib, name)(eng._h, *args) == -1
    assert (ok == 0x5A).all() and (out == 0x5A).all(), "a rejected call must not write its outputs"
    assert eng.kernel_launches == before
    big = list(args)
    big[len(head)] = C.c_size_t(1 << 31)
    assert getattr(eng._lib, name)(eng._h, *big) == -1
    assert (ok == 0x5A).all() and eng.kernel_launches == before


def test_pinned_and_pageable_buffers(eng, corpora):
    c = corpora[1][("pss", 384, ref.SHA384)]
    c1 = corpora[1][("pkcs1", 384, ref.SHA384)]
    want, want1 = pc.want(c, ref.SALT_EQUALS_HASH), c1["want"]
    lib = eng._lib
    lib.sbv_host_alloc.restype = C.c_void_p
    n, k = c["n"], 384
    arrays = [c["msgs"], c["off"], c["slot"], c["sig"], np.zeros(48 * n, np.uint8), np.zeros(n, np.uint8), c["digest"]]
    ptrs = []
    try:
        views = []
        for a in arrays:
            p = lib.sbv_host_alloc(C.c_size_t(max(a.nbytes, 1)))
            assert p
            ptrs.append(p)
            v = np.ctypeslib.as_array((C.c_uint8 * max(a.nbytes, 1)).from_address(p))
            v[:a.nbytes] = a.view(np.uint8).reshape(-1)
            views.append(v)
        eng.rsa_pss_hash_verify_registered_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, *ptrs[:6])
        assert np.array_equal(views[5][:n], want)
        assert np.array_equal(views[4].reshape(n, 48), c["digest"])
        assert np.array_equal(views[3], c["sig"].reshape(-1)), "the host signatures are never written"
        views[5][:] = 7
        eng.rsa_pss_verify_registered_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, ptrs[2], ptrs[6], ptrs[3], ptrs[5])
        assert np.array_equal(views[5][:n], want)
        ok = np.zeros(n, np.uint8)
        eng.rsa_pss_verify_registered_ptr(k, ref.SHA384, ref.SALT_EQUALS_HASH, n, c["slot"].ctypes.data, c["digest"].ctypes.data, c["sig"].ctypes.data,
                                          ok.ctypes.data)
        assert np.array_equal(ok, want)
        ok1 = np.zeros(c1["n"], np.uint8)
        eng.rsa_verify_registered_ptr(k, ref.SHA384, c1["n"], c1["slot"].ctypes.data, c1["digest"].ctypes.data, c1["sig"].ctypes.data, ok1.ctypes.data)
        assert np.array_equal(ok1, want1)
    finally:
        for p in ptrs:
            lib.sbv_host_free(C.c_void_p(p))


def test_six_concurrent_callers(eng, corpora):
    cs = corpora[1]
    jobs = [("pkcs1", 256, 0), ("pss", 384, 1), ("pkcs1", 512, 2), ("pss", 256, 2), ("pkcs1", 384, 0), ("pss", 512, 1)]
    cases = [(pad, h, _tiled(cs[(pad, k, h)], 600), cs[(pad, k, h)]) for pad, k, h in jobs]
    wants = [c["want"][t["idx"]] if pad == "pkcs1" else pc.want(c, ref.SALT_AUTO)[t["idx"]] for pad, _, t, c in cases]
    errs = []

    def run(i):
        try:
            pad, h, t, _ = cases[i]
            for _ in range(3):
                if pad == "pkcs1":
                    got = [eng.rsa_hash_verify_registered(h, t["msgs"], t["off"], t["slot"], t["sig"]), eng.rsa_verify_registered(h, t["slot"], t["digest"], t["sig"])]
                else:
                    got = [eng.rsa_pss_hash_verify_registered(h, ref.SALT_AUTO, t["msgs"], t["off"], t["slot"], t["sig"]),
                           eng.rsa_pss_verify_registered(h, ref.SALT_AUTO, t["slot"], t["digest"], t["sig"])]
                assert all(np.array_equal(g, wants[i]) for g in got), (pad, h)
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(6)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_set_keys_racing_registered_calls(corpora):
    """Registries A and B hold the same keys in opposite slot orders; while one thread swaps them, every registered call's
    verdicts equal, as a whole, A's expectation or B's."""
    _, cs = corpora
    c = cs[("pkcs1", 256, ref.SHA256)]
    reg, (slots,) = rr.corpus_registry(c)
    mb, mods, exp = reg.arrays()
    order = np.arange(reg.n)[::-1]
    offs = reg.offsets()
    mods_b = np.concatenate([mods[int(offs[j]):int(offs[j]) + 256] for j in order])
    t = _tiled(dict(c, slot=slots), 2000)
    want_a = c["want"][t["idx"]]
    b_key = order[t["slot"]]  # under B, slot s holds A's key order[s]
    want_b = np.array([ref.verify(256, 0, t["digest"][i].tobytes(), t["sig"][i].tobytes(), reg.keys[b_key[i]][0], reg.keys[b_key[i]][1])
                       for i in range(t["n"])], np.uint8)
    assert not np.array_equal(want_a, want_b)
    seen, errs, stop = set(), [], threading.Event()
    with _engine() as e:
        e.rsa_set_keys(mb, mods, exp)

        def caller():
            try:
                while not stop.is_set():
                    got = e.rsa_verify_registered(0, t["slot"], t["digest"], t["sig"])
                    if np.array_equal(got, want_a):
                        seen.add("a")
                    elif np.array_equal(got, want_b):
                        seen.add("b")
                    else:
                        raise AssertionError("verdicts of neither registry")
            except Exception as ex:  # noqa: BLE001
                errs.append(ex)

        ts = [threading.Thread(target=caller) for _ in range(4)]
        for th in ts:
            th.start()
        try:
            for r in range(12):
                if r % 2 == 0:
                    e.rsa_set_keys(mb, mods_b, exp[order])
                else:
                    e.rsa_set_keys(mb, mods, exp)
        finally:
            stop.set()
            for th in ts:
                th.join()
    assert not errs, errs
    assert seen, "no call completed"


def test_multi_device_sharding(corpora):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {torch.cuda.device_count()}")
    reg, cs = corpora
    c1, c2 = cs[("pkcs1", 512, ref.SHA512)], cs[("pss", 256, ref.SHA256)]
    t1, t2 = _tiled(c1, 301), _tiled(c2, 301)
    with _engine(2) as e2:
        e2.rsa_set_keys(*reg.arrays())
        assert np.array_equal(e2.rsa_verify_registered(2, t1["slot"], t1["digest"], t1["sig"]), c1["want"][t1["idx"]])
        ok, dig = e2.rsa_pss_hash_verify_registered(0, ref.SALT_AUTO, t2["msgs"], t2["off"], t2["slot"], t2["sig"], want_digest=True)
        assert np.array_equal(ok, pc.want(c2, ref.SALT_AUTO)[t2["idx"]]) and np.array_equal(dig, t2["digest"])
