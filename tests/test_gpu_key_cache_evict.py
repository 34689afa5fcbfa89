"""The evicting grouped-key cache (sbv_key_cache_reserve_evicting / sbv_key_cache_stats_ex) on the H100.  Churn over a key
population four times the capacity with a hot subset, through every keys-per-item entry point, with verdicts equal to an
engine without a cache and to OpenSSL on every call and the statistics counted from the corpora; admission after a full
cache, exactly sum(min(c_b, 16)) hits from the per-set counts c_b of the engine's own hash (0 in fill-once mode); six
concurrent callers on a cache of two sets; switching modes and freeing; argument faults; two devices."""
import ctypes as C
import hashlib
import os
import threading

import numpy as np
import pytest

import kca_sets
import mixed_keys_cases as mk
import oracle
from oracle import ecdsa_ref as ref

pytestmark = pytest.mark.gpu

P256, P384, ED = mk.P256, mk.P384, mk.ED
ALL = (P256, P384, ED)
SBV_ERR_ARG = -1
KEY_BYTES = {P256: 64, P384: 96, ED: 32}
K = 64    # keys per scheme in the population
PER = 20  # items per key: every key of a call is grouped (SBV_GROUP_THRESHOLD 16)
WAYS = 16


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _engine(devices=(0,)):
    import consensus_b200 as sbv
    return sbv.Engine(devices=list(devices))


@pytest.fixture(scope="module")
def pop():
    """PER items on each of K keys per scheme, shuffled, a fifth of them corrupted in ways that keep the key; P-384 items
    also carry a signature over SHA-384 of the message (for sbv_hash384_verify_batch)."""
    rng = np.random.default_rng(404)
    scheme = np.repeat(np.array(ALL, np.uint8), K * PER)
    key_idx = np.tile(np.repeat(np.arange(K), PER), 3)
    order = rng.permutation(scheme.size)
    scheme, key_idx = scheme[order], key_idx[order]
    pools = mk.key_pools(k256=K, k384=K, k_ed=K, seed=404)
    cp = mk.make_corpus(scheme, pools, seed=405, corrupt=0.2, key_idx=key_idx, classes=[mk.FLIP_MSG, mk.FLIP_SIG, mk.R_ZERO, mk.S_ZERO])
    cp["want"] = mk.expected_ok(cp)
    idx = np.flatnonzero(scheme == P384)
    m, o = mk.gather(cp["msgs"], cp["off"], idx)
    d384 = np.stack([np.frombuffer(hashlib.sha384(m[int(o[i]):int(o[i + 1])].tobytes()).digest(), np.uint8) for i in range(idx.size)])
    nonces = rng.integers(0, 256, (idx.size, 48), dtype=np.uint8)
    nonces[:, 0] &= 0x7F
    nonces[:, -1] |= 1
    r, s = oracle.sign_batch(P384, pools[P384][0], key_idx[idx].astype(np.uint32), d384, nonces)
    r[::7, 3] ^= 1
    cp["sig384"] = np.zeros((scheme.size, 96), np.uint8)
    cp["sig384"][idx, :48], cp["sig384"][idx, 48:] = r, s
    cp["want384"] = np.zeros(scheme.size, np.uint8)
    xy = cp["key96"][idx]
    cp["want384"][idx] = oracle.verify_batch(P384, r, s, xy[:, :48], xy[:, 48:96], d384)
    assert 0 < cp["want384"][idx].sum() < idx.size
    return cp


@pytest.fixture(scope="module")
def plain():
    e = _engine()
    yield e
    e.close()


def _sub(cp, keys):
    """The items whose key index is in keys[scheme], in corpus order."""
    sel = np.zeros(cp["scheme"].size, bool)
    for c, ks in keys.items():
        sel |= (cp["scheme"] == c) & np.isin(cp["key_idx"], list(ks))
    idx = np.flatnonzero(sel)
    m, o = mk.gather(cp["msgs"], cp["off"], idx)
    out = {k: cp[k][idx] for k in ("scheme", "sig96", "key96", "want", "sig384", "want384", "key_idx")}
    out.update(msgs=m, off=o)
    return out


def _fam(s, c):
    idx = np.flatnonzero(s["scheme"] == c)
    m, o = mk.gather(s["msgs"], s["off"], idx)
    sig, key = s["sig96"][idx], s["key96"][idx]
    if c == ED:
        return idx, m, o, np.ascontiguousarray(sig[:, :64]), np.ascontiguousarray(key[:, :32])
    Lc = mk.L[c]
    return idx, m, o, (np.ascontiguousarray(sig[:, :Lc]), np.ascontiguousarray(sig[:, Lc:2 * Lc])), (np.ascontiguousarray(key[:, :Lc]),
                                                                                                       np.ascontiguousarray(key[:, Lc:2 * Lc]))


def _der(r, s):
    return [ref.der_encode(int.from_bytes(a.tobytes(), "big"), int.from_bytes(b.tobytes(), "big")) for a, b in zip(r, s)]


# every keys-per-item entry point: call -> (schemes it groups, run(eng, sub) -> (verdicts, OpenSSL's verdicts))
def _hash(c):
    def run(eng, s):
        idx, m, o, sig, key = _fam(s, c)
        return eng.hash_verify_batch(c, m, o, *sig, *key), s["want"][idx]
    return (c,), run


def _digest(eng, s):
    idx, m, o, sig, key = _fam(s, P256)
    return eng.verify_batch(P256, *sig, *key, oracle.sha256_batch(m, o)), s["want"][idx]


def _device(eng, s):
    import torch
    idx, m, o, sig, key = _fam(s, P256)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (*sig, *key, oracle.sha256_batch(m, o))]
    ok = torch.zeros(idx.size, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    eng.verify_batch_device(P256, idx.size, *(t.data_ptr() for t in dev), 32, ok.data_ptr(), stream=st.cuda_stream)
    st.synchronize()
    return ok.cpu().numpy(), s["want"][idx]


def _der_call(eng, s):
    idx, m, o, sig, key = _fam(s, P384)
    der = _der(*sig)
    off = np.concatenate([[0], np.cumsum([len(d) for d in der])]).astype(np.uint32)
    return eng.verify_batch_der(P384, np.frombuffer(b"".join(der), np.uint8), off, np.concatenate(key, axis=1), oracle.sha256_batch(m, o)), s["want"][idx]


def _hash384(eng, s):
    idx, m, o, _, key = _fam(s, P384)
    r, sg = np.ascontiguousarray(s["sig384"][idx, :48]), np.ascontiguousarray(s["sig384"][idx, 48:])
    return eng.hash384_verify_batch(P384, m, o, r, sg, *key), s["want384"][idx]


def _verify_mixed(eng, s):
    idx = np.flatnonzero(s["scheme"] != ED)
    tag = s["scheme"][idx]
    f48 = [np.zeros((idx.size, 48), np.uint8) for _ in range(4)]
    for c in (P256, P384):
        j = np.flatnonzero(tag == c)
        Lc = mk.L[c]
        sig, key = s["sig96"][idx[j]], s["key96"][idx[j]]
        for f, a in zip(f48, (sig[:, :Lc], sig[:, Lc:2 * Lc], key[:, :Lc], key[:, Lc:2 * Lc])):
            f[j, 48 - Lc:] = a
    m, o = mk.gather(s["msgs"], s["off"], idx)
    return eng.verify_mixed(tag, *f48, oracle.sha256_batch(m, o)), s["want"][idx]


def _quorum(eng, s):
    idx, m, o, sig, key = _fam(s, P256)
    n = idx.size
    voter = (np.arange(n) % 500 + 1).astype(np.uint16)
    ok, _, _ = eng.verify_quorum(P256, *sig, *key, oracle.sha256_batch(m, o), np.zeros(n, np.uint32), voter, voter, np.ones(n, np.uint8), 1, 1)
    return ok, s["want"][idx]


def _ed(eng, s):
    idx, m, o, sig, key = _fam(s, ED)
    return eng.ed25519_verify_batch(m, o, sig, key), s["want"][idx]


def _mixed(eng, s):
    return eng.mixed_verify_batch(s["scheme"], s["msgs"], s["off"], s["sig96"], s["key96"]), s["want"]


CALLS = {
    "sbv_verify_batch": ((P256,), _digest), "sbv_verify_batch_device": ((P256,), _device), "sbv_verify_batch_der": ((P384,), _der_call),
    "sbv_hash_verify_batch/p256": _hash(P256), "sbv_hash_verify_batch/p384": _hash(P384), "sbv_hash384_verify_batch": ((P384,), _hash384),
    "sbv_verify_mixed": ((P256, P384), _verify_mixed), "sbv_verify_quorum": ((P256,), _quorum), "sbv_ed25519_verify_batch": ((ED,), _ed),
    "sbv_mixed_verify_batch": (ALL, _mixed),
}


def _stats(eng):
    return {c: eng.key_cache_stats_ex(c) for c in ALL}


def _draw(rng, hot=6, cold=10):
    return {c: set(range(hot)) | set(rng.choice(np.arange(hot, K), cold, replace=False).tolist()) for c in ALL}


def test_churn_on_every_entry_point(pop, plain):
    """Calls over 6 hot and 10 random keys of 64 per scheme against 16 ways: verdicts exact on every call; hits + misses
    count every grouped key of every call; the hot keys keep being hit while the others are evicted."""
    rng = np.random.default_rng(5)
    eng = _engine()
    try:
        eng.key_cache_reserve_evicting(16, 16, 16)
        grouped = dict.fromkeys(ALL, 0)
        for rep in range(3):
            for name, (schemes, run) in CALLS.items():
                s = _sub(pop, _draw(rng))
                got, want = run(eng, s)
                assert np.array_equal(got, want), (name, rep, np.flatnonzero(got != want)[:10])
                base, _ = run(plain, s)
                assert np.array_equal(got, base), (name, rep)
                for c in schemes:
                    grouped[c] += 16
        for c, st in _stats(eng).items():
            assert st["capacity"] == 16 and st["resident"] <= 16, (c, st)
            assert st["hits"] + st["misses"] == grouped[c], (c, st, grouped[c])
            assert st["hits"] > 0 and st["evictions"] > 0 and st["evictions"] <= st["misses"], (c, st)
    finally:
        eng.close()


@pytest.mark.parametrize("evicting", [True, False], ids=["evicting", "fill-once"])
def test_admission_after_full(pop, evicting):
    """32 ways (two sets) filled by key set A, then two calls over a disjoint set B: the second call hits exactly
    sum(min(c_b, 16)) keys of B evicting, and none fill-once."""
    A, B = set(range(32)), set(range(32, 64))
    eng = _engine()
    try:
        if evicting:
            eng.key_cache_reserve_evicting(32, 32, 32)
        else:
            eng.key_cache_reserve(32, 32, 32)
        runs = {P256: _hash(P256)[1], P384: _hash(P384)[1], ED: _ed}
        for c in ALL:
            for keys, rep in ((A, 0), (B, 0), (B, 1)):
                before = eng.key_cache_stats_ex(c)
                got, want = runs[c](eng, _sub(pop, {c: keys}))
                assert np.array_equal(got, want), (c, rep)
                hits = eng.key_cache_stats_ex(c)["hits"] - before["hits"]
            if evicting:
                geo = np.zeros(2, np.uint32)
                assert eng._lib.sbv_debug_key_cache_sets(eng._h, C.c_int(0), C.c_uint8(c), _p(geo)) == 1
                seed, sets = int(geo[0]), int(geo[1])
                assert sets == 2
                rows = [pop["key96"][np.flatnonzero((pop["scheme"] == c) & (pop["key_idx"] == k))[0], :KEY_BYTES[c]].tobytes() for k in sorted(B)]
                cb = kca_sets.per_set_counts(rows, seed, sets)
                assert hits == int(np.minimum(cb, WAYS).sum()), (c, hits, cb)
            else:
                assert hits == 0, c
            st = eng.key_cache_stats_ex(c)
            assert st["capacity"] == 32 and st["resident"] <= 32
            assert st["evictions"] == (st["misses"] - st["resident"] - st["given_up"] if evicting else 0), (c, st)
            if not evicting:
                assert st["given_up"] == 0
    finally:
        eng.close()


def test_six_concurrent_callers_on_two_sets(pop):
    eng = _engine()
    results, errors = {}, []
    try:
        eng.key_cache_reserve_evicting(32, 32, 32)
        subs = [[_sub(pop, _draw(np.random.default_rng(100 + 10 * t + i), hot=8, cold=12)) for i in range(4)] for t in range(6)]

        def work(t):
            try:
                for i, s in enumerate(subs[t]):
                    results[(t, i)] = _mixed(eng, s)
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)

        th = [threading.Thread(target=work, args=(t,)) for t in range(6)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors
        for key, (got, want) in results.items():
            assert np.array_equal(got, want), key
        for c, st in _stats(eng).items():
            assert st["capacity"] == 32 and st["resident"] <= 32, (c, st)
            assert st["hits"] + st["misses"] == 6 * 4 * 20, (c, st)
            assert st["evictions"] <= st["misses"], (c, st)
    finally:
        eng.close()


def test_mode_switching_and_freeing(pop, plain):
    s = _sub(pop, _draw(np.random.default_rng(9)))

    def launches(e):
        before = e.kernel_launches
        got, want = _mixed(e, s)
        assert np.array_equal(got, want)
        return e.kernel_launches - before

    launches(plain)
    uncached = launches(plain)
    eng = _engine()
    try:
        launches(eng)  # + k_ed_btab_init on the engine's first Ed25519 call
        assert launches(eng) == uncached
        zero = {"capacity": 0, "resident": 0, "hits": 0, "misses": 0, "evictions": 0, "given_up": 0}
        for mode in ("evicting", "fill-once", "evicting"):
            (eng.key_cache_reserve_evicting if mode == "evicting" else eng.key_cache_reserve)(20, 20, 20)
            cap = 32 if mode == "evicting" else 20  # rounded up to a multiple of 16 ways
            for c in ALL:
                assert eng.key_cache_stats_ex(c) == dict(zero, capacity=cap), (mode, c)
            assert launches(eng) == uncached + 2 * 3, mode  # lookup and insert per grouped scheme
            assert launches(eng) == uncached + 2 * 3, mode
            for c in ALL:
                st = eng.key_cache_stats_ex(c)
                assert st["hits"] == st["misses"] == st["resident"] == 16, (mode, c, st)
                assert eng.key_cache_stats(c) == {k: st[k] for k in ("capacity", "resident", "hits", "misses")}
        eng.key_cache_reserve(0, 0, 0)
        assert launches(eng) == uncached
        for c in ALL:
            assert eng.key_cache_stats_ex(c) == zero
    finally:
        eng.close()


def test_argument_faults(pop):
    import consensus_b200 as sbv
    eng = _engine()
    try:
        eng.key_cache_reserve_evicting(8, 8, 8)
        assert eng.key_cache_stats_ex(P256)["capacity"] == 16
        with pytest.raises(sbv.EngineFault, match=r"\(-4\)"):
            eng.key_cache_reserve_evicting(1 << 28, 0, 0)  # 8 TiB of P-256 tables
        with pytest.raises(sbv.EngineFault, match=r"\(-4\)"):
            eng.key_cache_reserve_evicting(0, 0, 1 << 62)
        for c in ALL:
            assert eng.key_cache_stats_ex(c)["capacity"] == 0
        got, want = _mixed(eng, _sub(pop, _draw(np.random.default_rng(3))))
        assert np.array_equal(got, want)
        out = (C.c_uint64 * 6)()
        assert eng._lib.sbv_key_cache_stats_ex(eng._h, C.c_uint8(3), out) == SBV_ERR_ARG
        assert eng._lib.sbv_key_cache_stats_ex(eng._h, C.c_uint8(0), None) == SBV_ERR_ARG
        assert eng._lib.sbv_key_cache_reserve_evicting(None, C.c_size_t(1), C.c_size_t(0), C.c_size_t(0)) == SBV_ERR_ARG
    finally:
        eng.close()


def test_two_devices(pop):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    eng = _engine(devices=(0, 1))
    try:
        eng.key_cache_reserve_evicting(16, 16, 16)
        rng = np.random.default_rng(11)
        for _ in range(4):
            got, want = _mixed(eng, _sub(pop, _draw(rng)))
            assert np.array_equal(got, want)
        for c, st in _stats(eng).items():
            assert st["capacity"] == 32 and st["resident"] <= 32 and st["hits"] > 0, (c, st)
    finally:
        eng.close()
