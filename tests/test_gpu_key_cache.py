"""The grouped-key cache (sbv_key_cache_reserve / sbv_key_cache_stats) on the H100.  For P-256, P-384, Ed25519 and
sbv_mixed_verify_batch, a cold call (inserts) and a warm call (hits) give verdicts equal to the same engine without a cache
and to OpenSSL, on corpora with flipped messages, r or s = 0 and = n, S >= L, an off-curve key and an undecodable Ed25519
key repeated past the threshold, and the y >= p and "-0" encodings of one point.  The statistics count the grouped valid
keys; a cached table equals the table a fresh launch builds; a full cache, a chunked engine, _device calls on a caller
stream, six concurrent callers, re-reserving, freeing, argument faults and a two-device engine; the kernel launches of
each call, with and without a cache, grouped or not, chunked or not (tests/launch_counts.py)."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import ecdsa_keys as ek
import ed25519_edges as edges
import launch_counts as lc
import mixed_keys_cases as mk
import oracle
from oracle.ecdsa_ref import CURVES
from oracle_ed25519 import corpus as edcorpus, ref

pytestmark = pytest.mark.gpu

P256, P384, ED = mk.P256, mk.P384, mk.ED
SBV_ERR_ARG, SBV_ERR_NOMEM = -1, -4
T = 16  # SBV_GROUP_THRESHOLD's default
KEY_BYTES = {P256: 64, P384: 96, ED: 32}
TABLE_WORDS = {P256: 512 * 16, P384: ek.windows(P384, 5) * 16 * 24, ED: 510 * 24}


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _engine(env=None, devices=(0,)):
    import consensus_b200 as sbv
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        os.environ.update({k: str(v) for k, v in (env or {}).items()})
        return sbv.Engine(devices=list(devices))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _corpus(seed=71, n=6000):
    """Mixed items over 20 keys per scheme, a third of them corrupted; then 40 P-256 and 40 P-384 items on one off-curve
    key, 40 Ed25519 items on one undecodable encoding, 24 items on each of three encodings of the identity (canonical,
    y = 1 + p, "-0"), and s = n on a few ECDSA items."""
    rng = np.random.default_rng(seed)
    pools = mk.key_pools(k256=20, k384=20, k_ed=20, seed=seed)
    cl = [mk.FLIP_MSG, mk.FLIP_SIG, mk.R_ZERO, mk.S_ZERO, mk.R_EQ_N, mk.S_PLUS_L, mk.WRONG_KEY, mk.HIGH_S]
    cp = mk.make_corpus(mk.tag_pattern("random", n, rng), pools, seed=seed + 1, corrupt=0.3, classes=cl)
    sch, key, sig = cp["scheme"], cp["key96"], cp["sig96"]
    for c in (P256, P384):
        Lc = mk.L[c]
        idx = rng.permutation(np.flatnonzero(sch == c))
        bad = key[idx[0], :2 * Lc].copy()
        bad[-1] ^= 1  # y + 1 (or - 1): off the curve
        key[idx[:40], :2 * Lc] = bad
        nb = CURVES[c].n.to_bytes(Lc, "big")
        sig[idx[40:44], Lc:2 * Lc] = np.frombuffer(nb, np.uint8)  # s = n
    idx = rng.permutation(np.flatnonzero(sch == ED))
    y = 2
    while ref.decode(edcorpus._enc_y(y)) is not None:
        y += 1
    key[idx[:40], :32] = np.frombuffer(edcorpus._enc_y(y), np.uint8)
    for j, A in enumerate(edges.IDENTITY_KEYS):
        for i in idx[40 + 24 * j:64 + 24 * j]:
            S = int.from_bytes(rng.bytes(32), "little") % ref.L
            key[i, :32] = np.frombuffer(A, np.uint8)
            sig[i, :64] = np.frombuffer(edges._sig(ref.encode(edges.bmul(S)), S), np.uint8)
    cp["want"] = mk.expected_ok(cp)
    return cp


@pytest.fixture(scope="module")
def cp():
    return _corpus()


@pytest.fixture(scope="module")
def plain():
    e = _engine()
    yield e
    e.close()


def _family(eng, cp, c):
    idx, m, o, sig, key = mk.family_arrays(cp, c)
    if c == ED:
        return idx, eng.ed25519_verify_batch(m, o, sig[0], key[0])
    return idx, eng.hash_verify_batch(c, m, o, sig[0], sig[1], key[0], key[1])


def _run(eng, cp, call):
    """Verdicts of `call` over the items it covers, and those items."""
    if call == "mixed":
        return np.arange(cp["scheme"].size), eng.mixed_verify_batch(cp["scheme"], cp["msgs"], cp["off"], cp["sig96"], cp["key96"])
    if call == "p256_digest":
        idx, m, o, sig, key = mk.family_arrays(cp, P256)
        return idx, eng.verify_batch(P256, sig[0], sig[1], key[0], key[1], oracle.sha256_batch(m, o))
    return _family(eng, cp, {"p256": P256, "p384": P384, "ed": ED}[call])


def _counted(eng, cp, call):
    """_run, and the kernels it launched."""
    before = eng.kernel_launches
    idx, ok = _run(eng, cp, call)
    return idx, ok, eng.kernel_launches - before


def _want_launches(cp, call, cached=(), env=None):
    n = [int((cp["scheme"] == c).sum()) for c in (P256, P384, ED)]
    if call == "mixed":
        return lc.mixed(n, env, cached)
    if call == "ed":
        return lc.ed25519(n[ED], env, cached)
    c = P384 if call == "p384" else P256
    return lc.ecdsa(c, n[c], call != "p256_digest", env, cached)


ALL = (P256, P384, ED)


def _schemes(call):
    return {"mixed": (P256, P384, ED), "p256": (P256,), "p256_digest": (P256,), "p384": (P384,), "ed": (ED,)}[call]


def _grouped_valid(eng, cp, c):
    """{key bytes: table} of the keys a launch over scheme c's items groups and finds valid, as a fresh launch builds them
    (sbv_debug_grouped_key_table / sbv_debug_ed25519_comb_tab on an engine without a cache)."""
    idx = np.flatnonzero(cp["scheme"] == c)
    rows = np.ascontiguousarray(cp["key96"][idx, :KEY_BYTES[c]])
    uniq, first = np.unique(rows, axis=0, return_index=True)
    first = np.ascontiguousarray(first, np.uint32)
    status = np.full(first.size, -1, np.int32)
    out = np.zeros((first.size, TABLE_WORDS[c]), np.uint32)
    if c == ED:
        rc = eng._lib.sbv_debug_ed25519_comb_tab(eng._h, C.c_size_t(rows.shape[0]), _p(rows), C.c_size_t(first.size), _p(first), _p(status), _p(out))
    else:
        Lc = mk.L[c]
        qx, qy = np.ascontiguousarray(rows[:, :Lc]), np.ascontiguousarray(rows[:, Lc:])
        rc = eng._lib.sbv_debug_grouped_key_table(eng._h, C.c_uint8(c), C.c_size_t(rows.shape[0]), _p(qx), _p(qy), C.c_size_t(first.size), _p(first),
                                                 _p(status), _p(out))
    assert rc == 0
    assert (status == 2).any(), "the corpus has no invalid grouped key"
    return {uniq[i].tobytes(): out[i] for i in np.flatnonzero(status == 0)}


@pytest.fixture(scope="module")
def grouped(plain, cp):
    return {c: _grouped_valid(plain, cp, c) for c in (P256, P384, ED)}


def _cache_entry(eng, c, key, device=0):
    out = np.zeros(TABLE_WORDS[c], np.uint32)
    k = np.frombuffer(key, np.uint8).copy()
    rc = eng._lib.sbv_debug_key_cache_entry(eng._h, C.c_int(device), C.c_uint8(c), _p(k), _p(out))
    assert rc in (0, 1)
    return out if rc == 1 else None


def _check(got, cp, idx, what):
    want = cp["want"][idx]
    assert np.array_equal(got, want), (what, np.flatnonzero(got != want)[:20])


@pytest.mark.parametrize("call", ["p256", "p256_digest", "p384", "ed", "mixed"])
def test_cold_and_warm_calls(plain, cp, grouped, call):
    idx, base = _run(plain, cp, call)
    _check(base, cp, idx, "uncached")
    assert 0 < base.sum() < base.size
    assert _counted(plain, cp, call)[2] == _want_launches(cp, call)
    eng = _engine()
    try:
        eng.key_cache_reserve(64, 64, 64)
        _, cold, k = _counted(eng, cp, call)
        _check(cold, cp, idx, "cold")
        assert k == _want_launches(cp, call, ALL) + (ED in _schemes(call))  # + k_ed_btab_init: the engine's first Ed25519 call
        G = {c: len(grouped[c]) for c in _schemes(call)}
        for c in (P256, P384, ED):
            st = eng.key_cache_stats(c)
            g = G.get(c, 0)
            assert st == {"capacity": 64, "resident": g, "hits": 0, "misses": g}, (c, st)
        _, warm, k = _counted(eng, cp, call)
        _check(warm, cp, idx, "warm")
        assert k == _want_launches(cp, call, ALL)
        for c, g in G.items():
            assert eng.key_cache_stats(c) == {"capacity": 64, "resident": g, "hits": g, "misses": g}, c
            for key, table in grouped[c].items():
                got = _cache_entry(eng, c, key)
                assert got is not None and np.array_equal(got, table), (c, key.hex())
    finally:
        eng.close()


def test_invalid_keys_are_never_cached(cp, grouped):
    eng = _engine()
    try:
        eng.key_cache_reserve(64, 64, 64)
        for _ in range(2):
            _run(eng, cp, "mixed")
        for c in (P256, P384, ED):
            idx = np.flatnonzero(cp["scheme"] == c)
            keys = {cp["key96"][i, :KEY_BYTES[c]].tobytes() for i in idx}
            for key in keys - set(grouped[c]):
                assert _cache_entry(eng, c, key) is None, (c, key.hex())
    finally:
        eng.close()


def test_full_cache(cp, grouped):
    eng = _engine()
    try:
        eng.key_cache_reserve(5, 5, 5)
        for rep in range(2):
            idx, got = _run(eng, cp, "mixed")
            _check(got, cp, idx, f"call {rep}")
            for c in (P256, P384, ED):
                st = eng.key_cache_stats(c)
                assert st["capacity"] == 5 and st["resident"] == 5, (c, st)
                assert st["hits"] == 5 * rep and st["misses"] == len(grouped[c]) * (rep + 1) - 5 * rep, (c, st)
    finally:
        eng.close()


def test_chunked_engine(cp, grouped):
    env = {"SBV_CHUNK_ITEMS": 256}
    eng = _engine(env)
    try:
        for call in ("p256", "p256_digest", "p384", "mixed"):
            idx, got, k = _counted(eng, cp, call)
            _check(got, cp, idx, call)
            assert k == _want_launches(cp, call, (), env) + (call == "mixed"), call  # + k_ed_btab_init
        eng.key_cache_reserve(64, 64, 64)
        for call in ("p256", "p384", "mixed"):
            for _ in range(2):
                idx, got, k = _counted(eng, cp, call)
                _check(got, cp, idx, call)
                assert k == _want_launches(cp, call, ALL, env), call
        assert eng.key_cache_stats(P256)["resident"] == len(grouped[P256])
        assert eng.key_cache_stats(P384)["hits"] == 3 * len(grouped[P384])
    finally:
        eng.close()


def test_device_calls_on_a_caller_stream(cp, grouped):
    import torch
    idx, m, o, sig, key = mk.family_arrays(cp, P256)
    dig = oracle.sha256_batch(m, o)
    n = idx.size
    eng = _engine()
    try:
        eng.key_cache_reserve(64, 0, 0)
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (sig[0], sig[1], key[0], key[1], dig)]
        st = torch.cuda.Stream()
        outs = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(3)]
        with torch.cuda.stream(st):
            for ok in outs:  # cold, then two warm launches queued behind it on the same stream
                eng.verify_batch_device(P256, n, *(t.data_ptr() for t in dev), 32, ok.data_ptr(), stream=st.cuda_stream)
        st.synchronize()
        for ok in outs:
            _check(ok.cpu().numpy(), cp, idx, "device call")
        g = len(grouped[P256])
        assert eng.key_cache_stats(P256) == {"capacity": 64, "resident": g, "hits": 2 * g, "misses": g}
    finally:
        eng.close()


def test_six_concurrent_callers_share_keys(cp, grouped):
    eng = _engine()
    idx, m, o, sig, key = mk.family_arrays(cp, P256)
    results, errors = [None] * 6, []
    try:
        eng.key_cache_reserve(64, 0, 0)

        def work(t):
            try:
                results[t] = eng.hash_verify_batch(P256, m, o, sig[0], sig[1], key[0], key[1])
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)

        th = [threading.Thread(target=work, args=(t,)) for t in range(6)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors
        for r in results:
            _check(r, cp, idx, "concurrent")
        g = len(grouped[P256])
        st = eng.key_cache_stats(P256)
        assert st["resident"] == g, st
        assert st["hits"] + st["misses"] == 6 * g and st["misses"] >= g, st
        for k in grouped[P256]:
            assert _cache_entry(eng, P256, k) is not None
    finally:
        eng.close()


def test_reserve_again_empties_and_zero_frees(plain, cp, grouped):
    eng = _engine()
    try:
        def launches(e):
            before = e.kernel_launches
            _run(e, cp, "p256")
            return e.kernel_launches - before

        uncached = launches(plain)
        assert uncached == _want_launches(cp, "p256")
        eng.key_cache_reserve(64, 64, 64)
        assert launches(eng) == uncached + 2 == _want_launches(cp, "p256", ALL)  # k_kc_lookup and k_kc_insert
        g = len(grouped[P256])
        assert eng.key_cache_stats(P256)["resident"] == g
        eng.key_cache_reserve(64, 64, 64)
        assert eng.key_cache_stats(P256) == {"capacity": 64, "resident": 0, "hits": 0, "misses": 0}
        _run(eng, cp, "p256")
        assert eng.key_cache_stats(P256) == {"capacity": 64, "resident": g, "hits": 0, "misses": g}
        eng.key_cache_reserve(0, 0, 0)
        assert launches(eng) == uncached
        for c in (P256, P384, ED):
            assert eng.key_cache_stats(c) == {"capacity": 0, "resident": 0, "hits": 0, "misses": 0}
        idx, got = _run(eng, cp, "mixed")
        _check(got, cp, idx, "freed")
    finally:
        eng.close()


@pytest.mark.parametrize("env", [{"SBV_GROUP_THRESHOLD": 0}, {"SBV_GROUP_THRESHOLD": 0, "SBV_CHUNK_ITEMS": 256}], ids=["one-chunk", "chunked"])
def test_a_launch_that_does_not_group_never_reads_the_cache(cp, env):
    eng = _engine(env)
    try:
        for reserve in ((0, 0, 0), (64, 64, 64)):
            eng.key_cache_reserve(*reserve)
            for call in ("p256", "p256_digest", "p384", "ed", "mixed"):
                idx, got, k = _counted(eng, cp, call)
                _check(got, cp, idx, call)
                first_ed = call == "ed" and reserve == (0, 0, 0)  # + k_ed_btab_init
                assert k == _want_launches(cp, call, ALL if reserve[0] else (), env) + first_ed, (reserve, call)
            for c in ALL:
                assert eng.key_cache_stats(c) == {"capacity": reserve[c], "resident": 0, "hits": 0, "misses": 0}
    finally:
        eng.close()


def test_argument_faults(cp):
    import consensus_b200 as sbv
    eng = _engine()
    try:
        eng.key_cache_reserve(8, 8, 8)
        with pytest.raises(sbv.EngineFault, match=r"\(-4\)"):
            eng.key_cache_reserve(1 << 28, 0, 0)  # 8 TiB of P-256 tables
        with pytest.raises(sbv.EngineFault, match=r"\(-4\)"):
            eng.key_cache_reserve(0, 0, 1 << 62)
        for c in (P256, P384, ED):
            assert eng.key_cache_stats(c)["capacity"] == 0
        idx, got = _run(eng, cp, "mixed")
        _check(got, cp, idx, "after NOMEM")
        out = (C.c_uint64 * 4)()
        assert eng._lib.sbv_key_cache_stats(eng._h, C.c_uint8(3), out) == SBV_ERR_ARG
        assert eng._lib.sbv_key_cache_stats(eng._h, C.c_uint8(0), None) == SBV_ERR_ARG
        assert eng._lib.sbv_key_cache_reserve(None, C.c_size_t(1), C.c_size_t(0), C.c_size_t(0)) == SBV_ERR_ARG
    finally:
        eng.close()


def test_two_devices(cp, grouped):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    eng = _engine(devices=(0, 1))
    try:
        eng.key_cache_reserve(64, 64, 64)
        for _ in range(2):
            idx, got = _run(eng, cp, "mixed")
            _check(got, cp, idx, "two devices")
        for c in (P256, P384, ED):
            st = eng.key_cache_stats(c)
            assert st["capacity"] == 128 and st["hits"] == st["misses"] > 0, (c, st)
    finally:
        eng.close()
