"""Ed25519 keys grouped inside a keys-per-item launch (sbv_ed25519_verify_batch) on the device: engines at
SBV_GROUP_THRESHOLD = 0, 1, 2 and 16 give verdicts byte-identical to OpenSSL and to each other on every corpus shape;
the comb tables (sbv_debug_ed25519_comb_tab) and the comb kernel with crafted k (sbv_debug_ed25519_verify_comb_k) equal
the CPU simulation's; which keys get a table; the kernel launches of each call; pinned and pageable input, concurrent
callers, the fault convention and a two-device engine.  tests/test_hostsim_ed25519_grouped.py runs the same sets on the CPU simulation."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

import ed25519_edges as edges
import ed25519_grouped as grp
import launch_counts as lc
import oracle_ed25519 as oe
from oracle_ed25519 import corpus, ref
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRESHOLDS = (0, 1, 2, 16)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def engines():
    es = {T: _engine(SBV_GROUP_THRESHOLD=T) for T in THRESHOLDS}
    c = corpus.make_corpus(64, seed=499, n_keys=2, crafted_max=0)
    for T, e in es.items():  # the first Ed25519 call of a device also builds the table of B (k_ed_btab_init)
        assert _launches(e, c)[1] == lc.ed25519(64, {"SBV_GROUP_THRESHOLD": T}) + 1, T
    yield es
    for e in es.values():
        e.close()


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    """The CPU simulation, built outside the tree."""
    out = str(tmp_path_factory.mktemp("hostsim") / "libhostsim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-DSBV_P384_GW=8", "-pthread", "-o", out,
                           os.path.join(ROOT, "tools", "hostsim", "hostsim.cpp")])
    return C.CDLL(out)


def _launches(e, c):
    """The verdicts of c, and the kernels the call launched."""
    before = e.kernel_launches
    got = e.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    return got, e.kernel_launches - before


def _all_equal(engines, c, want=None):
    if want is None:
        want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    for T, e in engines.items():
        got, k = _launches(e, c)
        assert np.array_equal(got, want), (T, np.nonzero(got != want)[0][:10])
        assert k == lc.ed25519(len(c["sig"]), {"SBV_GROUP_THRESHOLD": T}), (T, k)
    return want


def _rows_corpus(rows):
    a = rows.arrays()
    return {"msgs": a["msgs"], "off": a["off"], "sig": a["sig"], "pub": a["pub"]}


def comb_tab(eng, pub, items):
    pub = np.ascontiguousarray(pub, np.uint8)
    items = np.ascontiguousarray(items, np.uint32)
    status = np.full(items.size, -1, np.int32)
    out = np.zeros((items.size, 510, 24), np.uint32)
    rc = eng._lib.sbv_debug_ed25519_comb_tab(eng._h, C.c_size_t(pub.size // 32), _p(pub), C.c_size_t(items.size), _p(items), _p(status), _p(out))
    assert rc == 0
    return status, out


@pytest.mark.parametrize("n_keys", [64, 1024])
def test_full_corpus(engines, n_keys):
    c = corpus.make_corpus(65536, seed=500 + n_keys, n_keys=n_keys, crafted_max=64)
    want = _all_equal(engines, c)
    assert 0 < want.sum() < want.size


def test_every_class_and_edge_key(engines):
    """Every corruption class; y >= p, "-0", small-order and mixed-order keys repeated; S >= L under grouped keys."""
    c = grp.mixed_corpus(6000, seed=501, n_keys=48)
    want = _all_equal(engines, c)
    m = c["cls"] == corpus.CLASS_NAMES.index("s_plus_l")
    assert m.sum() > 16 and not want[m].any()


def test_one_key_and_all_distinct(engines):
    c = corpus.make_corpus(5000, seed=502, n_keys=1, crafted_max=0)
    _all_equal(engines, c)
    c = corpus.make_corpus(5000, seed=503, n_keys=5000, crafted_max=16)
    _all_equal(engines, c)


def test_threshold_boundary_and_undecodable_key(engines):
    """At T = 16: a key with 15 items (generic), one with 16 (comb), and an off-curve key repeated 40 times."""
    rows = edges._subset(grp.comb_rows(), range(64))
    keys = grp.table_keys()
    bad = [A for A in keys if ref.decode(A) is None][0]
    c = corpus.make_corpus(31, seed=504, n_keys=2, crafted_max=0)
    pub = c["pub"].copy()
    k0, k1 = np.unique(pub, axis=0)[:2]
    pub[:15], pub[15:] = k0, k1
    c2 = {"msgs": c["msgs"], "off": c["off"], "sig": c["sig"], "pub": pub}
    _all_equal(engines, c2)
    big = edges.Rows()
    for i in range(len(rows)):
        big.add(rows.A[i], rows.M[i], rows.sig[i], rows.want[i], rows.tag[i])
    for _ in range(40):
        big.add(bad, b"m", rows.sig[0], False, "off-curve")
    _all_equal(engines, _rows_corpus(big))
    st, _ = comb_tab(engines[16], pub, [0, 15])
    assert list(st) == [1, 0], st
    pubs = np.frombuffer(b"".join([bad] * 20 + [keys[0]] * 20), np.uint8)
    st, _ = comb_tab(engines[16], pubs, [0, 20])
    assert list(st) == [2, 0]


def test_encodings_of_one_point_are_separate_keys(engines):
    """The identity as canonical, y = 1 + p and "-0": three keys.  At T = 2 each reaches T only on its own count."""
    ids = edges.IDENTITY_KEYS
    pub = np.frombuffer(b"".join([ids[0], ids[1], ids[1], ids[2]]), np.uint8)
    st, out = comb_tab(engines[2], pub, [0, 1, 3])
    assert list(st) == [1, 0, 1]
    assert np.array_equal(out[1], grp.comb_words(ids[1]))
    rows = edges.Rows()
    rng = np.random.default_rng(505)
    for i in range(300):
        A = ids[i % 3]
        S = int.from_bytes(rng.bytes(32), "little") % ref.L
        R = ref.encode(edges.bmul(S))  # [k]O = O whatever k
        rows.add(A, bytes([i % 251]) * (i % 7), edges._sig(R if i % 5 else edges._flip(R, 3), S), i % 5 != 0, "identity")
    want = _all_equal(engines, _rows_corpus(rows))
    assert np.array_equal(want, np.array(rows.want, np.uint8))


def test_tables_equal_the_simulation_and_the_model(engines, hs):
    keys = grp.table_keys()
    pub = np.frombuffer(b"".join(keys), np.uint8)
    items = np.arange(len(keys), dtype=np.uint32)
    st, out = comb_tab(engines[1], pub, items)
    hst = np.full(items.size, -1, np.int32)
    hout = np.zeros_like(out)
    assert hs.hs_ed25519_comb_tab(C.c_size_t(len(keys)), _p(pub), C.c_uint32(1), C.c_uint32(8192), C.c_size_t(items.size), _p(items), _p(hst),
                                  _p(hout)) == 0
    assert np.array_equal(st, hst) and np.array_equal(out, hout)
    for i, A in enumerate(keys):
        w = grp.comb_words(A)
        assert (st[i] == 2) if w is None else np.array_equal(out[i], w), i


def test_crafted_k_equals_the_simulation(engines, hs):
    rows = grp.comb_rows()
    a = rows.arrays()
    n = len(rows)
    ok = np.full(n, 7, np.uint8)
    eng = engines[0]
    assert eng._lib.sbv_debug_ed25519_verify_comb_k(eng._h, C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) == 0
    hok = np.full(n, 7, np.uint8)
    assert hs.hs_ed25519_verify_comb_k(C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(hok)) == 0
    assert np.array_equal(ok, hok) and np.array_equal(ok, a["want"])
    acc, n2 = edges.check(edges.crafted_k(), verify_k=lambda b: _verify_comb_k(eng, b), ref_n=20, seed=9)
    assert 0 < acc < n2
    bad = a["k"].copy()
    bad[1] = np.frombuffer(ref.L.to_bytes(32, "little"), "<u4")
    assert eng._lib.sbv_debug_ed25519_verify_comb_k(eng._h, C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(bad), _p(ok)) != 0


def _verify_comb_k(eng, a):
    n = a["sig"].shape[0]
    ok = np.full(n, 7, np.uint8)
    assert eng._lib.sbv_debug_ed25519_verify_comb_k(eng._h, C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) == 0
    return ok


def test_max_keys_overflow_goes_generic():
    """With 4 table slots, exactly 4 of the keys that reach T hold one.  Which 4 is the order in which k_kg_assign's
    atomic counter hands them out, so a slot may go to a key that does not decode (status 2: a slot, no table; the
    corpus repeats off-curve keys)."""
    c = corpus.make_corpus(8192, seed=506, n_keys=64, crafted_max=32)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    e = _engine(SBV_GROUP_THRESHOLD=16, SBV_GROUP_MAX_KEYS=4)
    try:
        got, k = _launches(e, c)
        assert np.array_equal(got, want)
        assert k == lc.ed25519(8192, {"SBV_GROUP_MAX_KEYS": 4}) + 1  # + k_ed_btab_init
        uniq, first, cnt = np.unique(c["pub"], axis=0, return_index=True, return_counts=True)
        items = first[cnt >= 16]
        assert items.size > 4
        st, out = comb_tab(e, c["pub"], items)
        assert (st != 1).sum() == 4 and set(st.tolist()) <= {0, 1, 2}
        for q in np.nonzero(st != 1)[0]:
            A = bytes(c["pub"][items[q]])
            w = grp.comb_words(A)
            assert (st[q] == 2) if w is None else (st[q] == 0 and np.array_equal(out[q], w)), (q, A.hex())
        st, _ = comb_tab(e, c["pub"], first[cnt < 16]) if (cnt < 16).any() else (np.ones(1), None)
        assert (st == 1).all()
    finally:
        e.close()


def test_empty_ragged_and_pinned(engines):
    """Empty and ragged messages (edge lengths up to 10 KiB), from pageable and from pinned buffers."""
    import torch
    rng = np.random.default_rng(507)
    c = corpus.make_corpus(3000, seed=508, n_keys=20, crafted_max=16)
    lens = np.array([corpus.EDGE_LENGTHS[i % len(corpus.EDGE_LENGTHS)] for i in range(400)])
    seeds = np.frombuffer(b"".join(bytes([s]) * 32 for s in range(5)), np.uint8).reshape(5, 32)
    pubs = np.stack([np.frombuffer(oe.pubkey(bytes(s)), np.uint8) for s in seeds])
    key_idx = (np.arange(400) % 5).astype(np.int64)
    msgs = rng.integers(0, 256, int(lens.sum()) + 16, dtype=np.uint8)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    sig = oe.sign_batch(seeds, key_idx, msgs, off)
    sig[::7, 3] ^= 1
    r = {"msgs": msgs, "off": off, "sig": sig, "pub": pubs[key_idx].copy()}
    for cc in (c, r):
        want = _all_equal(engines, cc)
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
        pc = {k: pin(v) for k, v in cc.items() if k in ("msgs", "off", "sig", "pub")}
        for T in (0, 16):
            assert np.array_equal(engines[T].ed25519_verify_batch(pc["msgs"], pc["off"], pc["sig"], pc["pub"]), want)


def test_six_threads_at_once(engines):
    cs = [corpus.make_corpus(8192, seed=510 + t, n_keys=32 if t % 2 else 300, crafted_max=32) for t in range(6)]
    wants = [oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]) for c in cs]
    eng = engines[16]
    gots, errs = [None] * 6, []

    def work(t):
        try:
            for _ in range(3):
                gots[t] = eng.ed25519_verify_batch(cs[t]["msgs"], cs[t]["off"], cs[t]["sig"], cs[t]["pub"])
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=work, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for g, w in zip(gots, wants):
        assert np.array_equal(g, w)


def test_fault_convention_and_empty_launch(engines):
    eng = engines[16]
    c = corpus.make_corpus(64, seed=511, n_keys=2, crafted_max=4)
    lib, h = eng._lib, eng._h
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    assert np.array_equal(eng.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]), want)
    ok = np.full(64, 7, np.uint8)
    before = eng.kernel_launches
    assert lib.sbv_ed25519_verify_batch(h, C.c_size_t(0), _p(c["msgs"]), _p(c["off"][:1]), _p(c["sig"]), _p(c["pub"]), _p(ok)) == 0
    assert eng.kernel_launches == before and (ok == 7).all()
    assert lib.sbv_ed25519_verify_batch(h, C.c_size_t(64), _p(c["msgs"]), _p(c["off"]), _p(c["sig"]), None, _p(ok)) < 0
    bad = c["off"].copy()
    bad[10], bad[11] = bad[11], bad[10]
    assert lib.sbv_ed25519_verify_batch(h, C.c_size_t(64), _p(c["msgs"]), _p(bad), _p(c["sig"]), _p(c["pub"]), _p(ok)) < 0
    assert (ok == 7).all() and b"" != lib.sbv_last_error(h)
    assert np.array_equal(eng.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]), want)


def test_two_devices():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    c = corpus.make_corpus(40000, seed=512, n_keys=256, crafted_max=64)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    import consensus_b200 as sbv
    with sbv.Engine(devices=[0, 1]) as e:
        assert np.array_equal(e.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]), want)
