"""The device-pointer calls (sbv_verify_batch_device, sbv_verify_registered_device) as a caller that keeps the GPU busy
drives them: many distinct batches in flight on the caller's streams with no synchronisation between them, more launches
than scratch sets, scratch sets that grow while earlier launches are still queued and that Ed25519 launches share,
inputs written and verdicts read on the caller's stream only, and a key registry replaced behind queued launches.

Every verdict buffer has 64 bytes more than the batch and starts filled with 0xAB: each case checks the verdicts
against the OpenSSL oracle, that every one of the n bytes was written, and that the tail still holds 0xAB.

A case that tests ordering also checks that it can see a failure.  The batches of a sequence use disjoint key sets and
flip r on a random subset of their items, alternately about 35 % and about 65 % of them, each batch with its own subset.
So the expected verdicts of any two batches differ in at least a quarter of their positions, and so do all-accept and
all-reject: a launch that read another batch's inputs, tables or verdicts, or scratch data left by another launch,
fails its check.  _assert_detectable asserts this for the vectors each case compares."""
import ctypes as C
import functools
import threading

import numpy as np
import pytest

import edges
import oracle
import oracle_ed25519
from oracle import FIELD_BYTES, P256, P384, corpus
from oracle_ed25519 import corpus as ed_corpus
from test_gpu_round2 import _engine, _signed_requests

pytestmark = pytest.mark.gpu

SENTINEL = 0xAB
TAIL = 64
FIELDS = ("r", "s", "qx", "qy", "digest")
SLEEP_CYCLES = 500_000_000        # holds a stream long enough for the host to enqueue everything behind it
SIZES = [1, 15, 16, 17, 31, 32, 33, 2047, 2048, 2049, 70001]
SBV_ERR_ARG, SBV_ERR_NCCL = -1, -3


# ---- batches ------------------------------------------------------------------------------------------------------
def _signed(curve, m, K, seed, dlen):
    """m valid signatures over digests of dlen bytes, item i by key i % K of K keys of the batch's own (seeded)"""
    L = FIELD_BYTES[curve]
    d, kxy = corpus.make_keys(curve, K, seed)
    kidx = (np.arange(m) % K).astype(np.uint32)
    dig = corpus._blocks(seed + 1, m, dlen, b"dig")
    r, s = oracle.sign_batch(curve, d, kidx, dig, corpus._blocks(seed + 2, m, L, b"k"))
    return {"r": r, "s": s, "qx": kxy[kidx, :L].copy(), "qy": kxy[kidx, L:].copy(), "digest": dig, "keys": kxy, "key_idx": kidx,
            "priv": d}


def _oracle(curve, b):
    return oracle.verify_batch(curve, *(b[k] for k in FIELDS))


@functools.lru_cache(maxsize=None)
def _sweep(curve, dlen):
    """max(SIZES) items for the parity sweep: m signed items over 37 keys, 1/5 corrupted over every class, repeated; the
    batch of n items is the first n.  The oracle runs on the m distinct rows."""
    m = 4099 if curve == P256 else 1531
    b = _signed(curve, m, 37, 7000 + 10 * dlen + curve, dlen)
    corpus.corrupt(curve, b, seed=7100 + dlen + curve, rate=5)
    want = _oracle(curve, b)
    rows = np.arange(300_000) % m
    return {k: b[k][rows] for k in FIELDS}, want[rows]


def _pattern_batch(curve, n, K, seed, heavy, dlen=32):
    """n items over K keys of their own, r flipped on a seeded random ~65 % (heavy) or ~35 % of them.  Below n = K every
    item has its own key; above, at most UNIQUE[curve] distinct signatures repeat.  The oracle runs on the distinct rows.
    Returns the arrays, "want", the key index of every item ("kidx") and the keys ("keys")."""
    L = FIELD_BYTES[curve]
    m = n if K >= n else min(n, 4096 if curve == P256 else 400)
    base = _signed(curve, m, min(K, m), seed, dlen)
    rows = np.arange(n) % m
    flip = np.random.default_rng(seed).random(n) < (0.65 if heavy else 0.35)
    code, inv = np.unique(rows * 2 + flip, return_inverse=True)
    uniq = {k: base[k][code // 2].copy() for k in FIELDS}
    uniq["r"][code % 2 == 1, L - 1] ^= 1
    want = _oracle(curve, uniq)[inv.reshape(-1)]
    out = {k: base[k][rows].copy() for k in FIELDS}
    out["r"][flip, L - 1] ^= 1
    out.update(want=want, kidx=base["key_idx"][rows], keys=base["keys"], curve=curve, n=n, dlen=dlen)
    return out


# keys-per-item sequence: curves alternate, some launches build tables (few keys) and some do not (a key per item), and
# the sizes grow from the 13th batch on (past the headroom of every scratch buffer)
KP_SEQ = [(P256, 700, 3), (P384, 800, 3), (P256, 300, 300), (P384, 500, 500), (P256, 900, 3), (P384, 1000, 2),
          (P256, 2500, 2500), (P384, 400, 400), (P256, 1800, 4), (P384, 700, 3), (P256, 600, 600), (P384, 500, 500),
          (P256, 20000, 4), (P384, 9000, 3), (P256, 10000, 10000), (P384, 12000, 2), (P256, 40000, 5), (P384, 16000, 3),
          (P256, 12000, 12000), (P384, 8000, 3), (P256, 35000, 6), (P384, 18000, 2), (P256, 9000, 9000), (P384, 6000, 3)]
# registered-key sequence: the warp kernel (n <= 2048) first, then the thread kernel; digest lengths vary
REG_SIZES = [300, 1500, 700, 2048, 1000, 1800, 500, 1200, 900, 2000, 600, 1600,
             20000, 9000, 30000, 5000, 12000, 40000, 7000, 16000, 25000, 3000, 18000, 10000]


@functools.lru_cache(maxsize=None)
def _kp_seq():
    return [_pattern_batch(c, n, K, seed=8000 + 17 * i, heavy=i % 2 == 1) for i, (c, n, K) in enumerate(KP_SEQ)]


# registered-key parity: both curves, the warp kernel (n <= 2,048) and the thread kernel, three digest lengths
REG_PARITY = [(c, n, dlen) for c in (P256, P384) for n in (1500, 5000) for dlen in (20, 32, 64)]


@functools.lru_cache(maxsize=None)
def _registry():
    """The registered sequence, the registered parity batches and one registry with the keys of all of them: every batch
    owns the slots of its own keys (its "slot" column).  Returns (sequence, {(curve, n, dlen): batch}, curves, xy)."""
    curves, xy = [], []

    def register(b):
        b["slot"] = (len(curves) + b["kidx"]).astype(np.uint32)
        L = FIELD_BYTES[b["curve"]]
        for k in b["keys"]:
            row = np.zeros((2, 48), np.uint8)
            row[0, 48 - L:], row[1, 48 - L:] = k[:L], k[L:]
            curves.append(b["curve"])
            xy.append(row)
        return b

    seq = [register(_pattern_batch(P256 if i % 2 == 0 else P384, n, 2 + i % 5, seed=9000 + 17 * i, heavy=i % 2 == 1, dlen=(32, 20, 64)[i % 3]))
           for i, n in enumerate(REG_SIZES)]
    par = {(c, n, dlen): register(_pattern_batch(c, n, 5, seed=1200 + n + dlen + c, heavy=False, dlen=dlen)) for c, n, dlen in REG_PARITY}
    return seq, par, np.array(curves, np.uint8), np.stack(xy)


def _assert_detectable(wants):
    """Every vector differs from every other one, from all-accept and from all-reject in >= 1/4 of its positions (the
    0xAB left in an unwritten byte differs from both verdicts)."""
    for i, w in enumerate(wants):
        assert 0.25 <= w.mean() <= 0.75, (i, w.mean())
        for j, o in enumerate(wants):
            if j != i:
                m = min(w.size, o.size)
                assert (w[:m] != o[:m]).mean() >= 0.25, (i, j)


# ---- device buffers -----------------------------------------------------------------------------------------------
def _dev(b, keys=FIELDS, device="cuda:0"):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(b[k]).view(np.int32 if b[k].dtype == np.uint32 else np.uint8)).to(device)
            for k in keys}


def _ok_buf(n, device="cuda:0"):
    import torch
    return torch.full((n + TAIL,), SENTINEL, dtype=torch.uint8, device=device)


def _check(ok, want, what):
    got = ok.cpu().numpy() if hasattr(ok, "cpu") else ok
    n = want.size
    assert got.size == n + TAIL
    assert (got[n:] == SENTINEL).all(), f"{what}: written past d_ok[n): {np.flatnonzero(got[n:] != SENTINEL)[:8]}"
    unwritten = np.flatnonzero(got[:n] == SENTINEL)
    assert unwritten.size == 0, f"{what}: {unwritten.size} verdicts not written, first {unwritten[:8]}"
    bad = np.flatnonzero(got[:n] != want)
    assert bad.size == 0, f"{what}: {bad.size} wrong verdicts, first {bad[:8]} got {got[bad[:8]]} want {want[bad[:8]]}"


def _verify(eng, b, d, ok, n=None, stream=0, device_index=0):
    n = b["n"] if n is None else n
    eng.verify_batch_device(b["curve"], n, d["r"].data_ptr(), d["s"].data_ptr(), d["qx"].data_ptr(), d["qy"].data_ptr(),
                            d["digest"].data_ptr(), b["dlen"], ok.data_ptr(), stream=stream, device_index=device_index)


def _verify_reg(eng, b, d, ok, stream=0, slot_key="slot"):
    eng.verify_registered_device(b["curve"], b["n"], d[slot_key].data_ptr(), d["r"].data_ptr(), d["s"].data_ptr(), d["digest"].data_ptr(),
                                 b["dlen"], ok.data_ptr(), stream=stream)


def _raw_verify(eng, device_index, curve, n, d, dlen, ok, stream=0):
    vp = C.c_void_p
    return eng._lib.sbv_verify_batch_device(eng._h, C.c_int(device_index), C.c_uint8(curve), C.c_size_t(n), *(vp(d[k].data_ptr()) for k in FIELDS),
                                            C.c_uint8(dlen), vp(ok.data_ptr()), vp(stream))


@pytest.fixture(scope="module")
def engines():
    es = {thr: _engine(SBV_GROUP_THRESHOLD=thr) for thr in (0, 1, 2, 16)}
    yield es
    for e in es.values():
        e.close()


# ---- 1. parity of sbv_verify_batch_device ---------------------------------------------------------------------------
@pytest.mark.parametrize("thr", [0, 1, 16])
@pytest.mark.parametrize("dlen", [4, 20, 32, 48, 64])
@pytest.mark.parametrize("curve", [P256, P384])
def test_device_form_parity_sweep(engines, curve, dlen, thr):
    """Every size around the warp (32), block and SBV_KEYED_WARP_LIMIT (2,048) boundaries and one of 70,001 items, with
    grouping off (0), a table for every key (1) and the default threshold (16), one launch per size on the caller's
    stream and one synchronisation at the end."""
    import torch
    eng = engines[thr]
    arrs, want = _sweep(curve, dlen)
    nmax = max(SIZES)
    d = _dev({k: arrs[k][:nmax] for k in FIELDS})
    oks = [_ok_buf(n) for n in SIZES]
    st = torch.cuda.current_stream().cuda_stream
    for n, ok in zip(SIZES, oks):
        _verify(eng, {"curve": curve, "n": n, "dlen": dlen}, d, ok, stream=st)
    torch.cuda.synchronize()
    assert 0 < want[:nmax].sum() < nmax
    for n, ok in zip(SIZES, oks):
        _check(ok, want[:n], f"curve {curve} dlen {dlen} thr {thr} n {n}")


@pytest.mark.parametrize("curve", [P256, P384])
def test_edge_sets_through_the_device_form(engines, curve):
    """R.x >= n, the crafted comb and fixed-base scalars, and digests at and past the field size, on the generic kernel
    and with per-key tables (thresholds 1 and 2)."""
    import torch
    sets = {"big_x": edges.big_x_signatures(curve, 24, seed=400 + curve),
            "crafted": edges.crafted(curve, edges.comb_cases(curve) + edges.fixed_base_cases(curve))}
    for dlen in (20, 48, 64):
        sets[f"wide{dlen}"] = edges.wide_digest_signatures(curve, dlen, 6, seed=500 + dlen + curve)
    for name, b in sets.items():
        want = _oracle(curve, b)
        if "want" in b:
            assert np.array_equal(want, b["want"]), name
        assert 0 < want.sum() < want.size, name
        n, dlen = want.size, b["digest"].shape[1]
        d = _dev(b)
        for thr in (0, 1, 2):
            ok = _ok_buf(n)
            _verify(engines[thr], {"curve": curve, "n": n, "dlen": dlen}, d, ok)
            torch.cuda.synchronize()
            _check(ok, want, f"{name} thr {thr}")


def test_one_launch_larger_than_any_chunk():
    """300,000 P-256 items in one device call on an engine whose host-buffer calls would split them into chunks of
    1,000: the device form is one launch whatever SBV_CHUNK_ITEMS is."""
    import torch
    arrs, want = _sweep(P256, 32)
    n = 300_000
    e = _engine(SBV_CHUNK_ITEMS=1000)
    try:
        d = _dev(arrs)
        ok = _ok_buf(n)
        _verify(e, {"curve": P256, "n": n, "dlen": 32}, d, ok)
        torch.cuda.synchronize()
        _check(ok, want[:n], "300,000 items")
    finally:
        e.close()


def test_zero_items_and_bad_device_index(engines):
    """n = 0 returns 0 with no kernel launch; a device index out of range is SBV_ERR_ARG (for n = 0 as well).  Neither
    writes a verdict byte."""
    import torch
    eng = engines[16]
    arrs, _ = _sweep(P256, 32)
    d = _dev({k: arrs[k][:64] for k in FIELDS})
    ok = _ok_buf(64)
    torch.cuda.synchronize()
    before = eng.kernel_launches
    assert _raw_verify(eng, 0, P256, 0, d, 32, ok) == 0
    assert eng.kernel_launches == before
    for idx in (1, -1, 8):
        for n in (0, 64):
            assert _raw_verify(eng, idx, P256, n, d, 32, ok) == SBV_ERR_ARG, (idx, n)
    assert eng.kernel_launches == before
    torch.cuda.synchronize()
    assert (ok.cpu().numpy() == SENTINEL).all()


# ---- 2. distinct batches pipelined on the caller's streams ----------------------------------------------------------
def _run_pipelined(eng, items, streams, device_of=lambda i: 0):
    """items: [(kind, batch)], kind "kp" (sbv_verify_batch_device) or "reg" (sbv_verify_registered_device).  Uploads every
    batch, then enqueues item i on streams[i % len(streams)] behind one _sleep per stream (so that the first launches
    are still queued when the later ones take their scratch sets and grow them), synchronises once and checks every
    verdict buffer against its own batch."""
    import torch
    devs = [_dev(b, FIELDS + (("slot",) if kind == "reg" else ()), device=f"cuda:{device_of(i)}") for i, (kind, b) in enumerate(items)]
    oks = [_ok_buf(b["n"], device=f"cuda:{device_of(i)}") for i, (_, b) in enumerate(items)]
    torch.cuda.synchronize()
    for k in range(torch.cuda.device_count()):
        torch.cuda.synchronize(k)
    for s in streams:
        if s is None:
            torch.cuda._sleep(SLEEP_CYCLES // 5)     # the legacy default stream
        else:
            with torch.cuda.device(s.device), torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP_CYCLES // 5)
    for i, (kind, b) in enumerate(items):
        s = streams[i % len(streams)]
        st = s.cuda_stream if s is not None else 0
        if kind == "kp":
            _verify(eng, b, devs[i], oks[i], stream=st, device_index=device_of(i))
        else:
            _verify_reg(eng, b, devs[i], oks[i], stream=st)
    for k in range(torch.cuda.device_count()):
        torch.cuda.synchronize(k)
    for i, (kind, b) in enumerate(items):
        _check(oks[i], b["want"], f"launch {i} ({kind}, curve {b['curve']}, n {b['n']})")


@pytest.mark.parametrize("mode", ["four_streams", "one_stream", "legacy_stream", "with_registered"])
def test_pipelined_distinct_batches(mode):
    """24 keys-per-item batches (three times the scratch sets), P-256 and P-384 alternating, with and without per-key
    tables, growing from the 13th on, enqueued back to back with one synchronisation at the end: round robin on four
    streams, all on one stream, all on the legacy default stream, or on four streams interleaved with 24 registered-key
    launches, which take scratch sets too.  A fresh engine each time, so the buffers grow while launches are queued."""
    import torch
    items = [("kp", b) for b in _kp_seq()]
    e = _engine()
    try:
        if mode == "with_registered":
            reg, _, curves, xy = _registry()
            e.set_keys(curves, xy)
            items = [x for pair in zip(items, [("reg", b) for b in reg]) for x in pair]
        _assert_detectable([b["want"] for _, b in items])
        streams = {"four_streams": 4, "with_registered": 4, "one_stream": 1}.get(mode)
        streams = [torch.cuda.Stream() for _ in range(streams)] if streams else [None]
        _run_pipelined(e, items, streams)
    finally:
        e.close()


# ---- 3. inputs and outputs ordered by the caller's stream alone -----------------------------------------------------
def _mixed_key_batch(n, seed, heavy):
    """P-256, n items: the first half over 6 keys (tables at threshold 2), every item of the second half its own key"""
    half = n // 2
    a = _pattern_batch(P256, half, 6, seed, heavy)
    b = _pattern_batch(P256, n - half, n - half, seed + 1, heavy)
    out = {k: np.concatenate([a[k], b[k]]) for k in FIELDS + ("want",)}
    out.update(curve=P256, n=n, dlen=32)
    return out


@pytest.mark.parametrize("reader", ["same_stream", "event_on_second_stream"])
@pytest.mark.parametrize("thr", [0, 2])
def test_inputs_and_verdicts_follow_the_callers_stream(engines, thr, reader):
    """The call's buffers hold batch B.  On a fresh stream: _sleep, batch A copied over them, the call, and the verdicts
    copied to pinned host memory without blocking — either on the same stream, or on a second stream that waits on an
    event recorded after the call.  Only that stream is synchronised.  At threshold 2 the table construction (side
    stream s_tab) reads qx / qy and the generic kernel (side stream s_gen) reads every input of the keys that occur once,
    so both side streams must be ordered behind the copies."""
    import torch
    n = 3000
    A, B = _mixed_key_batch(n, 600 + thr, heavy=False), _mixed_key_batch(n, 700 + thr, heavy=True)
    _assert_detectable([A["want"], B["want"]])
    dA, bufs = _dev(A), _dev(B)
    ok = _ok_buf(n)
    host = torch.empty(n + TAIL, dtype=torch.uint8).pin_memory()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for k in FIELDS:
            bufs[k].copy_(dA[k], non_blocking=True)
        _verify(engines[thr], A, bufs, ok, stream=s.cuda_stream)
        if reader == "same_stream":
            host.copy_(ok, non_blocking=True)
        else:
            ev = torch.cuda.Event()
            ev.record(s)
    if reader == "same_stream":
        s.synchronize()
    else:
        s2 = torch.cuda.Stream()
        s2.wait_event(ev)
        with torch.cuda.stream(s2):
            host.copy_(ok, non_blocking=True)
        s2.synchronize()
    _check(host.numpy(), A["want"], f"thr {thr} {reader}")
    torch.cuda.synchronize()


# ---- 4. sbv_verify_registered_device --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def reg_engine():
    _, par, curves, xy = _registry()
    e = _engine()
    e.set_keys(curves, xy)
    yield e, par, curves
    e.close()


@pytest.mark.parametrize("dlen", [20, 32, 64])
@pytest.mark.parametrize("n", [1500, 5000])
@pytest.mark.parametrize("curve", [P256, P384])
def test_registered_device_parity(reg_engine, curve, n, dlen):
    """The warp kernel (n <= 2,048) and the thread kernel: the batch's own slots, and a tenth of the items each on slot
    n_slots, on slot 2^32 - 1 and on slots of keys of the other curve (these reject)."""
    import torch
    eng, par, curves = reg_engine
    b = dict(par[(curve, n, dlen)])
    slot, want = b["slot"].copy(), b["want"].copy()
    other = np.flatnonzero(curves != curve).astype(np.uint32)
    idx = np.random.default_rng(n + dlen + curve).permutation(n)[: 3 * (n // 10)].reshape(3, -1)
    slot[idx[0]] = curves.size
    slot[idx[1]] = 0xFFFFFFFF
    slot[idx[2]] = other[idx[2] % other.size]
    want[idx.reshape(-1)] = 0
    assert 0 < want.sum() < n
    b["slot"] = slot
    d = _dev(b, ("r", "s", "digest", "slot"))
    ok = _ok_buf(n)
    _verify_reg(eng, b, d, ok)
    torch.cuda.synchronize()
    _check(ok, want, f"registered curve {curve} n {n} dlen {dlen}")


def test_registered_device_empty_registry():
    """No key of the call's curve (an empty registry, or keys of the other curve only): every item rejects, written by
    the memset path, and nothing past n."""
    import torch
    b = _pattern_batch(P384, 700, 3, seed=1300, heavy=False)
    b["slot"] = b["kidx"].astype(np.uint32)
    d = _dev(b, ("r", "s", "digest", "slot"))
    e = _engine()
    try:
        for keys in ("none", "p256_only"):
            if keys == "none":
                e.set_keys(np.zeros(0, np.uint8), np.zeros((0, 96), np.uint8))
            else:
                _, kxy = corpus.make_keys(P256, 4, 1301)
                e.set_keys(np.zeros(4, np.uint8), kxy.reshape(4, 2, 32))
            ok = _ok_buf(b["n"])
            _verify_reg(e, b, d, ok)
            torch.cuda.synchronize()
            _check(ok, np.zeros(b["n"], np.uint8), f"registry {keys}")
    finally:
        e.close()


def test_registered_device_pipelined():
    """24 registered-key batches with their own slots, P-256 and P-384 alternating, growing from the 13th on (warp kernel,
    then thread kernel), on four streams with one synchronisation at the end."""
    import torch
    reg, _, curves, xy = _registry()
    _assert_detectable([b["want"] for b in reg])
    e = _engine()
    try:
        e.set_keys(curves, xy)
        _run_pipelined(e, [("reg", b) for b in reg], [torch.cuda.Stream() for _ in range(4)])
    finally:
        e.close()


def test_registry_swap_behind_queued_launches():
    """Launches enqueued behind a _sleep, then sbv_set_keys maps the same slots to other keys, then more launches: the
    first ones verify against the old keys, the later ones against the new (sbv_set_keys waits for the launches that
    may still read the old tables)."""
    import torch
    n, K = 1500, 4
    dold, old = corpus.make_keys(P256, K, 1400)
    dnew, new = corpus.make_keys(P256, K, 1500)
    batches = []
    for i in range(6):
        # each item signed by the old or the new key of its slot, at random: the two registries give opposite verdicts
        rng = np.random.default_rng(1600 + i)
        slot = rng.integers(0, K, n).astype(np.uint32)
        by_new = rng.random(n) < 0.5
        dig = corpus._blocks(1700 + i, n, 32, b"dig")
        r, s = oracle.sign_batch(P256, np.concatenate([dold, dnew]), (slot + K * by_new).astype(np.uint32), dig, corpus._blocks(1800 + i, n, 32, b"k"))
        batches.append({"curve": P256, "n": n, "dlen": 32, "r": r, "s": s, "digest": dig, "slot": slot,
                        "old": oracle.verify_batch(P256, r, s, old[slot, :32], old[slot, 32:], dig),
                        "new": oracle.verify_batch(P256, r, s, new[slot, :32], new[slot, 32:], dig)})
    for b in batches:
        assert (b["old"] != b["new"]).mean() >= 0.25
    _assert_detectable([b["old"] for b in batches[:3]] + [b["new"] for b in batches[3:]])
    e = _engine()
    try:
        e.set_keys(np.zeros(K, np.uint8), old.reshape(K, 2, 32))
        ds = [_dev(b, ("r", "s", "digest", "slot")) for b in batches]
        oks = [_ok_buf(n) for _ in batches]
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
        for i in range(3):
            _verify_reg(e, batches[i], ds[i], oks[i], stream=s.cuda_stream)
        e.set_keys(np.zeros(K, np.uint8), new.reshape(K, 2, 32))
        for i in range(3, 6):
            _verify_reg(e, batches[i], ds[i], oks[i], stream=s.cuda_stream)
        s.synchronize()
        for i, b in enumerate(batches):
            _check(oks[i], b["old"] if i < 3 else b["new"], f"launch {i} ({'before' if i < 3 else 'after'} the swap)")
    finally:
        e.close()


# ---- 5 / 6. ECDSA and Ed25519 on the same scratch sets, from several threads ----------------------------------------
def _threads(fns):
    errs = []

    def run(f):
        try:
            f()
        except BaseException as ex:  # noqa: BLE001 - reported below
            errs.append(repr(ex))
    th = [threading.Thread(target=run, args=(f,)) for f in fns]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs


def _device_worker(eng, items, n_launches, n_streams, out):
    """n_launches device-form launches over items [(kind, batch)] in turn, round robin on n_streams streams of the
    worker's own, each with its own verdict buffer; checked after those streams are synchronised.  out: one entry per
    launch."""
    import torch
    ds = [_dev(b, FIELDS + (("slot",) if kind == "reg" else ())) for kind, b in items]
    oks = [_ok_buf(items[i % len(items)][1]["n"]) for i in range(n_launches)]
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    torch.cuda.current_stream().synchronize()
    for i in range(n_launches):
        kind, b = items[i % len(items)]
        (_verify if kind == "kp" else _verify_reg)(eng, b, ds[i % len(items)], oks[i], stream=streams[i % n_streams].cuda_stream)
        out.append(kind)
    for s in streams:
        s.synchronize()
    for i, ok in enumerate(oks):
        kind, b = items[i % len(items)]
        _check(ok, b["want"], f"{kind} launch {i}")


def _hash_jobs():
    jobs = []
    for curve, n, K, seed in [(P256, 1500, 7, 2100), (P256, 5000, 3, 2200), (P384, 700, 3, 2300), (P256, 9000, 5, 2400)]:
        msgs, off, r, s, qx, qy = _signed_requests(curve, n, K, seed=seed)
        jobs.append((curve, msgs, off, r, s, qx, qy, oracle.verify_batch(curve, r, s, qx, qy, oracle.sha256_batch(msgs, off))))
    return jobs


def _hash_worker(eng, jobs, rounds, out):
    for _ in range(rounds):
        for curve, msgs, off, r, s, qx, qy, want in jobs:
            got = eng.hash_verify_batch(curve, msgs, off, r, s, qx, qy)
            assert np.array_equal(got, want), (curve, want.size, np.flatnonzero(got != want)[:8])
            out.append(1)


def test_ecdsa_and_ed25519_share_scratch_sets():
    """One engine at SBV_GROUP_THRESHOLD=2 with SBV_CHUNK_ITEMS=256 (host-buffer calls hold a scratch set open between
    their halves): grouped Ed25519 batches (few keys: comb tables in the scratch sets), device-form ECDSA launches on
    two streams and chunked hash-and-verify calls, from three threads at once.  Both families grow the shared buffers
    after the other has used them: the Ed25519 tables (49 KiB per key) outgrow the ECDSA ones, the ECDSA per-item
    buffers outgrow the Ed25519 ones."""
    ed = [ed_corpus.make_corpus(n, seed=2500 + n, n_keys=6, crafted_max=16) for n in (800, 2500, 6000, 1500)]
    ed_want = [oracle_ed25519.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"]) for c in ed]
    kp = _kp_seq()
    dev_batches = [kp[i] for i in (0, 1, 4, 5, 12, 13, 16, 17)]
    jobs = _hash_jobs()
    _assert_detectable(ed_want + [b["want"] for b in dev_batches])
    for j in jobs:
        assert 0.25 <= j[-1].mean() <= 0.75
    e = _engine(SBV_GROUP_THRESHOLD=2, SBV_CHUNK_ITEMS=256)
    try:
        def ed_worker():
            for _ in range(2):
                for c, want in zip(ed, ed_want):
                    got = e.ed25519_verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
                    assert np.array_equal(got, want), (want.size, np.flatnonzero(got != want)[:8])
        done = []
        _threads([ed_worker, lambda: _device_worker(e, [("kp", b) for b in dev_batches], 24, 2, done), lambda: _hash_worker(e, jobs, 2, done)])
    finally:
        e.close()


def test_profiling_under_concurrent_launches():
    """Profiling on while chunked host-buffer calls (SBV_CHUNK_ITEMS=256) are held open between their halves and other
    threads make well over 25 launches (the event pool grows by 25 launches at a time): verdicts unchanged, and
    sbv_profile_read counts one launch per keys-per-item launch (chunked or not) and per registered launch."""
    import torch
    reg, _, curves, xy = _registry()
    kp = _kp_seq()
    jobs = _hash_jobs()
    e = _engine(SBV_GROUP_THRESHOLD=2, SBV_CHUNK_ITEMS=256)
    try:
        e.set_keys(curves, xy)
        torch.cuda.synchronize()
        e.profile_enable(True)
        dev_done, hash_done, reg_done = [], [], []
        _threads([lambda: _device_worker(e, [("kp", b) for b in kp[:12]], 60, 2, dev_done),
                  lambda: _device_worker(e, [("reg", b) for b in reg[:12]], 36, 1, reg_done),
                  lambda: _hash_worker(e, jobs, 2, hash_done), lambda: _hash_worker(e, jobs[::-1], 2, hash_done)])
        torch.cuda.synchronize()
        prep_ms, verify_ms, pairs = e.profile_read()
        assert pairs == len(dev_done) + len(reg_done) + len(hash_done), (pairs, len(dev_done), len(reg_done), len(hash_done))
        assert pairs > 3 * 25
        assert prep_ms > 0 and verify_ms > 0
        e.profile_enable(False)
    finally:
        e.close()


# ---- 7. the second device of a two-device engine --------------------------------------------------------------------
def _two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


@pytest.mark.parametrize("curve", [P256, P384])
def test_second_device_parity_sweep(curve):
    """The parity sweep at device_index = 1 of a two-device engine, on device 1's buffers and legacy stream."""
    _two_gpus()
    import torch
    import consensus_b200 as sbv
    with sbv.Engine(n_devices=2) as e2:
        for dlen in (4, 20, 32, 48, 64):
            arrs, want = _sweep(curve, dlen)
            nmax = max(SIZES)
            d = _dev({k: arrs[k][:nmax] for k in FIELDS}, device="cuda:1")
            oks = [_ok_buf(n, device="cuda:1") for n in SIZES]
            torch.cuda.synchronize(1)
            for n, ok in zip(SIZES, oks):
                _verify(e2, {"curve": curve, "n": n, "dlen": dlen}, d, ok, device_index=1)
            torch.cuda.synchronize(1)
            for n, ok in zip(SIZES, oks):
                _check(ok, want[:n], f"device 1 curve {curve} dlen {dlen} n {n}")


def test_second_device_pipelined():
    """The keys-per-item sequence on a two-device engine, batches alternating between the devices, two streams on each."""
    _two_gpus()
    import torch
    import consensus_b200 as sbv
    items = [("kp", b) for b in _kp_seq()]
    streams = []
    for k in (0, 1):
        with torch.cuda.device(k):
            streams.append([torch.cuda.Stream(), torch.cuda.Stream()])
    # item i on device i % 2 and its stream (i // 2) % 2 of that device
    order = [streams[i % 2][(i // 2) % 2] for i in range(4)]
    with sbv.Engine(n_devices=2) as e2:
        _run_pipelined(e2, items, order, device_of=lambda i: i % 2)


# ---- 8. the device-form gather on one rank --------------------------------------------------------------------------
def test_gather_verdicts_device_on_one_rank():
    """sbv_gather_verdicts_device on the stream of a device-form call, on a one-rank channel: the packed mask (bit i of
    word i / 32) of the verdicts, the padding bits of the last word zero, nothing written past it;
    sbv_gather_words_device leaves its words as they are."""
    import torch
    import consensus_b200 as sbv
    uid = (C.c_uint8 * 128)()
    rc = sbv.load_library().sbv_comm_unique_id(uid)
    if rc == SBV_ERR_NCCL:
        pytest.skip("NCCL is not available")
    assert rc == 0
    arrs, want_all = _sweep(P256, 32)
    e = _engine()
    try:
        ch = e.comm_init_rank(bytes(uid), 1, 0)
        s = torch.cuda.Stream()
        for n in (1, 31, 33, 5000):
            words = (n + 31) // 32
            d = _dev({k: arrs[k][:n] for k in FIELDS})
            ok = _ok_buf(n)
            mask = torch.full((words + TAIL // 4,), -1, dtype=torch.int32, device="cuda:0")
            torch.cuda.synchronize()
            _verify(e, {"curve": P256, "n": n, "dlen": 32}, d, ok, stream=s.cuda_stream)
            e.gather_verdicts_device(ch, ok.data_ptr(), n, mask.data_ptr(), stream=s.cuda_stream)
            s.synchronize()
            want = want_all[:n]
            _check(ok, want, f"gather n {n}")
            bits = np.zeros(words * 32, np.uint8)
            bits[:n] = want
            want_words = np.packbits(bits, bitorder="little").view("<u4")
            got = mask.cpu().numpy().view(np.uint32)
            assert np.array_equal(got[:words], want_words), n
            assert (got[words:] == 0xFFFFFFFF).all(), n
        rng = np.random.default_rng(3)
        w = rng.integers(-2**31, 2**31, 100, dtype=np.int64).astype(np.int32)
        dw = torch.from_numpy(w).to("cuda:0")
        e.gather_words_device(ch, dw.data_ptr(), 100, stream=s.cuda_stream)
        s.synchronize()
        assert np.array_equal(dw.cpu().numpy(), w)
    finally:
        e.close()
