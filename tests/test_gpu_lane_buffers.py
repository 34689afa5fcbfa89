"""The buffers of a host-buffer call's lane on the GPU (engine.cu: each_lane_buffer, sbv_lane_reserve, lane_free).

A lane has one carve area, which the mixed calls (sbv_mix_carve) and the RSA calls (rsa_carve) each lay out in full.  One
engine alternates the two users: mixed384 calls with SHA-384 items, and RSA PKCS #1 v1.5 and PSS calls over 2048-, 3072-
and 4096-bit keys.  Their sizes are chosen so that calls of either kind grow the carve over the other's layout and reuse
a carve the other has grown.  The same sequence then runs from several threads at once, so that several lanes hold carves.
Every verdict array is checked against OpenSSL (mixed) and oracle_rsa.ref (RSA).  Last, three engines in turn run a
chunked call (SBV_CHUNK_ITEMS, which creates the lane's chunk events) and are destroyed; each one's verdicts are checked."""
import os
import threading

import numpy as np
import pytest

import mixed384_cases as mc
import oracle
import rsa_cases as rc
import rsa_pss_cases as pc
from oracle import corpus
from oracle_rsa import ref

pytestmark = pytest.mark.gpu


def _engine(env=None):
    """An engine on device 0, created with the settings of env (read once, by sbv_create)."""
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
def reg():
    return mc.registries(n256=5, n384=5, n_ed=6, seed=41)


def _mixed(reg, n, seed):
    """A mixed384 call over n items of every tag: about 400 bytes of carve per item."""
    cp = mc.make_corpus(np.random.default_rng(seed).integers(0, 5, n).astype(np.uint8), reg, seed=seed, hi=250)
    want = mc.expected_ok(cp, reg)
    assert 0 < int(want.sum()) < n
    if seed % 2:
        return f"mixed384 registered {n}", lambda e: e.mixed384_verify_registered(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"]), want
    return f"mixed384 batch {n}", lambda e: e.mixed384_verify_batch(cp["scheme"], cp["msgs"], cp["off"], cp["sig96"], cp["key96"]), want


def _rsa(k, hash, n, pss):
    """An RSA call over n items of the k-byte corpus, repeated: 2k + 69 bytes of carve per item."""
    c = (pc if pss else rc).make_cases(k, hash)
    idx = np.arange(n) % c["n"]
    dig, sig, mod, exp = (np.ascontiguousarray(c[f][idx]) for f in ("digest", "sig", "mod", "exp"))
    if pss:
        want = pc.want(c, ref.SALT_AUTO)[idx]
        call = lambda e: e.rsa_pss_verify_batch(hash, ref.SALT_AUTO, dig, sig, mod, exp)
    else:
        want = ref.verify_batch(k, hash, c["digest"], c["sig"], c["mod"], c["exp"])[idx]
        call = lambda e: e.rsa_verify_batch(hash, dig, sig, mod, exp)
    assert 0 < int(want.sum()) < n
    return f"rsa {'pss' if pss else 'pkcs1'} {8 * k} x {n}", call, want


@pytest.fixture(scope="module")
def steps(reg):
    """(name, call, expected verdicts) in order; the carve each takes, roughly, and whether it grows the lane's carve."""
    return [
        _mixed(reg, 300, 1),                            # 120 KB, grows
        _rsa(256, ref.SHA256, 600, pss=False),          # 350 KB, grows over the mixed layout
        _mixed(reg, 600, 2),                            # 240 KB, reuses the RSA carve
        _rsa(256, ref.SHA256, 300, pss=True),           # 175 KB, reuses
        _mixed(reg, 1500, 3),                           # 600 KB, grows
        _rsa(384, ref.SHA384, 600, pss=False),          # 500 KB, reuses
        _rsa(384, ref.SHA384, 1200, pss=True),          # 1.0 MB, grows
        _mixed(reg, 2000, 4),                           # 800 KB, reuses
        _mixed(reg, 4000, 5),                           # 1.6 MB, grows
        _rsa(512, ref.SHA512, 1000, pss=False),         # 1.1 MB, reuses
        _rsa(512, ref.SHA512, 2500, pss=True),          # 2.7 MB, grows
        _mixed(reg, 3000, 6),                           # 1.2 MB, reuses
    ]


def _run(e, steps):
    for name, call, want in steps:
        got = call(e)
        assert np.array_equal(got, want), (name, np.flatnonzero(got != want)[:8])


def test_mixed_and_rsa_share_the_carve(reg, steps):
    with _engine() as e:
        mc.set_keys(e, reg)
        _run(e, steps)
        _run(e, steps[::-1])  # every call again, now on a carve the largest call has grown


def test_several_lanes_hold_carves(reg, steps):
    """Four threads run the sequence at once, each from a different step, so the lanes' carves differ in size and layout."""
    errors = []

    def worker(e, first):
        try:
            _run(e, steps[first:] + steps[:first])
        except BaseException as x:  # noqa: BLE001 - reported by the main thread
            errors.append(x)

    with _engine() as e:
        mc.set_keys(e, reg)
        ts = [threading.Thread(target=worker, args=(e, 3 * i)) for i in range(4)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
    assert not errors, errors[0]


def test_engines_after_a_chunked_call():
    """Three engines in turn: each verifies a batch in 11 chunks (SBV_CHUNK_ITEMS=256) and is destroyed."""
    b = corpus.make_batch(oracle.P256, n=3000, K=8, seed=23, corrupt_rate=4)
    want = oracle.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert 0 < int(want.sum()) < want.size
    for _ in range(3):
        with _engine({"SBV_CHUNK_ITEMS": 256}) as e:
            assert np.array_equal(e.verify_batch(oracle.P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"]), want)
