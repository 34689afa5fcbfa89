"""sbv_mixed384_verify_registered, sbv_mixed384_verify_batch and sbv_mixed384_verify_quorum on the GPU: mixed batches
whose ECDSA items are signed over SHA-256 (tags 0, 1) or SHA-384 (tags 3, 4) beside Ed25519 items (tag 2).  Verdicts
against OpenSSL over each item's own digest and item for item against the single-scheme calls; every SHA-384 item also
goes in under its SHA-256 tag and the reverse, so a swapped hash cannot pass.  The CPU twin of the new kernels is
test_hostsim_mixed384.py."""
import os

import numpy as np
import pytest

import mixed384_cases as mc
from mixed_cases import gather
from oracle import ecdsa_ref

pytestmark = pytest.mark.gpu

TAGS = ["random", "runs", "alternating", "sha384_only"]


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


def _tags(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 5, n).astype(np.uint8)
    if kind == "runs":
        return np.repeat(rng.integers(0, 5, n), rng.integers(1, 40, n))[:n].astype(np.uint8)
    if kind == "alternating":
        return (np.arange(n) % 5).astype(np.uint8)
    return rng.integers(3, 5, n).astype(np.uint8)


@pytest.fixture(scope="module")
def reg():
    return mc.registries(n256=5, n384=5, n_ed=6, seed=31)


@pytest.fixture(scope="module")
def eng(reg):
    e = _engine()
    mc.set_keys(e, reg)
    yield e
    e.close()


def _registered(e, cp, fn="mixed384_verify_registered"):
    return getattr(e, fn)(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"])


def _batch(e, cp, fn="mixed384_verify_batch"):
    return getattr(e, fn)(cp["scheme"], cp["msgs"], cp["off"], cp["sig96"], cp["key96"])


def _single(e, cp, keys):
    """Item by item, the single-scheme calls: sbv_hash384_verify_* (tags 3, 4), sbv_hash_verify_* (0, 1) and
    sbv_ed25519_verify_* (2), each over its items' messages."""
    out = np.full(cp["scheme"].size, 0xEE, np.uint8)
    for t in range(5):
        idx = np.flatnonzero(cp["scheme"] == t)
        if idx.size == 0:
            continue
        m, o = gather(cp["msgs"], cp["off"], idx)
        if t == mc.ED:
            sig = np.ascontiguousarray(cp["sig96"][idx, :64])
            out[idx] = (e.ed25519_verify_batch(m, o, sig, np.ascontiguousarray(cp["key96"][idx, :32])) if keys
                        else e.ed25519_verify_registered(m, o, cp["key_slot"][idx], sig))
            continue
        c, L = mc.CURVE[t], mc.L[mc.CURVE[t]]
        r, s = np.ascontiguousarray(cp["sig96"][idx, :L]), np.ascontiguousarray(cp["sig96"][idx, L:2 * L])
        wide = t >= mc.P256_SHA384
        if keys:
            qx, qy = np.ascontiguousarray(cp["key96"][idx, :L]), np.ascontiguousarray(cp["key96"][idx, L:2 * L])
            out[idx] = (e.hash384_verify_batch if wide else e.hash_verify_batch)(c, m, o, r, s, qx, qy)
        else:
            out[idx] = (e.hash384_verify_registered if wide else e.hash_verify_registered)(c, m, o, cp["key_slot"][idx], r, s)
    return out


@pytest.mark.parametrize("kind", TAGS)
def test_all_tags_against_openssl_and_the_single_scheme_calls(eng, reg, kind):
    cp = mc.make_corpus(_tags(kind, 700, seed=len(kind)), reg, seed=len(kind) + 100)
    want = mc.expected_ok(cp, reg)
    assert 0 < int(want.sum()) < want.size
    got_reg = _registered(eng, cp)
    got_keys = _batch(eng, cp)
    assert np.array_equal(got_reg, want)
    assert np.array_equal(got_keys, want)
    assert np.array_equal(got_reg, _single(eng, cp, keys=False))
    assert np.array_equal(got_keys, _single(eng, cp, keys=True))


def test_hash_twins_reject_under_the_other_hash(eng, reg):
    """Every item twice: under its own tag and under the same curve's other hash.  The twin of a valid ECDSA item must
    reject, so an item hashed with the wrong function cannot pass; Ed25519 twins are identical items."""
    cp = mc.make_corpus(_tags("random", 600, seed=3), reg, seed=44, corrupt=0.0)
    both = mc.concat(cp, mc.with_scheme(cp, mc.SWAP[cp["scheme"]]))
    want = mc.expected_ok(both, reg)
    n = cp["scheme"].size
    ecdsa = cp["scheme"] != mc.ED
    assert want[:n].all()
    assert not want[n:][ecdsa].any() and want[n:][~ecdsa].all()
    for got in (_registered(eng, both), _batch(eng, both)):
        assert np.array_equal(got, want)


@pytest.mark.parametrize("fn", ["registered", "batch"])
def test_tags_0_to_2_match_the_existing_call_and_its_launches(eng, reg, fn):
    """A batch without SHA-384 items: the verdicts and the kernel launches of the sbv_mixed_* call."""
    cp = mc.make_corpus(np.random.default_rng(5).integers(0, 3, 3000).astype(np.uint8), reg, seed=55, hi=200)
    call = _registered if fn == "registered" else _batch
    old_fn, new_fn = f"mixed_verify_{fn}", f"mixed384_verify_{fn}"
    l0 = eng.kernel_launches
    old = call(eng, cp, old_fn)
    l1 = eng.kernel_launches
    new = call(eng, cp, new_fn)
    l2 = eng.kernel_launches
    assert np.array_equal(new, old)
    assert np.array_equal(new, mc.expected_ok(cp, reg))
    assert l2 - l1 == l1 - l0


@pytest.mark.parametrize("fn", ["registered", "batch"])
def test_sha384_items_add_one_launch(eng, reg, fn):
    """With SHA-384 items the call launches what the sbv_mixed_* call launches on the same items under their SHA-256 tags,
    plus k_mix_alg (k_sha2_sel takes the place of k_sha256)."""
    cp = mc.make_corpus(_tags("random", 2500, seed=8), reg, seed=66, hi=150)
    call = _registered if fn == "registered" else _batch
    as256 = mc.with_scheme(cp, np.where(cp["scheme"] >= 3, cp["scheme"] - 3, cp["scheme"]))
    l0 = eng.kernel_launches
    call(eng, as256, f"mixed_verify_{fn}")
    l1 = eng.kernel_launches
    got = call(eng, cp, f"mixed384_verify_{fn}")
    l2 = eng.kernel_launches
    assert l2 - l1 == l1 - l0 + 1
    assert np.array_equal(got, mc.expected_ok(cp, reg))


@pytest.mark.parametrize("env", [{}, {"SBV_GROUP_THRESHOLD": 0}])
def test_grouped_keys_under_both_hashes(reg, env):
    """Keys per item, each key repeating well past the grouping threshold under both hashes (one group per key whichever
    hash), with grouping on and off, and with a key cache reserved."""
    tags = _tags("random", 1600, seed=9)
    cp = mc.make_corpus(tags, reg, seed=77, hi=120, key_choice=2)
    for c in (0, 1):
        for t in (c, c + 3):
            for k in np.unique(cp["key_slot"][tags == t]):
                assert ((tags == t) & (cp["key_slot"] == k)).sum() >= 16
    want = mc.expected_ok(cp, reg)
    with _engine(env) as e:
        assert np.array_equal(_batch(e, cp), want)
        e.key_cache_reserve(64, 64, 64)
        assert np.array_equal(_batch(e, cp), want)
        assert np.array_equal(_batch(e, cp), want)  # the second call hits the cache


def test_quorum_c4_shape(eng, reg):
    """Commit votes of a consenter set of 16 with every tag (SHA-384 signers of both curves among them): verdicts and
    counts against OpenSSL and ecdsa_ref.count_commit_votes_batch."""
    tags = [0, 0, 0, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 0, 2, 3]
    n_inst = 64
    scheme, who, inst, sender, signer, dm = mc.vote_stream(tags, n_inst, seed=12)
    slot_of = []
    seen = {0: 0, 1: 0, 2: 0}
    for t in tags:
        c = mc.CURVE.get(t, mc.ED)
        own = np.flatnonzero(reg["ecdsa_curve"] == c) if c != mc.ED else np.arange(reg["ed_pub"].shape[0])
        slot_of.append(own[seen[c] % own.size])
        seen[c] += 1
    cp = mc.make_corpus(scheme, reg, seed=88, lo=100, hi=400, corrupt=0.1, key_slot=np.array(slot_of, np.uint32)[who])
    want = mc.expected_ok(cp, reg)
    threshold = 10  # n = 16: Q = 11, the caller passes Q - 1
    want_cnt, want_reached = ecdsa_ref.count_commit_votes_batch(inst, sender, signer, dm, want, n_inst, threshold)
    ok, cnt, reached = eng.mixed384_verify_quorum(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"], inst, sender, signer, dm,
                                                  n_inst, threshold)
    assert np.array_equal(ok, want)
    assert np.array_equal(cnt, np.asarray(want_cnt)) and np.array_equal(reached, np.asarray(want_reached))
    assert 0 < int(np.asarray(want_reached).sum()) < n_inst


def test_empty_and_multi_kib_messages(eng, reg):
    tags = _tags("alternating", 400, seed=0)
    lens = np.where(np.arange(400) % 4 == 0, 0, np.where(np.arange(400) % 4 == 1, 5000 + np.arange(400), 111 + np.arange(400) % 3))
    cp = mc.make_corpus(tags, reg, seed=99, lens=lens)
    want = mc.expected_ok(cp, reg)
    assert np.array_equal(_registered(eng, cp), want)
    assert np.array_equal(_batch(eng, cp), want)


def test_bad_tags_are_argument_faults_with_nothing_written_or_launched(eng, reg):
    import consensus_b200 as sbv
    cp = mc.make_corpus(_tags("random", 64, seed=1), reg, seed=5)
    for bad in (5, 255):
        for at in (0, 37):
            scheme = cp["scheme"].copy()
            scheme[at] = bad
            x = mc.with_scheme(cp, scheme)
            out = np.full(64, 7, np.uint8)
            l0 = eng.kernel_launches
            with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at {at}"):
                eng.mixed384_verify_registered(x["scheme"], x["msgs"], x["off"], x["key_slot"], x["sig96"], out=out)
            with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at {at}"):
                eng.mixed384_verify_batch(x["scheme"], x["msgs"], x["off"], x["sig96"], x["key96"], out=out)
            with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at {at}"):
                eng.mixed384_verify_quorum(x["scheme"], x["msgs"], x["off"], x["key_slot"], x["sig96"], np.zeros(64, np.uint32),
                                           np.ones(64, np.uint16), np.ones(64, np.uint16), np.ones(64, np.uint8), 1, 1)
            assert eng.kernel_launches == l0
            assert (out == 7).all()
    # the sbv_mixed_* calls keep rejecting both SHA-384 tags
    for bad in (3, 4):
        scheme = np.zeros(64, np.uint8)
        scheme[9] = bad
        x = mc.with_scheme(cp, scheme)
        with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at 9"):
            eng.mixed_verify_registered(x["scheme"], x["msgs"], x["off"], x["key_slot"], x["sig96"])
        with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at 9"):
            eng.mixed_verify_batch(x["scheme"], x["msgs"], x["off"], x["sig96"], x["key96"])
        with pytest.raises(sbv.EngineFault, match=f"bad scheme tag {bad} at 9"):
            eng.mixed_verify_quorum(x["scheme"], x["msgs"], x["off"], x["key_slot"], x["sig96"], np.zeros(64, np.uint32),
                                    np.ones(64, np.uint16), np.ones(64, np.uint16), np.ones(64, np.uint8), 1, 1)


def test_multi_device_sharding(reg):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {torch.cuda.device_count()}")
    import consensus_b200 as sbv
    cp = mc.make_corpus(_tags("runs", 900, seed=4), reg, seed=101)
    want = mc.expected_ok(cp, reg)
    with sbv.Engine(n_devices=2) as e2:
        mc.set_keys(e2, reg)
        assert np.array_equal(_registered(e2, cp), want)
        assert np.array_equal(_batch(e2, cp), want)
        n = cp["scheme"].size
        inst = (np.arange(n) * 7 // n).astype(np.uint32)
        sender = (np.arange(n) % 13 + 1).astype(np.uint16)
        dm = np.ones(n, np.uint8)
        ok, cnt, reached = e2.mixed384_verify_quorum(cp["scheme"], cp["msgs"], cp["off"], cp["key_slot"], cp["sig96"], inst, sender, sender, dm, 7, 5)
        want_cnt, want_reached = ecdsa_ref.count_commit_votes_batch(inst, sender, sender, dm, want, 7, 5)
        assert np.array_equal(ok, want)
        assert np.array_equal(cnt, np.asarray(want_cnt)) and np.array_equal(reached, np.asarray(want_reached))
