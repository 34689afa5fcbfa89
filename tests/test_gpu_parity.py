"""GPU parity: libsbv.so (through the C ABI) vs the CPU oracle on identical seeded inputs.
Integer work — the bar is bit-exact verdicts / digests / counts."""
import hashlib

import numpy as np
import pytest

import edges
import oracle
from oracle import P256, P384, corpus
from oracle import ecdsa_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(n_devices=1)
    yield e
    e.close()


def _be(v, L):
    return np.frombuffer(int(v).to_bytes(L, "big"), np.uint8)


def test_rfc6979_vectors(eng):
    from vectors import RFC6979
    for curve, ux, uy, msg, r, s in RFC6979:
        L = 32 if curve == P256 else 48
        dig = np.frombuffer(hashlib.sha256(msg).digest(), np.uint8)
        args = [_be(int(r, 16), L), _be(int(s, 16), L), _be(int(ux, 16), L), _be(int(uy, 16), L)]
        assert eng.verify_batch(curve, *args, dig).tolist() == [1]
        bad = args[0].copy(); bad[7] ^= 4
        assert eng.verify_batch(curve, bad, *args[1:], dig).tolist() == [0]


@pytest.mark.parametrize("n,K,seed,rate", [(1, 1, 3, 0), (33, 3, 5, 2), (4096, 64, 7, 4), (20011, 257, 9, 16)])
def test_p256_corrupted_corpus_bit_exact(eng, n, K, seed, rate):
    b = corpus.make_batch(P256, n=n, K=K, seed=seed, corrupt_rate=rate)
    want = oracle.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    got = eng.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    bad = np.nonzero(want != got)[0]
    assert bad.size == 0, (bad[:10], b["labels"][bad[:10]], want[bad[:10]], got[bad[:10]])
    if rate:
        assert want.min() == 0 and want.max() == 1


def test_empty_batch(eng):
    z = np.zeros((0, 32), np.uint8)
    assert eng.verify_batch(P256, z, z, z, z, z).size == 0


@pytest.mark.parametrize("curve", [P256, P384])
def test_exceptional_points_inside_the_scalar_multiplication(eng, curve):
    c = ref.CURVES[curve]
    n = c.n
    cases = []
    for k in [1, 2, 3, n - 1, n - 2, 5, 256, 2**8 + 1, 2**128]:
        for u1, u2 in [(1, 1), (k, 1), (n - k, 1), (k, n - 1), (2, n - 1), (1, 2), (7, 3), (2**255, 2**255), (n - 1, n - 1),
                       (k * 5 % n, 5), (n - (k * 5 % n), 5), (2**64, 2**64), (0x1111, 0x1111), (16, 1), (1, 16), (0, 1), (0, 77)]:
            cases.append((u1, u2, k))
    b = edges.crafted(curve, cases)
    want = oracle.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    got = eng.verify_batch(curve, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert want.tolist() == got.tolist()
    assert 0 < want.sum() < want.size  # both accept and reject (R = infinity) cases present


def test_p384_corrupted_corpus_bit_exact(eng):
    b = corpus.make_batch(P384, n=1500, K=16, seed=13, corrupt_rate=3)
    want = oracle.verify_batch(P384, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    got = eng.verify_batch(P384, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert (want == got).all(), np.nonzero(want != got)[0][:10]
    assert want.min() == 0 and want.max() == 1


def test_sha256_ragged_batch(eng):
    rng = np.random.default_rng(5)
    lens = list(range(0, 200)) + [255, 256, 257, 1000, 4095, 10240] + rng.integers(0, 3000, 300).tolist()
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    got = eng.sha256_batch(msgs, off)
    want = oracle.sha256_batch(msgs, off)
    assert (got == want).all()
    assert bytes(got[0]).hex() == hashlib.sha256(b"").hexdigest()


def test_hash_then_verify_fused(eng):
    n = 3000
    msgs, off = corpus.make_requests(n, seed=5, fixed_len=None, lo=64, hi=2048)
    dig = oracle.sha256_batch(msgs, off)
    d, kxy = corpus.make_keys(P256, 32, seed=41)
    key_idx = (np.arange(n) % 32).astype(np.uint32)
    nonces = corpus._blocks(43, n, 32, b"k")
    r, s = oracle.sign_batch(P256, d, key_idx, dig, nonces)
    qx, qy = np.ascontiguousarray(kxy[key_idx, :32]), np.ascontiguousarray(kxy[key_idx, 32:])
    # corrupt: flip one payload bit in every 5th message, one signature bit in every 7th
    msgs = msgs.copy()
    for i in range(0, n, 5):
        msgs[int(off[i]) + (i % int(off[i + 1] - off[i]))] ^= 1
    for i in range(0, n, 7):
        s[i, 9] ^= 2
    want_dig = oracle.sha256_batch(msgs, off)
    want = oracle.verify_batch(P256, r, s, qx, qy, want_dig)
    got, got_dig = eng.hash_verify_batch(P256, msgs, off, r, s, qx, qy, want_digest=True)
    assert (got_dig == want_dig).all()
    assert (got == want).all()
    assert 0 < want.sum() < n


def test_der_front_end(eng):
    b = corpus.make_batch(P256, n=400, K=8, seed=17, corrupt_rate=5)
    sigs, off = [], [0]
    for i in range(b["n"]):
        rv, sv = int.from_bytes(b["r"][i].tobytes(), "big"), int.from_bytes(b["s"][i].tobytes(), "big")
        sg = ref.der_encode(rv, sv)
        m = i % 10
        if m == 3: sg = sg + b"\x00"
        elif m == 4: sg = sg[:-1]
        elif m == 5: sg = b"\x30\x81" + sg[1:]
        elif m == 6: sg = sg[:2] + b"\x02\x21\x00" + sg[4:] if sg[3] == 0x20 and not sg[4] & 0x80 else sg
        elif m == 7: sg = b""
        sigs.append(sg); off.append(off[-1] + len(sg))
    blob = np.frombuffer(b"".join(sigs) + b"\x00", np.uint8)
    off = np.array(off, np.uint32)
    qxy = np.concatenate([b["qx"], b["qy"]], axis=1)
    want = oracle.verify_batch_der(P256, blob, off, qxy, b["digest"])
    got = eng.verify_batch_der(P256, blob, off, qxy, b["digest"])
    assert (want == got).all(), np.nonzero(want != got)[0][:10]
    assert 0 < want.sum() < want.size


def test_mixed_curve_batch(eng):
    n = 600
    b256 = corpus.make_batch(P256, n=n, K=8, seed=51, corrupt_rate=4)
    b384 = corpus.make_batch(P384, n=n, K=8, seed=53, corrupt_rate=4)
    tag = (np.arange(n) * 7 % 5 % 2).astype(np.uint8)
    def slot(a256, a384):
        out = np.zeros((n, 48), np.uint8)
        out[tag == 0, 16:] = a256[tag == 0]
        out[tag == 1] = a384[tag == 1]
        return out
    r, s, qx, qy = (slot(b256[k], b384[k]) for k in ("r", "s", "qx", "qy"))
    dig = np.where(tag[:, None] == 0, b256["digest"], b384["digest"])
    r[5, 3] = 1  # a P-256 item (tag[5]==0?) with a non-zero pad byte must reject
    want = np.zeros(n, np.uint8)
    w256 = oracle.verify_batch(P256, b256["r"], b256["s"], b256["qx"], b256["qy"], b256["digest"])
    w384 = oracle.verify_batch(P384, b384["r"], b384["s"], b384["qx"], b384["qy"], b384["digest"])
    want[tag == 0] = w256[tag == 0]; want[tag == 1] = w384[tag == 1]
    if tag[5] == 0:
        want[5] = 0
    else:
        r[5, 3] = b384["r"][5, 3]
    got = eng.verify_mixed(tag, r, s, qx, qy, dig)
    assert (want == got).all()


def test_quorum_counting_matches_reference_rules(eng):
    rng = np.random.default_rng(9)
    N, I = 16, 2000
    q, f = ref.compute_quorum(N)
    inst, snd, sig, dm, ok, selfs = [], [], [], [], [], []
    want = []
    for i in range(I):
        self_id = int(rng.integers(0, N))
        k = int(rng.integers(0, 24))
        votes = []
        for _ in range(k):
            a = int(rng.integers(0, N))
            g = a if rng.random() < 0.85 else int(rng.integers(0, N))
            votes.append((a, g, int(rng.random() < 0.9), int(rng.random() < 0.85)))
        want.append(ref.count_commit_votes(votes, self_id=self_id))
        selfs.append(self_id)
        for a, g, m, o in votes:
            inst.append(i); snd.append(a); sig.append(g); dm.append(m); ok.append(o)
    cnt, reached = eng.quorum(inst, snd, sig, dm, ok, I, q - 1, self_id=selfs)
    assert cnt.tolist() == want
    assert reached.tolist() == [int(w >= q - 1) for w in want]
    import consensus_b200 as sbv
    for n in range(1, 40):
        assert sbv.compute_quorum(n) == ref.compute_quorum(n)


def test_multi_device_engine_nccl_gather():
    """sbv_create with 2 devices: shards + ncclAllGather of the packed verdict mask (needs >= 2 GPUs)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import consensus_b200 as sbv
    b = corpus.make_batch(P256, n=5003, K=16, seed=23, corrupt_rate=4)
    want = oracle.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    with sbv.Engine(n_devices=2) as e2:
        got = e2.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    assert (got == want).all()


@pytest.mark.parametrize("curve", [P256, P384])
def test_registered_key_path_bit_exact(eng, curve):
    """sbv_set_keys + sbv_verify_registered (fixed-base comb per key) must give the oracle's verdicts,
    including for an invalid registered key, a slot of the other curve and an unknown slot."""
    L = 32 if curve == P256 else 48
    n, K = 3000, 12
    b = corpus.make_batch(curve, n=n, K=K, seed=61 + curve, corrupt_rate=0)
    keys = b["keys"].reshape(K, 2, L).copy()
    other = corpus.make_keys(1 - curve, 2, seed=5)[1].reshape(2, 2, 32 if curve == P384 else 48)
    slots_xy = np.zeros((K + 3, 2, 48), np.uint8)
    slots_xy[:K, :, 48 - L:] = keys
    slots_xy[K, :, 48 - L:] = keys[0]; slots_xy[K, 1, 47] ^= 1            # slot K: off-curve key
    Lo = other.shape[2]
    slots_xy[K + 1, :, 48 - Lo:] = other[0]                                # slot K+1: key of the other curve
    slots_xy[K + 2, :, 48 - L:] = keys[1]                                  # slot K+2: valid duplicate of key 1
    curves = np.full(K + 3, curve, np.uint8); curves[K + 1] = 1 - curve
    eng.set_keys(curves, slots_xy, verification_seq=7)
    slot = b["key_idx"].astype(np.uint32).copy()
    r, s, dig = b["r"].copy(), b["s"].copy(), b["digest"].copy()
    rng = np.random.default_rng(3)
    qx, qy = b["qx"].copy(), b["qy"].copy()
    for i in range(n):
        m = i % 16
        if m == 1: r[i, rng.integers(L)] ^= 1 << rng.integers(8)
        elif m == 2: s[i, rng.integers(L)] ^= 1 << rng.integers(8)
        elif m == 3: dig[i, rng.integers(32)] ^= 1 << rng.integers(8)
        elif m == 4:                                   # signed by key k, verified against another registered key
            slot[i] = (slot[i] + 1) % K; qx[i] = keys[slot[i], 0]; qy[i] = keys[slot[i], 1]
        elif m == 5: slot[i] = K; qy[i] = slots_xy[K, 1, 48 - L:]      # invalid key
        elif m == 6: slot[i] = K + 1                                      # other-curve slot  -> reject
        elif m == 7: slot[i] = K + 3 + 11                                 # unknown slot      -> reject
        elif m == 8: r[i] = 0
        elif m == 9 and slot[i] == 1: slot[i] = K + 2                     # duplicate registration of the same key
    want = oracle.verify_batch(curve, r, s, qx, qy, dig)
    want[np.isin(np.arange(n) % 16, [6, 7])] = 0
    got = eng.verify_registered(curve, slot, r, s, dig)
    bad = np.nonzero(want != got)[0]
    assert bad.size == 0, (bad[:10], (bad[:10] % 16))
    assert 0 < want.sum() < n
    # agrees with the keys-per-item entry point wherever the slot is a valid key of this curve
    sel = ~np.isin(np.arange(n) % 16, [5, 6, 7])
    generic = eng.verify_batch(curve, r[sel], s[sel], qx[sel], qy[sel], dig[sel])
    assert (generic == got[sel]).all()
    # small batches take the one-signature-per-warp kernel: same verdicts, item by item
    for lo, cnt in [(0, 1), (1, 2), (16, 77), (100, 1000), (33, 2048)]:
        sl = slice(lo, lo + cnt)
        assert (eng.verify_registered(curve, slot[sl], r[sl], s[sl], dig[sl]) == want[sl]).all(), (lo, cnt)
    eng.set_keys(np.zeros(0, np.uint8), np.zeros((0, 96), np.uint8))      # empty registry: everything rejects
    assert eng.verify_registered(curve, slot[:50], r[:50], s[:50], dig[:50]).sum() == 0


def test_concurrent_callers_share_the_engine(eng):
    """Two host threads each keep a synchronous call in flight (per-call lanes); verdicts stay exact."""
    import threading
    bs = [corpus.make_batch(P256, n=6000 + 37 * k, K=8, seed=101 + k, corrupt_rate=3) for k in range(4)]
    wants = [oracle.verify_batch(P256, b["r"], b["s"], b["qx"], b["qy"], b["digest"]) for b in bs]
    errs = []
    def worker(k):
        try:
            for _ in range(6):
                got = eng.verify_batch(P256, bs[k]["r"], bs[k]["s"], bs[k]["qx"], bs[k]["qy"], bs[k]["digest"])
                if not (got == wants[k]).all():
                    errs.append(k)
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ths: t.start()
    for t in ths: t.join()
    assert not errs, errs


def test_hash_verify_registered_fused(eng):
    """SHA-256 on the device feeding the registered-key verify (the call GpuVerifier / the Go shim make)."""
    n, K = 1500, 6
    msgs, off = corpus.make_requests(n, seed=15, fixed_len=None, lo=1, hi=900)
    dig = oracle.sha256_batch(msgs, off)
    d, kxy = corpus.make_keys(P256, K, seed=111)
    key_idx = (np.arange(n) % K).astype(np.uint32)
    r, s = oracle.sign_batch(P256, d, key_idx, dig, corpus._blocks(113, n, 32, b"k"))
    msgs = msgs.copy()
    for i in range(0, n, 6):
        msgs[int(off[i])] ^= 0x80            # tampered message
    for i in range(3, n, 9):
        r[i, 31] ^= 1                        # tampered signature
    slot = key_idx.copy(); slot[5::50] = (slot[5::50] + 1) % K   # wrong signer
    eng.set_keys(np.zeros(K, np.uint8), kxy.reshape(K, 2, 32))
    keys_of = kxy[slot]
    want = oracle.verify_batch(P256, r, s, np.ascontiguousarray(keys_of[:, :32]), np.ascontiguousarray(keys_of[:, 32:]),
                               oracle.sha256_batch(msgs, off))
    got = eng.hash_verify_registered(P256, msgs, off, slot, r, s)
    assert (got == want).all()
    assert 0 < want.sum() < n
    assert (eng.hash_verify_registered(P256, msgs, off[:8], slot[:7], r[:7], s[:7]) == want[:7]).all()   # warp path
