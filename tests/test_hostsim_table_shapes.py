"""The per-key table builds at the key counts where their grids turn over, on the CPU simulation of the device code
(tools/hostsim), every entry against the models of tests/table_shapes.py:

  - Ed25519 comb tables of keys grouped in a launch (k_edc_bases, k_edc_fill, k_edc_inv, k_edc_final) around their
    64-thread blocks, each key once or twice, so that the launch capacity is the key count or twice it;
  - registered ECDSA tables (the 8-bit window build of sbv_set_keys, k_kt_bases4 included) around its 32-key and
    64-thread blocks, for both curves;
  - registered Ed25519 tables built in chunks (k_ed_ktab_build) with undecodable slots at and next to the chunk
    boundaries, and a last chunk shorter than the others.

tests/test_gpu_table_shapes.py runs the same shapes, and larger ones, on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ecdsa_keys as ek
import table_shapes as ts
from oracle import ecdsa_ref as eref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")
W8 = 1  # hs_tables / hs_ktab_words: 8-bit windows


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    lib = C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))
    lib.hs_ktab_words.restype = C.c_size_t
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------- Ed25519 comb tables of keys grouped in a launch
@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("K", [1, 31, 33, 63, 64, 65, 129])
def test_every_entry_of_grouped_ed25519_comb_tables(hs, K, R):
    """K keys, R items each, at threshold 1 (R * K table slots): every item's table equals its key's model; the last key
    does not decode and reports status 2."""
    keys, pub = ts.comb_launch(K, R)
    n = K * R
    items = np.arange(n, dtype=np.uint32)
    status = np.full(n, -1, np.int32)
    out = np.zeros((n, 510, 24), np.uint32)
    assert hs.hs_ed25519_comb_tab(C.c_size_t(n), _p(pub), C.c_uint32(1), C.c_uint32(8192), C.c_size_t(n), _p(items), _p(status), _p(out)) == 0
    ts.check_comb_tables(keys, [keys[i % K] for i in range(n)], status, out)


# ---------------------------------------------------------------- registered ECDSA tables
@pytest.mark.parametrize("K", [31, 33, 65])
@pytest.mark.parametrize("curve", [ts.P256, ts.P384])
def test_every_entry_of_registered_ecdsa_tables(hs, curve, K):
    """The 8-bit window tables of K keys built in one launch, as sbv_set_keys builds the keys of a curve (the four-lane
    doubling chain of k_kt_bases4): every entry of every key equals the model; an off-curve last key gets no table."""
    L = eref.CURVES[curve].size
    pool = ts.ecdsa_pool(curve, K)
    qx = np.stack([ek._be(Q[0], L) for _, Q in pool])
    qy = np.stack([ek._be(Q[1], L) for _, Q in pool])
    qy[K - 1, L - 1] ^= 1                                                   # off the curve
    words = hs.hs_ktab_words(C.c_int(curve), C.c_int(W8), C.c_size_t(K))
    kt, fl = np.zeros(words, np.uint32), np.zeros(K, np.uint8)
    assert hs.hs_tables(C.c_int(curve), C.c_int(W8), C.c_size_t(K), _p(qx), _p(qy), C.c_int(1), _p(kt), _p(fl)) == 0
    assert fl.tolist() == [1] * (K - 1) + [0]
    per = words // K
    for k in range(K - 1):
        want = ts.window_model(curve, pool[k][1])
        bad = np.nonzero(kt[k * per:(k + 1) * per] != want)[0]
        assert bad.size == 0, f"K={K}, key {k}: {bad.size} words differ, first {bad[:8].tolist()}"


# ---------------------------------------------------------------- registered Ed25519 tables built in chunks
# (keys, undecodable slots before these local indices, keys per k_ed_ktab_build launch): chunks of 3 with an
# undecodable slot right before the first key of the second chunk and of the last (shorter) one; two in a row inside a
# chunk; a last chunk of one key; one key per launch; one launch for all
CHUNKS = [(8, (0, 3, 3, 5, 6), 3), (8, (2, 4), 7), (8, (3, 7), 1), (8, (1, 6), 0)]


@pytest.mark.parametrize("n_good,bad_at,chunk", CHUNKS)
def test_every_entry_of_registered_ed25519_tables_in_chunks(hs, n_good, bad_at, chunk):
    """Every entry of every decodable slot's table equals its key's model, wherever the chunk boundaries and the
    undecodable slots fall; undecodable slots and the slot past the registry have no table."""
    pub, slot_of, _ = ts.ed_chunk_order(n_good, bad_at)
    assert hs.hs_ed25519_set_keys(C.c_size_t(pub.shape[0]), _p(pub), C.c_uint32(chunk)) == 0
    keys = ts.ed_pool(n_good)[1]
    out = np.zeros((32, 128, 24), np.uint32)
    for slot in range(pub.shape[0] + 1):
        rc = hs.hs_ed25519_ktab(C.c_uint32(slot), _p(out))
        if slot not in slot_of:
            assert rc != 0, slot
            continue
        assert rc == 0
        local = slot_of.index(slot)
        bad = np.nonzero((out != ts.ktab_model(keys[local])).any(axis=2))
        assert bad[0].size == 0, f"chunk {chunk}, slot {slot} (local {local}): {bad[0].size} entries differ, first (win, j - 1) " \
                                 f"{list(zip(bad[0][:4].tolist(), bad[1][:4].tolist()))}"
