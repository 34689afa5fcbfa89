"""Ed25519 keys grouped inside a keys-per-item launch, on the CPU simulation of the device code (tools/hostsim): the comb
tables k_edc_* build, k_ed_verify_comb with crafted k, and the whole grouped pipeline against OpenSSL and the ungrouped
one.  tests/test_gpu_ed25519_grouped.py runs the same sets on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ed25519_edges as edges
import ed25519_grouped as grp
import oracle_ed25519 as oe
from oracle_ed25519 import corpus, ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def comb_tab(hs, pub, items, T=1, max_keys=8192):
    pub = np.ascontiguousarray(pub, np.uint8)
    items = np.ascontiguousarray(items, np.uint32)
    status = np.full(items.size, -1, np.int32)
    out = np.zeros((items.size, 510, 24), np.uint32)
    assert hs.hs_ed25519_comb_tab(C.c_size_t(pub.size // 32), _p(pub), C.c_uint32(T), C.c_uint32(max_keys), C.c_size_t(items.size), _p(items),
                                  _p(status), _p(out)) == 0
    return status, out


def verify_comb_k(hs):
    def run(a):
        n = a["sig"].shape[0]
        ok = np.full(n, 7, np.uint8)
        assert hs.hs_ed25519_verify_comb_k(C.c_size_t(n), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) == 0
        return ok
    return run


def verify_grouped(hs, c, T, max_keys=8192):
    n = c["off"].size - 1
    ok = np.full(n, 7, np.uint8)
    stats = np.zeros(3, np.uint32)
    assert hs.hs_ed25519_verify_grouped(C.c_size_t(n), _p(c["msgs"]), _p(c["off"]), _p(c["sig"]), _p(c["pub"]), C.c_uint32(T),
                                        C.c_uint32(max_keys), _p(ok), _p(stats)) == 0
    return ok, stats


def test_every_entry_of_every_kind_of_key(hs):
    """Random keys, B, the three identity encodings, small-order, mixed-order and y >= p keys against the model; an
    off-curve key gets a slot but no table."""
    keys = grp.table_keys()
    status, out = comb_tab(hs, np.frombuffer(b"".join(keys), np.uint8), np.arange(len(keys)))
    for i, A in enumerate(keys):
        want = grp.comb_words(A)
        if want is None:
            assert status[i] == 2, i
        else:
            assert status[i] == 0 and np.array_equal(out[i], want), (i, A.hex())


def test_a_table_exactly_at_the_threshold(hs):
    """At T = 4 a key with 4 items gets a table, one with 3 does not; with 2 table slots the third key over T has none."""
    keys = grp.table_keys()[:4]
    pub = np.frombuffer(b"".join([keys[0]] * 4 + [keys[1]] * 3 + [keys[2]] * 5 + [keys[3]] * 6), np.uint8)
    status, out = comb_tab(hs, pub, [0, 4, 7, 12], T=4)
    assert list(status) == [0, 1, 0, 0]
    assert np.array_equal(out[0], grp.comb_words(keys[0])) and np.array_equal(out[3], grp.comb_words(keys[3]))
    status, _ = comb_tab(hs, pub, [0, 4, 7, 12], T=4, max_keys=2)
    assert (status == 0).sum() == 2 and status[1] == 1
    status, _ = comb_tab(hs, pub, [0, 7], T=0)
    assert list(status) == [1, 1]


def test_comb_kernel_crafted_k(hs):
    """k = 0, 1, L - 1, 2^252, masks 0x00 / 0xFF in either block and single bits at every comb position."""
    acc, n = edges.check(grp.comb_rows(), verify_k=verify_comb_k(hs), ref_n=40, seed=7)
    assert 0 < acc < n


def test_comb_kernel_crafted_k_of_the_window_kernels(hs):
    acc, n = edges.check(edges.crafted_k(), verify_k=verify_comb_k(hs), ref_n=40, seed=8)
    assert 0 < acc < n


def test_comb_kernel_rejects_k_at_least_L(hs):
    a = edges._subset(grp.comb_rows(), range(4)).arrays()
    a["k"][1] = np.frombuffer(ref.L.to_bytes(32, "little"), "<u4")
    ok = np.zeros(4, np.uint8)
    assert hs.hs_ed25519_verify_comb_k(C.c_size_t(4), _p(a["sig"]), _p(a["pub"]), _p(a["k"]), _p(ok)) != 0


@pytest.mark.parametrize("T", [1, 2, 16])
def test_grouped_pipeline_equals_openssl_and_ungrouped(hs, T):
    """Every corpus class and the repeated edge keys: the verdicts at threshold T equal OpenSSL's and T = 0's, and the
    two work lists cover the batch."""
    c = grp.mixed_corpus(2500, seed=70 + T, n_keys=40)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    got, stats = verify_grouped(hs, c, T)
    base, stats0 = verify_grouped(hs, c, 0)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
    assert np.array_equal(base, want) and stats0[1] == 0
    n = want.size
    assert stats[1] + stats[2] == n and stats[1] > n // 2 and stats[0] > 0
    assert 0 < want.sum() < n
    for cls in (corpus.CLASS_NAMES.index("small_order_a"), corpus.CLASS_NAMES.index("a_y_ge_p")):
        assert (c["cls"] == cls).any()


def test_overflow_keys_go_generic(hs):
    c = grp.mixed_corpus(1200, seed=81, n_keys=24)
    want = oe.verify_batch(c["msgs"], c["off"], c["sig"], c["pub"])
    got, stats = verify_grouped(hs, c, 2, max_keys=3)
    assert np.array_equal(got, want)
    assert 0 < stats[1] < want.size // 4 and stats[0] > 3
