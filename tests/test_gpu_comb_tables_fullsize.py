"""The per-launch P-256 comb tables at the benchmark's full size: the 1,024 keys of bench.py's corpus (seed 1), 65,536
items at the default grouping threshold, built by the grouped path on the device.  A table is a pure function of its key,
so the build kernels (two lanes per key for the doubling chain, one thread per chain for the fill and the conversion) must
reproduce the Python-integer model word for word, whatever the launch shape."""
import numpy as np
import pytest

import ecdsa_keys as ek
from oracle import P256, corpus
from oracle import ecdsa_ref as ref
from test_gpu_key_tables import _assert_table, _grouped_tables
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu

RM = 1 << 256


def test_every_key_of_the_benchmark_corpus():
    """Every one of the 1,024 keys gets a table (keyflags set), slot 1 of every table is the key itself (affine
    Montgomery form), and every entry of 32 sampled keys' tables equals the model."""
    b = corpus.make_batch(P256, n=65536, K=1024, seed=1)
    kxy = b["keys"]
    item_key = {bytes(b["qx"][i]) + bytes(b["qy"][i]): i for i in range(b["qx"].shape[0] - 1, -1, -1)}  # first item of each key
    items = np.array([item_key[bytes(kxy[k])] for k in range(1024)], np.uint32)
    eng = _engine(SBV_GROUP_THRESHOLD=16)
    try:
        status, out = _grouped_tables(eng, P256, b["qx"], b["qy"], items)
    finally:
        eng.close()
    assert status.tolist() == [0] * 1024
    p = ref.CURVES[P256].p
    for k in range(1024):
        Q = (int.from_bytes(kxy[k, :32].tobytes(), "big"), int.from_bytes(kxy[k, 32:].tobytes(), "big"))
        assert np.array_equal(out[k, 16:32], ek.limbs((Q[0] * RM % p, Q[1] * RM % p), 32)), f"key {k}: slot 1 is not Q"
    for k in np.sort(np.random.default_rng(5).choice(1024, 32, replace=False)):
        Q = (int.from_bytes(kxy[k, :32].tobytes(), "big"), int.from_bytes(kxy[k, 32:].tobytes(), "big"))
        _assert_table(out[k], ek.comb_table(Q), f"key {k}")
