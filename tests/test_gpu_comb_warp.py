"""The per-launch P-256 comb tables as the device builds them (a warp per key: k_comb_fill_warp, k_comb_final) at key
counts around the two keys of a block and the warp (1, 31, 33) and at the benchmark's 1,024: every entry of every key's
table equals the Python-integer model, the same model the one-thread-per-chain kernels were checked against."""
import numpy as np
import pytest

import ecdsa_keys as ek
from oracle import P256, corpus
from test_gpu_key_tables import _assert_table, _grouped_tables
from test_gpu_round2 import _engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _engine(SBV_GROUP_THRESHOLD=1)
    yield e
    e.close()


@pytest.mark.parametrize("nkeys", [1, 31, 33, 1024])
def test_every_entry_of_every_key(eng, nkeys):
    _, kxy = corpus.make_keys(P256, nkeys, seed=900 + nkeys)
    status, out = _grouped_tables(eng, P256, kxy[:, :32], kxy[:, 32:], np.arange(nkeys, dtype=np.uint32))
    assert status.tolist() == [0] * nkeys
    for k in range(nkeys):
        Q = (int.from_bytes(kxy[k, :32].tobytes(), "big"), int.from_bytes(kxy[k, 32:].tobytes(), "big"))
        _assert_table(out[k], ek.comb_table(Q), f"{nkeys} keys, key {k}")
