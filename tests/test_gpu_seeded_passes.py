"""The first addition of each fixed-base pass is a load (pt_seed) on the device: k_gpart seeds from u1's comb digit 0 of
G, k_verify_comb from the mask of its step 0, the registered-key k_verify_kt from u2's Booth digit 0.  Verdicts against
the oracle on scalars that make those digits and masks 0, negative or equal to the other pass's first entry, on every
path; and the grouped path's verdicts against the generic kernel's on the benchmark's batch."""
import numpy as np
import pytest

import oracle
import seeded_cases
from oracle import P256, P384, corpus
from test_gpu_edges import _every_path, engines  # noqa: F401  (engines: generic, threshold 1 and threshold 2)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("curve,seed", [(P256, 5), (P256, 6), (P384, 7)])
def test_seeded_passes_on_every_path(engines, curve, seed):
    """The signatures accept and their copies with r + 1 reject: generic kernel, a table for every key (threshold 1 and
    2), registered keys on the warp and the thread kernel."""
    b = seeded_cases.seeded_batch(curve, seed)
    m = b["r"].shape[0] // 2
    _every_path(engines, curve, b, want=np.repeat(np.array([1, 0], np.uint8), m), thresholds=("grouped", "grouped2"))


def test_bench_batch_grouped_equals_generic():
    """65,536 signatures over 1,024 keys, 1/16 corrupted (bench.py's batch): the default engine (every key grouped:
    k_gpart and k_verify_comb) gives the generic kernel's verdicts and the oracle's."""
    from test_gpu_round2 import _engine
    b = corpus.make_batch(P256, n=65536, K=1024, seed=1)
    args = (b["r"], b["s"], b["qx"], b["qy"], b["digest"])
    want = oracle.verify_batch(P256, *args)
    assert 0 < int(want.sum()) < want.size
    grouped, generic = _engine(), _engine(SBV_GROUP_THRESHOLD=0)
    try:
        assert np.array_equal(grouped.verify_batch(P256, *args), want)
        assert np.array_equal(generic.verify_batch(P256, *args), want)
    finally:
        grouped.close()
        generic.close()
