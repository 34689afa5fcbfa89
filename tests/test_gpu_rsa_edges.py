"""RSA verdicts on the H100 for the sets of tests/rsa_edges.py, every item, for every modulus size and hash, bit-exact
against oracle_rsa.ref: keys of bit lengths 8k, 8k - 1, 8k - 4 and 8k - 7, odd exponents of every bit length, accepted
even exponents, and the encoding changed at every position.  Each set goes through sbv_rsa_verify_batch as built and
shifted by one item; the bit-length set also through sbv_rsa_hash_verify_batch."""
import numpy as np
import pytest

import rsa_edges as edges

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    with sbv.Engine(n_devices=1) as e:
        yield e


def _check(eng, c):
    got = eng.rsa_verify_batch(c["hash"], c["digest"], c["sig"], c["mod"], c["exp"])
    bad = [(cl, int(g), int(w)) for cl, g, w in zip(c["cls"], got, c["want"]) if g != w]
    assert not bad, bad


@pytest.mark.parametrize("name", sorted(edges.SETS))
@pytest.mark.parametrize("k", edges.SIZES)
@pytest.mark.parametrize("hash", edges.HASHES)
def test_set_as_built_and_shifted(eng, name, k, hash):
    c = edges.SETS[name](k, hash)
    assert 0 < int(c["want"].sum())
    _check(eng, c)
    _check(eng, edges.shifted(c))


@pytest.mark.parametrize("k", edges.SIZES)
@pytest.mark.parametrize("hash", edges.HASHES)
def test_bit_lengths_through_the_fused_call(eng, k, hash):
    c = edges.bitlen(k, hash)
    for cc in (c, edges.shifted(c)):
        got, dig = eng.rsa_hash_verify_batch(hash, cc["msgs"], cc["off"], cc["sig"], cc["mod"], cc["exp"], want_digest=True)
        assert np.array_equal(dig, cc["digest"])
        assert np.array_equal(got, cc["want"]), list(zip(cc["cls"], got, cc["want"]))
