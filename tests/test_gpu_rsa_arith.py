"""The RSA arithmetic of rsa.cuh on the H100: the sets of tests/rsa_arith.py through sbv_debug_rsa (k_rsa_debug of
rsa_debug.cuh, the production primitives in the production layout), bit for bit against Python integers, on every
modulus shape, as test_hostsim_rsa.py checks a subset of them on the CPU.  Every set runs twice: as built, and shifted by
one dummy item, so that each case also lands in the other half of its warp."""
import ctypes as C

import pytest

import rsa_arith as arith

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _call(eng):
    return lambda mb, op, n, *bufs: eng._lib.sbv_debug_rsa(eng._h, C.c_uint32(mb), C.c_int(op), C.c_size_t(n), *map(_p, bufs))


@pytest.fixture(scope="module", params=[0, 1], ids=["as_built", "shifted"])
def run(eng, request):
    return arith.runner(_call(eng), shift=request.param)


@pytest.mark.parametrize("k", arith.SIZES)
def test_montgomery_products_every_outcome(run, k):
    assert arith.check_products(run, k) > 400


@pytest.mark.parametrize("k", arith.SIZES)
def test_r2_and_ninv_every_doubling_count(run, k):
    arith.check_r2_ninv(run, k)


@pytest.mark.parametrize("k", arith.SIZES)
def test_subtraction_borrow_every_lane(run, k):
    arith.check_sub(run, k)


@pytest.mark.parametrize("k", arith.SIZES)
def test_carry_resolution_every_lane(run, k):
    arith.check_resolve(run, k)


@pytest.mark.parametrize("k", arith.SIZES)
def test_pow_every_exponent_and_modulus(run, k):
    assert arith.check_pow(run, k) > 10000


def test_hook_refuses_bad_calls(eng):
    arith.check_refused(_call(eng))
