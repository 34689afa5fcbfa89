"""The Ed25519 field, scalar and point arithmetic at its carry boundaries on the H100: the sets of tests/ed25519_arith.py
through sbv_debug_ed25519 (field and mod-L ops) and sbv_debug_ed25519_point (double, add, cached form, encode), bit for
bit against the limb models and against Python integers, as test_hostsim_ed25519_arith.py checks them on the CPU."""
import ctypes as C

import numpy as np
import pytest

import ed25519_arith as arith
import ed25519_cases as cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(devices=[0])
    yield e
    e.close()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _runner(eng, fn):
    def run(op, inp):
        inp = np.ascontiguousarray(inp, np.uint32)
        out = np.zeros_like(inp)
        assert fn(eng._h, C.c_int(op), C.c_size_t(inp.shape[0]), _p(inp), _p(out)) == 0
        return out
    return run


@pytest.fixture(scope="module")
def field(eng):
    return _runner(eng, eng._lib.sbv_debug_ed25519)


@pytest.fixture(scope="module")
def point(eng):
    return _runner(eng, eng._lib.sbv_debug_ed25519_point)


def test_fold_second_carry_every_c1(field):
    arith.check_fold(field)


def test_add_sub_carry_and_wrap(field):
    arith.check_addsub(field)


def test_canon_every_case_at_both_ends(field):
    arith.check_canon(field)


def test_inverse_of_non_canonical_values(field):
    arith.check_inv(field)


def test_reduce_mod_L_quotient_error_zero_and_one(field):
    arith.check_reduce(field)


def test_sqrt_ratio_edges(field):
    arith.check_sqrt(field)


def test_point_double(point):
    assert arith.check_double(point) > 100


def test_point_add_every_form(point):
    assert arith.check_add(point) > 1000


def test_point_cached(point):
    arith.check_cached(point)


def test_point_encode(point):
    arith.check_encode(point)


def test_point_op_refused(eng):
    inp = np.zeros((1, arith.PT_WORDS), np.uint32)
    out = np.full_like(inp, 7)
    lib, h = eng._lib, eng._h
    for op in (4, 255, arith.PT_ENCODE | arith.PT_NEG, arith.PT_DOUBLE | arith.PT_AFFINE, arith.PT_CACHED | arith.PT_NO_T,
               arith.PT_ADD | 0x800, -1):
        assert lib.sbv_debug_ed25519_point(h, C.c_int(op), C.c_size_t(1), _p(inp), _p(out)) != 0, op
    assert lib.sbv_debug_ed25519_point(h, C.c_int(arith.PT_DOUBLE), C.c_size_t(1), None, _p(out)) != 0
    assert lib.sbv_debug_ed25519_point(h, C.c_int(arith.PT_DOUBLE), C.c_size_t(1), _p(inp), None) != 0
    assert (out == 7).all()
    assert lib.sbv_debug_ed25519_point(h, C.c_int(arith.PT_DOUBLE), C.c_size_t(0), _p(inp), _p(out)) == 0
    assert (out == 7).all()
