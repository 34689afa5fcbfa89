"""The Ed25519 field, scalar and point arithmetic at its carry boundaries in the CPU simulation (tools/hostsim: ed25519.cuh
compiled with g++), bit for bit against the limb models of tests/ed25519_arith.py and against Python integers.  The
`-m gpu` file test_gpu_ed25519_arith.py runs the same sets on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ed25519_arith as arith
import ed25519_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS_DIR = os.path.join(ROOT, "tools", "hostsim")


@pytest.fixture(scope="module")
def hs():
    subprocess.check_call(["make", "-s", "-C", HS_DIR, "libhostsim.so"])
    return C.CDLL(os.path.join(HS_DIR, "libhostsim.so"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _runner(fn):
    def run(op, inp):
        inp = np.ascontiguousarray(inp, np.uint32)
        out = np.zeros_like(inp)
        assert fn(C.c_int(op), C.c_size_t(inp.shape[0]), _p(inp), _p(out)) == 0
        return out
    return run


@pytest.fixture(scope="module")
def field(hs):
    return _runner(hs.hs_ed25519_op)


@pytest.fixture(scope="module")
def point(hs):
    return _runner(hs.hs_ed25519_point)


def test_barrett_quotient_error_is_at_most_one():
    """Exactly (Fraction): x / L - q3 < B < 2 for every x < 2^512, so q - q3 <= 1, t < B L < 2L, and sc_reduce512's
    second conditional subtraction never runs."""
    B = arith.barrett_bound()
    assert 1 < B < 2
    assert arith.Fraction(12249, 10000) < B < arith.Fraction(12250, 10000)
    print(f"\nBarrett: x/L - q3 < {float(B):.6f} for every x < 2^512")


def test_fold_second_carry_every_c1(field):
    counts = arith.check_fold(field)
    for op, name in ((cases.MUL, "mul"), (cases.SQR, "sqr")):
        c = counts[op]
        print(f"\n{name} fold (c1, second carry): operands per branch "
              + " ".join(f"{k[0]}/{k[1]}:{c[k]}" for k in sorted(c)))


def test_add_sub_carry_and_wrap(field):
    counts = arith.check_addsub(field)
    for op, name in ((cases.ADD, "add"), (cases.SUB, "sub")):
        c = counts[op]
        print(f"\n{name}: none {c[(0, 0)]}, carry {c[(1, 0)]}, carry and wrap {c[(1, 1)]}")


def test_canon_every_case_at_both_ends(field):
    c = arith.check_canon(field)
    print(f"\ncanon (bit 255, t >= p): {dict(sorted(c.items()))}")


def test_inverse_of_non_canonical_values(field):
    arith.check_inv(field)


def test_reduce_mod_L_quotient_error_zero_and_one(field):
    c, tmax = arith.check_reduce(field)
    print(f"\nreduce: quotient error 0: {c[0]}, error 1: {c[1]}; largest t = {float(tmax):.6f} L")


def test_sqrt_ratio_edges(field):
    print(f"\nsqrt_ratio: {dict(arith.check_sqrt(field))}")


def test_point_double(point):
    assert arith.check_double(point) > 100


def test_point_add_every_form(point):
    assert arith.check_add(point) > 1000


def test_point_cached(point):
    arith.check_cached(point)


def test_point_encode(point):
    print(f"\nencode: {dict(arith.check_encode(point))}")


def test_point_op_refused(hs):
    inp = np.zeros((1, arith.PT_WORDS), np.uint32)
    out = np.zeros_like(inp)
    for op in (4, 255, arith.PT_ENCODE | arith.PT_NEG, arith.PT_DOUBLE | arith.PT_AFFINE, arith.PT_CACHED | arith.PT_NO_T,
               arith.PT_ADD | 0x800, -1):
        assert hs.hs_ed25519_point(C.c_int(op), C.c_size_t(1), _p(inp), _p(out)) == -1, op
