"""GPU arithmetic layer (Montgomery field ops, Jacobian group law) vs Python big integers.
Bit-exact.  Uses the sbv_debug_op test hook of libsbv.so."""
import ctypes as C

import numpy as np
import pytest

import edges
from oracle import ecdsa_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import consensus_b200 as sbv
    e = sbv.Engine(n_devices=1)
    yield e
    e.close()


def _limbs(vals, N):
    out = np.zeros((len(vals), 2 * N), np.uint32)
    for i, pair in enumerate(vals):
        for h, v in enumerate(pair):
            for k in range(N):
                out[i, h * N + k] = (v >> (32 * k)) & 0xFFFFFFFF
    return out


def _ints(arr, N):
    res = []
    for row in arr:
        res.append(tuple(sum(int(row[h * N + k]) << (32 * k) for k in range(N)) for h in range(2)))
    return res


def _run(eng, curve, op, a, b):
    N = 8 if curve == 0 else 12
    A, B = _limbs(a, N), _limbs(b, N)
    out = np.zeros_like(A)
    p32 = lambda x: x.ctypes.data_as(C.POINTER(C.c_uint32))
    rc = eng._lib.sbv_debug_op(eng._h, C.c_uint8(curve), C.c_int(op), C.c_size_t(len(a)), p32(A), p32(B), p32(out))
    assert rc == 0
    return _ints(out, N)


@pytest.mark.parametrize("curve", [0, 1])
def test_field_ops(eng, curve):
    """The CPU simulation's cases (edges.montgomery_cases) on the device, out of line and with the inlined multiplications
    of Inl<C> (k_verify_comb, the P-256 k_verify_kt): edge values, operands that put P256::redc / P384::redc /
    mont_reduce_sos on each side of the final subtraction, operands in [m, R); then the inverses."""
    c = ref.CURVES[curve]
    N = c.size // 4
    R = 1 << (32 * N)
    rng = np.random.default_rng(curve + 1)
    for label, op, xs, ys, want in edges.montgomery_cases(curve, rng, 300):
        a = [(x, 0) for x in xs]; b = [(y, 0) for y in ys]
        for flag in (0, edges.INL):
            assert [g[0] for g in _run(eng, curve, op | flag, a, b)] == want, (label, op | flag)
    # inverses (Montgomery in/out): inv(aR) = a^-1 R
    xs = [v for v in edges.edge_values(c.p, rng, 20) if v]
    got = _run(eng, curve, 4, [(x * R % c.p, 0) for x in xs], [(0, 0)] * len(xs))
    assert [g[0] for g in got] == [pow(x, -1, c.p) * R % c.p for x in xs]
    xs = [v for v in edges.edge_values(c.p, rng, 600) if v] + [pow(2, k, c.p) for k in (1, 31, 32, 33, 64, 96, 128, 224, 255, 256, 300)]
    xs += [a * pow(R, -1, c.p) % c.p for a in edges.longest_inverse_inputs(c.p, N)]   # 32N - 1 passes, the most
    got = _run(eng, curve, 10, [(x * R % c.p, 0) for x in xs], [(0, 0)] * len(xs))   # binary-GCD field inverse (table construction)
    assert [g[0] for g in got] == [pow(x, -1, c.p) * R % c.p for x in xs]
    # scalar-field inverse (binary extended GCD): many random values plus powers of two and their
    # neighbours, which exercise long runs of trailing zeros (tz = 31 passes, zero low words)
    xs = [v for v in edges.edge_values(c.n, rng, 1500) if v]
    xs += [pow(2, k, c.n) for k in (1, 31, 32, 33, 63, 64, 65, 96, 128, 255, 256, 300, 383)]
    xs += [(pow(2, k, c.n) * pow(R, -1, c.n)) % c.n for k in (32, 64, 96, 200)]   # residue itself a power of two
    xs += [(c.n - pow(2, k, c.n)) % c.n for k in (1, 32, 64, 128)]
    xs += [a * pow(R, -1, c.n) % c.n for a in edges.longest_inverse_inputs(c.n, N)]
    xs = [v for v in xs if v]
    got = _run(eng, curve, 8, [(x * R % c.n, 0) for x in xs], [(0, 0)] * len(xs))
    assert [g[0] for g in got] == [pow(x, -1, c.n) * R % c.n for x in xs]


@pytest.mark.parametrize("curve", [0, 1])
def test_group_law(eng, curve):
    """Doubling, mixed add (P == Q: the doubling branch; P == -Q: infinity -> (0, 0)) and general add 2P + Q with
    non-trivial Z on both sides, each with the neg / skip flags of the verification loops and from an accumulator at
    infinity, out of line and inlined."""
    c = ref.CURVES[curve]
    ks = [1, 2, 3, 4, 5, 7, 8, 255, 256, c.n - 1, c.n - 2, 2**100 + 3, 0xDEADBEEF]
    for op, a, b, want in edges.group_cases(curve, ks):
        for flag in (0, edges.INL):
            assert _run(eng, curve, op | flag, a, b) == want, op | flag
