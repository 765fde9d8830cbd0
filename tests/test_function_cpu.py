"""Table-defined function ops without a GPU: the numpy emulator of tests/function_ref.py pinned to the plain-C
restatement of the reference iterator's row rule (so the bit convention is the reference's after flip_bits), the path
plan (qipb200_function_plan) and its validation, the NULL refusals, the C++ mirror, and the Shor closed form against a
dense simulation."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import function_ref as fr
from oracle import qip_oracle as qo
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import FUNCTION_PAIR, FUNCTION_TILE, function_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7


def random_psi(n, seed, dtype):
    rng = np.random.default_rng(seed)
    psi = ((rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.4).astype(dtype)
    psi[rng.integers(0, 1 << n, size=4)] = complex(-0.0, -0.0)  # signed zeros must move as they are
    return psi


def random_case(n, rng, phase_only=False):
    """Random, unsorted, interleaved registers: n_in >= 1, n_out >= 0 (0 for phase_only)."""
    perm = [int(q) for q in rng.permutation(n)]
    n_in = int(rng.integers(1, n + 1)) if phase_only else int(rng.integers(1, n))
    n_out = 0 if phase_only else int(rng.integers(1, n - n_in + 1))
    return perm[:n_in], perm[n_in:n_in + n_out]


@pytest.mark.parametrize("dtype", [C128, C64])
@pytest.mark.parametrize("n", range(3, 11))
def test_emulator_matches_reference_row_rule(n, dtype):
    rng = np.random.default_rng(100 * n + (dtype == C64))
    for case in range(6):
        in_q, out_q = random_case(n, rng, phase_only=case == 5)
        f = rng.integers(0, 1 << len(out_q), size=1 << len(in_q), dtype=np.uint64) if out_q else None
        theta = rng.uniform(-7, 7, size=1 << len(in_q)) if case % 2 or not out_q else None
        psi = random_psi(n, 7 * n + case, dtype)
        want = fr.apply(psi, n, in_q, out_q, f, theta)
        got = fr.oracle_apply(psi, n, in_q, out_q, f, theta)
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (n, case, in_q, out_q)
    # without theta the op is a pure move and an involution
    in_q, out_q = random_case(n, rng)
    f = rng.integers(0, 1 << len(out_q), size=1 << len(in_q), dtype=np.uint64)
    psi = random_psi(n, n, dtype)
    once = fr.apply(psi, n, in_q, out_q, f)
    assert np.array_equal(fr.apply(once, n, in_q, out_q, f).view(np.uint8), psi.view(np.uint8))


def test_bit_convention_on_basis_states():
    """|x>|0> -> |x>|f(x)> with bit i of x on in_q[i] and bit i of f(x) on out_q[i]."""
    n, in_q, out_q = 6, [4, 0, 2], [5, 1]
    f = np.array([3, 1, 0, 2, 1, 3, 2, 0], dtype=np.uint64)
    for x in range(8):
        j = int(fr.scatter(np.array([x]), n, in_q)[0])
        psi = np.zeros(1 << n, dtype=C128)
        psi[j] = 1
        out = fr.oracle_apply(psi, n, in_q, out_q, f)
        want = j | int(fr.scatter(np.array([f[x]]), n, out_q)[0])
        assert np.flatnonzero(out).tolist() == [want]


# ---- the path plan -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_paths(dtype):
    tmax = 11 if dtype == C128 else 12
    n = 30
    low10 = list(range(20, 30))  # index bits 9..0
    high20 = list(range(0, 20))
    # out bits in the low bits: tile
    assert function_plan(n, dtype, high20, low10) == (FUNCTION_TILE, tmax)
    assert function_plan(n, dtype, high20, [29, 27]) == (FUNCTION_TILE, tmax)
    # out bits on high bits, within T_max: tile
    assert function_plan(n, dtype, [29, 28, 20], list(range(tmax - 4))) == (FUNCTION_TILE, tmax)
    # more out bits above the 4 low bits than a tile holds: pair
    assert function_plan(n, dtype, low10 + high20[10:], high20[:10]) == (FUNCTION_PAIR, 0)
    assert function_plan(n, dtype, [29], list(range(tmax - 3))) == (FUNCTION_PAIR, 0)
    assert function_plan(40, dtype, [0], list(range(1, 33))) == (FUNCTION_PAIR, 0)
    # phase only: tile, whatever the in register
    assert function_plan(n, dtype, list(range(4, n)), []) == (FUNCTION_TILE, tmax)
    assert function_plan(n, dtype, [0], []) == (FUNCTION_TILE, tmax)
    # small states are one tile
    assert function_plan(5, dtype, [0, 1], [2, 3, 4]) == (FUNCTION_TILE, 5)
    assert function_plan(1, dtype, [0], []) == (FUNCTION_TILE, 1)


def _plan_raw(n, in_q, out_q, prec=1, n_in=None, n_out=None, null_in=False, null_out=False):
    ia = (C.c_uint64 * max(1, len(in_q)))(*in_q)
    oa = (C.c_uint64 * max(1, len(out_q)))(*out_q)
    v = (C.c_uint32 * 2)(99, 99)
    st = _lib.lib().qipb200_function_plan(prec, n, None if null_in else ia, len(in_q) if n_in is None else n_in,
                                          None if null_out else oa, len(out_q) if n_out is None else n_out, v)
    return st, _lib.lib().qipb200_last_error(None).decode(), (v[0], v[1])


def test_plan_validation_errors():
    assert _plan_raw(8, [0, 1], [2])[0] == 0
    for prec, n in ((7, 8), (1, 0), (1, 41)):
        st, msg, _ = _plan_raw(n, [0], [], prec=prec)
        assert st == INVALID_ARG and msg.startswith("function_plan:"), msg
    v = (C.c_uint32 * 2)()
    ia = (C.c_uint64 * 1)(0)
    assert _lib.lib().qipb200_function_plan(1, 8, ia, 1, None, 0, None) == INVALID_ARG
    st, msg, _ = _plan_raw(8, [], [1])
    assert st == INVALID_ARG and "n_in must be at least 1" in msg
    st, msg, _ = _plan_raw(40, list(range(27)), [])
    assert st == UNSUPPORTED and "at most 26 input qubits" in msg
    st, msg, _ = _plan_raw(40, [0], list(range(1, 34)))
    assert st == UNSUPPORTED and "at most 32 output qubits" in msg
    st, msg, _ = _plan_raw(8, [0], [1], null_in=True)
    assert st == INVALID_ARG and "NULL qubit array" in msg
    st, msg, _ = _plan_raw(8, [0], [1], null_out=True)
    assert st == INVALID_ARG and "NULL qubit array" in msg
    assert _lib.lib().qipb200_function_plan(1, 8, ia, 1, None, 0, v) == 0  # no out register: NULL is fine
    st, msg, _ = _plan_raw(8, [0, 8], [1])
    assert st == BAD_INDEX and "qubit 8 out of range for 8 qubits" in msg
    st, msg, _ = _plan_raw(8, [0, 3, 0], [1])
    assert st == BAD_INDEX and "qubit 0 repeated" in msg
    st, msg, _ = _plan_raw(8, [0, 3], [1, 3])
    assert st == BAD_INDEX and "qubit 3 repeated" in msg
    with pytest.raises(CircuitError) as e:
        function_plan(8, C128, [0, 1], [1])
    assert e.value.status == BAD_INDEX


def test_null_handles_are_refused():
    L = _lib.lib()
    ia = (C.c_uint64 * 1)(0)
    assert L.qipb200_state_apply_function(None, None, ia, None) == INVALID_ARG
    assert "apply_function: NULL state or function" in L.qipb200_last_error(None).decode()
    out = C.c_void_p()
    f = (C.c_uint64 * 2)(0, 1)
    assert L.qipb200_function_new(None, 1, 1, f, None, C.byref(out)) == INVALID_ARG
    assert "function_new: NULL context" in L.qipb200_last_error(None).decode()
    L.qipb200_function_free(None)  # a no-op


def test_cpp_mirror_apply_function_compiles(tmp_path):
    src = tmp_path / "use_function.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::Context &ctx, qip::B200State<double> &a, qip::B200State<float> &b) {\n"
                   "  qip::B200Function f(ctx, 2, 1, {0, 1, 1, 0});\n"
                   "  qip::B200Function g(ctx, 2, 0, {}, {0.1, 0.2, 0.3, 0.4});\n"
                   "  a.apply_function(f, {0, 1}, {2});\n"
                   "  b.apply_function(g, {2, 0});\n"
                   "  const qipb200_function *h = f.get();\n"
                   "  (void)h;\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr


# ---- Shor's period finding: the closed form the GPU test uses ------------------------------------------------------

def test_shor_closed_form_against_dense_simulation():
    """n = 12: x on qubits 0..7 (m = 8, qubit 0 the most significant bit of x, so in_qubits = [7, ..., 0]), y on qubits
    8..11, N = 15, a = 7 (r = 4).  H on x, |x>|0> -> |x>|7^x mod 15>, the MatrixOp QFT on qubits 0..7, then the
    probabilities of x read with the same bit order."""
    n, m, N, a = 12, 8, 15, 7
    r = fr.order(a, N)
    assert r == 4
    in_q, out_q = list(range(m - 1, -1, -1)), list(range(n - 1, m - 1, -1))
    psi = np.zeros(1 << n, dtype=C128)
    psi[0] = 1
    psi = qo.run_pipeline(n, [gates.h(q) for q in range(m)], state=psi, dtype=C128)
    psi = fr.apply(psi, n, in_q, out_q, fr.modexp_table(a, N, m))
    psi = qo.run_pipeline(n, circuits.qft(m), state=psi, dtype=C128)
    probs = np.zeros(1 << m)
    np.add.at(probs, fr.register_value(np.arange(1 << n, dtype=np.uint64), n, in_q).astype(np.int64),
              np.abs(psi) ** 2)
    want = fr.shor_probs(m, r)
    assert np.max(np.abs(probs - want)) <= 1e-12
    assert np.flatnonzero(want > 1e-12).tolist() == [0, 64, 128, 192]
    # a period that does not divide 2^m: N = 21, a = 2 (r = 6)
    N, a = 21, 2
    r = fr.order(a, N)
    assert r == 6
    psi = np.zeros(1 << n, dtype=C128)
    psi[0] = 1
    psi = qo.run_pipeline(n, [gates.h(q) for q in range(m)], state=psi, dtype=C128)
    psi = fr.apply(psi, n, in_q, out_q, fr.modexp_table(a, N, m) & np.uint64(15))  # a 4-bit register keeps a^x mod 16
    psi = qo.run_pipeline(n, circuits.qft(m), state=psi, dtype=C128)
    probs = np.zeros(1 << m)
    np.add.at(probs, fr.register_value(np.arange(1 << n, dtype=np.uint64), n, in_q).astype(np.int64),
              np.abs(psi) ** 2)
    assert abs(probs.sum() - 1) <= 1e-12
    # continued fractions on the peaks of the N = 15 case recover r
    assert fr.period_from_shot(64, m, 7, 15) == 4 and fr.period_from_shot(192, m, 7, 15) == 4
