"""exp(-iHt) by a Chebyshev series without a GPU: the plan's coefficients against scipy.special.jv, its degree against an
independent tail from scipy, the long-double series reference of tests/evolve_ref.py against scipy.linalg.expm of
Kronecker products, the emulator within its documented bound, the plan counts, every validation error, the NULL-state
refusal and the C++ mirror."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg

import evolve_ref as er
import pauli_rot_ref as rr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import _marshal_paulis, _ptr, pauli_evolution_plan, pauli_sum_plan
from test_gradient_cpu import dense_h, random_terms
from test_pauli_rotation_cpu import random_psi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7


@pytest.mark.parametrize("bt", [0.1, 1.0, 37.5, 200.0, 5000.0])
@pytest.mark.parametrize("sign", [1, -1])
def test_coefficients_match_scipy(bt, sign):
    terms = [[("X", 0), ("Z", 1)], [], [("Y", 2)], []]
    coeffs = np.array([0.75 * bt, 0.4, -0.25 * bt, -1.1])
    t = float(sign)
    K, s, k, tail, c = pauli_evolution_plan(3, C128, terms, coeffs, t, 1e-12)
    a, b, _, _ = er.split(terms, coeffs)
    assert b == bt and k == K * s and c.shape == (K + 1,)
    want = er.series_coeffs(a, b, t, K)
    # scipy.special.jv itself errs by up to ~6e-14 at x = 5000 (against mpmath), 1.2e-13 in C_k = 2 J_k; the library's
    # J_k are checked against mpmath there instead
    assert np.max(np.abs(c - want)) <= (1e-14 if bt <= 200 else 2.5e-13)
    if bt == 5000.0:
        mp = pytest.importorskip("mpmath")
        mp.mp.dps = 30
        for j in (0, 1, 102, 681, 2500, 4999, K - 3):
            jv = float(mp.besselj(j, sign * bt, maxprec=20000))
            got = (c[j] * np.exp(1j * (a * t)) * 1j ** j).real / (1 if j == 0 else 2)
            assert abs(got - jv) <= 1e-15, (j, got, jv)


@pytest.mark.parametrize("x", [0.3, 2.0, 11.0, 64.0, 200.0])
@pytest.mark.parametrize("tol", [1e-4, 1e-9, 1e-12, 1e-15])
def test_degree_is_the_smallest_with_tail_below_tol(x, tol):
    K, _, _, tail, _ = pauli_evolution_plan(2, C128, [[("Z", 0)], [("X", 1)]], [x / 2, -x / 2], 1.0, tol)
    want, tau = er.degree_policy(x, tol)
    if K != want:  # an off-by-one only where tau sits at tol
        assert abs(K - want) == 1 and abs(tau[min(K, want)] - tol) <= 1e-9 * tol, (K, want)
    assert abs(tail - tau[K]) <= 1e-6 * tau[K] + 1e-17 and tail <= tol


def hamiltonians(n, rng):
    """The families of tests/test_gpu_gradient.py plus identity-only and single-term H."""
    out = {"ising": rr.ising_step(n)}
    if n >= 4 and n % 2 == 0:
        out["qaoa"] = rr.qaoa_layer(n)[: n + n // 2]
    rand = random_terms(n, 2 * n + 3, rng)
    out["random"] = rand + rand[:2] + [[]]
    out["identity"] = [[], []]
    out["single"] = [[("Y", n - 1)]]
    return {k: (v, rng.normal(size=len(v))) for k, v in out.items()}


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_reference_matches_expm_and_emulator_within_bound(n):
    rng = np.random.default_rng(60 + n)
    psi = random_psi(n, 5 * n)
    norm = float(np.linalg.norm(psi))
    for name, (terms, coeffs) in sorted(hamiltonians(n, rng).items()):
        H = dense_h(n, terms, coeffs)
        for t in (0.45, -3.0, 17.0 / max(1.0, float(np.sum(np.abs(coeffs))) / 4)):
            want = scipy.linalg.expm(-1j * t * H) @ psi
            for dtype, tol in ((C128, 1e-12), (C64, 1e-6)):
                K, s, k, tail, c = pauli_evolution_plan(n, dtype, terms, coeffs, t, tol)
                ref = er.cheb_ref(psi, n, terms, coeffs, t, c)
                err = float(np.linalg.norm((ref - want).astype(C128)))
                assert err <= tail * norm + er.exact_allowance(terms, coeffs, t, c, norm) + 1e-15, (name, t, err, tail)
                got = er.emulate(psi, n, terms, coeffs, t, tol, dtype)
                e2 = float(np.linalg.norm((got.astype(np.clongdouble) - ref).astype(C128)))
                assert e2 <= er.bound(n, terms, coeffs, c, dtype, norm), (name, t, np.dtype(dtype).name, e2)


def test_plan_counts_and_special_cases():
    for dtype in (C128, C64):
        tfim = rr.ising_step(30)
        K, s, k, tail, c = pauli_evolution_plan(30, dtype, tfim + [[]], np.ones(61), 1.0, None)
        assert s == pauli_sum_plan(30, dtype, tfim) == 4 and k == K * s and K >= 2
        qaoa = rr.qaoa_layer(30)[:45]
        K, s, k, _, _ = pauli_evolution_plan(30, dtype, qaoa, np.ones(45), 1.0, None)
        assert s == pauli_sum_plan(30, dtype, qaoa) == 1 and k == K
        rand = random_terms(12, 40, np.random.default_rng(3))
        coeffs = np.linspace(-1, 1, 40)
        nonid = [t for t in rand if t]
        K, s, k, _, _ = pauli_evolution_plan(12, dtype, rand, coeffs, 0.8, None)
        assert s == pauli_sum_plan(12, dtype, nonid) and k == K * s
        # t = 0, no terms: a no-op; identity only: one kernel, the phase
        assert pauli_evolution_plan(30, dtype, tfim, np.ones(60), 0.0, None)[:4] == (0, 0, 0, 0.0)
        assert pauli_evolution_plan(30, dtype, [], [], 2.0, None)[:4] == (0, 0, 0, 0.0)
        K, s, k, tail, c = pauli_evolution_plan(30, dtype, [[], []], [0.25, 0.5], 2.0, None)
        assert (K, s, k, tail) == (0, 0, 1, 0.0) and c[0] == complex(np.cos(1.5), -np.sin(1.5))
        K, s, k, tail, c = pauli_evolution_plan(30, dtype, [[("Z", 3)], []], [0.0, 0.5], 2.0, None)
        assert (K, k) == (0, 1)  # zero coefficients only: b == 0


def _plan_raw(n, terms, coeffs, t, tol, prec=1, out3=True, tail=True):
    qs, ls, lens = _marshal_paulis(terms)
    c = np.ascontiguousarray(np.asarray(coeffs, dtype=np.float64))
    v, tl = (C.c_uint32 * 3)(), C.c_double()
    st = _lib.lib().qipb200_pauli_evolution_plan(prec, n, _ptr(qs), ls, _ptr(lens), len(terms),
                                                 _ptr(c) if c.size else None, t, tol, v if out3 else None,
                                                 C.byref(tl) if tail else None, None, 0)
    return st, _lib.lib().qipb200_last_error(None).decode()


def test_plan_validation_errors():
    x = [[("X", 0)]]
    st, msg = _plan_raw(4, [[("W", 0)]], [1.0], 1.0, 1e-9)
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg
    st, msg = _plan_raw(4, [[("X", 4)]], [1.0], 1.0, 1e-9)
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg = _plan_raw(4, [[("X", 1), ("Z", 1)]], [1.0], 1.0, 1e-9)
    assert st == BAD_INDEX and "qubit 1 repeated" in msg
    assert _plan_raw(4, x, [], 1.0, 1e-9)[0] == INVALID_ARG  # NULL coeffs
    assert _plan_raw(4, x, [np.nan], 1.0, 1e-9)[0] == INVALID_ARG
    assert _plan_raw(4, x, [np.inf], 1.0, 1e-9)[0] == INVALID_ARG
    st, msg = _plan_raw(4, x, [1.0], np.inf, 1e-9)
    assert st == INVALID_ARG and "time is not finite" in msg
    assert _plan_raw(4, x, [1.0], np.nan, 1e-9)[0] == INVALID_ARG
    for tol in (0.0, 1.0, -1e-3, 2.0, np.nan):
        st, msg = _plan_raw(4, x, [1.0], 1.0, tol)
        assert st == INVALID_ARG and "tol must be in (0, 1)" in msg
    assert _plan_raw(4, x, [1.0], 1.0, 1e-9, out3=False)[0] == INVALID_ARG
    assert _plan_raw(4, x, [1.0], 1.0, 1e-9, tail=False)[0] == INVALID_ARG
    for prec, n in ((7, 4), (1, 0), (1, 41)):
        assert _plan_raw(n, x, [1.0], 1.0, 1e-9, prec=prec)[0] == INVALID_ARG
    # the degree cap: the message says to split the time
    st, msg = _plan_raw(4, x, [1.0], 70000.0, 1e-9)
    assert st == UNSUPPORTED and "split the time over several calls" in msg
    st, msg = _plan_raw(4, x, [1.0], 1e6, 1e-9)
    assert st == UNSUPPORTED and "split the time" in msg
    assert pauli_evolution_plan(4, C128, x, [1.0], 65000.0, 1e-3)[0] <= 65536
    with pytest.raises(CircuitError) as e:
        pauli_evolution_plan(4, C128, x, [1.0], 65536.0, 1e-15)
    assert e.value.status == UNSUPPORTED


def test_null_states_are_refused():
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    c = np.ones(1)
    d, tl = C.c_uint32(), C.c_double()
    L = _lib.lib()
    assert L.qipb200_state_evolve_pauli_sum(None, None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(c), 1.0, 1e-9,
                                            C.byref(d), C.byref(tl)) == INVALID_ARG
    assert "evolve_pauli_sum: NULL state" in L.qipb200_last_error(None).decode()


def test_cpp_mirror_evolve_compiles(tmp_path):
    src = tmp_path / "use_evolve.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &st, qip::B200State<double> &a, qip::B200State<double> &b) {\n"
                   "  std::pair<uint32_t, double> kt =\n"
                   "      st.evolve_pauli_sum(a, b, {{{'Z', 0}, {'Z', 1}}, {{'X', 2}}, {}}, {0.1, -0.2, 0.3}, 1.5, 1e-12);\n"
                   "  (void)kt;\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
