"""The Lanczos ground state without a GPU: the library's tridiagonal solve against scipy.linalg.eigh_tridiagonal, the
numpy emulation of the device recurrence (tests/lanczos_ref.py) reaching eigh's lowest eigenvalue within its returned
residual at the default tolerances, the open-chain TFIM closed form against eigh, the plan counts, every validation
error of the host-only entries, the NULL-state refusal and the C++ mirror."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg

import lanczos_ref as lr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import _marshal_paulis, _ptr, lanczos_ritz, pauli_lanczos_plan
from test_gradient_cpu import dense_h, random_terms
from test_pauli_rotation_cpu import random_psi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3
TOL = {C128: 1e-8, C64: 1e-3}
EPS = np.finfo(np.float64).eps


def tridiagonals(rng):
    """(name, alpha, beta[0..m]) : random, graded, near-degenerate lowest pair, Lanczos-like."""
    out = []
    for m in (1, 2, 3, 5, 17, 64, 200, 500):
        out.append(("random", rng.normal(size=m), np.abs(rng.normal(size=m + 1))))
        g = 10.0 ** -np.linspace(0, 8, m)
        out.append(("graded", rng.normal(size=m) * g, np.append(np.abs(rng.normal(size=m)) * g, 0.3)))
        if m >= 4:  # two weakly coupled blocks with the same lowest eigenvalue
            h = m // 2
            a = np.concatenate([np.full(h, 2.0), np.full(m - h, 2.0)])
            a[0] = a[h] = -1.0
            b = np.full(m + 1, 0.5)
            b[h] = 1e-9
            out.append(("near-degenerate", a, b))
        out.append(("positive beta, clustered", np.cos(np.arange(m) * 0.7), np.full(m + 1, 0.5)))
    return out


def test_ritz_matches_eigh_tridiagonal():
    rng = np.random.default_rng(7)
    for name, a, b in tridiagonals(rng):
        m = len(a)
        theta, y, est = lanczos_ritz(a, b)
        w, V = scipy.linalg.eigh_tridiagonal(a, b[1:m]) if m > 1 else (a.copy(), np.ones((1, 1)))
        tn = max(np.max(np.abs(a)) + 2 * np.max(np.abs(b[1:m]), initial=0.0), 1e-300)
        assert abs(theta - w[0]) <= 8 * m * EPS * tn, (name, m, theta, w[0])
        gap = w[1] - w[0] if m > 1 else np.inf
        v = V[:, 0] * (1 if V[0, 0] >= 0 else -1)
        ytol = 1e-9 + 64 * m * EPS * tn / max(gap, 1e-300)
        if ytol < 0.1:
            # the sign rule y[0] >= 0 decides only where |y[0]| stands above the vector's absolute accuracy (a
            # random tridiagonal may localise the eigenvector far from row 0; Lanczos' never is, since v_0 overlaps it)
            if abs(v[0]) <= ytol:
                v = v if np.max(np.abs(y - v)) <= np.max(np.abs(y + v)) else -v
            assert np.max(np.abs(y - v)) <= ytol, (name, m, np.max(np.abs(y - v)), gap)
            assert abs(est - b[m] * abs(v[-1])) <= b[m] * ytol
        assert abs(np.linalg.norm(y) - 1) <= 1e-13 and y[0] >= 0
        assert abs(est - b[m] * abs(y[-1])) <= 1e-15 * b[m]


def test_ritz_validation_errors():
    L = _lib.lib()
    a, b = np.ones(3), np.ones(4)
    t, e = C.c_double(), C.c_double()
    assert L.qipb200_lanczos_ritz(None, _ptr(b), 3, C.byref(t), None, C.byref(e)) == INVALID_ARG
    assert L.qipb200_lanczos_ritz(_ptr(a), None, 3, C.byref(t), None, C.byref(e)) == INVALID_ARG
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 3, None, None, C.byref(e)) == INVALID_ARG
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 3, C.byref(t), None, None) == INVALID_ARG
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 0, C.byref(t), None, C.byref(e)) == INVALID_ARG
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 3, C.byref(t), None, C.byref(e)) == 0  # y may be NULL
    a[1] = np.nan
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 3, C.byref(t), None, C.byref(e)) == INVALID_ARG
    assert "alpha 1 is not finite" in L.qipb200_last_error(None).decode()
    a[1], b[3] = 1.0, np.inf
    assert L.qipb200_lanczos_ritz(_ptr(a), _ptr(b), 3, C.byref(t), None, C.byref(e)) == INVALID_ARG
    with pytest.raises(ValueError):
        lanczos_ritz([1.0, 2.0], [1.0, 1.0])


def hamiltonians(n, rng):
    """The open TFIM, the XXX chain (n >= 2), random strings with repeats and identities, and a single term."""
    out = {"tfim": lr.tfim(rng.uniform(0.2, 1.0, size=n - 1), rng.uniform(0.5, 1.5, size=n)),
           "single": ([[("Y", n // 2)]], np.array([0.7]))}
    if n >= 2:
        out["xxx"] = lr.heisenberg(n)
    rand = random_terms(n, 2 * n + 3, rng)
    rand = rand + rand[:2] + [[]]
    out["random"] = (rand, rng.normal(size=len(rand)))
    return out


@pytest.mark.parametrize("dtype", [C128, C64])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 10])
def test_emulated_lanczos_reaches_eigh_within_residual(n, dtype):
    rng = np.random.default_rng(90 + n)
    psi = random_psi(n, 3 * n + 1)
    for name, (terms, coeffs) in sorted(hamiltonians(n, rng).items()):
        lam = np.linalg.eigvalsh(dense_h(n, terms, coeffs))[0]
        a, b = lr.split(terms, coeffs)
        r = lr.lanczos(psi, n, terms, coeffs, dtype, TOL[dtype])
        assert r["converged"] and r["steps"] <= min(300, 2 ** n + 40), (name, r["steps"])
        assert r["estimate"] <= TOL[dtype] * b
        # the state's own rounding: |x| carries u relative error per amplitude, so E and the residual move by ~u b
        allow = 8 * lr.rr.U[dtype] * (b + abs(a)) + 1e-13
        assert abs(r["energy"] - lam) <= r["residual"] + allow, (name, r["energy"], lam, r["residual"])
        assert r["residual"] <= 4 * TOL[dtype] * b + allow, (name, r["residual"], TOL[dtype] * b)
        assert abs(r["theta"] - lam) <= r["estimate"] + allow


def test_emulator_is_consistent_with_its_lanczos():
    """Given the alpha and beta of the numpy run, the emulator rebuilds vectors whose norms are those betas."""
    n = 6
    terms, coeffs = lr.heisenberg(n)
    psi = random_psi(n, 11)
    for dtype in (C128, C64):
        r = lr.lanczos(psi, n, terms, coeffs, dtype, TOL[dtype])
        e = lr.emulate(psi, n, terms, coeffs, dtype, r["alpha"], r["beta"], xnorm=1.0)
        for j in range(r["steps"] + 1):
            nu = float(np.linalg.norm(e["u"][j].astype(C128)))
            assert abs(nu - r["beta"][j]) <= 1e-12 * nu
        assert e["state"].dtype == dtype


@pytest.mark.parametrize("n", [2, 3, 5, 8, 10])
def test_tfim_closed_form_matches_eigh(n):
    rng = np.random.default_rng(200 + n)
    J, h = rng.uniform(-1.5, 1.5, size=n - 1), rng.uniform(-1.5, 1.5, size=n)
    terms, coeffs = lr.tfim(J, h)
    lam = np.linalg.eigvalsh(dense_h(n, terms, coeffs))[0]
    assert abs(lr.tfim_ground(J, h) - lam) <= 1e-12 * n


def test_sector_ground_state_from_neel():
    """The XXX chain conserves S_z: from the Neel state Lanczos finds the S_z = 0 ground energy."""
    n = 8
    terms, coeffs = lr.heisenberg(n)
    neel = np.zeros(1 << n, dtype=C128)
    neel[int("01" * (n // 2), 2)] = 1.0
    H = dense_h(n, terms, coeffs)
    sz0 = [i for i in range(1 << n) if bin(i).count("1") == n // 2]
    lam0 = np.linalg.eigvalsh(H[np.ix_(sz0, sz0)])[0]
    r = lr.lanczos(neel, n, terms, coeffs, C128, 1e-8)
    assert r["converged"] and abs(r["energy"] - lam0) <= r["residual"] + 1e-12
    # the antiferromagnet's ground state is in S_z = 0; a sector of S_z != 0 has a higher ground energy
    one = [i for i in range(1 << n) if bin(i).count("1") == n // 2 + 1]
    assert np.linalg.eigvalsh(H[np.ix_(one, one)])[0] > lam0 + 1e-3
    up = np.zeros(1 << n, dtype=C128)
    up[int("11" + "01" * (n // 2 - 1), 2)] = 1.0  # n/2 + 1 ones
    r1 = lr.lanczos(up, n, terms, coeffs, C128, 1e-8)
    assert abs(r1["energy"] - np.linalg.eigvalsh(H[np.ix_(one, one)])[0]) <= r1["residual"] + 1e-12


def test_plan_counts():
    rng = np.random.default_rng(5)
    cases = [lr.tfim(np.ones(29), np.ones(30))[0], lr.heisenberg(30)[0], lr.rr.ucc_strings(30, 64, 64),
             random_terms(12, 40, rng), [[("Z", 0)]], lr.rr.qaoa_layer(30)[:45] + [[]], [], [[], []]]
    for dtype in (C128, C64):
        for terms in cases:
            n = 30 if terms and len(terms) > 3 and terms is not cases[3] else 12
            assert pauli_lanczos_plan(n, dtype, terms) == lr.plan_policy(n, terms), terms[:3]
    s, k1, k2, k0 = pauli_lanczos_plan(30, C128, cases[0])
    assert (s, k1, k2, k0) == (4, 5, 5, 8)  # the TFIM: 4 sum sweeps
    assert pauli_lanczos_plan(30, C128, [[], []]) == (0, 0, 0, 2)


def _plan_raw(n, terms, prec=1, out=True):
    qs, ls, lens = _marshal_paulis(terms)
    v = (C.c_uint32 * 4)()
    st = _lib.lib().qipb200_pauli_lanczos_plan(prec, n, _ptr(qs), ls, _ptr(lens), len(terms), v if out else None)
    return st, _lib.lib().qipb200_last_error(None).decode()


def test_plan_validation_errors():
    st, msg = _plan_raw(4, [[("W", 0)]])
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg
    st, msg = _plan_raw(4, [[("X", 4)]])
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg = _plan_raw(4, [[("X", 1), ("Z", 1)]])
    assert st == BAD_INDEX and "qubit 1 repeated" in msg
    assert _plan_raw(4, [[("X", 0)]], out=False)[0] == INVALID_ARG
    for prec, n in ((7, 4), (1, 0), (1, 41)):
        assert _plan_raw(n, [[("X", 0)]], prec=prec)[0] == INVALID_ARG
    with pytest.raises(CircuitError) as e:
        pauli_lanczos_plan(3, C128, [[("Q", 0)]])
    assert e.value.status == INVALID_ARG


def test_null_states_are_refused():
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    c, out3 = np.ones(1), np.zeros(3)
    m, cv = C.c_uint32(), C.c_uint32()
    L = _lib.lib()
    assert L.qipb200_state_lanczos_pauli_sum(None, None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(c), 10, 1e-8, 1,
                                             C.byref(m), C.byref(cv), None, None, _ptr(out3)) == INVALID_ARG
    assert "lanczos_pauli_sum: NULL state" in L.qipb200_last_error(None).decode()


def test_cpp_mirror_lanczos_compiles(tmp_path):
    src = tmp_path / "use_lanczos.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &st, qip::B200State<double> &a, qip::B200State<double> &b) {\n"
                   "  auto r = st.lanczos_pauli_sum(a, b, {{{'Z', 0}, {'Z', 1}}, {{'X', 2}}, {}}, {0.1, -0.2, 0.3}, 300,\n"
                   "                                1e-8, true);\n"
                   "  double e = r.energy + r.residual + r.ritz_norm + r.alpha.size() + r.beta.size();\n"
                   "  (void)e;\n"
                   "  (void)r.converged;\n"
                   "  (void)r.steps;\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
