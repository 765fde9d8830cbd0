"""Pauli sums and the adjoint gradient without a GPU: the long-double adjoint reference of tests/gradient_ref.py pinned to
scipy.linalg.expm of Kronecker products (central finite differences) and to the exact parameter-shift rule; the sum
references and the emulators; the closed form of the full-size tests; the plans (qipb200_pauli_sum_plan,
qipb200_pauli_gradient_plan) against the policy copies; the validation, the NULL-state refusals and the C++ mirror."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg

import gradient_ref as gr
import pauli_rot_ref as rr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import _marshal_paulis, _ptr, pauli_gradient_plan, pauli_sum_plan
from test_pauli_rotation_cpu import kron_matrix, random_psi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3


def random_terms(n, count, rng, weights=None):
    """Random strings of every weight 0..n (the identity included)."""
    out = []
    for i in range(count):
        w = (i % (n + 1)) if weights is None else int(rng.choice(weights))
        qs = rng.choice(n, size=w, replace=False)
        out.append([(str(rng.choice(list("XYZ"))), int(q)) for q in qs])
    return out


def dense_h(n, ham, coeffs):
    return sum(float(c) * kron_matrix(n, t) for t, c in zip(ham, coeffs))


def energy_expm(n, psi0, ansatz, angles, H):
    v = psi0.astype(C128)
    for t, th in zip(ansatz, angles):
        v = scipy.linalg.expm(-0.5j * th * kron_matrix(n, t)) @ v
    return float(np.vdot(v, H @ v).real)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_adjoint_reference_matches_expm_finite_differences_and_parameter_shift(n):
    rng = np.random.default_rng(40 + n)
    T = 12 if n < 8 else 6
    ansatz = random_terms(n, T, rng)
    angles = rng.uniform(-3, 3, size=T)
    ham = random_terms(n, 7, rng)
    coeffs = rng.normal(size=len(ham))
    psi0 = random_psi(n, 7 * n)
    H = dense_h(n, ham, coeffs)
    e, g = gr.adjoint_ref(psi0, n, ansatz, angles, ham, coeffs)
    scale = float(np.sum(np.abs(coeffs))) * float(np.linalg.norm(psi0)) ** 2
    assert abs(float(e) - energy_expm(n, psi0, ansatz, angles, H)) <= 1e-12 * scale
    h = 1e-5
    for t in range(T):
        d = np.zeros(T)
        d[t] = h
        fd = (energy_expm(n, psi0, ansatz, angles + d, H) - energy_expm(n, psi0, ansatz, angles - d, H)) / (2 * h)
        assert abs(float(g[t]) - fd) <= 1e-7 * scale, (t, float(g[t]), fd)
        d[t] = math.pi / 2  # exact for a Pauli string: P^2 = 1
        ps = (energy_expm(n, psi0, ansatz, angles + d, H) - energy_expm(n, psi0, ansatz, angles - d, H)) / 2
        assert abs(float(g[t]) - ps) <= 1e-12 * scale, (t, float(g[t]), ps)


def test_one_qubit_spot_check():
    psi0 = np.array([1, 0], dtype=C128)
    for th in (0.0, 0.3, -1.7, 2.9):
        e, g = gr.adjoint_ref(psi0, 1, [[("Y", 0)]], [th], [[("Z", 0)]], [1.0])
        assert abs(float(e) - math.cos(th)) <= 1e-15 and abs(float(g[0]) + math.sin(th)) <= 1e-15


@pytest.mark.parametrize("n", [1, 3, 6])
def test_sum_references_match_kronecker_products(n):
    rng = np.random.default_rng(n)
    ham = random_terms(n, 3 * n + 4, rng) + [[("Z", 0)], [("Z", 0)], []]  # repeated and identity terms
    coeffs = rng.normal(size=len(ham))
    psi = random_psi(n, n + 1)
    want = dense_h(n, ham, coeffs) @ psi
    assert np.max(np.abs(gr.sum_ref(psi, n, ham, coeffs).astype(C128) - want)) <= 1e-13
    for dtype in (C128, C64):
        src = psi.astype(dtype)
        ref = gr.sum_ref(src, n, ham, coeffs)
        got = gr.emulate_sum(src, n, ham, coeffs, dtype)
        lim = gr.sum_bound(n, ham, dtype) * gr.sum_weights(src, n, ham, coeffs)
        assert np.all(np.abs(got.astype(np.clongdouble) - ref) <= lim)
    assert not np.any(gr.emulate_sum(psi, n, [], [], C128))


def test_emulated_gradient_states_match_expm():
    n = 5
    rng = np.random.default_rng(5)
    ansatz = random_terms(n, 10, rng)
    angles = rng.uniform(-3, 3, size=10)
    ham = random_terms(n, 6, rng)
    coeffs = rng.normal(size=6)
    psi0 = random_psi(n, 3)
    U = np.eye(1 << n, dtype=C128)
    for t, th in zip(ansatz, angles):
        U = scipy.linalg.expm(-0.5j * th * kron_matrix(n, t)) @ U
    st, wk = gr.emulate_gradient(psi0, n, ansatz, angles, ham, coeffs, C128)
    assert np.max(np.abs(st - psi0)) <= 1e-13
    assert np.max(np.abs(wk - U.conj().T @ dense_h(n, ham, coeffs) @ U @ psi0)) <= 1e-12


@pytest.mark.parametrize("n", [3, 4, 5, 6])
def test_closed_form_matches_expm_and_adjoint_reference(n):
    rng = np.random.default_rng(90 + n)
    theta, phi = rng.uniform(-3, 3, size=n), rng.uniform(-3, 3, size=n)
    a, b, c = rng.normal(size=n), rng.normal(size=n), rng.normal(size=n)
    ansatz = gr.product_ansatz(n)
    angles = np.concatenate([theta, phi])
    ham, coeffs = gr.product_hamiltonian(n, a, b, c)
    e, gt, gp = gr.closed_form(n, theta, phi, a, b, c)
    psi0 = np.zeros(1 << n, dtype=C128)
    psi0[0] = 1
    assert abs(float(e) - energy_expm(n, psi0, ansatz, angles, dense_h(n, ham, coeffs))) <= 1e-12
    er, g = gr.adjoint_ref(psi0, n, ansatz, angles, ham, coeffs)
    assert abs(float(er - e)) <= 1e-15 * n
    assert np.max(np.abs(g - np.concatenate([gt, gp]))) <= 1e-15 * n


# ---- plans ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [C128, C64])
def test_sum_plan_matches_policy(dtype):
    rng = np.random.default_rng(11)
    diag = [[("Z", int(q)) for q in np.flatnonzero(rng.random(30) < 0.5)] for _ in range(2000)] + [[]]
    assert pauli_sum_plan(30, dtype, diag) == gr.sum_sweeps(30, diag) == 1
    assert pauli_sum_plan(30, dtype, []) == gr.sum_sweeps(30, []) == 0
    tfim = rr.ising_step(30)
    assert pauli_sum_plan(30, dtype, tfim) == gr.sum_sweeps(30, tfim) == 4
    qaoa = rr.qaoa_layer(30)[:45]
    assert pauli_sum_plan(30, dtype, qaoa) == 1
    for seed in range(6):
        r = np.random.default_rng(seed)
        n = int(r.integers(1, 34))
        terms = random_terms(n, 60, r)
        assert pauli_sum_plan(n, dtype, terms) == gr.sum_sweeps(n, terms)
    ucc = rr.ucc_strings(30, 64, 64)
    assert pauli_sum_plan(30, dtype, ucc) == gr.sum_sweeps(30, ucc)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_gradient_plan_matches_policy(dtype):
    rng = np.random.default_rng(12)
    cases = [(rr.ising_step(30) * 2, rr.ising_step(30)), (rr.qaoa_layer(30), rr.qaoa_layer(30)[:45]),
             (rr.ucc_strings(30, 64, 64), rr.ising_step(30)), ([], rr.ising_step(30)), (rr.z_pairs(30), []),
             ([[("X", 27)]] * 600, [[("Z", 0)]])]
    for seed in range(4):
        r = np.random.default_rng(seed)
        n = int(r.integers(1, 34))
        cases.append((random_terms(n, 40, r), random_terms(n, 10, r)))
    for ansatz, ham in cases:
        n = 30 if all(q < 30 for t in ansatz + ham for _, q in t) else 34
        n = max([n] + [q + 1 for t in ansatz + ham for _, q in t])
        assert pauli_gradient_plan(n, dtype, ansatz, ham) == gr.gradient_plan_policy(n, ansatz, ham)
    assert pauli_gradient_plan(30, dtype, [], [])[2] == 1  # the energy alone is one backward sweep
    assert pauli_gradient_plan(30, dtype, [[("X", 27)]] * 600, [])[2] == 3  # cut every 256 terms


def _sum_plan_raw(n, qubits, letters, lens, prec=1):
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    la = C.create_string_buffer(bytes(letters), max(1, len(letters)))
    ln = (C.c_uint32 * max(1, len(lens)))(*lens)
    v = C.c_uint32(99)
    st = _lib.lib().qipb200_pauli_sum_plan(prec, n, qa, la, ln, len(lens), C.byref(v))
    return st, _lib.lib().qipb200_last_error(None).decode(), v.value


def test_plan_validation_errors():
    st, msg, _ = _sum_plan_raw(4, [0], b"W", [1])
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg and "term 0" in msg
    st, msg, _ = _sum_plan_raw(4, [4], b"X", [1])
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg, _ = _sum_plan_raw(4, [0, 2, 2], b"XYZ", [3])
    assert st == BAD_INDEX and "qubit 2 repeated" in msg
    for prec, n in ((7, 4), (1, 0), (1, 41)):
        assert _sum_plan_raw(n, [0], b"X", [1], prec=prec)[0] == INVALID_ARG
    v = C.c_uint32()
    assert _lib.lib().qipb200_pauli_sum_plan(1, 4, None, None, None, 1, C.byref(v)) == INVALID_ARG
    assert _lib.lib().qipb200_pauli_sum_plan(1, 4, None, None, None, 0, C.byref(v)) == 0 and v.value == 0
    # the gradient plan validates both lists
    for ansatz, ham, code in (([[("Q", 0)]], [], INVALID_ARG), ([], [[("X", 5)]], BAD_INDEX),
                              ([[("X", 1), ("Y", 1)]], [[("Z", 0)]], BAD_INDEX)):
        with pytest.raises(CircuitError) as e:
            pauli_gradient_plan(4, C128, ansatz, ham)
        assert e.value.status == code
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    assert _lib.lib().qipb200_pauli_gradient_plan(1, 4, _ptr(qs), ls, _ptr(lens), 1, _ptr(qs), ls, _ptr(lens), 1,
                                                  None) == INVALID_ARG
    with pytest.raises(CircuitError) as e:
        pauli_sum_plan(3, C128, [[("X", 0)], [("Q", 1)]])
    assert e.value.status == INVALID_ARG


def test_null_states_are_refused():
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    c = np.ones(1)
    L = _lib.lib()
    assert L.qipb200_state_apply_pauli_sum(None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(c)) == INVALID_ARG
    assert "apply_pauli_sum: NULL state" in L.qipb200_last_error(None).decode()
    e, g = np.zeros(1), np.zeros(1)
    assert L.qipb200_state_pauli_energy_gradient(None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(c), _ptr(qs), ls,
                                                 _ptr(lens), 1, _ptr(c), _ptr(e), _ptr(g)) == INVALID_ARG
    assert "pauli_energy_gradient: NULL state" in L.qipb200_last_error(None).decode()


def test_cpp_mirror_gradient_compiles(tmp_path):
    src = tmp_path / "use_grad.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &st, qip::B200State<double> &w) {\n"
                   "  w.apply_pauli_sum(st, {{{'Z', 0}, {'Z', 1}}, {{'X', 2}}, {}}, {0.1, -0.2, 0.3});\n"
                   "  std::pair<double, std::vector<double>> eg =\n"
                   "      st.energy_gradient(w, {{{'Y', 0}}, {}}, {0.4, 0.1}, {{{'Z', 0}}}, {1.0});\n"
                   "  (void)eg;\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
