"""The quantum geometric tensor without a GPU: the long-double fork-and-segment reference of tests/qgt_ref.py pinned to
the definition (d_t psi from scipy.linalg.expm of Kronecker products), to the parameter-shift rule for the fidelity
Hessian and to the product-ansatz closed form; the end-state emulation; the error bound against a precision-faithful
numpy run of the algorithm; the plan (qipb200_pauli_geometric_tensor_plan) against the policy; the validation, the NULL
refusals and the C++ mirror."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg

import gradient_ref as gr
import pauli_rot_ref as rr
import qgt_ref as qr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import _marshal_paulis, _ptr, pauli_geometric_tensor_plan
from test_gradient_cpu import random_terms
from test_pauli_rotation_cpu import kron_matrix, random_psi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7


def unit_psi(n, seed):
    v = random_psi(n, seed)
    return v / np.linalg.norm(v)


def qgt_definition(n, psi0, ansatz, angles):
    """(G, e) from the definition: d_t psi = R_(T-1) .. R_(t+1) (-i/2) P_t psi_t with every R_t = expm(-i theta/2 P_t)."""
    P = [kron_matrix(n, t) for t in ansatz]
    R = [scipy.linalg.expm(-0.5j * th * p) for th, p in zip(angles, P)]
    T = len(ansatz)
    psis, v = [], psi0.astype(C128)
    for t in range(T):
        v = R[t] @ v
        psis.append(v)
    d = []
    for t in range(T):
        w = -0.5j * (P[t] @ psis[t])
        for k in range(t + 1, T):
            w = R[k] @ w
        d.append(w)
    psi = psis[-1]
    G = np.array([[np.vdot(d[i], d[j]) - np.vdot(d[i], psi) * np.vdot(psi, d[j]) for j in range(T)] for i in range(T)])
    e = np.array([np.vdot(psis[t], P[t] @ psis[t]).real for t in range(T)])
    return G, e


def fidelity_hessian(n, psi0, ansatz, angles):
    """d_i d_j |<psi(theta)|psi(theta')>|^2 at theta' = theta by the parameter-shift rule: R_t(theta) = cos(theta/2) -
    i sin(theta/2) P_t is a trigonometric polynomial of frequency 1/2 in each angle, so the fidelity has frequencies
    0 and 1 and four overlaps shifted by +-pi/2 give each second derivative exactly (shifts add when i == j)."""
    P = [kron_matrix(n, t) for t in ansatz]
    eye = np.eye(1 << n)

    def state(th):
        v = psi0.astype(C128)
        for a, p in zip(th, P):
            v = (math.cos(a / 2) * eye - 1j * math.sin(a / 2) * p) @ v
        return v

    ref = state(angles)
    T = len(ansatz)
    H = np.zeros((T, T))
    for i in range(T):
        for j in range(T):
            f = 0.0
            for si, sj, w in ((1, 1, 1), (1, -1, -1), (-1, 1, -1), (-1, -1, 1)):
                th = np.array(angles, dtype=np.float64)
                th[i] += si * math.pi / 2
                th[j] += sj * math.pi / 2
                f += w * abs(np.vdot(ref, state(th))) ** 2
            H[i, j] = f / 4
    return H


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_reference_matches_definition_and_parameter_shift(n):
    rng = np.random.default_rng(60 + n)
    T = 9 if n < 8 else 6
    ansatz = random_terms(n, T, rng)  # every weight, the empty string included
    ansatz[2] = ansatz[1]  # a repeated string
    angles = rng.uniform(-3, 3, size=T)
    psi0 = unit_psi(n, 5 * n)
    G, e = qr.qgt_ref(psi0, n, ansatz, angles)
    Gd, ed = qgt_definition(n, psi0, ansatz, angles)
    assert np.max(np.abs(G.astype(C128) - Gd)) <= 1e-13
    assert np.max(np.abs(e.astype(np.float64) - ed)) <= 1e-13
    assert np.array_equal(G, np.conj(G.T))
    H = fidelity_hessian(n, psi0, ansatz, angles)
    assert np.max(np.abs(-2 * G.real.astype(np.float64) - H)) <= 1e-12
    for t, term in enumerate(ansatz):  # an empty string is a global phase
        if not term:
            assert np.max(np.abs(G[t].astype(C128))) <= 1e-15 and np.max(np.abs(G[:, t].astype(C128))) <= 1e-15


def test_one_qubit_spot_check():
    """R_Y(a) then R_Z(b) on |0>: G = [[1/4, (i/4) sin a], [-(i/4) sin a, (1 - cos^2 a)/4]], e = (0, cos a)."""
    psi0 = np.array([1, 0], dtype=C128)
    for a, b in ((0.3, 1.1), (-1.7, 0.4), (2.9, -2.2)):
        G, e = qr.qgt_ref(psi0, 1, [[("Y", 0)], [("Z", 0)]], [a, b])
        want = np.array([[0.25, 0.25j * math.sin(a)], [-0.25j * math.sin(a), (1 - math.cos(a) ** 2) / 4]])
        assert np.max(np.abs(G.astype(C128) - want)) <= 1e-16
        assert abs(float(e[0])) <= 1e-16 and abs(float(e[1]) - math.cos(a)) <= 1e-16


@pytest.mark.parametrize("n", [3, 4, 5, 6])
def test_closed_form_matches_definition_and_reference(n):
    rng = np.random.default_rng(80 + n)
    theta, phi = rng.uniform(-3, 3, size=n), rng.uniform(-3, 3, size=n)
    ansatz = gr.product_ansatz(n)
    angles = np.concatenate([theta, phi])
    psi0 = np.zeros(1 << n, dtype=C128)
    psi0[0] = 1
    G, e = qr.closed_form(n, theta, phi)
    Gd, ed = qgt_definition(n, psi0, ansatz, angles)
    assert np.max(np.abs(G.astype(C128) - Gd)) <= 1e-13
    assert np.max(np.abs(e.astype(np.float64) - ed)) <= 1e-13
    Gr, er = qr.qgt_ref(psi0, n, ansatz, angles)
    assert np.max(np.abs(G - Gr)) <= 1e-16 * n and np.max(np.abs(e - er)) <= 1e-16 * n


def test_emulated_end_states():
    n = 6
    rng = np.random.default_rng(6)
    ansatz = random_terms(n, 11, rng) + [[("Y", 1), ("X", 4)]]
    angles = rng.uniform(-3, 3, size=len(ansatz))
    psi0 = unit_psi(n, 9)
    U = np.eye(1 << n, dtype=C128)
    for t, th in zip(ansatz, angles):
        U = scipy.linalg.expm(-0.5j * th * kron_matrix(n, t)) @ U
    for dtype in (C128, C64):
        st, wa, wb = qr.emulate_end_states(psi0.astype(dtype), n, ansatz, angles, dtype)
        assert st.dtype == wa.dtype == wb.dtype == dtype
        split = psi0.astype(dtype)
        for t, th in zip(ansatz, angles):  # rotation results do not depend on how the terms are grouped
            split = rr.emulate(split, n, [t], [th], dtype)
        assert np.array_equal(st, split) and np.array_equal(wa, st)
        assert np.array_equal(gr.apply_pauli(wb, n, ansatz[-1]), st)  # P^2 = 1, exactly
        tol = 1e-13 if dtype == C128 else 1e-5
        assert np.max(np.abs(st - U @ psi0)) <= tol
        assert np.max(np.abs(wb - kron_matrix(n, ansatz[-1]) @ U @ psi0)) <= tol


def emulate_values(psi0, n, ansatz, angles, dtype):
    """The call's algorithm with the device's precisions: states rounded to dtype after every rotation (the emulator's
    arithmetic), inner products in double (numpy's order, not the device's)."""
    T = len(ansatz)
    psi = np.asarray(psi0).astype(dtype)
    M = np.zeros((T, T), dtype=C128)
    e, nrm = np.zeros(T), np.zeros(T)
    for i in range(T):
        psi = rr.emulate(psi, n, [ansatz[i]], [angles[i]], dtype)
        mu = gr.apply_pauli(psi, n, ansatz[i]).astype(dtype)
        nrm[i] = float(np.sum(np.abs(psi.astype(C128)) ** 2))
        e[i] = float(np.vdot(psi.astype(C128), mu.astype(C128)).real)
        phi = psi
        for j in range(i + 1, T):
            M[i, j] = np.vdot(mu.astype(C128), gr.apply_pauli(phi.astype(C128), n, ansatz[j]))
            phi = rr.emulate(phi, n, [ansatz[j]], [angles[j]], dtype)
            mu = rr.emulate(mu, n, [ansatz[j]], [angles[j]], dtype)
    G = np.zeros((T, T), dtype=C128)
    for i in range(T):
        G[i, i] = 0.25 * (nrm[i] - e[i] * e[i])
        for j in range(i + 1, T):
            G[i, j] = complex(0.25 * (M[i, j].real - e[i] * e[j]), 0.25 * M[i, j].imag)
            G[j, i] = np.conj(G[i, j])
    return G, e


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bound_covers_the_precision_of_the_algorithm(dtype):
    n = 7
    rng = np.random.default_rng(70)
    ansatz = rr.ising_step(n) + rr.ucc_strings(n, 6, 7) + [[]]
    angles = rng.uniform(-6, 6, size=len(ansatz))
    psi0 = unit_psi(n, 71).astype(dtype)
    G, e = emulate_values(psi0, n, ansatz, angles, dtype)
    Gr, er = qr.qgt_ref(psi0, n, ansatz, angles)
    norm = float(np.linalg.norm(psi0.astype(C128)))
    bg, be = qr.qgt_bound(n, len(ansatz), norm, dtype)
    dg = float(np.max(np.abs(G.astype(np.clongdouble) - Gr)))
    de = float(np.max(np.abs(e.astype(np.longdouble) - er)))
    assert dg <= bg and de <= be, (dg, bg, de, be)
    # not vacuous: the f32 run errs by more than an f64 unit roundoff and within a few hundred of its own bound
    if dtype == C64:
        assert dg >= 1e-9 and dg >= bg / 1000, (dg, bg)


# ---- the plan ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_matches_policy(dtype):
    cases = [rr.qaoa_layer(30), rr.ising_step(30), rr.ucc_strings(30, 64, 64), [], [[("Z", 3)]], rr.z_pairs(12),
             [[("X", 27)]] * 300, [[("X", 2), ("Y", 20)], [("Y", 29)]] * 150]
    for seed in range(6):
        r = np.random.default_rng(seed)
        n = int(r.integers(1, 34))
        cases.append(random_terms(n, int(r.integers(1, 300)), r))
    for ansatz in cases:
        n = max([30] + [q + 1 for t in ansatz for _, q in t])
        got = pauli_geometric_tensor_plan(n, dtype, ansatz)
        assert got == qr.plan_policy(n, ansatz), (n, len(ansatz))
    assert pauli_geometric_tensor_plan(30, dtype, []) == (0, 0, 0)
    assert pauli_geometric_tensor_plan(30, dtype, [[("Y", 0)]]) == (1, 0, 2)
    # 300 joinable terms: the segments of the first 43 forks hold more than 256 terms and take two sweeps
    assert pauli_geometric_tensor_plan(30, dtype, [[("X", 27)]] * 300)[1] == 299 + 43


def _plan_raw(n, qubits, letters, lens, prec=1, out=True):
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    la = C.create_string_buffer(bytes(letters), max(1, len(letters)))
    ln = (C.c_uint32 * max(1, len(lens)))(*lens)
    v = (C.c_uint32 * 3)(9, 9, 9)
    st = _lib.lib().qipb200_pauli_geometric_tensor_plan(prec, n, qa, la, ln, len(lens), v if out else None)
    return st, _lib.lib().qipb200_last_error(None).decode(), list(v)


def test_plan_validation_errors():
    st, msg, _ = _plan_raw(4, [0], b"W", [1])
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg and "term 0" in msg
    st, msg, _ = _plan_raw(4, [4], b"X", [1])
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg, _ = _plan_raw(4, [0, 2, 2], b"XYZ", [3])
    assert st == BAD_INDEX and "qubit 2 repeated" in msg
    for prec, n in ((7, 4), (1, 0), (1, 41)):
        assert _plan_raw(n, [0], b"X", [1], prec=prec)[0] == INVALID_ARG
    st, msg, _ = _plan_raw(4, [0], b"X", [1], out=False)
    assert st == INVALID_ARG and "pauli_geometric_tensor_plan: NULL out3" in msg
    v = (C.c_uint32 * 3)()
    assert _lib.lib().qipb200_pauli_geometric_tensor_plan(1, 4, None, None, None, 1, v) == INVALID_ARG
    with pytest.raises(CircuitError) as e:
        pauli_geometric_tensor_plan(4, C128, [[("Z", 0)]] * 2049)
    assert e.value.status == UNSUPPORTED and "2049 terms, at most 2048" in str(e.value)
    assert pauli_geometric_tensor_plan(4, C128, [[("Z", 0)]] * 2048)[0] == 2048


def test_null_states_are_refused():
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    a, g = np.ones(1), np.zeros(2)
    L = _lib.lib()
    assert L.qipb200_state_pauli_geometric_tensor(None, None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(a), _ptr(g),
                                                  None) == INVALID_ARG
    assert "pauli_geometric_tensor: NULL state" in L.qipb200_last_error(None).decode()


def test_cpp_mirror_geometric_tensor_compiles(tmp_path):
    src = tmp_path / "use_qgt.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &st, qip::B200State<double> &a, qip::B200State<double> &b) {\n"
                   "  auto ge = st.geometric_tensor(a, b, {{{'Y', 0}}, {{'Z', 0}, {'Z', 1}}, {}}, {0.4, 0.1, 0.2});\n"
                   "  std::vector<std::complex<double>> G = ge.first;\n"
                   "  std::vector<double> e = ge.second;\n"
                   "  (void)G;\n"
                   "  (void)e;\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
