"""Reduced density matrices without a GPU: the references of tests/rdm_ref.py pinned against np.einsum, against the
Pauli reference of tests/pauli_ref.py and against closed forms; the exact integer reference; the bound's sensitivity;
the NULL-state refusal of qipb200_state_reduced_density and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import pauli_ref as pr
import rdm_ref as rr
from exact_circuits import exact_state
from rustqip_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG = 1
PRODUCT_V = [(1, 0.5), (0.5, 1j), (0.5j, 0.5), (-0.5, 1), (1, -0.25j), (0.25, -1)]


def random_psi(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.3


def einsum_rdm(psi, n, qubits):
    """Tensor contraction over the reshaped state: axis q is qubit q; the kept axes are moved to the end in the order
    qubits[k-1], ..., qubits[0], so that qubits[0] is the least significant bit of the flattened index."""
    k = len(qubits)
    t = np.asarray(psi, dtype=np.complex128).reshape((2,) * n)
    rest = [q for q in range(n) if q not in qubits]
    t = np.transpose(t, rest + list(qubits)[::-1]).reshape(1 << (n - k), 1 << k)
    return np.einsum("ra,rb->ab", t, np.conj(t))


def subsets(n):
    out = []
    for k in (1, 2, 3):
        if k > n:
            continue
        for qs in itertools.combinations(range(n), k):
            for perm in itertools.permutations(qs):
                out.append(list(perm))
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_reference_matches_einsum(n):
    psi = random_psi(n, 100 + n)
    cases = subsets(n)
    if n > 5:
        cases = cases[:: max(1, len(cases) // 120)]
    if n <= 5:
        cases += [list(range(n)), list(range(n))[::-1]]
    for qs in cases:
        want = einsum_rdm(psi, n, qs)
        got = rr.rdm_ref(psi, n, qs).astype(np.complex128)
        assert np.max(np.abs(got - want)) <= 1e-13, (n, qs)


@pytest.mark.parametrize("n", [3, 5, 7])
def test_reference_matches_pauli_expectations(n):
    """Tr(rho P_A) == <psi|P|psi> for every Pauli string on A: fixes the Kronecker order of bit i <-> qubits[i]."""
    psi = random_psi(n, 200 + n)
    for qs in ([0], [n - 1], [2, 0], [0, n - 1], [n - 1, 1, 0], [1, n - 2, n - 1]):
        if len(set(qs)) < len(qs):
            continue
        rho = rr.rdm_ref(psi, n, qs).astype(np.complex128)
        for letters in itertools.product("IXYZ", repeat=len(qs)):
            term = [(l, q) for l, q in zip(letters, qs) if l != "I"]
            want = float(pr.expect_ref(psi, n, term))
            got = np.trace(rho @ rr.pauli_matrix(term, qs))
            assert abs(got.imag) <= 1e-12 and abs(got.real - want) <= 1e-12, (qs, term, got, want)


def test_diagonal_is_the_marginal_and_trace_is_norm2():
    n = 9
    psi = random_psi(n, 7)
    for qs in ([0, 4], [8, 3, 1], list(range(9))[::-1][:6]):
        rho = rr.rdm_ref(psi, n, qs)
        a, _ = rr.split_index(n, qs)
        marg = np.bincount(a, weights=np.abs(psi) ** 2, minlength=1 << len(qs))
        assert np.allclose(np.diag(rho).real.astype(float), marg, rtol=0, atol=1e-13)
        assert abs(float(np.trace(rho).real) - float(np.sum(np.abs(psi) ** 2))) <= 1e-12


@pytest.mark.parametrize("n", [4, 6])
def test_product_state_closed_form(n):
    psi = rr.product_state(n, [PRODUCT_V[q % 6] for q in range(n)])
    vs = [PRODUCT_V[q % 6] for q in range(n)]
    for qs in ([0], [n - 1, 0], [1, 3, 2], list(range(n))[::-1]):
        want = rr.product_rdm(n, qs, vs)
        got = rr.rdm_ref(psi, n, qs)
        assert np.max(np.abs(got - want)) <= 1e-15, qs


@pytest.mark.parametrize("n", [3, 6])
def test_ghz_closed_form(n):
    alpha, beta = 0.6, 0.8 * np.exp(0.7j)
    psi = np.zeros(1 << n, dtype=np.complex128)
    psi[0], psi[-1] = alpha, beta
    for qs in ([0], [n - 1, 1], list(range(n - 1)), list(range(n))[::-1]):
        want = rr.ghz_rdm(n, qs, alpha, beta)
        got = rr.rdm_ref(psi, n, qs)
        assert np.max(np.abs(got - want)) <= 1e-15, qs
        nz = np.count_nonzero(np.abs(want) > 0)
        assert nz == (4 if len(qs) == n else 2)


@pytest.mark.parametrize("n,bits", [(5, 20), (10, 16), (12, 8)])
def test_integer_reference_is_exact(n, bits):
    psi = exact_state(n, 300 + n, bits)
    assert rr.budget_ok(psi, n, 1)
    for qs in ([0], [n - 1, 0], [3, 1, 4], list(range(n))[::-1][: min(n, 8)]):
        exact = rr.rdm_int(psi, n, qs)
        assert np.array_equal(rr.rdm_exact(psi, n, qs), exact)
        assert np.max(np.abs(rr.rdm_ref(psi, n, qs) - exact)) == 0
        assert np.array_equal(exact, np.conj(exact.T))


def test_budget_refuses_states_over_53_bits():
    psi = exact_state(12, 1, 23)
    assert rr.budget_ok(psi, 12, 4) is False
    with pytest.raises(AssertionError):
        rr.rdm_int(psi, 12, [0, 1, 2, 3])


def test_bound_accepts_another_order_and_rejects_a_perturbation():
    n, qs = 14, [0, 13, 5]
    psi = random_psi(n, 99)
    want = rr.rdm_ref(psi, n, qs)
    W = rr.abs_weight(psi, n, qs)
    b = rr.bound(n, len(qs), W)
    # plain double matrix product: another summation order, well inside the bound
    X = rr.blocks(psi, n, qs, np.complex128)
    other = X.T @ np.conj(X)
    assert np.all(np.abs(other - want) <= b)
    bad = other.copy()
    bad[1, 2] += 1e-12 * W[1, 2]
    assert not np.all(np.abs(bad - want) <= b)
    assert rr.kernel_depth(30, 6) == 2 * 32 * 1986 + 1 + 264
    assert rr.kernel_depth(30, 1) == 2 * 4 * 1986 + 256 + 264


def test_null_state_is_refused():
    out = (C.c_double * 8)()
    qs = (C.c_uint64 * 1)(0)
    assert _lib.lib().qipb200_state_reduced_density(None, qs, 1, out) == INVALID_ARG
    assert "reduced_density" in _lib.lib().qipb200_last_error(None).decode()


def test_cpp_mirror_reduced_density_compiles(tmp_path):
    src = tmp_path / "use_rdm.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::B200State<double> &st) {\n"
                   "  std::vector<std::complex<double>> rho = st.reduced_density({0, 3});\n"
                   "  return rho[0].real() + rho[5].imag();\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
