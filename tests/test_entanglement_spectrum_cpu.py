"""Entanglement spectrum without a GPU: the references of tests/spectrum_ref.py pinned against closed forms (product
states, Bell pairs, GHZ, Schmidt-form states with a chosen spectrum) and against purity_ref; the plan
(qipb200_entanglement_spectrum_plan) for every route, side size and kernel count, and every refusal; cuSOLVER loads in
this process; the NULL-state refusal of qipb200_state_entanglement_spectrum."""
import math

import numpy as np
import pytest

import purity_ref as pu
import rdm_ref as rr
import spectrum_ref as sr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import entanglement_spectrum_plan

C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
PRODUCT_V = [(1, 0.5), (0.5, 1j), (0.5j, 0.5), (-0.5, 1), (1, -0.25j), (0.25, -1)]


def bell_state(m, extra):
    """Qubit i paired with qubit m + i (i < m) as |00> + |11>, `extra` qubits after them in |0>; unnormalised."""
    n = 2 * m + extra
    j = np.arange(1 << n)
    ok = np.ones(1 << n, dtype=bool)
    for i in range(m):
        ok &= ((j >> (n - 1 - i)) & 1) == ((j >> (n - 1 - (m + i))) & 1)
    for q in range(2 * m, n):
        ok &= ((j >> (n - 1 - q)) & 1) == 0
    return n, ok.astype(np.complex128)


@pytest.mark.parametrize("n", [4, 7])
def test_product_state_has_one_eigenvalue(n):
    vs = [PRODUCT_V[q % 6] for q in range(n)]
    psi = rr.product_state(n, vs)
    T = float(np.prod([sum(abs(complex(x)) ** 2 for x in v) for v in vs]))
    for qs in ([0], [n - 1, 1], list(range(n // 2)), list(range(1, n))):
        lam, t = sr.schmidt_ref(psi, n, qs)
        s = min(len(qs), n - len(qs))
        assert lam.size == 1 << s
        assert abs(t - T) <= 1e-14 * T
        assert abs(lam[0] - T) <= 1e-13 * T and np.all(np.abs(lam[1:]) <= 1e-13 * T), qs
        assert sr.entropy([T] + [0.0] * (lam.size - 1), T) == 0.0


@pytest.mark.parametrize("m", [1, 2, 3, 5])
def test_bell_pairs_give_flat_spectrum(m):
    n, psi = bell_state(m, 2)
    for qs in (list(range(m)), list(range(m, 2 * m)), list(range(m)) + [2 * m]):
        lam, T = sr.schmidt_ref(psi, n, qs)
        assert T == 2 ** m
        nz = lam[: 1 << m]
        assert np.allclose(nz, 1.0, rtol=0, atol=1e-13), (qs, lam)
        assert np.all(np.abs(lam[1 << m:]) <= 1e-13)
        S = sr.entropy(np.where(lam > 1e-9, lam, 0.0), T)
        assert abs(S - m * math.log(2)) <= 1e-13
        # the exact G of this integer state: 2^m eigenvalues 1 (one per Bell-pair pattern), the rest 0
        G = sr.gram_exact(psi, n, qs, 0)
        assert np.array_equal(np.sort(np.linalg.eigvalsh(G))[::-1][: 1 << m], np.ones(1 << m))


@pytest.mark.parametrize("n", [3, 8])
def test_ghz_is_two_halves(n):
    psi = np.zeros(1 << n, dtype=np.complex128)
    psi[0] = psi[-1] = 1 / math.sqrt(2)
    for qs in ([0], [n - 1, 0], list(range(1, n))):
        lam, T = sr.schmidt_ref(psi, n, qs)
        assert np.allclose(lam[:2], 0.5, atol=1e-15) and np.all(np.abs(lam[2:]) <= 1e-15), qs
        assert abs(sr.entropy(lam[:2], T) - math.log(2)) <= 1e-15


@pytest.mark.parametrize("n,side", [(6, [0, 1, 2]), (9, [8, 2, 5, 0]), (10, [1, 3, 5, 7, 9]), (12, [11, 4])])
def test_schmidt_form_states(n, side):
    d = 1 << len(side)
    for lam in (sr.geometric_spectrum(d, 0.6), sr.geometric_spectrum(d - 1, 0.9), np.array([0.7, 0.3])):
        psi = sr.schmidt_state(n, side, lam, 100 + n)
        got, T = sr.schmidt_ref(psi, n, side)
        want = np.zeros(d)
        want[: lam.size] = lam
        b = sr.svd_ref_bound(n, len(side), 1.0) + 1e-15
        assert abs(T - 1.0) <= 1e-13
        assert np.max(np.abs(got - want)) <= b, (n, side, np.max(np.abs(got - want)), b)
        # the complement sees the same nonzero values
        rest = [q for q in range(n) if q not in side]
        got_b, _ = sr.schmidt_ref(psi, n, rest) if len(rest) <= len(side) else (None, None)
        if got_b is not None:
            assert np.max(np.abs(got_b[: lam.size] - lam)) <= sr.svd_ref_bound(n, len(rest), 1.0) + 1e-15
        S = -float(np.sum(lam * np.log(lam)))
        assert abs(sr.entropy(got, T) - S) <= sr.entropy_bound(len(side), T, b, 1e-13, S)


@pytest.mark.parametrize("n,qs", [(6, [0, 2]), (9, [8, 1, 4]), (11, [0, 1, 2, 3, 4, 5])])
def test_sum_of_squares_is_purity(n, qs):
    rng = np.random.default_rng(n)
    psi = (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.2
    lam, T = sr.schmidt_ref(psi, n, qs)
    P, t, bp, bt, _, _ = pu.purity_ref(psi, n, qs)
    s = min(len(qs), n - len(qs))
    e = sr.svd_ref_bound(n, s, float(lam[0]))
    assert abs(float(np.sum(lam ** 2)) - P) <= sr.sum_sq_bound(s, T, e) + bp
    assert abs(T - t) <= 1e-13 * T


def test_gram_exact_matches_reduced_density_reference():
    n = 9
    rng = np.random.default_rng(5)
    psi = (rng.choice([-1.0, 0.0, 1.0], size=1 << n) + 1j * rng.choice([-1.0, 1.0], size=1 << n)) * 2.0 ** -5
    for qs in ([0, 4], [8, 1, 3], [2, 6, 5, 7]):
        G = sr.gram_exact(psi, n, qs, 5)
        assert np.array_equal(G, rr.rdm_ref(psi, n, qs).astype(np.complex128)), qs


def test_bounds_are_monotone_and_finite():
    for n, s in ((12, 6), (24, 12), (26, 13), (30, 13), (31, 13)):
        e = sr.eig_bound(n, s, 1.0, 1.0)
        assert 0 < e < 1e-6, (n, s, e)
        assert sr.entropy_bound(s, 1.0, e, sr.trace_bound(n, s, 1.0), 5.0) < 1e-2
    assert sr.gram_error_frobenius(30, 13, 2.0) == 2 * sr.gram_error_frobenius(30, 13, 1.0)
    assert sr.binary_entropy(0.0) == 0.0 and sr.binary_entropy(0.5) == math.log(2)


# ---- the plan -------------------------------------------------------------------------------------------------------

def test_plan_every_route_and_side():
    for n in (1, 2, 5, 12, 20, 26, 30, 31, 40):
        for k in range(1, n + 1):
            s = min(k, n - k)
            if s > sr.MAX_SIDE:
                continue
            for qs in (list(range(k)), list(range(n - k, n))[::-1]):
                for dtype in (C128, C64):
                    got = entanglement_spectrum_plan(n, dtype, qs)
                    assert got == sr.plan(n, qs), (n, qs, got)
    # the kernel counts by route, spelled out
    assert entanglement_spectrum_plan(8, C128, list(range(8))) == (0, 0, 1, 0, 1)
    assert entanglement_spectrum_plan(20, C128, [3]) == (1, 1, 2, 64, 1)
    assert entanglement_spectrum_plan(20, C128, list(range(7))) == (1, 7, 6, 16 * 4 ** 7, 1)
    assert entanglement_spectrum_plan(20, C128, list(range(10))) == (1, 10, 16 * 17, 16 << 20, 1)
    assert entanglement_spectrum_plan(30, C128, list(range(11))) == (2, 11, 1, 16 << 22, 1)
    assert entanglement_spectrum_plan(30, C64, list(range(17))) == (2, 13, 1, 1 << 30, 1)


def test_solver_loads_here():
    assert entanglement_spectrum_plan(4, C128, [0])[4] == 1


def test_plan_refusals():
    lib = _lib.lib()
    v = (np.zeros(5, dtype=np.uint32))
    qs = np.array([0, 1], dtype=np.uint64)
    for prec, n, out, code in ((0, 4, v.ctypes.data, 0), (5, 4, v.ctypes.data, INVALID_ARG), (0, 0, v.ctypes.data, INVALID_ARG),
                               (0, 41, v.ctypes.data, INVALID_ARG), (0, 4, None, INVALID_ARG)):
        assert lib.qipb200_entanglement_spectrum_plan(prec, n, qs.ctypes.data, 2, out) == code, (prec, n, out)
        if code:
            assert "entanglement_spectrum_plan: NULL out5, bad precision or n_qubits not in 1..40" in \
                lib.qipb200_last_error(None).decode()
    cases = (([], INVALID_ARG, "bad qubit list"), (list(range(9)), INVALID_ARG, "bad qubit list"),
             ([0, 8], BAD_INDEX, "qubit index out of range"), ([3, 1, 3], BAD_INDEX, "repeated qubit index"))
    for bad, code, msg in cases:
        with pytest.raises(CircuitError) as e:
            entanglement_spectrum_plan(8, C128, bad)
        assert e.value.status == code and "entanglement_spectrum_plan: " + msg in str(e.value), bad
    assert lib.qipb200_entanglement_spectrum_plan(0, 4, None, 1, v.ctypes.data) == INVALID_ARG
    for n, k in ((28, 14), (30, 15), (40, 20), (30, 16)):
        with pytest.raises(CircuitError) as e:
            entanglement_spectrum_plan(n, C128, list(range(k)))
        assert e.value.status == UNSUPPORTED, (n, k)
        assert "has %d qubits; at most 13 are supported (the matrix of 14 would be 4 GiB or more)" % min(k, n - k) \
            in str(e.value)


def test_null_state_refusal():
    lib = _lib.lib()
    qs = np.array([0], dtype=np.uint64)
    eigs, out2 = np.zeros(2), np.zeros(2)
    st = lib.qipb200_state_entanglement_spectrum(None, qs.ctypes.data, 1, eigs.ctypes.data, 2, None, out2.ctypes.data)
    assert st == INVALID_ARG
    assert lib.qipb200_last_error(None).decode() == "entanglement_spectrum: NULL state"
