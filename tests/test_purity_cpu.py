"""Purity of a bipartition without a GPU: the references of tests/purity_ref.py pinned against closed forms, against
sum |rdm_ref|^2 and against the symmetry between a side and its complement; the bound's sensitivity; the plan
(qipb200_purity_plan) and every validation code; the NULL-state refusal of qipb200_state_purity."""
import ctypes as C

import numpy as np
import pytest

import purity_ref as pu
import rdm_ref as rr
from exact_circuits import exact_state
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import purity_plan

C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3
PRODUCT_V = [(1, 0.5), (0.5, 1j), (0.5j, 0.5), (-0.5, 1), (1, -0.25j), (0.25, -1)]


def random_psi(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.3


@pytest.mark.parametrize("n", [4, 7])
def test_product_state_closed_form(n):
    vs = [PRODUCT_V[q % 6] for q in range(n)]
    psi = rr.product_state(n, vs)
    norms = [sum(abs(complex(x)) ** 2 for x in v) for v in vs]
    T = np.prod(norms)
    for qs in ([0], [n - 1, 1], list(range(n // 2)), list(range(n))):
        P, t = pu.purity_ld(psi, n, qs)
        assert abs(float(t) - T) <= 1e-14 * T
        assert abs(float(P) - T ** 2) <= 1e-13 * T ** 2, qs


@pytest.mark.parametrize("n", [3, 8])
def test_ghz_is_one_half(n):
    psi = np.zeros(1 << n, dtype=np.complex128)
    psi[0], psi[-1] = 1.0, 1.0
    for qs in ([0], [n - 1, 0], list(range(1, n))):
        P, T = pu.purity_ld(psi, n, qs)
        assert P / T ** 2 == 0.5, qs


@pytest.mark.parametrize("m", [1, 2, 4])
def test_bell_pairs_across_the_cut(m):
    n = 2 * m + 2
    j = np.arange(1 << n)
    ok = np.ones(1 << n, dtype=bool)
    for i in range(m):  # qubit i with qubit m + 1 + i; qubits m and n - 1 in |0>
        ok &= ((j >> (n - 1 - i)) & 1) == ((j >> (n - 1 - (m + 1 + i))) & 1)
    ok &= ((j >> (n - 1 - m)) & 1) == 0
    ok &= (j & 1) == 0
    psi = ok.astype(np.complex128)
    P, T = pu.purity_ld(psi, n, list(range(m + 1)))
    assert P / T ** 2 == 2.0 ** -m
    assert pu.purity_int(psi, n, list(range(m + 1))) == (2 ** m, 2 ** m)


@pytest.mark.parametrize("n", [5, 9])
def test_reference_is_the_frobenius_norm_of_rdm_ref(n):
    psi = random_psi(n, 40 + n)
    for qs in ([0], [n - 1, 2], [1, 3, 0], list(range(n // 2))):
        rho = rr.rdm_ref(psi, n, qs)
        want = np.sum(np.abs(rho) ** 2)
        P, T = pu.purity_ld(psi, n, qs)
        assert abs(P - want) <= 1e-15 * want, qs
        P2, T2, b, bt, _, _ = pu.purity_ref(psi, n, qs)
        assert abs(P2 - float(want)) <= b and abs(T2 - float(T)) <= bt + 1e-15


@pytest.mark.parametrize("n", [6, 9])
def test_side_and_complement_agree(n):
    psi = random_psi(n, 60 + n)
    rng = np.random.default_rng(n)
    for k in range(1, n):
        qs = [int(q) for q in rng.permutation(n)[:k]]
        comp = [q for q in range(n) if q not in qs]
        a = rr.rdm_ref(psi, n, qs)
        b = rr.rdm_ref(psi, n, comp)
        pa, pb = np.sum(np.abs(a) ** 2), np.sum(np.abs(b) ** 2)
        assert abs(pa - pb) <= 1e-14 * pa, (qs, pa, pb)
        assert abs(pu.purity_ld(psi, n, qs)[0] - pa) <= 1e-14 * pa


def test_integer_reference_is_exact():
    n = 12
    psi = exact_state(n, 5, 6)
    for qs in ([0, 1, 2], list(range(6)), [11, 3, 7, 0, 5]):
        P, T = pu.purity_int(psi, n, qs)
        Pl, Tl = pu.purity_ld(psi, n, qs)
        assert P == int(Pl) and T == int(Tl), qs


def test_bound_accepts_another_order_and_rejects_a_perturbation():
    n, qs = 14, list(range(7))
    psi = random_psi(n, 99)
    P, T = pu.purity_ld(psi, n, qs)
    M = pu.side_matrix(psi, n, qs, np.complex128)
    G = M @ np.conj(M.T)  # another summation order
    W = np.abs(M) @ np.abs(M).T
    b, _ = pu.device_bound(n, 7, G, W, float(P), float(T))
    other = float(np.sum(np.abs(G) ** 2))
    assert abs(other - P) <= b
    assert abs(other * (1 + 1e-12) - P) > b
    assert pu.bound_cs(n, 7, float(P), float(T))[0] >= b
    assert pu.gram_depths(30, 15) == (2 * 2 ** 15, 64 + 8 + 257 + 8)


def test_plan_routes_and_counts():
    n = 30
    cases = {
        "prefix s=11": list(range(11)),
        "suffix s=15": list(range(15, 30)),
        "scattered s=13": list(range(0, 26, 2)),
        "complement larger s=12": list(range(12, 30)),
        "k = n": list(range(30)),
        "s=1": [29],
        "s=10": list(range(10)),
        "complement s=6": list(range(24)),
    }
    for name, qs in cases.items():
        got = purity_plan(n, C128, qs)
        assert got == pu.plan(n, qs), name
        assert purity_plan(n, C64, qs) == got
    assert purity_plan(n, C128, list(range(30))) == (0, 0, 1, 0)
    assert purity_plan(n, C128, [5]) == (1, 1, 2, 0)
    assert purity_plan(n, C128, list(range(7))) == (1, 7, 6, 0)
    assert purity_plan(n, C128, list(range(10))) == (1, 10, 272, 0)
    assert purity_plan(n, C128, list(range(11))) == (2, 11, 2, 272)
    assert purity_plan(n, C128, list(range(15))) == (2, 15, 2, 256 * 257)
    assert purity_plan(32, C64, list(range(16))) == (2, 16, 2, 512 * 513)
    assert purity_plan(n, C128, list(range(1, 30))) == (1, 1, 2, 0)


def test_plan_validation():
    lib = _lib.lib()
    out = (C.c_uint32 * 4)()
    qs = (C.c_uint64 * 3)(0, 1, 2)
    assert lib.qipb200_purity_plan(1, 10, qs, 3, None) == INVALID_ARG
    assert lib.qipb200_purity_plan(7, 10, qs, 3, out) == INVALID_ARG  # precision
    assert lib.qipb200_purity_plan(1, 0, qs, 3, out) == INVALID_ARG
    assert lib.qipb200_purity_plan(1, 41, qs, 3, out) == INVALID_ARG
    assert lib.qipb200_purity_plan(1, 10, None, 3, out) == INVALID_ARG
    assert lib.qipb200_purity_plan(1, 10, qs, 0, out) == INVALID_ARG
    assert lib.qipb200_purity_plan(1, 2, qs, 3, out) == INVALID_ARG  # k > n
    for bad, word in (([0, 10], "out of range"), ([4, 1, 4], "repeated")):
        with pytest.raises(CircuitError) as e:
            purity_plan(10, C128, bad)
        assert e.value.status == BAD_INDEX and word in str(e.value)


def test_null_state_is_refused():
    out = (C.c_double * 2)()
    qs = (C.c_uint64 * 1)(0)
    assert _lib.lib().qipb200_state_purity(None, qs, 1, out) == INVALID_ARG
    assert "purity" in _lib.lib().qipb200_last_error(None).decode()
