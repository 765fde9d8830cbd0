"""Pauli-string expectation values without a GPU: the sweep plan (qipb200_expect_plan), the validation both C entries
share, and the long-double reference helper of tests/pauli_ref.py pinned against explicit Kronecker products."""
import ctypes as C
import itertools

import numpy as np
import pytest

import pauli_ref as pr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import expect_plan

C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3


def tfim(n):
    return [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_diagonal_terms_take_one_sweep(dtype):
    terms = [[("Z", i)] for i in range(30)] + [[("Z", i), ("Z", j)] for i, j in itertools.combinations(range(30), 2)]
    assert len(terms) == 465
    assert expect_plan(30, dtype, terms) == 1
    assert expect_plan(30, dtype, [[]]) == 1  # the identity
    assert expect_plan(30, dtype, []) == 0


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_equal_masks_share_one_sweep(dtype):
    # X/Y letters on qubits 0 and 29 (one X/Y mask), Z on every subset of 8 other qubits: 4 * 256 = 2^10 terms
    terms = []
    for a, b in itertools.product("XY", "XY"):
        for zs in range(256):
            terms.append([(a, 0), (b, 29)] + [("Z", 5 + k) for k in range(8) if (zs >> k) & 1])
    assert len(terms) == 1 << 10
    assert expect_plan(30, dtype, terms) == 1


def z_strings(n, count, seed):
    rng = np.random.default_rng(seed)
    return [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.5)] for _ in range(count)]


def one_mask(count):
    """count terms with X on qubits 0 and 29 and a distinct Z pattern on qubits 1..28 each."""
    return [[("X", 0), ("X", 29)] + [("Z", 1 + k) for k in range(28) if (i >> k) & 1] for i in range(count)]


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_many_terms_per_sweep(dtype):
    # a sweep carries up to 16384 terms (one reduction batch), however they split into groups
    for count in (1025, 4096, 16384):
        assert expect_plan(30, dtype, z_strings(30, count, count)) == 1
    assert expect_plan(30, dtype, z_strings(30, 16385, 1)) == 2
    assert expect_plan(30, dtype, one_mask(2048)) == 1
    assert expect_plan(30, dtype, one_mask(16384)) == 1
    assert expect_plan(30, dtype, one_mask(16385)) == 2
    # Z-only terms fill the room the other sweeps leave before opening one of their own
    assert expect_plan(30, dtype, one_mask(16000) + z_strings(30, 384, 2)) == 1
    assert expect_plan(30, dtype, one_mask(16000) + z_strings(30, 385, 3)) == 2
    assert expect_plan(30, dtype, tfim(30) + z_strings(30, 4096, 4)) == 4
    # more distinct masks in one tile than the kernel stages in shared memory (256)
    masks = [[("X", 30 - 1 - b) for b in range(11) if (r >> b) & 1] for r in range(1, 600)]
    assert expect_plan(30, dtype, masks) == 1


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_transverse_field_ising(dtype):
    # A tile is the 4 low index bits plus 7 chosen high bits.  The first sweep holds X_i on the 4 low bits and 7 high
    # bits, every later one 7 more: 4 + 7 + 7 + 7 + 5 = 30 single-bit masks in 4 sweeps; the Z_iZ_i+1 ride along.
    assert expect_plan(30, dtype, tfim(30)) == 4
    assert expect_plan(30, dtype, tfim(30)[:30]) == 4
    assert expect_plan(11, dtype, tfim(11)) == 1  # the whole state is one tile
    assert expect_plan(12, dtype, tfim(12)) == 2


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_all_x_and_pair_masks(dtype):
    assert expect_plan(30, dtype, [[("X", q) for q in range(30)]]) == 1
    assert expect_plan(32, dtype, [[("Y" if q % 3 else "X", q) for q in range(32)]]) == 1
    # masks differing in many high bits cannot share a tile: one sweep each
    terms = [[("X", 0), ("X", 1)], [("X", 2), ("X", 3), ("X", 4), ("X", 5), ("X", 6), ("X", 7), ("X", 8), ("X", 9)]]
    assert expect_plan(30, dtype, terms) == 2
    assert expect_plan(30, dtype, terms + [[("Z", 3)]]) == 2


def _plan_raw(n, qubits, letters, lens, n_terms=None, prec=1):
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    la = C.create_string_buffer(bytes(letters), max(1, len(letters)))
    ln = (C.c_uint32 * max(1, len(lens)))(*lens)
    v = C.c_uint32(99)
    st = _lib.lib().qipb200_expect_plan(prec, n, qa, la, ln, len(lens) if n_terms is None else n_terms, C.byref(v))
    return st, _lib.lib().qipb200_last_error(None).decode(), v.value


def test_plan_validation_errors():
    st, msg, _ = _plan_raw(4, [0], b"W", [1])
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg and "term 0" in msg
    st, msg, _ = _plan_raw(4, [0, 1], b"Zx", [1, 1])
    assert st == INVALID_ARG and "term 1" in msg
    st, msg, _ = _plan_raw(4, [4], b"X", [1])
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg, _ = _plan_raw(4, [0, 2, 2], b"XYZ", [3])
    assert st == BAD_INDEX and "qubit 2 repeated" in msg
    # the same qubit in two different terms is fine
    st, _, v = _plan_raw(4, [2, 2], b"XZ", [1, 1])
    assert st == 0 and v == 1
    for which in range(3):
        args = [(C.c_uint64 * 1)(0), C.create_string_buffer(b"X", 1), (C.c_uint32 * 1)(1)]
        args[which] = None
        v = C.c_uint32()
        assert _lib.lib().qipb200_expect_plan(1, 4, *args, 1, C.byref(v)) == INVALID_ARG
        assert "NULL" in _lib.lib().qipb200_last_error(None).decode()
        # n_terms == 0: a no-op whatever the arrays
        assert _lib.lib().qipb200_expect_plan(1, 4, *args, 0, C.byref(v)) == 0 and v.value == 0
    st, _, _ = _plan_raw(4, [0], b"X", [1], prec=7)
    assert st == INVALID_ARG
    with pytest.raises(CircuitError) as e:
        expect_plan(3, C128, [[("X", 0)], [("Q", 1)]])
    assert e.value.status == INVALID_ARG


# ---- the reference helper against explicit matrices --------------------------------------------------------------

PAULI = {"I": np.eye(2), "X": np.array([[0, 1], [1, 0]], dtype=complex),
         "Y": np.array([[0, -1j], [1j, 0]]), "Z": np.diag([1.0, -1.0]).astype(complex)}


def kron_matrix(n, term):
    letters = ["I"] * n
    for letter, q in term:
        letters[q] = letter
    m = np.array([[1.0 + 0j]])
    for q in range(n):  # qubit 0 is the most significant index bit
        m = np.kron(m, PAULI[letters[q]])
    return m


@pytest.mark.parametrize("n", [1, 2, 5, 8, 10])
def test_reference_helper_matches_kronecker_products(n):
    rng = np.random.default_rng(40 + n)
    psi = (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.7
    terms = [[]] + [[(l, q)] for q in range(n) for l in "XYZ"]
    for _ in range(12):
        k = int(rng.integers(1, n + 1))
        qs = rng.choice(n, size=k, replace=False)
        terms.append([(str(rng.choice(list("XYZ"))), int(q)) for q in qs])
    terms.append([("Y", q) for q in range(n)])
    for t in terms:
        want = np.vdot(psi, kron_matrix(n, t) @ psi)
        assert abs(want.imag) < 1e-9 * max(1.0, abs(want))
        got = float(pr.expect_ref(psi, n, t))
        assert abs(got - want.real) <= 1e-12 * np.sum(np.abs(psi) ** 2), (t, got, want)
        S = pr.abs_weight(psi, n, t)
        assert S >= abs(want) - 1e-12
