"""Transition elements <bra|P|ket> without a GPU: the sweep and kernel counts (qipb200_transition_plan), the validation
the C entries share with expect_paulis, the long-double reference of tests/transition_ref.py pinned against explicit
Kronecker products, and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import pauli_ref as pr
import transition_ref as tr
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import _marshal_paulis, _ptr, expect_plan, transition_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3


def tfim(n):
    return [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]


def z_strings(n, count, seed):
    rng = np.random.default_rng(seed)
    return [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.5)] for _ in range(count)]


def one_mask(count):
    """count terms with X on qubits 0 and 29 and a distinct Z pattern on qubits 1..28 each."""
    return [[("X", 0), ("X", 29)] + [("Z", 1 + k) for k in range(28) if (i >> k) & 1] for i in range(count)]


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_diagonal_terms_take_one_sweep(dtype):
    terms = [[("Z", i)] for i in range(30)] + [[("Z", i), ("Z", j)] for i, j in itertools.combinations(range(30), 2)]
    assert len(terms) == 465
    assert transition_plan(30, dtype, terms) == (1, 2)
    assert transition_plan(30, dtype, z_strings(30, 4000, 1)) == (1, 2)
    assert transition_plan(30, dtype, []) == (0, 0)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_overlap_alone(dtype):
    for n in (1, 11, 12, 30, 40):
        assert transition_plan(n, dtype, [[]]) == (1, 2)  # one sweep and its reduction


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_equal_masks_share_one_sweep(dtype):
    terms = []
    for a, b in itertools.product("XY", "XY"):
        for zs in range(256):
            terms.append([(a, 0), (b, 29)] + [("Z", 5 + k) for k in range(8) if (zs >> k) & 1])
    assert transition_plan(30, dtype, terms) == (1, 2)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_two_rows_per_term_halve_the_batch(dtype):
    # a sweep and a reduction batch carry 16384 rows: 8192 terms of two rows each
    assert transition_plan(30, dtype, z_strings(30, 8192, 2)) == (1, 2)
    assert transition_plan(30, dtype, z_strings(30, 8193, 3)) == (2, 4)
    assert expect_plan(30, dtype, z_strings(30, 8193, 3)) == 1
    assert transition_plan(30, dtype, one_mask(8192)) == (1, 2)
    assert transition_plan(30, dtype, one_mask(8193)) == (2, 4)
    # Z-only terms fill the room the other sweeps leave: 8000 + 192 terms fit one sweep, 8000 + 200 do not
    assert transition_plan(30, dtype, one_mask(8000) + z_strings(30, 192, 4)) == (1, 2)
    assert transition_plan(30, dtype, one_mask(8000) + z_strings(30, 200, 5)) == (2, 4)
    # several sweeps whose rows fit one batch share its reduction kernel
    assert transition_plan(30, dtype, tfim(30) + z_strings(30, 2000, 6)) == (4, 5)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_transverse_field_ising(dtype):
    # the masks of expect_plan's count (4 + 7 + 7 + 7 + 5 single-bit masks in 4 sweeps), one reduction
    assert transition_plan(30, dtype, tfim(30)) == (4, 5)
    assert transition_plan(30, dtype, tfim(30))[0] == expect_plan(30, dtype, tfim(30))
    assert transition_plan(11, dtype, tfim(11)) == (1, 2)
    assert transition_plan(12, dtype, tfim(12)) == (2, 3)
    assert transition_plan(30, dtype, [[("X", q) for q in range(30)]]) == (1, 2)


def _plan_raw(n, qubits, letters, lens, n_terms=None, prec=1, out=True):
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    la = C.create_string_buffer(bytes(letters), max(1, len(letters)))
    ln = (C.c_uint32 * max(1, len(lens)))(*lens)
    v = (C.c_uint32 * 2)(99, 99)
    st = _lib.lib().qipb200_transition_plan(prec, n, qa, la, ln, len(lens) if n_terms is None else n_terms,
                                            v if out else None)
    return st, _lib.lib().qipb200_last_error(None).decode(), tuple(v)


def test_plan_validation_errors():
    st, msg, _ = _plan_raw(4, [0], b"W", [1])
    assert st == INVALID_ARG and "not 'X', 'Y' or 'Z'" in msg and "term 0" in msg
    st, msg, _ = _plan_raw(4, [0, 1], b"Zx", [1, 1])
    assert st == INVALID_ARG and "term 1" in msg
    st, msg, _ = _plan_raw(4, [4], b"X", [1])
    assert st == BAD_INDEX and "qubit 4 out of range for 4 qubits" in msg
    st, msg, _ = _plan_raw(4, [0, 2, 2], b"XYZ", [3])
    assert st == BAD_INDEX and "qubit 2 repeated" in msg
    st, _, v = _plan_raw(4, [2, 2], b"XZ", [1, 1])
    assert st == 0 and v == (1, 2)
    for which in range(3):
        args = [(C.c_uint64 * 1)(0), C.create_string_buffer(b"X", 1), (C.c_uint32 * 1)(1)]
        args[which] = None
        v = (C.c_uint32 * 2)(7, 7)
        assert _lib.lib().qipb200_transition_plan(1, 4, *args, 1, v) == INVALID_ARG
        assert "NULL" in _lib.lib().qipb200_last_error(None).decode()
        assert _lib.lib().qipb200_transition_plan(1, 4, *args, 0, v) == 0 and tuple(v) == (0, 0)
    st, msg, _ = _plan_raw(4, [0], b"X", [1], out=False)
    assert st == INVALID_ARG and "NULL out2" in msg
    for n, prec in ((0, 1), (41, 1), (4, 7), (4, -1)):
        st, msg, _ = _plan_raw(n, [0], b"X", [1], prec=prec)
        assert st == INVALID_ARG and "transition_plan" in msg, (n, prec)
    with pytest.raises(CircuitError) as e:
        transition_plan(3, C128, [[("X", 0)], [("Q", 1)]])
    assert e.value.status == INVALID_ARG


def test_null_states_are_refused_without_a_device():
    qs, ls, lens = _marshal_paulis([[("X", 0)]])
    out = np.zeros(2)
    L = _lib.lib()
    assert L.qipb200_state_transition_paulis(None, None, _ptr(qs), ls, _ptr(lens), 1, _ptr(out)) == INVALID_ARG
    assert "transition_paulis: NULL state" in L.qipb200_last_error(None).decode()


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


def every_term(n, rng):
    """Every Pauli string for n <= 3; otherwise every single letter, every letter pair on two qubits, all-X/Y/Z and
    random strings of every weight."""
    if n <= 3:
        return [[(l, q) for q, l in enumerate(ls) if l != "I"] for ls in itertools.product("IXYZ", repeat=n)]
    terms = [[]] + [[(l, q)] for q in range(n) for l in "XYZ"]
    terms += [[(a, 0), (b, n - 1)] for a, b in itertools.product("XYZ", "XYZ")]
    terms += [[(l, q) for q in range(n)] for l in "XYZ"]
    for _ in range(12):
        qs = rng.choice(n, size=int(rng.integers(1, n + 1)), replace=False)
        terms.append([(str(rng.choice(list("XYZ"))), int(q)) for q in qs])
    return terms


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_reference_helper_matches_kronecker_products(n):
    rng = np.random.default_rng(60 + n)
    bra = (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.7
    ket = (rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.4
    scale = np.linalg.norm(bra) * np.linalg.norm(ket)
    for t in every_term(n, rng):
        want = np.vdot(bra, kron_matrix(n, t) @ ket)
        got = complex(tr.transition_ref(bra, ket, n, t))
        assert abs(got - want) <= 1e-12 * scale, (t, got, want)
        S = tr.abs_weight(bra, ket, n, t)
        assert S >= abs(want) - 1e-12 * scale
        # <bra|P|ket> = conj(<ket|P|bra>) (P is Hermitian)
        swapped = complex(tr.transition_ref(ket, bra, n, t))
        assert abs(swapped.conjugate() - got) <= 1e-12 * scale
        # bra == ket: the real part is expect_ref's value exactly, the imaginary part is 0 up to rounding
        same = tr.transition_ref(bra, bra, n, t)
        assert same.real == pr.expect_ref(bra, n, t), t
        assert abs(float(same.imag)) <= 1e-12 * np.sum(np.abs(bra) ** 2)


def test_cpp_mirror_transition_compiles(tmp_path):
    src = tmp_path / "use_transition.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &bra, qip::B200State<double> &ket) {\n"
                   "  std::vector<std::complex<double>> v = bra.transition_paulis(ket, {{{'Z', 0}, {'Z', 1}}, {{'X', 2}}, {}});\n"
                   "  std::complex<double> o = bra.overlap(ket);\n"
                   "  std::vector<std::complex<double>> none = bra.transition_paulis(bra, {});\n"
                   "  (void)v;\n"
                   "  (void)o;\n"
                   "  (void)none;\n"
                   "}\n"
                   "void run32(qip::B200State<float> &bra, qip::B200State<float> &ket) { (void)bra.overlap(ket); }\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
