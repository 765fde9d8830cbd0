"""Pauli-string rotations without a GPU: the emulator and the long-double reference of tests/pauli_rot_ref.py pinned to
scipy.linalg.expm of explicit Kronecker products and to the oracle run of the MatrixOp decomposition; the sweep plan
(qipb200_pauli_rotation_plan); the validation both C entries share; the NULL-state refusal and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg

import pauli_rot_ref as rr
from oracle import qip_oracle as qo
from rustqip_b200 import _lib, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import pauli_rotation_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3

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


def random_psi(n, seed, dtype=C128):
    rng = np.random.default_rng(seed)
    return ((rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)) * 0.4).astype(dtype)


def letter_mix_terms(n):
    """Every letter on every qubit, every letter mix on up to three qubits, all-X, all-Y, all-Z and the identity."""
    terms = [[], [("X", q) for q in range(n)], [("Y", q) for q in range(n)], [("Z", q) for q in range(n)]]
    terms += [[(l, q)] for q in range(n) for l in "XYZ"]
    for k in (2, 3):
        for qs in list(itertools.combinations(range(n), k))[:6]:
            terms += [list(zip(ls, qs)) for ls in itertools.product("XYZ", repeat=k)]
    return terms


@pytest.mark.parametrize("n", [1, 2, 3, 4, 6])
def test_references_match_expm_of_kronecker_products(n):
    terms = letter_mix_terms(n)
    rng = np.random.default_rng(500 + n)
    angles = rng.uniform(-7, 7, size=len(terms))
    psi = random_psi(n, n)
    want = psi.astype(C128)
    for t, th in zip(terms, angles):
        want = scipy.linalg.expm(-0.5j * th * kron_matrix(n, t)) @ want
        one = scipy.linalg.expm(-0.5j * th * kron_matrix(n, t)) @ psi.astype(C128)
        assert np.max(np.abs(rr.rotate_ref(psi, n, [t], [th]).astype(C128) - one)) <= 1e-13, t
        assert np.max(np.abs(rr.emulate(psi, n, [t], [th], C128) - one)) <= 1e-13, t
    norm = float(np.linalg.norm(psi))
    assert np.max(np.abs(rr.rotate_ref(psi, n, terms, angles).astype(C128) - want)) <= 1e-11 * norm
    assert np.max(np.abs(rr.emulate(psi, n, terms, angles, C128) - want)) <= 1e-11 * norm
    assert np.max(np.abs(rr.emulate(psi.astype(C64), n, terms, angles, C64) - want)) <= 2e-4 * norm


@pytest.mark.parametrize("dtype", [C128, C64])
def test_emulator_within_bound_of_long_double_reference(dtype):
    n = 10
    rng = np.random.default_rng(3)
    terms = letter_mix_terms(n) + rr.ucc_strings(n, 40, 9)
    angles = rng.uniform(-4, 4, size=len(terms))
    psi = random_psi(n, 8, dtype)
    ref = rr.rotate_ref(psi, n, terms, angles)
    got = rr.emulate(psi, n, terms, angles, dtype)
    b = rr.bound(len(terms), float(np.linalg.norm(psi.astype(C128))), dtype)
    err = float(np.max(np.abs(got.astype(np.clongdouble) - ref)))
    assert err <= b, (err, b)
    # one letter changed (X_0 -> Y_0) is far outside it
    bad = list(terms)
    assert bad[4] == [("X", 0)]
    bad[4] = [("Y", 0)]
    assert float(np.max(np.abs(rr.emulate(psi, n, bad, angles, dtype).astype(np.clongdouble) - ref))) > 100 * b


@pytest.mark.parametrize("n", [4, 5])
def test_references_match_oracle_run_of_decomposition(n):
    terms = letter_mix_terms(n) + rr.ucc_strings(n, 6, 1)
    rng = np.random.default_rng(60 + n)
    angles = rng.uniform(-5, 5, size=len(terms))
    psi = random_psi(n, 70 + n)
    want = qo.run_pipeline(n, rr.decompose_all(terms, angles), state=psi, dtype=C128)
    norm = float(np.linalg.norm(psi))
    assert np.max(np.abs(rr.emulate(psi, n, terms, angles, C128) - want)) <= 1e-11 * norm
    assert np.max(np.abs(rr.rotate_ref(psi, n, terms, angles).astype(C128) - want)) <= 1e-11 * norm


def test_single_z_term_is_rz():
    n = 4
    psi = random_psi(n, 4)
    for q in range(n):
        for th in (0.3, -2.0, 3.7):
            want = qo.run_pipeline(n, [gates.rz(q, th)], state=psi, dtype=C128)
            assert np.max(np.abs(rr.emulate(psi, n, [[("Z", q)]], [th], C128) - want)) <= 1e-15


# ---- the sweep plan ------------------------------------------------------------------------------------------------

def check_plan(n, dtype, terms, want):
    assert rr.plan_policy(n, terms) == want
    assert pauli_rotation_plan(n, dtype, terms) == want


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_invariants(dtype):
    rng = np.random.default_rng(12)
    # only diagonal terms, any length: one sweep
    diag = [[("Z", int(q)) for q in np.flatnonzero(rng.random(30) < 0.5)] for _ in range(5000)] + [[]] * 10
    check_plan(30, dtype, diag, 1)
    check_plan(30, dtype, [[]], 1)
    check_plan(30, dtype, [], 0)
    # any single term
    for term in ([("X", q) for q in range(30)], [("Y", q) for q in range(32)], [("X", 0), ("Y", 31)], [("Z", 3)]):
        n = max(q for _, q in term) + 1
        check_plan(n, dtype, [term], 1)
    # X/Y letters on the 4 low bits (qubits n-4..n-1) plus 7 others: one sweep however many terms
    others = [0, 3, 7, 11, 15, 20, 24]
    support = others + [26, 27, 28, 29]
    run = [[(str(rng.choice(list("XY"))), int(q)) for q in rng.choice(support, size=int(rng.integers(1, 6)),
                                                                          replace=False)] for _ in range(300)]
    check_plan(30, dtype, run + diag[:50], 1)
    # at most max(1, non-diagonal terms)
    for seed in range(5):
        r = np.random.default_rng(seed)
        terms = [[(str(r.choice(list("XYZ"))), int(q)) for q in r.choice(30, size=int(r.integers(0, 5)),
                                                                          replace=False)] for _ in range(80)]
        nd = sum(1 for t in terms if any(l != "Z" for l, _ in t))
        assert pauli_rotation_plan(30, dtype, terms) == rr.plan_policy(30, terms) <= max(1, nd)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_plan_counts_of_the_documented_policy(dtype):
    # Ising step: the 30 Z_iZ_i+1 ride in the first sweep; X_0..X_6 fill the 7 high tile bits, X_7 becomes its
    # out-of-tile mask, X_8 opens the next sweep: 8 X_i per sweep, and X_24, X_25 plus the 4 low bits in the fourth
    check_plan(30, dtype, rr.ising_step(30), 4)
    check_plan(30, dtype, rr.z_pairs(30), 1)
    assert len(rr.z_pairs(30)) == 465
    check_plan(30, dtype, [[("X", q) for q in range(30)]], 1)
    check_plan(30, dtype, rr.ucc_strings(30, 64, 64), 22)
    check_plan(30, dtype, [[("X", 3)]] * 1000, 1)
    check_plan(30, dtype, rr.qaoa_layer(30), 4)
    check_plan(11, dtype, rr.ising_step(11) + rr.ucc_strings(11, 20, 2), 1)  # the whole state is one tile


def _plan_raw(n, qubits, letters, lens, n_terms=None, prec=1):
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    la = C.create_string_buffer(bytes(letters), max(1, len(letters)))
    ln = (C.c_uint32 * max(1, len(lens)))(*lens)
    v = C.c_uint32(99)
    st = _lib.lib().qipb200_pauli_rotation_plan(prec, n, qa, la, ln, len(lens) if n_terms is None else n_terms,
                                                C.byref(v))
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
    st, _, v = _plan_raw(4, [2, 2], b"XZ", [1, 1])
    assert st == 0 and v == 1
    for which in range(3):
        args = [(C.c_uint64 * 1)(0), C.create_string_buffer(b"X", 1), (C.c_uint32 * 1)(1)]
        args[which] = None
        v = C.c_uint32()
        assert _lib.lib().qipb200_pauli_rotation_plan(1, 4, *args, 1, C.byref(v)) == INVALID_ARG
        assert "NULL" in _lib.lib().qipb200_last_error(None).decode()
        assert _lib.lib().qipb200_pauli_rotation_plan(1, 4, *args, 0, C.byref(v)) == 0 and v.value == 0
    for prec, n in ((7, 4), (1, 0), (1, 41)):
        st, _, _ = _plan_raw(n, [0], b"X", [1], prec=prec)
        assert st == INVALID_ARG
    with pytest.raises(CircuitError) as e:
        pauli_rotation_plan(3, C128, [[("X", 0)], [("Q", 1)]])
    assert e.value.status == INVALID_ARG


def test_null_state_is_refused():
    qs = (C.c_uint64 * 1)(0)
    ls = C.create_string_buffer(b"X", 1)
    ln = (C.c_uint32 * 1)(1)
    ang = (C.c_double * 1)(0.5)
    assert _lib.lib().qipb200_state_apply_pauli_rotations(None, qs, ls, ln, 1, ang) == INVALID_ARG
    assert "apply_pauli_rotations" in _lib.lib().qipb200_last_error(None).decode()


def test_cpp_mirror_apply_pauli_rotations_compiles(tmp_path):
    src = tmp_path / "use_rot.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "void run(qip::B200State<double> &st) {\n"
                   "  st.apply_pauli_rotations({{{'Z', 0}, {'Z', 1}}, {{'X', 2}}, {}}, {0.1, -0.2, 0.3});\n"
                   "  st.apply_pauli_rotations({{}}, {1.0});\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
