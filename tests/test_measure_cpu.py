"""qipb200_state_measure without a GPU: argument checks at the C boundary, the C++ mirror's wrapper, and the deferred
collapse.  The diagonal gates that carry a pending collapse into the next fused schedule are built by the library's
own qipb200_collapse_ops (opcompile.cpp), which the tile-kernel emulator build links as well: here they are planned
and run on the emulator in front of a mixed circuit and compared with the oracle's measure_state + fold."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200._abi import QipOp, marshal_ops, prec_of
from rustqip_b200.ops import make_control_op, make_matrix_op, make_swap_op

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "native", "_build", "libplan_emul.so")
SRCS = [os.path.join(HERE, "native", "plan_emulator.cpp"),
        os.path.join(ROOT, "rustqip_b200", "csrc", "planner.cpp"),
        os.path.join(ROOT, "rustqip_b200", "csrc", "opcompile.cpp"),
        os.path.join(ROOT, "rustqip_b200", "csrc", "jit_codegen.cpp")]
HDRS = [os.path.join(ROOT, "rustqip_b200", "csrc", "tile.cuh"),
        os.path.join(ROOT, "rustqip_b200", "csrc", "jit_codegen.h"),
        os.path.join(ROOT, "rustqip_b200", "csrc", "opcompile.h"),
        os.path.join(ROOT, "include", "qip_op.h")]
QIPB200_ERR_INVALID_ARG = 1


@pytest.fixture(scope="module")
def emul():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    stale = not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRCS + HDRS)
    if stale:
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SO] + SRCS + ["-ldl"])
    L = C.CDLL(SO)
    L.emul_schedule.restype = C.c_int
    L.emul_schedule.argtypes = [C.c_int, C.c_uint32, C.POINTER(QipOp), C.c_size_t, C.c_void_p, C.c_uint32,
                                C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_char_p, C.c_size_t]
    L.emul_plan_stats.restype = C.c_int
    L.emul_plan_stats.argtypes = [C.c_int, C.c_uint32, C.POINTER(QipOp), C.c_size_t, C.c_uint32, C.c_uint32,
                                  C.c_int, C.c_uint32, C.c_void_p]
    L.qipb200_collapse_ops.restype = None
    L.qipb200_collapse_ops.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_uint64, C.c_double, C.POINTER(QipOp),
                                       C.c_void_p]
    return L


def p_mult_of(p, dtype):
    """1 / sqrt(p) in the state's precision, as the library computes it for a collapse."""
    if dtype == np.complex64:
        return float(np.float32(1.0) / np.sqrt(np.float32(p)))
    return 1.0 / np.sqrt(p)


def collapse_then(L, prec, indices, measured, p_mult, ops):
    """The library's collapse ops followed by `ops`, as one marshalled array (plus what keeps it alive)."""
    k = len(indices)
    idx = np.ascontiguousarray(np.asarray(indices, dtype=np.uint64))
    dense = np.zeros(8 * k, dtype=np.float64)
    cops = (QipOp * max(k, 1))()
    L.qipb200_collapse_ops(prec, idx.ctypes.data, k, measured, p_mult, cops, dense.ctypes.data)
    rest, keep = marshal_ops(ops, prec)
    arr = (QipOp * (k + len(ops)))()
    for i in range(k):
        arr[i] = cops[i]
    for i in range(len(ops)):
        arr[k + i] = rest[i]
    return arr, (idx, dense, cops, rest, keep)


def rand_state(n, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return v / np.linalg.norm(v)


def rand_unitary(k, rng):
    a = rng.standard_normal((1 << k, 1 << k)) + 1j * rng.standard_normal((1 << k, 1 << k))
    q, r = np.linalg.qr(a)
    return q * (np.diag(r) / np.abs(np.diag(r)))


def mixed_circuit(n, count, seed):
    rng = np.random.default_rng(seed)
    ops = []
    for _ in range(count):
        q = [int(x) for x in rng.choice(n, 4, replace=False)]
        kind = int(rng.integers(12))
        ops.append([
            lambda: gates.h(q[0]), lambda: gates.t(q[0]), lambda: gates.x(q[0]), lambda: gates.cnot(q[0], q[1]),
            lambda: gates.cz(q[0], q[1]), lambda: gates.cphase(q[0], q[1], 0.37), lambda: gates.rz(q[0], 1.1),
            lambda: make_swap_op([q[0]], [q[1]]), lambda: gates.toffoli(q[0], q[1], q[2]),
            lambda: make_matrix_op([q[0], q[1]], rand_unitary(2, rng).reshape(-1)),
            lambda: make_control_op([q[0]], make_matrix_op([q[1]], rand_unitary(1, rng).reshape(-1))),
            lambda: make_control_op([q[3]], make_swap_op([q[0]], [q[1]])),
        ][kind]())
    return ops


def test_measure_rejects_null_state():
    L = _lib.lib()
    idx = (C.c_uint64 * 1)(0)
    m, p = C.c_uint64(0), C.c_double(0.0)
    assert L.qipb200_state_measure(None, idx, 1, 0.5, 0, C.byref(m), C.byref(p)) == QIPB200_ERR_INVALID_ARG
    assert b"measure" in L.qipb200_last_error(None)


def test_cpp_mirror_measure_compiles(tmp_path):
    src = tmp_path / "use_measure.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::B200State<double> &st) {\n"
                   "  auto drawn = st.measure({0, 2}, 0.25);\n"
                   "  auto forced = st.measure({1}, uint64_t(1), std::nullopt);\n"
                   "  auto known = st.measure({1}, uint64_t(0), 0.5);\n"
                   "  return drawn.second + forced.second + known.second + (double)(drawn.first + forced.first + known.first);\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr


def _cases(n):
    """(indices, measured): one, three and all qubits; outcomes with 0 and 1 bits; index bit 0 (qubit n-1) and the top
    index bit (qubit 0)."""
    return [([0], 0), ([0], 1), ([n - 1], 1), ([n - 1], 0), ([n - 1, 2, 0], 0b101), ([1, n - 2, 3], 0b010),
            (list(range(n)), 0b1011 % (1 << n)), (list(range(n))[::-1], (1 << n) - 2)]


@pytest.mark.parametrize("n,T,Lo", [(8, 5, 2), (9, 6, 3), (10, 7, 2), (10, 10, 4), (7, 3, 1), (11, 8, 5)])
@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-5)])
def test_collapse_ops_then_circuit_match_oracle(emul, n, T, Lo, dtype, tol):
    ops = mixed_circuit(n, 60, 4000 + n + T)
    psi = rand_state(n, 7 + n).astype(dtype)
    prec = prec_of(dtype)
    for indices, measured in _cases(n):
        p = qo.measure_prob(n, measured, indices, psi)
        assert p > 0
        collapsed = np.zeros_like(psi)
        qo.measure_state(n, indices, measured, p, psi, collapsed)
        want = qo.run_pipeline(n, ops, state=collapsed)
        arr, keep = collapse_then(emul, prec, indices, measured, p_mult_of(p, dtype), ops)
        st = np.ascontiguousarray(psi.astype(np.complex128))
        stats = np.zeros(64, dtype=np.uint64)
        err = C.create_string_buffer(256)
        rc = emul.emul_schedule(prec, n, arr, len(arr), st.ctypes.data, T, Lo, 1, 0, stats.ctypes.data, err, 256)
        assert rc == 0, err.value
        assert stats[0] > 0
        diff = float(np.max(np.abs(st - want.astype(np.complex128))))
        assert diff < tol, (indices, measured, diff)


def test_collapse_alone_matches_measure_state(emul):
    """Without a circuit after it the collapse ops are measure_state itself (and leave no stray scaling)."""
    n = 9
    psi = rand_state(n, 3)
    for indices, measured in _cases(n):
        p = qo.measure_prob(n, measured, indices, psi)
        want = np.zeros_like(psi)
        qo.measure_state(n, indices, measured, p, psi, want)
        arr, keep = collapse_then(emul, prec_of(np.complex128), indices, measured, p_mult_of(p, np.complex128), [])
        st = np.ascontiguousarray(psi.copy())
        stats = np.zeros(64, dtype=np.uint64)
        err = C.create_string_buffer(256)
        assert emul.emul_schedule(1, n, arr, len(arr), st.ctypes.data, 6, 3, 1, 0, stats.ctypes.data, err, 256) == 0
        assert float(np.max(np.abs(st - want))) < 1e-15, (indices, measured)
        assert int(stats[0] + stats[1]) == 1  # one sweep


def test_collapse_ops_add_no_sweep_to_headline_circuit(emul):
    n = 30
    ops = circuits.random_circuit(n, 40, 0x5EED0002)
    prec = prec_of(np.complex128)
    alone, keep = marshal_ops(ops, prec)
    stats = np.zeros(64, dtype=np.uint64)
    assert emul.emul_plan_stats(prec, n, alone, len(ops), 0, 0, 1, 0, stats.ctypes.data) == 0
    sweeps = int(stats[0] + stats[1])
    assert sweeps > 0
    for indices, measured in (([0], 1), ([n - 1], 0), ([3, 17, 25], 0b110), (list(range(n)), 12345)):
        arr, keep2 = collapse_then(emul, prec, indices, measured, 1.7, ops)
        stats = np.zeros(64, dtype=np.uint64)
        assert emul.emul_plan_stats(prec, n, arr, len(arr), 0, 0, 1, 0, stats.ctypes.data) == 0
        assert int(stats[0] + stats[1]) == sweeps, (indices, int(stats[0]), int(stats[1]), sweeps)
