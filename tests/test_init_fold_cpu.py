"""A schedule on a state that set_basis left pending: the first tile pass builds its tiles from the basis index
instead of loading them (jit_codegen.cpp, QIP_SYNTH).  Validated without a GPU: the generated source is compiled for the
HOST (g++ -DQIP_JIT_HOST) and run over a state filled with NaN by tests/native/init_fold_emulator.cpp; the result must
equal the oracle's per-entry fold from |init_index>.  An amplitude the synthesised pass read instead of writing would
turn the result into NaN."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import circuits, gates
from rustqip_b200._abi import QipOp, marshal_ops, prec_of

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "native", "_build", "libinit_fold_emul.so")
CSRC = os.path.join(ROOT, "rustqip_b200", "csrc")
SRCS = [os.path.join(HERE, "native", "init_fold_emulator.cpp")] + [os.path.join(CSRC, f) for f in
                                                                   ("planner.cpp", "opcompile.cpp", "jit_codegen.cpp")]
DEPS = SRCS + [os.path.join(HERE, "native", "plan_emulator.cpp")] + [
    os.path.join(CSRC, f) for f in ("tile.cuh", "opcompile.h", "jit_codegen.h")] + [os.path.join(ROOT, "include", "qip_op.h")]

TOL = {np.complex128: 1e-12, np.complex64: 2e-5}


@pytest.fixture(scope="module")
def emul():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in DEPS):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SO] + SRCS + ["-ldl"])
    L = C.CDLL(SO)
    L.emul_init_fold_jit.restype = C.c_int
    L.emul_init_fold_jit.argtypes = [C.c_int, C.c_uint32, C.c_uint64, C.POINTER(QipOp), C.c_size_t, C.c_void_p, C.c_uint32,
                                     C.c_uint32, C.c_char_p, C.c_void_p, C.c_char_p, C.c_size_t]
    return L


def run_from_basis(L, n, ops, init, dtype, T=0, Lb=0):
    prec = prec_of(dtype)
    arr, keep = marshal_ops(ops, prec)
    st = np.full(1 << n, np.nan + 1j * np.nan, dtype=dtype)  # nothing of this may survive
    stats = np.zeros(8, dtype=np.uint64)
    err = C.create_string_buffer(512)
    with tempfile.TemporaryDirectory() as d:
        rc = L.emul_init_fold_jit(prec, n, init, arr, len(ops), st.ctypes.data, T, Lb, d.encode(), stats.ctypes.data, err, 512)
    assert rc == 0, err.value
    return st, stats


def check(L, n, ops, init, dtype, T=0, Lb=0):
    got, stats = run_from_basis(L, n, ops, init, dtype, T, Lb)
    want = qo.run_pipeline(n, ops, init, dtype)
    assert stats[2] == 1 and stats[4] == 1, "the first pass was not generated as a synthesised pass"
    assert stats[0] >= 1
    assert not np.isnan(got).any()
    assert np.max(np.abs(got.astype(np.complex128) - want.astype(np.complex128))) <= TOL[dtype] * np.max(np.abs(want)) * 10
    return stats


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
@pytest.mark.parametrize("init", [0, 1, 0x2A5D, (1 << 15) - 1])
@pytest.mark.parametrize("geom", [(0, 0), (12, 4), (12, 5)])
def test_synthesised_first_pass_random_circuit(emul, dtype, init, geom):
    n = 15
    ops = circuits.random_circuit(n, 8, 0x5EED0002, "H,T,CNOT") + circuits.random_circuit(n, 3, 0x5EED0005, "H,CZ,CNOT")
    check(emul, n, ops, init, dtype, *geom)


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
@pytest.mark.parametrize("init", [0, 0x1234])
def test_synthesised_first_pass_qft(emul, dtype, init):
    # conditional-phase tables and CTA-uniform conditions in the first pass
    n = 14
    check(emul, n, circuits.qft(n), init, dtype)


@pytest.mark.parametrize("init", [0, 0x3C1])
def test_synthesised_first_pass_starts_with_diagonal_and_controlled_ops(emul, init):
    # phases and a controlled op whose control lies outside the tile act on the basis state before any mixing
    n = 14
    ops = [gates.t(0), gates.z(n - 1), gates.cnot(0, n - 1), gates.cnot(n - 2, 3)] + circuits.random_circuit(n, 4, 0x5EED0007, "H,T,CNOT")
    check(emul, n, ops, init, np.complex128)


def test_synthesised_pass_is_a_different_program(emul):
    """The synthesised first pass is keyed by its source text (the kernel cache maps source -> cubin): it must differ
    from the loading pass of the same plan, and the basis index must not be part of the text."""
    n = 15
    ops = circuits.random_circuit(n, 4, 0x5EED0002, "H,T,CNOT")
    _, s0 = run_from_basis(emul, n, ops, 0, np.complex128)
    _, s1 = run_from_basis(emul, n, ops, 0x155, np.complex128)
    assert s0[4] == 1 and s1[4] == 1
    assert s0[3] == s1[3]  # same source length: the index travels in the parameter block
