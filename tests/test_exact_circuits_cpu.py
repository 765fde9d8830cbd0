"""Exactly representable circuits (tests/exact_circuits.py) on the CPU: the reference pinned by an integer fold, and
the planner's passes -- run by the tile emulator and by the host-compiled generated kernels -- equal to it bit for bit
under every planner knob, with qubit rotation and on sharded states.  No tolerance anywhere: a wrong index, sign,
constant or fold shows up on any amplitude, however small."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import exact_circuits as xc
from oracle import qip_oracle as qo
from rustqip_b200._abi import QipOp, marshal_ops, prec_of
from rustqip_b200.ops import make_matrix_op

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "native", "_build", "libplan_emul.so")
CSRC = os.path.join(ROOT, "rustqip_b200", "csrc")
SRCS = [os.path.join(HERE, "native", "plan_emulator.cpp")] + [os.path.join(CSRC, f) for f in ("planner.cpp", "opcompile.cpp", "jit_codegen.cpp")]
HDRS = [os.path.join(CSRC, f) for f in ("tile.cuh", "opcompile.h", "jit_codegen.h")] + [os.path.join(ROOT, "include", "qip_op.h")]
DTYPES = [np.complex128, np.complex64]
BITS0 = {np.complex128: 8, np.complex64: 3}
KNOBS = [
    {"QIPB200_SEED_SEARCH": "1"}, {"QIPB200_KEEP_REAL": "1"}, {"QIPB200_NO_HAD": "1"}, {"QIPB200_NO_LOOKBACK": "1"},
    {"QIPB200_NO_FILL": "1"}, {"QIPB200_NO_PEEPHOLE": "1"}, {"QIPB200_NO_PHASEN": "1"}, {"QIPB200_X_MOVES": "1"},
    {"QIPB200_COMPOSE": "3"}, {"QIPB200_SEED_SEARCH": "1", "QIPB200_KEEP_REAL": "1", "QIPB200_NO_FILL": "1"},
    {"QIPB200_PLAN_LOOKAHEAD": "2"}, {"QIPB200_PLAN_LOOKAHEAD": "1", "QIPB200_SEED_SEARCH": "1"},
]


@pytest.fixture(scope="module")
def emul():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    stale = not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRCS + HDRS)
    if stale:
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SO] + SRCS + ["-ldl"])
    L = C.CDLL(SO)
    opp, u32, p, s = C.POINTER(QipOp), C.c_uint32, C.c_void_p, C.c_char_p
    L.emul_schedule.argtypes = [C.c_int, u32, opp, C.c_size_t, p, u32, u32, C.c_int, u32, p, s, C.c_size_t]
    L.emul_schedule_jit.argtypes = [C.c_int, u32, opp, C.c_size_t, p, u32, u32, s, p, s, C.c_size_t]
    L.emul_schedule_rotate.argtypes = [C.c_int, u32, opp, C.c_size_t, p, u32, u32, C.c_int, p, C.c_int, p, s, C.c_size_t]
    L.emul_sharded_uniform.argtypes = [C.c_int, u32, u32, opp, C.c_size_t, p, u32, u32, p, s, C.c_size_t]
    L.emul_plan_coverage.argtypes = [C.c_int, u32, opp, C.c_size_t, u32, u32, p]
    return L


def run(L, entry, n, ops, psi, *args):
    """Run one emulator entry point on a copy of psi (complex128 host buffer; the precision is psi's)."""
    prec = prec_of(psi.dtype)
    arr, keep = marshal_ops(ops, prec)
    st = np.ascontiguousarray(psi.astype(np.complex128))
    stats = np.zeros(8, dtype=np.uint64)
    err = C.create_string_buffer(512)
    if entry == "schedule":
        T, Lo = args
        rc = L.emul_schedule(prec, n, arr, len(ops), st.ctypes.data, T, Lo, 1, 0, stats.ctypes.data, err, 512)
    elif entry == "rotate":
        T, Lo = args
        rc = L.emul_schedule_rotate(prec, n, arr, len(ops), st.ctypes.data, T, Lo, 1, None, 0, stats.ctypes.data, err, 512)
    elif entry == "sharded":
        g, T, Lo = args
        rc = L.emul_sharded_uniform(prec, n, g, arr, len(ops), st.ctypes.data, T, Lo, stats.ctypes.data, err, 512)
    else:
        raise ValueError(entry)
    assert rc == 0, (rc, err.value)
    return st.astype(psi.dtype), stats


def run_jit(L, n, ops, psi):
    prec = prec_of(psi.dtype)
    arr, keep = marshal_ops(ops, prec)
    st = np.ascontiguousarray(psi.copy())
    stats = np.zeros(8, dtype=np.uint64)
    err = C.create_string_buffer(512)
    with tempfile.TemporaryDirectory() as d:
        rc = L.emul_schedule_jit(prec, n, arr, len(ops), st.ctypes.data, 0, 0, d.encode(), stats.ctypes.data, err, 512)
    assert rc == 0, (rc, err.value)
    return st, stats


def case(n, seed, dtype, count=150, wide=True):
    ops = xc.random_exact_circuit(n, count, seed, dtype, BITS0[dtype], wide=wide)
    psi = xc.exact_state(n, seed + 1, BITS0[dtype], shift=int(seed % 5), dtype=dtype)
    return ops, psi


# ---- the reference --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [5, 9, 12, 14])
def test_integer_fold_pins_both_oracle_folds(n, dtype):
    """int64 mantissas + one exponent (exact by construction) == the oracle's f64 fold == its f32 fold, bit for bit."""
    for seed in range(6 if n < 14 else 2):
        ops, psi = case(n, 100 * n + seed, dtype)
        exact = xc.integer_fold(n, ops, psi)
        assert xc.first_mismatch(qo.run_pipeline(n, ops, state=psi.astype(np.complex128)), exact) == ""
        if dtype == np.complex64:
            f32 = qo.run_pipeline(n, ops, state=psi, dtype=np.complex64)
            assert xc.first_mismatch(f32.astype(np.complex128), exact) == ""
        assert xc.first_mismatch(xc.reference(n, ops, psi).astype(np.complex128), exact) == ""


def test_budget_is_tight_and_enforced():
    """The generator never goes over budget, a circuit one bit over is refused, and the cost model is the documented one."""
    assert xc.op_bits(xc.bfly(0, 1.0)) == 1 and xc.op_bits(xc.bfly(0, 0.5)) == 1
    assert xc.op_bits(xc.diag_op([0], [1, 2 + 1j])) == 2 and xc.op_bits(xc.fredkin(0, 1, 2)) == 0
    assert xc.op_bits(make_matrix_op([0], xc.IBFLY)) == 1 and xc.op_bits(xc.x4([0, 1, 2, 3], 4)) == 0
    for dtype in DTYPES:
        lim = xc.LIMIT[np.dtype(dtype)]
        ops = [xc.bfly(0, 0.5)] * (lim - BITS0[dtype] - 1)
        assert xc.check_budget(ops, BITS0[dtype], dtype) == lim
        with pytest.raises(xc.BudgetError):
            xc.check_budget(ops + [xc.bfly(1, 1.0)], BITS0[dtype], dtype)
        for seed in range(4):
            ops = xc.random_exact_circuit(10, 300, seed, dtype, BITS0[dtype], wide=True)
            assert xc.check_budget(ops, BITS0[dtype], dtype) <= lim
    with pytest.raises(xc.BudgetError):  # not dyadic at all: refused, not approximated
        xc.op_bits(make_matrix_op([0], np.array([1, 0, 0, np.exp(0.25j * np.pi)])))


def test_negative_controls_are_reported():
    """One flipped last mantissa bit, or one matrix entry with the wrong sign, must show up as a mismatch."""
    n = 9
    ops, psi = case(n, 7, np.complex128)
    want = xc.reference(n, ops, psi)
    bad = want.copy()
    i = int(np.flatnonzero(np.abs(want) > 0)[-1])
    bad.real[i] = np.frombuffer((np.frombuffer(bad.real[i:i + 1].tobytes(), np.uint64) ^ np.uint64(1)).tobytes(), np.float64)[0]
    assert xc.first_mismatch(bad, want) != ""
    k = next(j for j, op in enumerate(ops) if op.kind == "matrix" and xc.op_bits(op) > 0)
    m = np.asarray(ops[k].data).copy()
    m[int(np.flatnonzero(m != 0)[0])] *= -1
    wrong = ops[:k] + [make_matrix_op(ops[k].indices(), m)] + ops[k + 1:]
    assert xc.first_mismatch(xc.integer_fold(n, wrong, psi), want) != ""


# ---- the planner's passes on the tile emulator -------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,T,Lo", [(5, 0, 0), (9, 6, 2), (10, 7, 3), (12, 12, 5), (12, 8, 3), (13, 10, 4), (14, 12, 5)])
def test_tile_emulator_exact(emul, n, T, Lo, dtype):
    for seed in range(3):
        ops, psi = case(n, 1000 * n + 10 * T + seed, dtype)
        got, stats = run(emul, "schedule", n, ops, psi, T, Lo)
        assert stats[0] > 0
        assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == "", (n, T, Lo, seed)


@pytest.mark.parametrize("knobs", KNOBS)
def test_planner_knobs_exact(emul, monkeypatch, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    for n, T, Lo, dtype, seed in [(10, 7, 3, np.complex128, 5), (11, 8, 2, np.complex64, 6), (12, 12, 4, np.complex128, 7)]:
        ops, psi = case(n, seed, dtype)
        got, _ = run(emul, "schedule", n, ops, psi, T, Lo)
        assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == "", (knobs, n)


def test_condition_table_overflow_exact(emul):
    """More than 63 distinct outside-tile conditions in one pass, mixed into an exact circuit."""
    n, T, Lo = 16, 8, 3
    ops = xc.condition_overflow_block(n, list(range(5, 13)), 21)
    psi = xc.exact_state(n, 22, 8)
    prec = prec_of(psi.dtype)
    arr, keep = marshal_ops(ops, prec)
    st = np.ascontiguousarray(psi.copy())
    stats = np.zeros(8, dtype=np.uint64)
    err = C.create_string_buffer(256)
    assert emul.emul_schedule(prec, n, arr, len(ops), st.ctypes.data, T, Lo, 1, 0, stats.ctypes.data, err, 256) == 0, err.value
    assert stats[5] == 63 and stats[4] >= 10
    assert xc.first_mismatch(st, xc.reference(n, ops, psi)) == ""
    more = xc.random_exact_circuit(n, 60, 23, wide=False) + ops + xc.random_exact_circuit(n, 60, 24, growing=8)
    got, _ = run(emul, "schedule", n, more, psi, T, Lo)
    assert xc.first_mismatch(got, xc.reference(n, more, psi)) == ""


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,T,Lo", [(10, 7, 3), (12, 8, 2), (13, 10, 4)])
def test_rotating_plans_exact(emul, n, T, Lo, dtype):
    for seed in range(2):
        ops, psi = case(n, 77 + seed, dtype)
        got, stats = run(emul, "rotate", n, ops, psi, T, Lo)
        assert stats[2] > 0  # the plan really relabelled qubits
        assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == ""


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,g,T,Lo", [(11, 1, 6, 2), (12, 2, 6, 2), (13, 3, 7, 3)])
def test_sharded_emulation_exact(emul, n, g, T, Lo, dtype):
    for seed in range(2):
        ops, psi = case(n, 300 + 10 * g + seed, dtype)
        got, stats = run(emul, "sharded", n, ops, psi, g, T, Lo)
        assert stats[0] > 0 and stats[2] > 0  # passes ran, qubits migrated
        assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == ""


def test_rotating_plan_single_step_between_passes_regression(emul):
    """A per-gate step (an 8-qubit diagonal) between two rotating passes: the next tile may carry over only the
    qubits then sitting in the low positions.  It used to carry over the whole previous tile, and planning failed
    with 'rotating plan lost track of the tile'."""
    n = 10
    ops = xc.random_exact_circuit(n, 150, 77, np.complex128, 8, wide=True)  # the diagonal is among the wide ops
    psi = xc.exact_state(n, 4, 8)
    got, stats = run(emul, "rotate", n, ops, psi, 7, 3)
    assert stats[1] >= 1  # per-gate steps ran between the passes
    assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == ""


# ---- the generated kernels, compiled for the host ----------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,seed", [(14, 1), (15, 2)])
def test_generated_kernels_exact(emul, n, seed, dtype):
    ops, psi = case(n, 500 + seed, dtype, count=200)
    ops = xc.narrow(ops)  # the host-compiled generator path refuses plans with interpreter passes
    got, stats = run_jit(emul, n, ops, psi)
    assert stats[0] > 0 and stats[1] == 0
    assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == ""


def test_generated_kernels_exact_rotating(emul, monkeypatch):
    monkeypatch.setenv("EMUL_ROTATE", "1")
    for n, dtype in [(14, np.complex128), (15, np.complex64)]:
        ops, psi = case(n, 600 + n, dtype, count=150, wide=False)
        ops = xc.narrow(ops)
        got, stats = run_jit(emul, n, ops, psi)
        assert stats[0] > 0
        assert xc.first_mismatch(got, xc.reference(n, ops, psi)) == ""


# ---- coverage ------------------------------------------------------------------------------------------------------
EC_NAMES = {1: "D1R_FULL", 4: "D1C_FULL", 7: "D1R_MASK", 10: "D1C_MASK", 13: "PHASE", 14: "DENSE3", 15: "X_FULL", 18: "X_MASK",
            21: "PHASEN", 22: "PHASE_J", 25: "D1R_C1", 31: "D1R_C2", 34: "PHASE_2", 37: "HAD"}
JELEM = ["D1", "X", "PH", "DK", "HAD"]
EXTRA = {45: "predicated phase (pm)", 46: "thread-term factors", 47: "CTA factor terms", 48: "conditional JElem",
         49: "conditional load address", 50: "conditional store address", 51: "condition-table overflow",
         53: "interpreter passes", 54: "per-gate steps", 55: "store-time phase terms", 56: "wide dense micro-op",
         57: "wide diagonal micro-op", 58: "wide exchange micro-op"}


def coverage(L, n, ops, dtype, T=0, Lo=0):
    arr, keep = marshal_ops(ops, prec_of(dtype))
    hist = np.zeros(64, dtype=np.uint64)
    assert L.emul_plan_coverage(prec_of(dtype), n, arr, len(ops), T, Lo, hist.ctypes.data) == 0
    return hist


def cpu_family_coverage(L, monkeypatch):
    """Histogram over the circuit family of this file (tile emulator geometries, X_MOVES, condition-table overflow)."""
    total = np.zeros(64, dtype=np.uint64)
    for n, dtype, T, Lo in [(9, np.complex128, 6, 2), (12, np.complex128, 8, 3), (14, np.complex128, 0, 0), (14, np.complex64, 0, 0),
                            (16, np.complex64, 0, 0), (22, np.complex128, 0, 0), (17, np.complex128, 0, 0)]:
        for seed in range(3):
            ops, _ = case(n, 1000 * n + seed, dtype)
            total += coverage(L, n, ops, dtype, T, Lo)
    total += coverage(L, 16, xc.condition_overflow_block(16, list(range(5, 13)), 21), np.complex128, 8, 3)
    monkeypatch.setenv("QIPB200_X_MOVES", "1")
    for seed in range(4):
        ops, _ = case(14, 3 + seed, np.complex128)
        total += coverage(L, 14, ops, np.complex128)
    monkeypatch.delenv("QIPB200_X_MOVES")
    return total


def device_coverage(L, monkeypatch):
    """Histogram over the plans of the circuits tests/test_gpu_exact.py runs, planned as the device plans them
    (QIPB200_JIT=sync; the switch cases under their switch)."""
    total = np.zeros(64, dtype=np.uint64)
    monkeypatch.setenv("QIPB200_JIT", "sync")
    for n, dtype in xc.DEVICE_GEOMETRIES:
        for seed, wide in ((0, True), (0, False), (1, True)):
            if n >= 24 and not wide:
                continue
            ops, _ = xc.device_case(n, dtype, seed, wide)
            total += coverage(L, n, ops, dtype)
    for dtype in DTYPES:
        total += coverage(L, xc.OVERFLOW_N, xc.device_overflow_block(), dtype)
    monkeypatch.setenv("QIPB200_X_MOVES", "1")
    for n, dtype in [(16, np.complex128), (17, np.complex64), (22, np.complex128)]:
        ops, _ = xc.device_case(n, dtype, 2)
        total += coverage(L, n, ops, dtype)
    monkeypatch.delenv("QIPB200_X_MOVES")
    return total


def shape_report(h):
    # EC_D1R_MASK (7-9) is unreachable by construction: a real 2x2 inside a 3-bit group has 0, 1 or 2 local controls,
    # whose pair masks (0xf, 0xA / 0xC, 0x8) all have case ids of their own (tile.cuh: elem_op)
    report = {("EC_%d" % i): int(h[i]) for i in range(1, 40) if i not in (7, 8, 9)}
    report.update({("J_" + k): int(h[40 + i]) for i, k in enumerate(JELEM)})
    report.update({v: int(h[k]) for k, v in EXTRA.items()})
    return report


@pytest.mark.parametrize("family", ["cpu", "device"])
def test_exact_circuits_reach_every_shape(emul, monkeypatch, family):
    """Every interpreter case id, every JElem kind and every special path of a pass is reached by the exact circuits of
    this file and, separately, by the circuits the device test runs (when a shape is added, these histograms show
    whether the exact suite covers it)."""
    h = cpu_family_coverage(emul, monkeypatch) if family == "cpu" else device_coverage(emul, monkeypatch)
    report = shape_report(h)
    print(family, report)
    missing = [k for k, v in report.items() if v == 0]
    assert not missing, missing


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("jit", ["sync", "off"])
def test_device_overflow_block_overflows(emul, monkeypatch, jit, dtype):
    """The overflow circuit of the device test plans, in the device's geometry, as ONE pass with more than 63 distinct
    CTA-uniform conditions: records on the interpreter's in-record path, and a generated kernel for it."""
    monkeypatch.setenv("QIPB200_JIT", jit)
    h = coverage(emul, xc.OVERFLOW_N, xc.device_overflow_block(), dtype)
    assert h[52] == 1 and h[54] == 0, (int(h[52]), int(h[54]))
    assert h[51] > 0 and h[59] > 63, (int(h[51]), int(h[59]))
    assert h[53] == 0


@pytest.mark.parametrize("n,dtype", [g for g in xc.DEVICE_GEOMETRIES if g[0] >= 13],
                         ids=["n%d_%s" % (n, np.dtype(d).name) for n, d in xc.DEVICE_GEOMETRIES if n >= 13])
def test_device_plans_decline_only_wide_passes(emul, monkeypatch, n, dtype):
    """In the device circuits' plans, the generator declines exactly the passes holding an op wider than a register
    group and the passes with no register-group work (only CTA-uniform store-time phases); both run the interpreter
    kernel by design.  The device test's njit == accepted passes then means every other pass ran a generated kernel."""
    monkeypatch.setenv("QIPB200_JIT", "sync")
    for seed in (0, 1, 2):
        ops, _ = xc.device_case(n, dtype, seed)
        h = coverage(emul, n, ops, dtype)
        assert h[61] == 0 and h[53] == h[62] + h[63], (seed, int(h[52]), int(h[53]), int(h[61]), int(h[62]), int(h[63]))
