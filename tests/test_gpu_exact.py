"""Fused tile passes on the device, bit for bit, on exactly representable circuits (tests/exact_circuits.py).

Every amplitude and matrix entry is a Gaussian integer times a power of two and no intermediate needs more mantissa
bits than the precision has, so every product and partial sum is exact in any order: the device must reproduce the
reference exactly (np.array_equal), in every tile geometry, generated-kernel shape and pass-kernel switch.  Switches
read once per process (QIPB200_JIT_PERSISTENT, QIPB200_JIT_PREFETCH, QIPB200_JIT_CTA_THREADS, QIPB200_ROTATE,
QIPB200_DENSE_DMMA) run in one child process each, sharing one NVRTC cache directory."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import exact_circuits as xc
from oracle import qip_oracle as qo
from rustqip_b200 import _lib
from rustqip_b200._abi import marshal_ops, prec_of
from rustqip_b200.state import State

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
GEOMETRIES = xc.DEVICE_GEOMETRIES
KNOBS = [
    {"QIPB200_SEED_SEARCH": "1"}, {"QIPB200_KEEP_REAL": "1"}, {"QIPB200_NO_HAD": "1"}, {"QIPB200_NO_LOOKBACK": "1"},
    {"QIPB200_NO_FILL": "1"}, {"QIPB200_NO_PEEPHOLE": "1"}, {"QIPB200_NO_PHASEN": "1"}, {"QIPB200_X_MOVES": "1"},
    {"QIPB200_COMPOSE": "3"}, {"QIPB200_PLAN_LOOKAHEAD": "2"},
    {"QIPB200_TILE_T": "10"}, {"QIPB200_TILE_L": "3"}, {"QIPB200_TILE_G": "2"}, {"QIPB200_NO_TMA": "1"},
    {"QIPB200_JIT_GROUP_BITS": "3"}, {"QIPB200_JIT_GROUP_BITS": "5"},
]


def planned_passes(n, ops, dtype):
    """(tile passes, passes the generator accepts) of the plan, computed on the host by the library itself."""
    arr, keep = marshal_ops(ops, prec_of(dtype))
    out = (C.c_double * 5)()
    log = C.create_string_buffer(2000)
    assert _lib.lib().qipb200_jit_precompile(prec_of(dtype), n, arr, len(ops), out, log, 2000) == 0, log.value
    return int(out[0]), int(out[1])


def run(ctx, n, ops, psi, fusion=True):
    j0 = ctx.jit_stats()
    with State(n, psi.dtype, ctx) as st:
        st.upload(psi)
        st.apply_schedule(ops, fusion=fusion)
        got = st.download()
    j1 = ctx.jit_stats()
    return got, j1["jit_passes"] - j0["jit_passes"], j1["tile_passes"] - j0["tile_passes"]


_REF = {}


def reference(n, dtype, seed, wide=True):
    key = (n, np.dtype(dtype).str, seed, wide)
    if key not in _REF:
        _REF.clear()
        ops, psi = xc.device_case(n, dtype, seed, wide)
        _REF[key] = (ops, psi, xc.reference(n, ops, psi))
    return _REF[key]


@pytest.mark.parametrize("n,dtype", GEOMETRIES, ids=["n%d_%s" % (n, np.dtype(d).name) for n, d in GEOMETRIES])
def test_modes_exact(ctx, monkeypatch, n, dtype):
    """sync (every plannable pass on its generated kernel), off, async (first and converged run), unfused."""
    ctx.release_pool()
    for wide in (True, False) if n < 24 else (True,):
        ops, psi, want = reference(n, dtype, 0, wide)
        monkeypatch.setenv("QIPB200_JIT", "sync")
        passes, gen = planned_passes(n, ops, dtype) if n >= 6 else (0, 0)  # schedule.cu fuses from 6 qubits
        got, njit, ntile = run(ctx, n, ops, psi)
        assert xc.first_mismatch(got, want) == "", ("sync", wide)
        assert njit == gen and ntile == passes, (njit, gen, ntile, passes)
        if not wide and n >= 13:
            assert gen == passes  # only the deliberately wide ops send passes to the interpreter (the plan-level check
            # that the declined passes are exactly the ones holding such ops: test_exact_circuits_cpu.py)
        monkeypatch.setenv("QIPB200_JIT", "off")
        got, njit, _ = run(ctx, n, ops, psi)
        assert njit == 0 and xc.first_mismatch(got, want) == "", ("off", wide)
        got, _, _ = run(ctx, n, ops, psi, fusion=False)
        assert xc.first_mismatch(got, want) == "", ("unfused", wide)
    monkeypatch.setenv("QIPB200_JIT", "async")
    ops, psi, want = reference(n, dtype, 1)
    got, _, _ = run(ctx, n, ops, psi)
    assert xc.first_mismatch(got, want) == "", "async first run"
    ctx.jit_stats(wait=True)
    got, _, _ = run(ctx, n, ops, psi)
    assert xc.first_mismatch(got, want) == "", "async converged"


@pytest.mark.parametrize("knobs", KNOBS, ids=["+".join("%s=%s" % (k[8:], v) for k, v in kb.items()) for kb in KNOBS])
def test_switches_exact(ctx, monkeypatch, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    for n, dtype, modes in [(16, C128, ("sync", "off")), (17, C64, ("sync",)), (22, C128, ("sync",))]:
        ops, psi, want = reference(n, dtype, 2)
        for jit in modes:
            monkeypatch.setenv("QIPB200_JIT", jit)
            got, _, _ = run(ctx, n, ops, psi)
            assert xc.first_mismatch(got, want) == "", (knobs, n, jit)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_condition_table_overflow_exact(ctx, monkeypatch, dtype):
    """One pass with 92 distinct outside-tile conditions: past the interpreter's 63-slot condition table (the rest on the
    in-record path) and past one 32-bit condition word of the generated kernel.  That the plan really is such a pass is
    checked on the CPU (test_exact_circuits_cpu.py::test_device_overflow_block_overflows)."""
    n = xc.OVERFLOW_N
    block = xc.device_overflow_block()
    tail = xc.random_exact_circuit(n, 40, 6, dtype, xc.DEVICE_BITS0[np.dtype(dtype)], wide=False)
    psi = xc.exact_state(n, 7, xc.DEVICE_BITS0[np.dtype(dtype)], dtype=dtype)
    want = xc.reference(n, block + tail, psi)
    for jit in ("sync", "off"):
        monkeypatch.setenv("QIPB200_JIT", jit)
        j0 = ctx.jit_stats()
        with State(n, dtype, ctx) as st:
            st.upload(psi)
            st.apply_schedule(block)  # a schedule of its own: the tail would change how the block is planned
            j1 = ctx.jit_stats()
            st.apply_schedule(tail)
            got = st.download()
        assert j1["tile_passes"] - j0["tile_passes"] == 1
        assert j1["jit_passes"] - j0["jit_passes"] == (1 if jit == "sync" else 0)
        assert xc.first_mismatch(got, want) == "", jit


@pytest.mark.parametrize("dtype", [C128, C64])
def test_measure_collapse_save_load_exact(ctx, monkeypatch, dtype, tmp_path):
    """measure forced with probability 1/4 (collapse scale 2: exact), its collapse folded into the next generated pass;
    collapse itself; save / load round trips."""
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 20
    ops, psi, _ = reference(n, dtype, 3)
    idx, m = [1, n - 1], 2
    coll = np.zeros_like(psi)
    qo.measure_state(n, idx, m, 0.25, psi, coll)
    assert np.array_equal(coll[coll != 0], (2 * psi[coll != 0]).astype(dtype))
    want = xc.reference(n, ops, coll)
    with State(n, dtype, ctx) as st:
        st.upload(psi)
        assert st.measure(idx, measured=m, prob=0.25)[0] == m
        st.apply_schedule(ops)
        assert xc.first_mismatch(st.download(), want) == ""
        st.save(str(tmp_path / "a.qipa"))
        st.upload(psi)
        st.collapse(idx, m, 0.25)
        assert xc.first_mismatch(st.download(), coll) == ""
        with State(n, dtype, ctx) as other:
            other.load(str(tmp_path / "a.qipa"))
            assert xc.first_mismatch(other.download(), want) == ""


# ---- process-static switches: one child process each ---------------------------------------------------------------
_WORKER = r"""
import ctypes as C, json, os, sys
import numpy as np
sys.path.insert(0, "tests")
import exact_circuits as xc
from rustqip_b200._abi import QipOp, marshal_ops, prec_of
from rustqip_b200.state import Context, State
emul = C.CDLL(os.path.join("tests", "native", "_build", "libplan_emul.so"))
emul.emul_plan_coverage.argtypes = [C.c_int, C.c_uint32, C.POINTER(QipOp), C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]


def fewest_tiles(n, ops, dtype):  # the plan of this process's environment, as the library makes it
    arr, keep = marshal_ops(ops, prec_of(dtype))
    hist = np.zeros(64, dtype=np.uint64)
    assert emul.emul_plan_coverage(prec_of(dtype), n, arr, len(ops), 0, 0, hist.ctypes.data) == 0
    return int(hist[60])


out = {}
with Context(0) as ctx:
    for n, dtype, bits in [(22, np.complex128, 8), (20, np.complex64, 3), (16, np.complex128, 8)]:
        ops = xc.random_exact_circuit(n, 80, 31 + n, dtype, bits, wide=True)
        psi = xc.exact_state(n, 32 + n, bits, dtype=dtype)
        want = xc.reference(n, ops, psi)
        for jit in ("sync", "off"):
            os.environ["QIPB200_JIT"] = jit
            tiles = fewest_tiles(n, ops, dtype)
            j0 = ctx.jit_stats()["jit_passes"]
            with State(n, dtype, ctx) as st:
                st.upload(psi)
                st.apply_schedule(ops)
                st.apply_schedule(xc.random_exact_circuit(n, 30, 33 + n, dtype, bits, growing=0))
                got = st.download()
            want2 = xc.reference(n, xc.random_exact_circuit(n, 30, 33 + n, dtype, bits, growing=0), want)
            out["n%d_%s_%s" % (n, np.dtype(dtype).name, jit)] = [xc.first_mismatch(got, want2), ctx.jit_stats()["jit_passes"] - j0, tiles]
print("RESULT " + json.dumps(out))
"""

STATIC = [{"QIPB200_JIT_PERSISTENT": "1"}, {"QIPB200_JIT_PERSISTENT": "7"}, {"QIPB200_JIT_PERSISTENT": "132"},
          {"QIPB200_JIT_PREFETCH": "1"}, {"QIPB200_JIT_PREFETCH": "4"}, {"QIPB200_JIT_CTA_THREADS": "256"},
          {"QIPB200_ROTATE": "1"}, {"QIPB200_DENSE_DMMA": "0"}]


@pytest.fixture(scope="module")
def jit_cache(tmp_path_factory):
    return str(tmp_path_factory.mktemp("jitcache"))


@pytest.mark.parametrize("env", STATIC, ids=["%s=%s" % (k[8:], v) for e in STATIC for k, v in e.items()])
def test_process_static_switches_exact(env, jit_cache):
    e = dict(os.environ, PYTHONPATH=ROOT, QIPB200_JIT_CACHE_DIR=jit_cache, **env)
    p = subprocess.run([sys.executable, "-c", _WORKER], cwd=ROOT, env=e, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
    print(env, res)
    for k, (mismatch, njit, tiles) in res.items():
        assert mismatch == "", (env, k, mismatch)
        if k.endswith("_sync") and not k.startswith("n16"):
            assert njit > 0, (env, k)
    if "QIPB200_JIT_PERSISTENT" in env:
        # every generated pass of the f64 n=22 circuit has more tiles than the grid has CTAs: each CTA walks several
        # (at f32 n=20, 128 tiles, only the 1- and 7-CTA grids do)
        assert res["n22_complex128_sync"][2] > int(env["QIPB200_JIT_PERSISTENT"]), res


# ---- full size: no host oracle, fused passes against per-gate kernels -----------------------------------------------
@pytest.mark.parametrize("jit", ["sync", "off"])
def test_full_size_n30_f64(ctx, monkeypatch, jit):
    monkeypatch.setenv("QIPB200_JIT", jit)
    n = 30
    ops = xc.random_exact_circuit(n, 120, 30, C128, 8, wide=True)
    ctx.release_pool()
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        w = 1 << 26
        block = xc.exact_state(26, 30, 8, dtype=C128)
        for k in range((1 << n) // w):
            blk = xc.exact_window(block, k)
            a.upload(blk, offset=k * w)
            b.upload(blk, offset=k * w)
        a.apply_schedule(ops)
        b.apply_schedule(ops, fusion=False)
        assert a.max_abs_diff(b) == 0.0
    ctx.release_pool()


def test_full_size_n31_f32(ctx, monkeypatch):
    """Targets, controls and tile bits at index bit 30 (qubit 0): amplitude indices >= 2^31."""
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 31
    ops = xc.random_exact_circuit(n, 60, 31, C64, 3, wide=False, qubits=[0, 1, 2, 3, 20, 25, 27, 28, 29, 30])
    ctx.release_pool()
    with State(n, C64, ctx) as a, State(n, C64, ctx) as b:
        w = 1 << 26
        block = xc.exact_state(26, 31, 3, dtype=C64)
        for k in range((1 << n) // w):
            blk = xc.exact_window(block, k)
            a.upload(blk, offset=k * w)
            b.upload(blk, offset=k * w)
        a.apply_schedule(ops)
        b.apply_schedule(ops, fusion=False)
        assert a.max_abs_diff(b) == 0.0
    ctx.release_pool()


def test_full_size_n32_f32_circuit_then_inverse(ctx, monkeypatch):
    """One 32 GiB state: C fused, then its exact inverse fused; the input must come back bit for bit."""
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 32
    ops = xc.reversible_circuit(n, 120, 32, growing=9)
    inv = xc.inverse_circuit(ops)
    xc.check_budget(ops + inv, 3, C64)
    ctx.release_pool()
    w = 1 << 27
    block = xc.exact_state(27, 32, 3, dtype=C64)
    with State(n, C64, ctx) as a:
        for k in range((1 << n) // w):
            a.upload(xc.exact_window(block, k), offset=k * w)
        a.apply_schedule(ops)
        a.apply_schedule(inv)
        for k in range((1 << n) // w):
            assert xc.first_mismatch(a.download(offset=k * w, length=w), xc.exact_window(block, k)) == "", k
    ctx.release_pool()
