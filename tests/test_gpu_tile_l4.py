"""f64 states from 22 local qubits plan their tiles with L = 4 (256-byte contiguous runs).  The generated kernels run
that plan, and so does the interpreter kernel: for the passes whose generated kernel is still compiling, and for every
pass where NVRTC or the driver API is missing.  Both on the device against the oracle (the per-entry fold of
apply_op_overwrite, qip/src/builder.rs:423-514)."""
import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import circuits

from test_gpu_jit import run
from test_gpu_parity import _mixed_circuit, assert_close, rand_state

pytestmark = pytest.mark.gpu

N = 22


def test_interpreter_on_the_l4_plan(ctx, monkeypatch):
    monkeypatch.setenv("QIPB200_TILE_L", "4")  # QIPB200_JIT=off alone would plan with L = 5
    ops = _mixed_circuit(N, 120, 7422) + circuits.random_circuit(N, 8, 0x5EED0002, "H,T,CNOT")
    psi = rand_state(N, np.complex128, 24)
    want = qo.run_pipeline(N, ops, state=psi, dtype=np.complex128)
    got, njit = run(ctx, N, ops, psi, monkeypatch, "off")
    assert njit == 0
    assert_close(got, want, np.complex128)


def test_default_async_plan_at_22_qubits(ctx, monkeypatch):
    """The default mode: the first run starts on the interpreter kernel while NVRTC compiles, the second runs the
    generated kernels; both equal to the oracle."""
    monkeypatch.delenv("QIPB200_TILE_L", raising=False)
    ops = circuits.random_circuit(N, 12, 0x5EED0422, "H,T,CNOT") + _mixed_circuit(N, 60, 7423)
    psi = rand_state(N, np.complex128, 25)
    want = qo.run_pipeline(N, ops, state=psi, dtype=np.complex128)
    t0 = ctx.jit_stats()
    first, njit0 = run(ctx, N, ops, psi, monkeypatch, "async")
    t1 = ctx.jit_stats()
    assert t1["tile_passes"] - t0["tile_passes"] > njit0  # some passes ran on the interpreter
    assert_close(first, want, np.complex128)
    ctx.jit_stats(wait=True)
    second, njit1 = run(ctx, N, ops, psi, monkeypatch, "async")
    assert njit1 > njit0
    assert_close(second, want, np.complex128)
