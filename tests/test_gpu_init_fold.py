"""set_basis on an unsharded state leaves the basis state pending: the next fused schedule's first tile pass builds its
tiles from the index instead of loading them, and every other access writes the basis state first.  Each check runs the
same calls twice, once pending and once with QIPB200_NO_INIT_FOLD=1 (the state written by set_basis at once), and the
two must agree."""
import ctypes as C

import numpy as np
import pytest

from rustqip_b200 import _lib, circuits
from rustqip_b200._abi import marshal_ops, prec_of
from rustqip_b200.state import State

pytestmark = pytest.mark.gpu

OPS22 = circuits.random_circuit(22, 6, 0x5EED0002, "H,T,CNOT") + circuits.random_circuit(22, 2, 0x5EED0005, "H,CZ,CNOT")


def _basis(ctx, n, dtype, index, fold, monkeypatch):
    if fold:
        monkeypatch.delenv("QIPB200_NO_INIT_FOLD", raising=False)
    else:
        monkeypatch.setenv("QIPB200_NO_INIT_FOLD", "1")
    st = State(n, dtype, ctx)
    st.set_basis(index)
    monkeypatch.delenv("QIPB200_NO_INIT_FOLD", raising=False)
    return st


def _pair(ctx, n, dtype, index, monkeypatch):
    return _basis(ctx, n, dtype, index, True, monkeypatch), _basis(ctx, n, dtype, index, False, monkeypatch)


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
@pytest.mark.parametrize("index", [0, 0x2A5D31])
def test_readers_of_a_pending_state(ctx, dtype, index, monkeypatch):
    n = 22
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        draws = np.random.default_rng(7).random(64)
        assert np.array_equal(a.sample([0, 5, 21], draws), b.sample([0, 5, 21], draws))
        terms = [[("Z", 0)], [("X", 3)], [("Z", 21), ("Z", 4)], []]
        assert np.array_equal(a.expect_paulis(terms), b.expect_paulis(terms))
        assert a.norm2() == b.norm2() == 1.0
        assert np.array_equal(a.download(), b.download())
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        assert a.measure([1, 7], r=0.3) == b.measure([1, 7], r=0.3)
        assert np.array_equal(a.download(), b.download())
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        want = np.zeros(1 << n, dtype=dtype)
        want[index] = 1
        assert np.array_equal(a.download(offset=index - 5 if index else 0, length=11),
                              want[index - 5 if index else 0:][:11])


def _run(ctx, n, dtype, index, ops, fold, monkeypatch, fusion=True):
    st = _basis(ctx, n, dtype, index, fold, monkeypatch)
    st.apply_schedule(ops, fusion=fusion)
    return st


@pytest.mark.parametrize("jit", ["sync", "async", "off"])
@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_fused_schedule_from_a_pending_state(ctx, jit, dtype, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", jit)
    n, index = 22, 0x155
    for rep in range(2):  # async: the first run takes the interpreter while the programs compile
        l0 = ctx.kernel_launches()
        j0 = ctx.jit_stats(wait=False)["jit_passes"]
        a = _run(ctx, n, dtype, index, OPS22, True, monkeypatch)
        l1 = ctx.kernel_launches()
        j1 = ctx.jit_stats(wait=False)["jit_passes"]
        b = _run(ctx, n, dtype, index, OPS22, False, monkeypatch)
        l2 = ctx.kernel_launches()
        with a, b:
            assert a.max_abs_diff(b) == 0.0
            assert np.array_equal(a.download(), b.download())
        if jit == "sync" or (jit == "async" and rep == 1):
            assert j1 > j0
            assert l2 - l1 == (l1 - l0) + 1  # the eager path launches the one-amplitude kernel
        if jit == "async":
            ctx.jit_stats(wait=True)


@pytest.mark.parametrize("n", [22, 24, 26, 28])
def test_headline_like_circuits_from_a_pending_state(ctx, n, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", "sync")
    ops = circuits.random_circuit(n, 6, 0x5EED0003, "H,T,CNOT")
    index = (1 << (n - 1)) | 3
    a = _run(ctx, n, np.complex128, index, ops, True, monkeypatch)
    b = _run(ctx, n, np.complex128, index, ops, False, monkeypatch)
    with a, b:
        assert a.max_abs_diff(b) == 0.0
        assert abs(a.norm2() - 1.0) < 1e-9


def test_n30_qft_f32_from_a_pending_state(ctx, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 30
    a = _run(ctx, n, np.complex64, 0, circuits.qft(n), True, monkeypatch)
    b = _run(ctx, n, np.complex64, 0, circuits.qft(n), False, monkeypatch)
    with a, b:
        assert a.max_abs_diff(b) == 0.0


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_writers_of_a_pending_state(ctx, dtype, monkeypatch):
    n, index = 22, 0x3001
    ops = OPS22[:40]
    # per-op application and an unfused schedule
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        for op in ops[:5]:
            a.apply_op(op)
            b.apply_op(op)
        assert a.max_abs_diff(b) == 0.0
    a = _run(ctx, n, dtype, index, ops, True, monkeypatch, fusion=False)
    b = _run(ctx, n, dtype, index, ops, False, monkeypatch, fusion=False)
    with a, b:
        assert a.max_abs_diff(b) == 0.0
    # a partial upload keeps the other amplitudes; a full upload replaces all of them
    part = (np.arange(8) + 1j).astype(dtype)
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        a.upload(part, offset=0x3000)
        b.upload(part, offset=0x3000)
        assert np.array_equal(a.download(), b.download())
    full = np.random.default_rng(3).standard_normal(1 << n).astype(dtype)
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    with a, b:
        a.upload(full)
        b.upload(full)
        a.apply_schedule(ops)
        b.apply_schedule(ops)
        assert a.max_abs_diff(b) == 0.0
    # out of place: a copy (identity Pauli sum) reads a pending source and overwrites a pending destination
    a, b = _pair(ctx, n, dtype, index, monkeypatch)
    c, d = _pair(ctx, n, dtype, 7, monkeypatch)
    with a, b, c, d:
        c.apply_pauli_sum(a, [[]], [1.0])
        d.apply_pauli_sum(b, [[]], [1.0])
        assert c.max_abs_diff(d) == 0.0
        c.apply_schedule(ops)
        d.apply_schedule(ops)
        assert c.max_abs_diff(d) == 0.0
        assert a.max_abs_diff(b) == 0.0


def test_set_basis_twice_and_an_empty_schedule(ctx, monkeypatch):
    n = 22
    a, b = _pair(ctx, n, np.complex128, 5, monkeypatch)
    with a, b:
        a.apply_schedule([])
        a.set_basis(9)
        b.set_basis(9)
        a.apply_schedule(OPS22)
        b.apply_schedule(OPS22)
        assert a.max_abs_diff(b) == 0.0


@pytest.mark.parametrize("jit", ["sync", "off"])
def test_calculate_state(ctx, jit, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", jit)
    n = 22
    p = prec_of(np.complex128)
    arr, keep = marshal_ops(OPS22, p)
    outs = []
    for fold in (True, False):
        if fold:
            monkeypatch.delenv("QIPB200_NO_INIT_FOLD", raising=False)
        else:
            monkeypatch.setenv("QIPB200_NO_INIT_FOLD", "1")
        out = np.zeros(1 << n, dtype=np.complex128)
        _lib.check(_lib.lib().qipb200_calculate_state(ctx.handle, p, n, 0x1F00F, arr, len(OPS22), 0,
                                                      C.c_void_p(out.ctypes.data)), ctx.handle)
        outs.append(out)
    monkeypatch.delenv("QIPB200_NO_INIT_FOLD", raising=False)
    assert np.array_equal(outs[0], outs[1])


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_writing_a_pending_state_launches_no_kernel(ctx, dtype, monkeypatch):
    """The first reader of a pending state launches the kernels it launches on a state written at once, no more."""
    n = 22
    a, b = _pair(ctx, n, dtype, 0x1234, monkeypatch)
    with a, b:
        l0 = ctx.kernel_launches()
        va = a.norm2()
        l1 = ctx.kernel_launches()
        vb = b.norm2()
        assert ctx.kernel_launches() - l1 == l1 - l0 and va == vb == 1.0
        assert np.array_equal(a.download(), b.download())
