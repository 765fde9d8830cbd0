"""qipb200_state_measure on the device: measure (measurement_ops.rs:190-214) in one call, and the collapse it leaves
pending on an unsharded state (folded into the next fused schedule, applied before any other access).

Draws are kept away from the cumulative boundaries: the device sums |a|^2 in another order than the serial scan."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.ops import from_reals
from rustqip_b200.state import Context, State

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QIPB200_ERR_INVALID_ARG = 1


def _index_lists(n):
    return [[0], [9, 0, 4], list(range(n)), list(range(n))[::-1]]


def _far_draws(psi, k, seed, tol=1e-9):
    cum = np.cumsum(np.abs(psi.astype(np.complex128)) ** 2)
    r = np.random.default_rng(seed).random(8 * k) * cum[-1] * 1.02
    pos = np.searchsorted(cum, r)
    near = np.minimum(np.abs(cum[np.clip(pos, 0, cum.size - 1)] - r), np.abs(cum[np.clip(pos - 1, 0, cum.size - 1)] - r))
    return r[(near > tol) & (r > tol)][:k]


def _three_calls(st, indices, r):
    m = st.soft_measure(indices, r)
    p = st.measure_prob(m, indices)
    st.collapse(indices, m, p)
    return m, p


def _agree(a, b):
    """(m, p) of measure against the three calls: p is summed in another order than measure_prob's."""
    return a[0] == b[0] and abs(a[1] - b[1]) <= 1e-12


def _collapsed(n, indices, m, p, psi):
    out = np.zeros_like(psi)
    qo.measure_state(n, indices, m, p, psi, out)
    return out


def test_reference_known_answers(ctx):
    # measurement_ops.rs:291-327 (test_measure_state, test_measure_state2), as forced outcomes with measure_prob
    half = np.sqrt(0.5)
    for m, want in ((0, [half, half, 0.0, 0.0]), (1, [0.0, 0.0, half, half])):
        with State(2, np.complex128, ctx) as st:
            st.upload(from_reals([0.5, 0.5, 0.5, 0.5]))
            got_m, p = st.measure([0], measured=m)
            assert got_m == m and abs(p - 0.5) < np.finfo(np.float64).eps
            assert np.allclose(st.download(), from_reals(want), atol=1e-10)
    # measurement_ops.rs:136-152: the doctest's draws, now through measure
    for indices, want in (([0], 1), ([1], 0), ([0, 1], 0b01), ([1, 0], 0b10)):
        with State(2, np.complex128, ctx) as st:
            st.upload(from_reals([0.0, 0.0, 1.0, 0.0]))
            assert st.measure(indices, 0.5) == (want, 1.0)
            assert np.array_equal(st.download(), from_reals([0.0, 0.0, 1.0, 0.0]))


@pytest.mark.parametrize("n", [10, 14])
@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-6)])
@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_oracle_parity(ctx, n, dtype, tol, scale):
    psi = (circuits.random_state(n, 100 + n, dtype) * scale).astype(dtype)
    wide = psi.astype(np.complex128)  # the library accumulates in double, as the f64 oracle does
    draws = _far_draws(psi, 6, n)
    assert draws.size == 6
    with State(n, dtype, ctx) as st:
        for indices in _index_lists(n):
            for r in draws:
                st.upload(psi)
                m, p = st.measure(indices, float(r))
                assert m == qo.soft_measure(n, indices, wide, float(r)), (indices, r)
                assert abs(p - qo.measure_prob(n, m, indices, wide)) <= 1e-12, (indices, r)
                got = st.download()
                want = _collapsed(n, indices, m, p, psi)
                assert float(np.max(np.abs(got - want))) <= tol, (indices, r)


@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-6)])
def test_forced_outcomes(ctx, dtype, tol):
    n = 12
    psi = circuits.random_state(n, 5, dtype)
    with State(n, dtype, ctx) as a, State(n, dtype, ctx) as b:
        for indices, m in (([0], 1), ([3, 11, 7], 0b110), (list(range(n)), 1234)):
            a.upload(psi)
            b.upload(psi)
            got_m, p = a.measure(indices, measured=m)
            assert got_m == m and abs(p - b.measure_prob(m, indices)) <= 1e-12
            b.collapse(indices, m, p)
            assert a.max_abs_diff(b) <= tol
            a.upload(psi)
            b.upload(psi)
            assert a.measure(indices, measured=m, prob=0.3) == (m, 0.3)
            b.collapse(indices, m, 0.3)
            assert a.max_abs_diff(b) <= tol
        # zero probability: a basis state measured against itself, and an outcome no index list can give
        a.set_basis(5)
        before = a.download()
        for indices, m in (([n - 1], 0), ([0, 1], 4)):
            assert a.measure(indices, measured=m) == (m, 0.0)
            assert a.download().tobytes() == before.tobytes()
        assert a.measure([n - 1], measured=0, prob=0.0) == (0, 0.0)
        assert a.download().tobytes() == before.tobytes()
        L = _lib.lib()
        idx = (C.c_uint64 * 1)(0)
        mm, pp = C.c_uint64(0), C.c_double(0.5)
        for flags in (4, _lib.MEASURE_FORCED_PROB, 8 | _lib.MEASURE_FORCED):
            assert L.qipb200_state_measure(a._h, idx, 1, 0.5, flags, C.byref(mm), C.byref(pp)) == QIPB200_ERR_INVALID_ARG
            assert "measure" in L.qipb200_last_error(ctx.handle).decode()
        for bad in ([], [0, 0], [n]):
            with pytest.raises(CircuitError) as e_meas:
                a.measure(bad, 0.5)
            with pytest.raises(CircuitError) as e_soft:
                a.soft_measure(bad, 0.5)
            assert e_meas.value.status == e_soft.value.status and str(e_meas.value) == str(e_soft.value)


def _entry_points(n, dtype, tmp_path):
    """(name, f(state) -> comparable result): every call that must see the collapse first."""
    rng = np.random.default_rng(77)
    part = (rng.standard_normal(40) + 1j * rng.standard_normal(40)).astype(dtype) * 0.01
    sched = circuits.random_circuit(n, 6, 0x5EED0004, "H,T,CNOT") + circuits.qft(n)[:20]
    return [
        ("download", lambda st: st.download()),
        ("upload", lambda st: (st.upload(part, offset=100), st.download())[1]),
        ("apply_op", lambda st: (st.apply_op(gates.h(1)), st.download())[1]),
        ("schedule_fused", lambda st: (st.apply_schedule(sched), st.download())[1]),
        ("schedule_unfused", lambda st: (st.apply_schedule(sched, fusion=False), st.download())[1]),
        ("norm2", lambda st: st.norm2()),
        ("measure_probs", lambda st: st.measure_probs([0, 5, n - 1])),
        ("measure_prob", lambda st: st.measure_prob(1, [2, 4])),
        ("soft_measure", lambda st: st.soft_measure([1, 3, n - 2], 0.3)),
        ("sample", lambda st: st.sample([1, 3, n - 2], [0.3, 0.7])),
        ("collapse", lambda st: (st.collapse([1], 1, 0.4), st.download())[1]),
        ("measure", lambda st: (st.measure([2, 7], 0.6), st.download())),
        ("save", lambda st: _saved(st, str(tmp_path / "s.qipa"), dtype)),
    ]


def _saved(st, path, dtype):
    """The amplitudes a state file holds (QIPA v1: a 40-byte header, then the amplitudes)."""
    st.save(path)
    with open(path, "rb") as f:
        return np.frombuffer(f.read()[40:], dtype=dtype)


def _same(x, y, tol):
    if isinstance(x, tuple):
        return all(_same(a, b, tol) for a, b in zip(x, y))
    if isinstance(x, np.ndarray) and x.dtype == np.uint64:
        return np.array_equal(x, y)
    if isinstance(x, int):
        return x == y
    return float(np.max(np.abs(np.asarray(x) - np.asarray(y)))) <= tol


@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-6)])
def test_deferral_is_invisible(ctx, dtype, tol, tmp_path):
    n = 12
    psi = circuits.random_state(n, 9, dtype)
    indices, r = [0, 6, n - 1], 0.41
    with State(n, dtype, ctx) as a, State(n, dtype, ctx) as b:
        for name, call in _entry_points(n, dtype, tmp_path):
            a.upload(psi)
            b.upload(psi)
            assert _agree(a.measure(indices, r), _three_calls(b, indices, r)), name
            got_b = call(b)
            got_a = call(a)
            assert _same(got_a, got_b, tol), name
        # max_abs_diff applies the collapse on both states
        a.upload(psi)
        b.upload(psi)
        a.measure(indices, r)
        b.measure(indices, r)
        assert a.max_abs_diff(b) == 0.0
        # set_basis and load overwrite every amplitude: the pending collapse is dropped
        a.upload(psi)
        a.measure(indices, r)
        a.set_basis(3)
        basis = np.zeros(1 << n, dtype=dtype)
        basis[3] = 1
        assert np.array_equal(a.download(), basis)
        b.upload(psi)
        b.save(str(tmp_path / "plain.qipa"))
        a.upload(psi)
        a.measure(indices, r)
        a.load(str(tmp_path / "plain.qipa"))
        assert np.array_equal(a.download(), psi)
        # a rejected schedule: nothing of it runs and the collapse stays pending; or the ops before the bad one run
        # after the collapse
        for sched in ([gates.h(n + 2)], [gates.h(1), gates.x(n)]):
            a.upload(psi)
            b.upload(psi)
            m, p = a.measure(indices, r)
            _three_calls(b, indices, r)
            with pytest.raises(CircuitError) as ea:
                a.apply_schedule(sched)
            with pytest.raises(CircuitError) as eb:
                b.apply_schedule(sched)
            assert ea.value.status == eb.value.status and str(ea.value) == str(eb.value)
            assert a.max_abs_diff(b) <= tol
            assert float(np.max(np.abs(a.download() - b.download()))) <= tol


def test_deferral_is_free(ctx, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 22
    first = circuits.random_circuit(n, 10, 0x5EED0002, "H,T,CNOT")
    nxt = circuits.random_circuit(n, 40, 0x5EED0006, "H,T,CNOT")
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for st in (a, b):
            st.set_basis(0)
            st.apply_schedule(first)
        for indices, r in (([0], 0.3), ([n - 1, 4, 11], 0.8)):
            assert _agree(a.measure(indices, r), _three_calls(b, indices, r))
            deltas = []
            for st in (a, b):
                s0, l0 = ctx.launch_stats(), ctx.kernel_launches()
                st.apply_schedule(nxt)
                s1, l1 = ctx.launch_stats(), ctx.kernel_launches()
                deltas.append((s1["tile_passes"] - s0["tile_passes"], l1 - l0))
            assert deltas[0] == deltas[1], deltas  # same passes, and no k_collapse sweep
            assert a.max_abs_diff(b) <= 1e-12
        js = ctx.jit_stats()
        assert js["jit_passes"] > 0, js["note"]


def test_repeatable(ctx):
    n = 16
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for st in (a, b):
            st.set_basis(3)
            st.apply_schedule(circuits.random_circuit(n, 10, 9, "H,T,CNOT"))
        for indices in ([0], [3, 15, 8, 1], list(range(n))):
            ra, rb = a.measure(indices, 0.37), b.measure(indices, 0.37)
            assert ra == rb
            assert a.max_abs_diff(b) == 0.0


def test_launch_count_is_fixed(ctx):
    counts = set()
    for n in (14, 22):
        psi = circuits.random_state(n, 31)
        for indices in ([0], list(range(8))):
            with State(n, np.complex128, ctx) as st:
                st.upload(psi)
                l0 = ctx.kernel_launches()
                st.measure(indices, 0.5)
                counts.add(ctx.kernel_launches() - l0)
    assert len(counts) == 1 and counts.pop() > 0


def test_headline_size(ctx):
    n = 28
    first = circuits.random_circuit(n, 8, 0x5EED0002, "H,T,CNOT")
    nxt = circuits.random_circuit(n, 6, 0x5EED0007, "H,T,CNOT")
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for st in (a, b):
            st.set_basis(0)
            st.apply_schedule(first)
        assert _agree(a.measure([0], 0.6), _three_calls(b, [0], 0.6))
        a.apply_schedule(nxt)
        b.apply_schedule(nxt)
        assert a.max_abs_diff(b) <= 1e-12


_ROTATE_WORKER = r"""
import os
import numpy as np
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State
from oracle import qip_oracle as qo

with Context(0) as ctx:
    for n, jit in [(16, "off"), (18, "sync")]:
        os.environ["QIPB200_JIT"] = jit
        a = circuits.random_circuit(n, 10, 11, "H,T,CNOT")
        b = circuits.qft(n)[:60] + circuits.random_circuit(n, 5, 12, "H,CZ,CNOT")
        c = circuits.random_circuit(n, 6, 13, "H,T,CNOT")
        want = qo.run_pipeline(n, a + b, 5, np.complex128)
        for indices, r in (([0], 0.3), ([9, 0, 4], 0.71)):
            with State(n, np.complex128, ctx) as st:
                st.set_basis(5)
                st.apply_schedule(a)
                st.apply_schedule(b)
                assert not np.array_equal(st.qubit_map(), np.arange(n)[::-1]), "the layout is not rotated"
                m, p = st.measure(indices, r)
                assert m == qo.soft_measure(n, indices, want, r), (m, indices, r)
                assert abs(p - qo.measure_prob(n, m, indices, want)) <= 1e-12
                coll = np.zeros_like(want)
                qo.measure_state(n, indices, m, p, want, coll)
                st.apply_schedule(c)  # the collapse runs inside this schedule's first pass, in a rotated layout
                got = st.download()
            err = float(np.max(np.abs(got - qo.run_pipeline(n, c, state=coll))))
            assert err <= 1e-10, err
        print("rotate measure n=%d jit=%s: OK" % (n, jit))
"""


def test_measure_on_rotated_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=420)
    sys.stdout.write(p.stdout[-3000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]


def test_multi_device_context():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n = 14
    psi = circuits.random_state(n, 41)
    with Context([0, 1]) as mctx:
        with State(n, np.complex128, mctx) as a, State(n, np.complex128, mctx) as b:
            for indices, r in (([0], 0.3), ([n - 1, 2], 0.55)):
                a.upload(psi)
                b.upload(psi)
                assert _agree(a.measure(indices, r), _three_calls(b, indices, r))
                assert float(np.max(np.abs(a.download() - b.download()))) <= 1e-12
