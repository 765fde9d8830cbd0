"""qipb200_state_sample on the device: many soft_measure draws (measurement_ops.rs:153-176) from one state.

The device sums |a|^2 in another order than the serial scan, so a draw within rounding distance of a cumulative
boundary may land on the neighbouring index; draws that close to a boundary are compared by bracketing instead."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import _lib, circuits
from rustqip_b200.errors import CircuitError
from rustqip_b200.ops import from_reals
from rustqip_b200.state import State

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QIPB200_ERR_INVALID_ARG, QIPB200_ERR_UNSUPPORTED = 1, 7

SPECIAL_DRAWS = [0.0, 1e-300, 0.5, 1.0 - 2.0 ** -53]


def _draws(seed, k):
    return np.concatenate([np.random.default_rng(seed).random(k), SPECIAL_DRAWS])


def _index_lists(n):
    return [[0], [9, 0, 4], list(range(n)), list(range(n))[::-1]]


def _check_against_oracle(n, psi, st_or_got, draws, tol):
    """Draws farther than `tol` from every boundary of the float64 cumulative sum equal the oracle; every draw
    brackets: the index i read back with all qubits measured has C(i-1) < r <= C(i) within tol (or is 0 when the
    draw never crosses).  f32 amplitudes are widened first: the library accumulates in double (as soft_measure
    does), while the oracle's f32 scan accumulates in float and drifts by ~1e-5 over 2^14 amplitudes."""
    psi = psi.astype(np.complex128)
    cum = np.cumsum(np.abs(psi) ** 2)
    pos = np.searchsorted(cum, draws)
    near = np.full(draws.shape, np.inf)
    for d in (-1, 0):
        j = np.clip(pos + d, 0, cum.size - 1)
        near = np.minimum(near, np.abs(cum[j] - draws))
    near = np.minimum(near, np.abs(draws))  # the boundary C(-1) = 0
    far = near > tol

    def got_for(indices):
        return st_or_got(indices) if callable(st_or_got) else st_or_got[tuple(indices)]

    for indices in _index_lists(n):
        got = got_for(indices)
        assert got.dtype == np.uint64 and got.shape == draws.shape
        for k in np.nonzero(far)[0]:
            assert int(got[k]) == qo.soft_measure(n, indices, psi, float(draws[k])), (indices, draws[k])
    idx = got_for(list(range(n))[::-1]).astype(np.int64)  # bit i <-> qubit n-1-i <-> index bit i: the index itself
    total = cum[-1]
    for r, i in zip(draws, idx):
        if i == 0:
            assert r <= cum[0] + tol or r > total - tol, (r, cum[0], total)
        else:
            assert cum[i - 1] - tol < r <= cum[i] + tol, (r, i, cum[i - 1], cum[i])


def test_reference_doctest_sampled(ctx):
    # measurement_ops.rs:136-152
    inp = from_reals([0.0, 0.0, 1.0, 0.0])
    with State(2, np.complex128, ctx) as st:
        st.upload(inp)
        draws = np.array([0.3, 0.5, 0.999])
        for indices, want in (([0], 1), ([1], 0), ([0, 1], 0b01), ([1, 0], 0b10)):
            got = st.sample(indices, draws)
            assert list(got) == [want] * 3, indices
            for r in draws:
                assert st.soft_measure(indices, r) == want == qo.soft_measure(2, indices, inp, r)
            assert list(st.sample(indices, [0.0])) == [0] == [st.soft_measure(indices, 0.0)]
            assert qo.soft_measure(2, indices, inp, 0.0) == 0


@pytest.mark.parametrize("n", [10, 14])
@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-6)])
def test_oracle_parity(ctx, n, dtype, tol):
    psi = circuits.random_state(n, 100 + n, dtype)
    draws = _draws(n, 4096)
    with State(n, dtype, ctx) as st:
        st.upload(psi)
        _check_against_oracle(n, psi, lambda ix: st.sample(ix, draws), draws, tol)


@pytest.mark.parametrize("dtype,tol", [(np.complex128, 1e-12), (np.complex64, 1e-6)])
def test_unnormalised_state(ctx, dtype, tol):
    n = 14
    psi = (circuits.random_state(n, 7, dtype) * 0.5).astype(dtype)  # total 0.25
    draws = np.concatenate([_draws(3, 2048), [0.2499, 0.26, 0.5, 0.99]])
    with State(n, dtype, ctx) as st:
        st.upload(psi)
        for indices in _index_lists(n):
            got = st.sample(indices, draws)
            assert np.all(got[draws > 0.25 + tol] == 0), indices
        _check_against_oracle(n, psi, lambda ix: st.sample(ix, draws), draws, tol)


def _far_draws(psi, k, seed, tol=1e-12):
    cum = np.cumsum(np.abs(psi) ** 2)
    r = np.random.default_rng(seed).random(4 * k)
    pos = np.searchsorted(cum, r)
    near = np.minimum(np.abs(cum[np.clip(pos, 0, cum.size - 1)] - r), np.abs(cum[np.clip(pos - 1, 0, cum.size - 1)] - r))
    return r[near > tol][:k]


def test_agrees_with_soft_measure_on_jit_path(ctx, monkeypatch):
    monkeypatch.setenv("QIPB200_JIT", "sync")
    n = 22
    with State(n, np.complex128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule(circuits.random_circuit(n, 12, 0x5EED0002, "H,T,CNOT"))
        draws = _far_draws(st.download(), 64, 5)
        assert draws.size == 64
        for indices in ([0], [21, 3, 10], list(range(n))):
            got = st.sample(indices, draws)
            assert [int(g) for g in got] == [st.soft_measure(indices, r) for r in draws], indices


def test_agrees_with_soft_measure_n28(ctx):
    # 4 GiB: no host copy.  With 2^28 boundaries a seeded uniform lies within rounding distance (~1e-16) of one
    # with probability ~1e-7, so the 64 fixed draws are compared one by one.
    n = 28
    with State(n, np.complex128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0002, "H,T,CNOT"))
        draws = np.random.default_rng(28).random(64)
        for indices in ([0], [27, 0, 13], list(range(n))):
            got = st.sample(indices, draws)
            assert [int(g) for g in got] == [st.soft_measure(indices, r) for r in draws], indices


def test_statistics_match_measure_probs(ctx):
    n, K = 24, 1 << 20
    indices = [0, 5, 17, 23]
    with State(n, np.complex128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule(circuits.random_circuit(n, 10, 0x5EED0003, "H,T,CNOT"))
        p = st.measure_probs(indices)
        got = st.sample(indices, shots=K, rng=np.random.default_rng(2024))
    freq = np.bincount(got.astype(np.int64), minlength=1 << len(indices)) / K
    bound = 6 * np.sqrt(p * (1 - p) / K) + 1e-9
    assert np.all(np.abs(freq - p) <= bound), (freq, p)


def test_state_untouched_and_deterministic(ctx):
    n = 16
    with State(n, np.complex128, ctx) as st:
        st.set_basis(3)
        st.apply_schedule(circuits.random_circuit(n, 10, 9, "H,T,CNOT"))
        before = st.download()
        draws = _draws(16, 1 << 14)
        a = st.sample(list(range(n)), draws)
        b = st.sample(list(range(n)), draws)
        after = st.download()
    assert np.array_equal(a, b)
    assert before.tobytes() == after.tobytes()


def test_launch_count_independent_of_draws(ctx):
    n = 20
    with State(n, np.complex128, ctx) as st:
        st.upload(circuits.random_state(n, 21))
        deltas = []
        for k in (1, 1 << 16):
            l0 = ctx.kernel_launches()
            st.sample([0, 7], shots=k, rng=np.random.default_rng(k))
            deltas.append(ctx.kernel_launches() - l0)
    assert deltas[0] == deltas[1] > 0, deltas


_ROTATE_WORKER = r"""
import os
import sys
import numpy as np
sys.path.insert(0, os.path.join(os.environ["PYTHONPATH"], "tests"))
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State
from oracle import qip_oracle as qo
from test_gpu_sample import _check_against_oracle, _draws

with Context(0) as ctx:
    # two schedules back to back leave the state in a rotated layout; sample before any download
    for n, jit in [(16, "off"), (18, "sync")]:
        os.environ["QIPB200_JIT"] = jit
        a = circuits.random_circuit(n, 10, 11, "H,T,CNOT")
        b = circuits.qft(n)[:60] + circuits.random_circuit(n, 5, 12, "H,CZ,CNOT")
        want = qo.run_pipeline(n, a + b, 5, np.complex128)
        draws = _draws(n, 512)
        with State(n, np.complex128, ctx) as st:
            st.set_basis(5)
            st.apply_schedule(a)
            st.apply_schedule(b)
            assert not np.array_equal(st.qubit_map(), np.arange(n)[::-1]), "the layout is not rotated"
            got = {tuple(ix): st.sample(ix, draws) for ix in ([0], [9, 0, 4], list(range(n)), list(range(n))[::-1])}
            psi = st.download()  # the amplitudes that were sampled, in canonical order
        assert float(np.max(np.abs(psi - want))) <= 1e-10
        _check_against_oracle(n, psi, got, draws, 1e-12)
        print("rotate sample n=%d jit=%s: OK" % (n, jit))
"""


def test_sample_on_rotated_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=420)
    sys.stdout.write(p.stdout[-3000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]


def test_errors(ctx):
    n = 6
    with State(n, np.complex128, ctx) as st:
        st.set_basis(1)
        for bad in ([], [0, 0], [n]):
            with pytest.raises(CircuitError) as e_soft:
                st.soft_measure(bad, 0.5)
            with pytest.raises(CircuitError) as e_sample:
                st.sample(bad, [0.5])
            assert str(e_sample.value) == str(e_soft.value)
            assert e_sample.value.status == e_soft.value.status
        L = _lib.lib()
        idx = (C.c_uint64 * 1)(0)
        out = (C.c_uint64 * 4)()
        assert L.qipb200_state_sample(st._h, idx, 1, None, 4, out) == QIPB200_ERR_INVALID_ARG
        draws = (C.c_double * 4)(0.1, 0.2, 0.3, 0.4)
        assert L.qipb200_state_sample(st._h, idx, 1, draws, 4, None) == QIPB200_ERR_INVALID_ARG
        l0 = ctx.kernel_launches()
        assert L.qipb200_state_sample(st._h, idx, 1, None, 0, None) == 0
        assert st.sample([0], []).shape == (0,)
        assert ctx.kernel_launches() == l0
    with State(n, np.complex128, ctx, rank=0, world_size=2) as sh:
        with pytest.raises(CircuitError) as e:
            sh.sample([0], [0.5])
        assert e.value.status == QIPB200_ERR_UNSUPPORTED
        assert "sharded" in str(e.value)
