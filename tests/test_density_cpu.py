"""Host-side checks of exact density-matrix simulation (qipb200_density_schedule, DensityMatrix, density_schedule):
the doubled schedule run by the oracle on 2n qubits against the numpy reference of tests/density_ref.py, the
superoperator bits, the generated kernels compiled on the host, NVRTC for the benchmark's noisy circuit, and the
refusals.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import density_ref as dr
from oracle import qip_oracle as qo
from rustqip_b200 import _lib, channels as ch, circuits, gates
from rustqip_b200._abi import marshal_ops, prec_of
from rustqip_b200.errors import CircuitError
from rustqip_b200.ops import MatrixOp, make_control_op, make_matrix_op, make_swap_op
from rustqip_b200.state import density_schedule

from test_jit_cpu import emul, run_jit  # noqa: F401  (the host-compiled generated kernels)

TOL = {np.complex128: 1e-12, np.complex64: 2e-5}


def rand_unitary(k, rng):
    a = rng.standard_normal((1 << k, 1 << k)) + 1j * rng.standard_normal((1 << k, 1 << k))
    return np.linalg.qr(a)[0]


def constructor_channels():
    return [ch.amplitude_damping(0.3), ch.generalized_amplitude_damping(0.2, 0.4), ch.phase_damping(0.25),
            ch.pauli_channel(0.1, 0.05, 0.2), ch.depolarizing(0.3), ch.reset(),
            ch.pauli_string_channel({"XZ": 0.1, "YY": 0.05}), ch.two_qubit_depolarizing(0.2)]


def random_items(n, rng, n_items):
    """Gates of every kind and channels (constructors and random Kraus sets on 1..min(n, 4) qubits), interleaved,
    with a channel at position 0 and one at the end; channels may share qubits."""
    cons = [c for c in constructor_channels() if c.n_qubits <= n]
    items = [(cons[int(rng.integers(len(cons)))], None)]
    for _ in range(n_items):
        kind = int(rng.integers(8))
        q = [int(x) for x in rng.permutation(n)]
        if kind == 0:
            k = int(rng.integers(1, min(n, 3) + 1))
            items.append(make_matrix_op(q[:k], rand_unitary(k, rng).reshape(-1)))
        elif kind == 1 and n >= 2:
            items.append(MatrixOp.new_sparse(q[:2], [[(1, 1j)], [(0, 1.0)], [(3, np.exp(0.3j))], [(2, -1.0)]]))
        elif kind == 2 and n >= 2:
            items.append(make_swap_op([q[0]], [q[1]]))
        elif kind == 3 and n >= 3:
            u = make_matrix_op([q[2]], rand_unitary(1, rng).reshape(-1))  # nested controls, not flattened
            inner = MatrixOp("control", [q[1], q[2]], n_control=1, inner=u)
            items.append(MatrixOp("control", [q[0], q[1], q[2]], n_control=1, inner=inner))
        elif kind == 4:
            items.append([gates.h, gates.t, gates.s][int(rng.integers(3))](q[0]))
        elif kind == 5:
            items.append((cons[int(rng.integers(len(cons)))], None))
        else:
            k = int(rng.integers(1, min(n, 4) + 1))
            items.append((dr.random_kraus(k, int(rng.integers(1, 5)), rng), None))
    items.append((cons[int(rng.integers(len(cons)))], None))
    out = []
    for it in items:  # give each channel its qubits
        if isinstance(it, tuple):
            chan = it[0]
            out.append((chan, [int(x) for x in rng.permutation(n)[: chan.n_qubits]]))
        else:
            out.append(it)
    return out


def run_emitted(n, items, dtype, rho0):
    ops = density_schedule(n, dtype, items)
    got = qo.run_pipeline(2 * n, ops, state=rho0.reshape(-1).astype(dtype), dtype=dtype)
    return got.reshape(1 << n, 1 << n), ops


def test_reference_is_pinned():
    """The reference equals KrausChannel.superop on the channel's own qubits, and unitary evolution of |psi><psi|."""
    rng = np.random.default_rng(1)
    for k in (1, 2, 3):
        kc = dr.random_kraus(k, 3, rng)
        a = rng.standard_normal((1 << k, 1 << k)) + 1j * rng.standard_normal((1 << k, 1 << k))
        rho = a @ a.conj().T
        assert np.allclose(dr.evolve(k, [(kc, list(range(k)))], rho), kc.superop(rho), atol=1e-13)
    n = 4
    ops = circuits.random_circuit(n, 3, 7)
    psi = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    u = qo.run_pipeline(n, ops, state=psi)
    assert np.allclose(dr.evolve(n, ops, np.outer(psi, psi.conj())), np.outer(u, u.conj()), atol=1e-12)


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_emitted_schedule_matches_reference(n, dtype):
    rng = np.random.default_rng(100 + n)
    items = random_items(n, rng, 14)
    rho0 = dr.basis(n, int(rng.integers(1 << n)))
    got, _ = run_emitted(n, items, dtype, rho0)
    want = dr.evolve(n, items, rho0)
    # f32: each of the ~30 doubled ops rounds every amplitude, error ~1e-7 relative per op
    assert np.max(np.abs(got.astype(np.complex128) - want)) <= TOL[dtype] * 10
    assert abs(np.trace(want) - 1.0) < 1e-12


def test_schedule_layout_of_gates_and_channels():
    """Each gate is followed by its conjugate on the column qubits; a channel is one MAT op on [q.., q + n..]."""
    n = 3
    ops = density_schedule(n, np.complex128, [(ch.depolarizing(0.1), [2]), gates.t(1),
                                              make_control_op([0], make_matrix_op([2], rand_unitary(1, np.random.default_rng(2)).reshape(-1))),
                                              make_swap_op([0], [1]), (ch.reset(), [2])])
    kinds = [(o.kind, o.indices()) for o in ops]
    assert kinds == [("matrix", [2, 5]), ("matrix", [1]), ("matrix", [4]), ("control", [0, 2]), ("control", [3, 5]),
                     ("swap", [0, 1]), ("swap", [3, 4]), ("matrix", [2, 5])]
    assert np.array_equal(ops[2].data, np.conj(ops[1].data))
    assert np.array_equal(ops[4].inner.data, np.conj(ops[3].inner.data))


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_superoperator_bits(dtype):
    rng = np.random.default_rng(5)
    chans = constructor_channels() + [dr.random_kraus(k, m, rng) for k, m in ((1, 3), (2, 5), (3, 2), (4, 2))]
    for chan in chans:
        k = chan.n_qubits
        qs = list(range(k))[::-1]
        ops = density_schedule(4, dtype, [(chan, qs)])
        assert len(ops) == 1 and ops[0].indices() == qs + [q + 4 for q in qs]
        want = dr.superop_bits(chan, dtype).reshape(-1)
        got = np.asarray(ops[0].data).astype(dtype)
        assert got.tobytes() == want.tobytes(), chan


def test_generated_kernels_on_host_match_oracle(emul):  # noqa: F811
    """n = 7 (a 14-qubit vector) with single-qubit channels: the host-compiled generated tile kernels give the
    oracle's result."""
    n = 7
    items = circuits.noisy_random_circuit(n, 3, 0x5EED0007, gamma=0.05, lam=0.03)
    ops = density_schedule(n, np.complex128, items)
    rho0 = dr.basis(n, 5).reshape(-1)
    want = qo.run_pipeline(2 * n, ops, state=rho0)
    got, stats = run_jit(emul, 2 * n, ops, rho0, np.complex128)
    assert stats[0] >= 1
    assert np.max(np.abs(got - want)) <= 1e-12
    assert np.max(np.abs(want.reshape(1 << n, 1 << n) - dr.evolve(n, items, dr.basis(n, 5)))) <= 1e-12


def test_nvrtc_compiles_every_pass_of_the_noisy_bench_circuit():
    """The benchmark's noisy circuit (n = 15, f64: a 30-qubit vector): every pass has a generated kernel and each
    compiles with NVRTC for sm_90a."""
    items = circuits.noisy_random_circuit(15, 20, 0x5EED0015)
    ops = density_schedule(15, np.complex128, items)
    arr, keep = marshal_ops(ops, prec_of(np.complex128))
    out = (C.c_double * 5)()
    log = C.create_string_buffer(4000)
    rc = _lib.lib().qipb200_jit_precompile(prec_of(np.complex128), 30, arr, len(ops), out, log, 4000)
    assert rc == 0, log.value
    assert out[0] >= 1 and out[1] == out[0] and out[2] == out[0], (list(out), log.value)


def _raw_schedule(n, ops, positions, chans, qubits, cap):
    prec = prec_of(np.complex128)
    arr, keep = marshal_ops(ops, prec)
    arity, n_kraus, kraus = ch.marshal([ch.KrausChannel(c) for c in chans])
    pos = np.ascontiguousarray(np.asarray(positions, dtype=np.uint64))
    qa = np.ascontiguousarray(np.asarray(qubits, dtype=np.uint64))
    buf = (C.c_ubyte * max(1, cap))()
    ln = C.c_size_t(0)
    nc = len(chans)
    st = _lib.lib().qipb200_density_schedule(
        prec, n, arr, len(ops), nc, pos.ctypes.data if nc else None, arity.ctypes.data if nc else None,
        qa.ctypes.data if nc else None, n_kraus.ctypes.data if nc else None, kraus.ctypes.data if nc else None,
        buf, cap, C.byref(ln))
    return st, ln.value


def test_host_refusals():
    ops = [gates.h(0), gates.cnot(0, 1)]
    damp = ch.amplitude_damping(0.1)
    assert _raw_schedule(2, ops, [1], [damp], [1], 1 << 16)[0] == 0
    assert _raw_schedule(0, [], [], [], [], 1 << 16)[0] == 1                 # n = 0
    assert _raw_schedule(2, [gates.h(2)], [], [], [], 1 << 16)[0] == 3       # an op's qubit >= n
    assert _raw_schedule(2, ops, [0], [damp], [2], 1 << 16)[0] == 3          # a channel's qubit >= n
    assert _raw_schedule(2, ops, [2, 1], [damp, damp], [0, 1], 1 << 16)[0] == 1  # decreasing positions
    assert _raw_schedule(2, ops, [3], [damp], [0], 1 << 16)[0] == 1          # position > n_ops
    st, need = _raw_schedule(2, ops, [1], [damp], [1], 16)                    # buffer too small
    assert st == 2 and need > 16
    assert _raw_schedule(2, ops, [1], [damp], [1], need) == (0, need)
    # an incomplete channel (KrausChannel refuses it too, so marshal the raw operator)
    prec = prec_of(np.complex128)
    arity = np.array([1], dtype=np.uint32)
    n_kraus = np.array([1], dtype=np.uint32)
    kraus = np.ascontiguousarray(np.array([[1, 0], [0, 0.5]], dtype=np.complex128).reshape(-1).view(np.float64))
    pos, qa = np.array([0], dtype=np.uint64), np.array([0], dtype=np.uint64)
    ln = C.c_size_t(0)
    st = _lib.lib().qipb200_density_schedule(prec, 2, None, 0, 1, pos.ctypes.data, arity.ctypes.data,
                                             qa.ctypes.data, n_kraus.ctypes.data, kraus.ctypes.data, None, 0,
                                             C.byref(ln))
    assert st == 1
    assert b"not complete" in _lib.lib().qipb200_last_error(None)
    # a qubit repeated inside one channel is refused; in two channels it is not
    with pytest.raises(CircuitError):
        density_schedule(3, np.complex128, [(ch.two_qubit_depolarizing(0.1), [1, 1])])
    assert len(density_schedule(3, np.complex128, [(damp, [1]), (damp, [1])])) == 2


def test_kraus_layer_rule_unchanged():
    """apply_kraus_channels still refuses a qubit in two channels of one layer (its plan checks the same rule)."""
    from rustqip_b200.state import kraus_channels_plan
    damp = ch.amplitude_damping(0.1)
    with pytest.raises(CircuitError):
        kraus_channels_plan(3, np.complex128, [damp, damp], [[1], [1]])
