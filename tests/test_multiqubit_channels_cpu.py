"""Channels on one to four qubits along quantum trajectories without a GPU: the sampling argument by exact enumeration
over layers that mix arities and straddle an index byte, the emulation of tests/multiqubit_channel_ref.py against
dense Kraus products and against channel_ref for single-qubit layers, the constructors, tensor and compose, every
refusal of qipb200_multiqubit_channels_plan, the plan's counts, and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import channel_ref as cr
import multiqubit_channel_ref as mr
from rustqip_b200 import _lib
from rustqip_b200 import channels as ch
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import channels_plan, multiqubit_channels_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG, BAD_INDEX = 1, 3
F64 = 1  # QIP_F64


def random_channel(rng, k, m=None):
    """m random operators d(b)|b ^ f> on k qubits (random masks and zeros), completed column by column."""
    D = 1 << k
    m = m or int(rng.integers(1, 4))
    for _ in range(100):
        ks = []
        for _ in range(m):
            f = int(rng.integers(0, D))
            d = rng.normal(size=D) + 1j * rng.normal(size=D)
            d[rng.random(D) < (0.2 if m > 1 else 0.0)] = 0
            if not np.any(d):
                d[0] = 1.0
            K = np.zeros((D, D), dtype=np.complex128)
            K[np.arange(D) ^ f, np.arange(D)] = d
            ks.append(K)
        s = np.array([sum(mr.weights(K)[b] for K in ks) for b in range(D)])
        if min(s) == 0:
            continue
        try:
            return ch.Channel([K / np.sqrt(s)[None, :] for K in ks])
        except ValueError:
            continue
    raise AssertionError("no random channel")


def random_state(n, rng):
    v = rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)
    return v / np.linalg.norm(v)


def random_layer(rng, n, straddle=True):
    """Disjoint qubit groups of sizes 1..4 with random channels; with straddle, one group holds qubits n - 9 and n - 8
    (physical bits 8 and 7, across the first index-byte boundary)."""
    free = [int(q) for q in rng.permutation(n)]
    groups = []
    if straddle:
        g = [n - 9, n - 8] if rng.random() < 0.5 else [n - 8, n - 9]
        free = [q for q in free if q not in g]
        groups.append(g)
    while free and len(groups) < 4:
        k = min(int(rng.integers(1, 5)), len(free))
        groups.append(free[:k])
        free = free[k:]
    chans = [random_channel(rng, len(g), m=int(rng.integers(1, 3))) for g in groups]
    return groups, chans


def marginal(psi, n, qubits):
    P = np.zeros(1 << len(qubits))
    idx = np.arange(1 << n)
    x = np.zeros(1 << n, dtype=np.int64)
    for k, q in enumerate(qubits):
        x |= ((idx >> (n - 1 - q)) & 1) << k
    np.add.at(P, x, np.abs(psi) ** 2)
    return P


def dep_qubits(groups, chans):
    return [q for g, c in zip(groups, chans) if c.state_dependent for q in g]


@pytest.mark.parametrize("seed", range(6))
def test_sampling_by_enumeration(seed):
    """Every tuple's probability from x ~ P and the per-channel weights equals <psi|(x)_c K^dagger K|psi>, and the
    emulated state for that tuple is K psi / sqrt(p)."""
    rng = np.random.default_rng(seed)
    n = 9 + seed % 2
    groups, chans = random_layer(rng, n)
    psi = random_state(n, rng)
    dep = dep_qubits(groups, chans)
    P = marginal(psi, n, dep)
    for tup in itertools.product(*[range(len(c)) for c in chans]):
        ops = [c.kraus[i] for c, i in zip(chans, tup)]
        phi = mr.apply_dense(psi, n, groups, ops)
        p = float(np.vdot(phi, phi).real)
        induced = 0.0
        for x in np.flatnonzero(P):
            w, kd = P[x], 0
            for g, c, i in zip(groups, chans, tup):
                b = 0
                if c.state_dependent:
                    b = mr.channel_value((int(x) >> (kd + j)) & 1 for j in range(len(g)))
                    kd += len(g)
                w *= mr.weights(c.kraus[i])[b]
            induced += w
        assert abs(induced - p) <= 1e-12, (tup, induced, p)
    # the emulated trajectory step for random draws
    for _ in range(4):
        draws = rng.random(1 + len(groups))
        x = int(np.searchsorted(np.cumsum(P), draws[0], side="right")) if dep else 0
        chosen, prob, out = mr.emulate(psi, n, groups, [c.kraus for c in chans], x, draws)
        phi = mr.apply_dense(psi, n, groups, [c.kraus[i] for c, i in zip(chans, chosen)])
        p = float(np.vdot(phi, phi).real)
        assert abs(prob - p) <= 1e-12
        assert np.max(np.abs(out - phi / np.sqrt(p))) <= 1e-12


def test_dense_product_matches_kron():
    """apply_dense and full_op agree with a Kronecker product for adjacent qubits in order."""
    rng = np.random.default_rng(3)
    a, b = random_channel(rng, 2).kraus[0], random_channel(rng, 1).kraus[0]
    M = mr.full_op(4, [[1, 2], [3]], [a, b])
    assert np.allclose(M, np.kron(np.eye(2), np.kron(a, b)))
    swap = mr.full_op(2, [[1, 0]], [np.kron(ch._X, ch._Z)])
    assert np.allclose(swap, np.kron(ch._Z, ch._X))


@pytest.mark.parametrize("seed", range(4))
def test_single_qubit_emulation_is_channel_ref(seed):
    """Every arity 1: the choices, prob and state equal channel_ref.emulate bit for bit."""
    rng = np.random.default_rng(50 + seed)
    n = 10
    psi = random_state(n, rng)
    psi[rng.integers(0, 1 << n, size=2)] = complex(-0.0, -0.0)
    nc = int(rng.integers(2, n + 1))
    qubits = [int(q) for q in rng.permutation(n)[:nc]]
    chans = [random_channel(rng, 1) for _ in qubits]
    chans[0] = ch.depolarizing(0.3)
    draws = rng.random(1 + nc)
    dep = [q for q, c in zip(qubits, chans) if c.state_dependent]
    x = int(np.searchsorted(np.cumsum(marginal(psi, n, dep)), draws[0], side="right")) if dep else 0
    a = cr.emulate(psi, n, qubits, [c.kraus for c in chans], x, draws)
    b = mr.emulate(psi, n, [[q] for q in qubits], [c.kraus for c in chans], x, draws)
    assert a[0] == b[0]
    assert np.float64(a[1]).tobytes() == np.float64(b[1]).tobytes()
    assert np.array_equal(a[2].view(np.uint8), b[2].view(np.uint8))


def test_constructors_tensor_and_compose():
    rng = np.random.default_rng(9)
    X, Y, Z, I = ch._X, ch._Y, ch._Z, ch._I
    paulis = [np.kron(a, b) for a in (I, X, Y, Z) for b in (I, X, Y, Z)]
    v = rng.normal(size=4) + 1j * rng.normal(size=4)
    rho = np.outer(v, v.conj()) / np.vdot(v, v).real
    for p in (0.0, 0.01, 0.3, 1.0):
        d = ch.two_qubit_depolarizing(p)
        assert d.n_qubits == 2 and not d.state_dependent
        assert sum(k.conj().T @ k for k in d.kraus) == pytest.approx(np.eye(4), abs=1e-12)
        want = (1 - p) * rho + p / 15 * sum(P @ rho @ P for P in paulis[1:])
        assert np.allclose(d.superop(rho), want, atol=1e-14)
    zz = ch.pauli_string_channel({"ZZ": 0.2})
    assert len(zz) == 2 and np.allclose(zz.superop(rho), 0.8 * rho + 0.2 * paulis[15] @ rho @ paulis[15])
    three = ch.pauli_string_channel({"XYZ": 0.1, "zzi": 0.05})
    assert three.n_qubits == 3 and sum(k.conj().T @ k for k in three.kraus) == pytest.approx(np.eye(8), abs=1e-12)
    for bad in ({"II": 0.1}, {"XQ": 0.1}, {"X": 0.1, "XX": 0.1}, {"XXXXX": 0.1}):
        with pytest.raises(ValueError):
            ch.pauli_string_channel(bad)
    a, b = ch.amplitude_damping(0.3), ch.phase_damping(0.2)
    t = a.tensor(b)
    assert t.n_qubits == 2 and t.state_dependent and len(t) == len(a) * len(b)
    assert np.array_equal(t.kraus, np.array([np.kron(x, y) for x in a.kraus for y in b.kraus]))
    sep = np.kron(np.diag([0.6, 0.4]), np.diag([0.3, 0.7])).astype(np.complex128)
    assert np.allclose(t.superop(sep), np.kron(a.superop(np.diag([0.6, 0.4])), b.superop(np.diag([0.3, 0.7]))))
    c = t.compose(ch.two_qubit_depolarizing(0.1))
    assert np.allclose(c.superop(rho), ch.two_qubit_depolarizing(0.1).superop(t.superop(rho)), atol=1e-14)
    reset2 = ch.Channel([np.outer(np.eye(4)[0], np.eye(4)[b]) for b in range(4)])
    assert reset2.state_dependent and np.allclose(reset2.superop(rho), np.diag([1.0, 0, 0, 0]))
    assert ch.reset().tensor(ch.reset()).n_qubits == 2
    with pytest.raises(ValueError):
        a.compose(t)
    with pytest.raises(ValueError):
        t.tensor(t).tensor(a)
    for bad in ([np.ones((4, 4)) / 2], [np.eye(3)], [np.zeros((4, 4))], [np.diag([1.0, 1.0, 1.0, 0.5])],
                [np.eye(4)] * 257):
        with pytest.raises(ValueError):
            ch.Channel(bad)
    assert ch.Channel([np.eye(2)] * 1).n_qubits == 1
    with pytest.raises(ValueError):  # a single-qubit channel keeps the limit of 16
        ch.Channel([np.eye(2) / 17 ** 0.5] * 17)


def _plan_call(n, arity, qubits, n_kraus, kraus, prec=F64, out=True):
    L = _lib.lib()
    aa = (C.c_uint32 * max(1, len(arity)))(*arity) if arity is not None else None
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits) if qubits is not None else None
    na = (C.c_uint32 * max(1, len(n_kraus)))(*n_kraus) if n_kraus is not None else None
    ka = (C.c_double * max(1, len(kraus)))(*kraus) if kraus is not None else None
    v = (C.c_uint32 * 4)()
    nc = len(n_kraus) if n_kraus is not None else len(arity)
    st = L.qipb200_multiqubit_channels_plan(prec, n, nc, aa, qa, na, ka, v if out else None)
    return st, L.qipb200_last_error(None).decode()


def _flat(*ops):
    return [float(v) for k in ops for v in np.asarray(k, dtype=np.complex128).reshape(-1).view(np.float64)]


def test_plan_refusals():
    I2, I4 = np.eye(2), np.eye(4)
    cx = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]])  # columns 2 and 3 swap, 0 and 1 stay
    w = "multiqubit_channels_plan"
    cases = [
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(I2), out=False), INVALID_ARG,
         w + ": NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=41, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=4, arity=None, qubits=[0], n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL arity, qubits, n_kraus or kraus"),
        (dict(n=4, arity=[1], qubits=None, n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL arity, qubits, n_kraus or kraus"),
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[1], kraus=None), INVALID_ARG,
         w + ": NULL arity, qubits, n_kraus or kraus"),
        (dict(n=6, arity=[2, 0], qubits=[0, 1], n_kraus=[1, 1], kraus=_flat(I4, I2)), INVALID_ARG,
         w + ": channel 1: arity must be 1..4, got 0"),
        (dict(n=6, arity=[5], qubits=[0, 1, 2, 3, 4], n_kraus=[1], kraus=[1.0]), INVALID_ARG,
         w + ": channel 0: arity must be 1..4, got 5"),
        (dict(n=4, arity=[2], qubits=[1, 4], n_kraus=[1], kraus=_flat(I4)), BAD_INDEX,
         w + ": channel 0: qubit 4 out of range for 4 qubits"),
        (dict(n=4, arity=[2], qubits=[2, 2], n_kraus=[1], kraus=_flat(I4)), BAD_INDEX,
         w + ": channel 0: qubit 2 repeated"),
        (dict(n=4, arity=[1, 2], qubits=[3, 0, 3], n_kraus=[1, 1], kraus=_flat(I2, I4)), BAD_INDEX,
         w + ": channel 1: qubit 3 repeated"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[0], kraus=_flat(I4)), INVALID_ARG,
         w + ": channel 0: n_kraus must be 1..256, got 0"),
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[257], kraus=_flat(*([I2] * 257))), INVALID_ARG,
         w + ": channel 0: n_kraus must be 1..256, got 257"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[2], kraus=_flat(I4, np.diag([np.inf, 0, 0, 0]))),
         INVALID_ARG, w + ": channel 0, operator 1: an entry is not finite"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[2], kraus=_flat(I4, np.zeros((4, 4)))), INVALID_ARG,
         w + ": channel 0, operator 1: the zero matrix"),
        (dict(n=4, arity=[1, 2], qubits=[3, 0, 1], n_kraus=[1, 1], kraus=_flat(I2, cx)), INVALID_ARG,
         w + ": channel 1, operator 0: not of the form K|b> = d(b)|b ^ f> (one nonzero entry per column, one f)"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[1], kraus=_flat(np.ones((4, 4)) / 2)), INVALID_ARG,
         w + ": channel 0, operator 0: not of the form K|b> = d(b)|b ^ f> (one nonzero entry per column, one f)"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[1], kraus=_flat(np.diag([1.0, 1.0, 0.5, 1.0]))), INVALID_ARG,
         w + ": channel 0: the operators are not complete (sum of |d_i(2)|^2 - 1 = -0.75)"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[1], kraus=_flat(np.diag([1.0, 1.0, 1.0, 1.0 + 1e-11]))),
         INVALID_ARG, w + ": channel 0: the operators are not complete (sum of |d_i(3)|^2 - 1 = 2e-11)"),
    ]
    for kw, code, msg in cases:
        assert _plan_call(**kw) == (code, msg), kw
    reset2 = [np.outer(np.eye(4)[0], np.eye(4)[b]) for b in range(4)]  # zero columns are allowed
    assert _plan_call(4, [2], [0, 3], [4], _flat(*reset2))[0] == 0
    assert _plan_call(4, [], [], [], [])[0] == 0
    with pytest.raises(CircuitError):
        multiqubit_channels_plan(4, np.complex128, ch.two_qubit_depolarizing(0.1), [[0, 1], [1, 2]])
    with pytest.raises(ValueError):
        multiqubit_channels_plan(4, np.complex128, ch.two_qubit_depolarizing(0.1), [[0]])
    with pytest.raises(ValueError):
        channels_plan(4, np.complex128, ch.two_qubit_depolarizing(0.1), [0])


def test_plan_counts():
    c128 = np.complex128
    dep2 = ch.two_qubit_depolarizing(0.01)
    pairs = [[2 * i, 2 * i + 1] for i in range(15)]
    assert multiqubit_channels_plan(30, c128, dep2, pairs) == (0, 0, 1, 1)
    ad2 = ch.amplitude_damping(0.01).tensor(ch.amplitude_damping(0.02))
    assert multiqubit_channels_plan(30, c128, [dep2, ad2], [[0, 1], [2, 17]]) == (1, 3, 1, 12)
    assert multiqubit_channels_plan(30, c128, ch.two_qubit_depolarizing(0.0), [[4, 5]]) == (0, 0, 0, 0)
    assert multiqubit_channels_plan(8, c128, [], []) == (0, 0, 0, 0)
    # single-qubit layers count as channels_plan does
    assert multiqubit_channels_plan(30, c128, ch.amplitude_damping(0.01), [[q] for q in range(30)]) == \
        channels_plan(30, c128, ch.amplitude_damping(0.01), range(30))
    rng = np.random.default_rng(5)
    for _ in range(20):
        groups, chans = random_layer(rng, 10)
        assert multiqubit_channels_plan(10, c128, chans, groups) == mr.plan([c.kraus for c in chans])


def test_tables_fold_one_byte_and_gather_the_rest():
    """Groups inside one index byte fold into that byte's table, the others are gathered in operator order."""
    ops = [np.diag([1, 1j, -1, 1]), np.kron(ch._X, ch._Z), np.diag([1, -1]), np.eye(8)[:, [1, 0, 3, 2, 5, 4, 7, 6]]]
    tabs, F = mr.tables([[3, 1], [8, 7], [2], [33, 20, 9]], ops)
    assert [(t[0], t[1]) for t in tabs] == [("byte", 0), ("gat", [8, 7]), ("gat", [33, 20, 9])]
    assert F == (1 << 8) | (1 << 9)
    # byte 0: value v has bit 3 -> b's top bit, bit 1 -> its low bit, bit 2 -> the Z
    v = (1 << 3) | (1 << 2)
    assert (tabs[0][2][v], tabs[0][3][v]) == (1.0, 0.0)  # d(2) = -1 times Z(1) = -1


def test_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "use_multiqubit_channels.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::B200State<double> &st) {\n"
                   "  std::vector<double> k(32, 0.0);\n"
                   "  for (int i = 0; i < 4; ++i) k[2 * (4 * i + i)] = 1.0;  // the identity on two qubits\n"
                   "  auto r = st.apply_multiqubit_channels({2}, {0, 1}, {1}, k, {0.5, 0.25});\n"
                   "  return r.second + (double)r.first.at(0);\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
