"""Single-qubit channels along quantum trajectories without a GPU: the sampling argument by exact enumeration, the
emulation of tests/channel_ref.py against dense Kraus products, the constructors and compose of rustqip_b200.channels,
every refusal of qipb200_channels_plan, the plan's counts, and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import channel_ref as cr
from rustqip_b200 import _lib
from rustqip_b200 import channels as ch
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import channels_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG, BAD_INDEX = 1, 3
F64 = 1  # QIP_F64


def random_channel(rng, m=None):
    """m random monomial operators (random diagonal / anti-diagonal patterns and zeros), completed column by column."""
    m = m or int(rng.integers(1, 5))
    for _ in range(100):
        ks = []
        for _ in range(m):
            d = rng.normal(size=2) + 1j * rng.normal(size=2)
            d[rng.random(2) < 0.2] = 0
            if not np.any(d):
                d[0] = 1.0
            ks.append(np.array([[0, d[1]], [d[0], 0]]) if rng.random() < 0.4 else np.diag(d))
        s = [sum(cr.weights(k)[b] for k in ks) for b in (0, 1)]
        if min(s) == 0:
            continue
        scale = np.array([1 / np.sqrt(s[0]), 1 / np.sqrt(s[1])])  # column b of every operator times 1/sqrt(s_b)
        ks = [k * scale[None, :] for k in ks]
        try:
            return ch.Channel(ks)
        except ValueError:
            continue
    raise AssertionError("no random channel")


def random_state(n, rng):
    v = rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)
    return v / np.linalg.norm(v)


def marginal(psi, n, qubits):
    """P(x) of the qubits (bit k of x <-> qubits[k])."""
    P = np.zeros(1 << len(qubits))
    idx = np.arange(1 << n)
    x = np.zeros(1 << n, dtype=np.int64)
    for k, q in enumerate(qubits):
        x |= ((idx >> (n - 1 - q)) & 1) << k
    np.add.at(P, x, np.abs(psi) ** 2)
    return P


@pytest.mark.parametrize("seed", range(8))
def test_sampling_argument_by_enumeration(seed):
    rng = np.random.default_rng(seed)
    n = 5 + seed % 2
    nc = 1 + seed % 4
    qubits = [int(q) for q in rng.permutation(n)[:nc]]
    chans = [random_channel(rng) for _ in range(nc)]
    psi = random_state(n, rng)
    rho = np.outer(psi, psi.conj())
    dep = [q for q, c in zip(qubits, chans) if c.state_dependent]
    P = marginal(psi, n, dep)
    want = np.zeros_like(rho)
    got = np.zeros_like(rho)
    total = 0.0
    for tup in itertools.product(*[range(len(c)) for c in chans]):
        K = cr.full_op(n, qubits, [c.kraus[i] for c, i in zip(chans, tup)])
        phi = K @ psi
        p = float(np.vdot(phi, phi).real)
        want += K @ rho @ K.conj().T
        # the distribution the call draws from: x ~ P, then i_c ~ |d_i(x_c)|^2 independently
        induced = 0.0
        for x in range(len(P)):
            w, kd = P[x], 0
            for c, i in zip(chans, tup):
                if c.state_dependent:
                    b = (x >> kd) & 1
                    kd += 1
                else:
                    b = 0
                w *= cr.weights(c.kraus[i])[b]
            induced += w
        assert abs(induced - p) <= 1e-12, (tup, induced, p)
        total += p
        if p > 0:
            got += p * np.outer(phi / np.sqrt(p), (phi / np.sqrt(p)).conj())
    assert abs(total - 1.0) <= 1e-12
    assert np.max(np.abs(got - want)) <= 1e-12


@pytest.mark.parametrize("seed", range(6))
def test_choice_follows_the_weights(seed):
    """chosen = i on a u-interval of length e_i / S_b: a fine grid of u lands on i in that proportion."""
    rng = np.random.default_rng(100 + seed)
    c = random_channel(rng, m=int(rng.integers(1, 9)))
    grid = (np.arange(1 << 14) + 0.5) / (1 << 14)
    for b in (0, 1):
        e = np.array([cr.weights(k)[b] for k in c.kraus])
        counts = np.bincount([cr.choose(c.kraus, b, u) for u in grid], minlength=len(c)) / len(grid)
        assert np.max(np.abs(counts - e / e.sum())) <= 2.0 / len(grid)
        assert all(e[cr.choose(c.kraus, b, u)] > 0 for u in (0.0, 1 - 2 ** -53))


@pytest.mark.parametrize("seed", range(10))
def test_emulation_is_the_normalised_kraus_product(seed):
    """The emulated trajectory step equals K psi / sqrt(p) for the tuple it chose, and prob equals p."""
    rng = np.random.default_rng(200 + seed)
    n = 5 + seed % 2
    nc = 1 + seed % 4
    qubits = [int(q) for q in rng.permutation(n)[:nc]]
    chans = [random_channel(rng) for _ in range(nc)]
    if seed % 3 == 0:
        chans[0] = ch.depolarizing(0.3)
    psi = random_state(n, rng)
    dep = [q for q, c in zip(qubits, chans) if c.state_dependent]
    draws = rng.random(1 + nc)
    P = np.cumsum(marginal(psi, n, dep))
    x = int(np.searchsorted(P, draws[0], side="right")) if dep else 0
    chosen, prob, out = cr.emulate(psi, n, qubits, [c.kraus for c in chans], x, draws)
    K = cr.full_op(n, qubits, [c.kraus[i] for c, i in zip(chans, chosen)])
    phi = K @ psi
    p = float(np.vdot(phi, phi).real)
    assert abs(prob - p) <= 1e-12
    assert np.max(np.abs(out - phi / np.sqrt(p))) <= 1e-12


def test_constructors_are_complete_and_compose_matches_dense_products():
    rho = np.array([[0.6, 0.2 - 0.1j], [0.2 + 0.1j, 0.4]])
    g, lam, p = 0.3, 0.2, 0.15
    made = [ch.amplitude_damping(g), ch.generalized_amplitude_damping(g, 0.7), ch.phase_damping(lam),
            ch.depolarizing(p), ch.pauli_channel(0.1, 0.05, 0.2), ch.reset(), ch.amplitude_damping(0.0),
            ch.amplitude_damping(1.0), ch.depolarizing(0.0)]
    for c in made:
        assert sum(k.conj().T @ k for k in c.kraus) == pytest.approx(np.eye(2), abs=1e-12)
    assert np.allclose(ch.reset().superop(rho), np.diag([1.0, 0.0]))
    assert np.allclose(ch.depolarizing(p).superop(rho), (1 - 4 * p / 3) * rho + (2 * p / 3) * np.eye(2))
    ad = ch.amplitude_damping(g).superop(rho)
    assert ad == pytest.approx(np.array([[rho[0, 0] + g * rho[1, 1], np.sqrt(1 - g) * rho[0, 1]],
                                         [np.sqrt(1 - g) * rho[1, 0], (1 - g) * rho[1, 1]]]), abs=1e-15)
    assert [c.state_dependent for c in made[:6]] == [True, True, True, False, False, True]
    a, b = ch.amplitude_damping(g), ch.phase_damping(lam)
    t = a.compose(b)
    assert t.superop(rho) == pytest.approx(b.superop(a.superop(rho)), abs=1e-15)
    dense = [kb @ ka for kb in b.kraus for ka in a.kraus]
    assert len(t) == sum(1 for k in dense if np.any(k != 0))
    assert np.array_equal(t.kraus, np.array([k for k in dense if np.any(k != 0)]))
    t2 = ch.reset().compose(ch.depolarizing(0.1))
    assert t2.superop(rho) == pytest.approx(ch.depolarizing(0.1).superop(np.diag([1.0, 0.0])), abs=1e-15)
    for bad in ([np.zeros((2, 2))], [np.ones((2, 2))], [np.diag([1.0, 0.5])], [np.diag([np.nan, 1])], []):
        with pytest.raises(ValueError):
            ch.Channel(bad)


def _plan_call(n, qubits, n_kraus, kraus, prec=F64, out=True):
    L = _lib.lib()
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits) if qubits is not None else None
    na = (C.c_uint32 * max(1, len(n_kraus)))(*n_kraus) if n_kraus is not None else None
    ka = (C.c_double * max(1, len(kraus)))(*kraus) if kraus is not None else None
    v = (C.c_uint32 * 4)()
    nc = len(qubits) if qubits is not None else len(n_kraus or [])
    st = L.qipb200_channels_plan(prec, n, nc, qa, na, ka, v if out else None)
    return st, L.qipb200_last_error(None).decode()


def _flat(*ops):
    return [float(v) for k in ops for v in np.asarray(k, dtype=np.complex128).reshape(-1).view(np.float64)]


def test_plan_refusals():
    I, X = np.eye(2), np.array([[0, 1], [1, 0]])
    ad = ch.amplitude_damping(0.2).kraus
    half = np.sqrt(0.5)
    cases = [
        (dict(n=4, qubits=[0], n_kraus=[1], kraus=_flat(I), out=False), INVALID_ARG,
         "channels_plan: NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=4, qubits=[0], n_kraus=[1], kraus=_flat(I), prec=7), INVALID_ARG,
         "channels_plan: NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=41, qubits=[0], n_kraus=[1], kraus=_flat(I)), INVALID_ARG,
         "channels_plan: NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=4, qubits=None, n_kraus=[1], kraus=_flat(I)), INVALID_ARG,
         "channels_plan: NULL qubits, n_kraus or kraus"),
        (dict(n=4, qubits=[0], n_kraus=None, kraus=_flat(I)), INVALID_ARG,
         "channels_plan: NULL qubits, n_kraus or kraus"),
        (dict(n=4, qubits=[0], n_kraus=[1], kraus=None), INVALID_ARG, "channels_plan: NULL qubits, n_kraus or kraus"),
        (dict(n=4, qubits=[1, 4], n_kraus=[1, 1], kraus=_flat(I, I)), BAD_INDEX,
         "channels_plan: channel 1: qubit 4 out of range for 4 qubits"),
        (dict(n=4, qubits=[2, 2], n_kraus=[1, 1], kraus=_flat(I, I)), BAD_INDEX,
         "channels_plan: channel 1: qubit 2 repeated"),
        (dict(n=4, qubits=[0], n_kraus=[0], kraus=_flat(I)), INVALID_ARG,
         "channels_plan: channel 0: n_kraus must be 1..16, got 0"),
        (dict(n=4, qubits=[0], n_kraus=[17], kraus=_flat(*([I] * 17))), INVALID_ARG,
         "channels_plan: channel 0: n_kraus must be 1..16, got 17"),
        (dict(n=4, qubits=[0, 1], n_kraus=[1, 2], kraus=_flat(I, half * I, np.diag([np.inf, 0]))), INVALID_ARG,
         "channels_plan: channel 1, operator 1: an entry is not finite"),
        (dict(n=4, qubits=[0], n_kraus=[2], kraus=_flat(I, np.zeros((2, 2)))), INVALID_ARG,
         "channels_plan: channel 0, operator 1: the zero matrix"),
        (dict(n=4, qubits=[0], n_kraus=[2], kraus=_flat(half * I, half * np.array([[1, 1], [0, 1]]))), INVALID_ARG,
         "channels_plan: channel 0, operator 1: neither diagonal nor anti-diagonal"),
        (dict(n=4, qubits=[3], n_kraus=[2], kraus=_flat(I, X)), INVALID_ARG,
         "channels_plan: channel 0: the operators are not complete (sum of |d_i(0)|^2 - 1 = 1)"),
        (dict(n=4, qubits=[3], n_kraus=[1], kraus=_flat(np.diag([1.0, 1.0 + 1e-11]))), INVALID_ARG,
         "channels_plan: channel 0: the operators are not complete (sum of |d_i(1)|^2 - 1 = 2e-11)"),
        (dict(n=4, qubits=[3, 0], n_kraus=[2, 1], kraus=_flat(ad[0], ad[1], 0.5 * I)), INVALID_ARG,
         "channels_plan: channel 1: the operators are not complete (sum of |d_i(0)|^2 - 1 = -0.75)"),
    ]
    for kw, code, msg in cases:
        st, err = _plan_call(**kw)
        assert (st, err) == (code, msg), kw
    # within the tolerance, and the empty list
    assert _plan_call(4, [0], [1], _flat(np.diag([1.0, 1.0 + 4e-13])))[0] == 0
    assert _plan_call(4, [], [], [])[0] == 0
    with pytest.raises(CircuitError):
        channels_plan(4, np.complex128, ch.reset(), [0, 0])


def test_plan_counts():
    c128 = np.complex128
    assert channels_plan(30, c128, ch.amplitude_damping(0.01), range(30)) == (30, 3, 1, 12)
    assert channels_plan(30, c128, ch.depolarizing(0.01), range(30)) == (0, 0, 1, 1)
    assert channels_plan(30, c128, ch.reset(), range(10)) == (10, 3, 1, 12)
    assert channels_plan(30, c128, ch.depolarizing(0.0), [5]) == (0, 0, 0, 0)
    assert channels_plan(8, np.complex64, [ch.depolarizing(0.1), ch.phase_damping(0.2)], [0, 5]) == (1, 3, 1, 12)
    assert channels_plan(8, c128, [], []) == (0, 0, 0, 0)
    rng = np.random.default_rng(5)
    for _ in range(20):
        chans = [random_channel(rng) for _ in range(3)]
        assert channels_plan(6, c128, chans, [0, 2, 5]) == cr.plan([c.kraus for c in chans])


def test_cpp_mirror_apply_channels_compiles(tmp_path):
    src = tmp_path / "use_channels.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::B200State<double> &st) {\n"
                   "  std::vector<double> k = {1, 0, 0, 0, 0, 0, 0, 0,  0, 0, 1, 0, 0, 0, 0, 0};  // reset\n"
                   "  auto r = st.apply_channels({0}, {2}, k, {0.5, 0.25});\n"
                   "  return r.second + (double)r.first.at(0);\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
