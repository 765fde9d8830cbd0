"""General Kraus channels along quantum trajectories without a GPU: the grouped sequential rule by exact enumeration over
random Stinespring channels with mixed arities and group boundaries, the apply emulation of tests/kraus_channel_ref.py
against dense Kraus products, the grouping rule, KrausChannel's checks, every refusal of qipb200_kraus_channels_plan,
the plan's counts, and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import kraus_channel_ref as kr
from rustqip_b200 import _lib
from rustqip_b200 import channels as ch
from rustqip_b200.state import kraus_channels_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG, BAD_INDEX = 1, 3
F64 = 1  # QIP_F64

CX = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]], dtype=np.complex128)


def random_state(n, rng):
    v = rng.normal(size=1 << n) + 1j * rng.normal(size=1 << n)
    return v / np.linalg.norm(v)


def x_damping(g):
    """Amplitude damping along X: |-> decays to |+>."""
    H = np.array([[1, 1], [1, -1]]) / np.sqrt(2)
    return ch.KrausChannel([H @ k @ H for k in ch.amplitude_damping(g).kraus])


@pytest.mark.parametrize("seed", range(4))
def test_grouped_rule_by_enumeration(seed):
    """Every outcome tuple gets probability Tr[(x)_c M_{i_c} rho] from the grouped sequential rule, and the average of
    the post-states over all tuples is (x)_c E_c(rho)."""
    rng = np.random.default_rng(100 + seed)
    n = 8 if seed % 2 else 6 + seed % 3
    free = [int(q) for q in rng.permutation(n)]
    qubit_groups, chans = [], []
    for k in (1, 2, 1, 2, 1)[: 4 + seed % 2]:  # groups close at 4 qubits: {1, 2, 1}, {2, 1}
        g = [free.pop() for _ in range(k)]
        qubit_groups.append(g)
        chans.append(kr.stinespring(k, 2, rng))
    if seed % 2:  # a state-independent channel among them
        qubit_groups.append([free.pop()])
        chans.append(ch.KrausChannel(ch.depolarizing(0.2)))
    psi = random_state(n, rng)
    rho = np.outer(psi, psi.conj())
    total = np.zeros_like(rho)
    ptot = 0.0
    for tup in itertools.product(*[range(len(c)) for c in chans]):
        p, post = kr.trajectory_step(psi, n, qubit_groups, chans, tup)
        direct = kr.apply_dense(psi, n, qubit_groups, [chans[c].kraus[i] for c, i in enumerate(tup)])
        want = float(np.vdot(direct, direct).real)
        assert abs(p - want) <= 1e-12, (tup, p, want)
        ptot += p
        if p > 0:
            total += p * np.outer(post, post.conj())
    assert abs(ptot - 1.0) <= 1e-12
    # (x)_c E_c(rho) by the superoperators on the dense density matrix
    want = rho
    for g, c in zip(qubit_groups, chans):
        out = np.zeros_like(want)
        for K in c.kraus:
            Kf = np.stack([kr.apply_dense(e, n, [g], [K]) for e in np.eye(1 << n, dtype=np.complex128)], axis=1)
            out += Kf @ want @ Kf.conj().T
        want = out
    assert np.max(np.abs(total - want)) <= 1e-12


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_apply_emulation_matches_dense(dtype):
    rng = np.random.default_rng(7)
    n = 7
    qubit_groups = [[6, 0], [1], [5, 4, 3], [2]]  # physical bits {0, 6}, {5}, {0..2} ... straddling the low tile bits
    chans = [kr.stinespring(2, 3, rng), kr.stinespring(1, 2, rng), kr.stinespring(3, 2, rng),
             kr.stinespring(1, 3, rng)]
    psi = random_state(n, rng).astype(dtype)
    chosen = [1, 0, 1, 2]
    cond = [0.25, 0.5, 0.125, 0.3]
    got = kr.emulate_groups(psi, n, qubit_groups, chans, chosen, cond)
    ops = [chans[c].kraus[chosen[c]] / np.sqrt(cond[c]) for c in range(4)]
    want = kr.apply_dense(psi.astype(np.complex128), n, qubit_groups, ops)
    tol = 1e-13 if dtype == np.complex128 else 2e-6
    assert np.max(np.abs(got - want)) <= tol * 8


def test_grouping_rule():
    rng = np.random.default_rng(3)
    s1, s2, s3, s4 = (kr.stinespring(k, 2, rng) for k in (1, 2, 3, 4))
    dep = ch.KrausChannel(ch.depolarizing(0.1))
    assert kr.groups([s1, s2, s1, s1]) == [[0, 1, 2], [3]]
    assert kr.groups([s2, s2, s2]) == [[0, 1], [2]]
    assert kr.groups([s4, s1, s3]) == [[0], [1, 2]]
    assert kr.groups([s1, dep, s2, dep, s1, s1]) == [[0, 2, 4], [5]]
    assert kr.groups([dep, dep]) == []
    for chans, want in (([s1, s2, s1, s1], (2, 1, 2, 5)), ([s2] * 15, (8, 1, 8, 17)), ([dep] * 3, (0, 0, 0, 0)),
                        ([s4, s1, s3], (2, 1, 2, 5))):
        k = [c.n_qubits for c in chans]
        qs, q = [], 0
        for a in k:
            qs.append(list(range(q, q + a)))
            q += a
        assert kraus_channels_plan(max(q, 1), np.complex128, chans, qs) == want == kr.plan(chans)


def test_kraus_channel_checks():
    K = ch.KrausChannel(ch.amplitude_damping(0.3))
    assert K.n_qubits == 1 and len(K) == 2 and not K.state_independent
    assert ch.KrausChannel(ch.depolarizing(0.3)).state_independent
    U = ch.KrausChannel([CX])
    assert U.state_independent and U.n_qubits == 2
    noisy = U.compose(ch.two_qubit_depolarizing(0.05))
    assert len(noisy) == 16 and noisy.state_independent
    adcx = U.compose(ch.amplitude_damping(0.1).tensor(ch.amplitude_damping(0.2)))
    assert len(adcx) == 4 and not adcx.state_independent
    rho = np.diag([0.0, 0.0, 0.0, 1.0]).astype(np.complex128)
    out = adcx.superop(rho)
    assert abs(np.trace(out) - 1) < 1e-14
    t = ch.KrausChannel(ch.amplitude_damping(0.1)).tensor(x_damping(0.2))
    assert t.n_qubits == 2 and len(t) == 4
    with pytest.raises(ValueError, match="not complete .entry .0, 1. of sum"):
        ch.KrausChannel([np.array([[1, 0.5], [0, 1]])])
    with pytest.raises(ValueError, match="zero matrix"):
        ch.KrausChannel([np.eye(2), np.zeros((2, 2))])
    with pytest.raises(ValueError, match="non-finite"):
        ch.KrausChannel([np.array([[np.nan, 0], [0, 1]])])
    with pytest.raises(ValueError, match="1 to 256"):
        ch.KrausChannel([np.eye(2) / 257 ** 0.5] * 257)
    with pytest.raises(ValueError, match="2.k x 2.k"):
        ch.KrausChannel([np.eye(3)])
    with pytest.raises(ValueError, match="at most 4"):
        ch.KrausChannel(np.eye(8)[None]).tensor(ch.KrausChannel(np.eye(4)[None]))
    with pytest.raises(ValueError, match="compose"):
        U.compose(ch.amplitude_damping(0.1))


def _plan_call(n, arity, qubits, n_kraus, kraus, prec=F64, out=True):
    L = _lib.lib()
    aa = (C.c_uint32 * max(1, len(arity)))(*arity) if arity is not None else None
    qa = (C.c_uint64 * max(1, len(qubits)))(*qubits) if qubits is not None else None
    na = (C.c_uint32 * max(1, len(n_kraus)))(*n_kraus) if n_kraus is not None else None
    ka = (C.c_double * max(1, len(kraus)))(*kraus) if kraus is not None else None
    v = (C.c_uint32 * 4)()
    nc = len(n_kraus) if n_kraus is not None else len(arity)
    st = L.qipb200_kraus_channels_plan(prec, n, nc, aa, qa, na, ka, v if out else None)
    return st, L.qipb200_last_error(None).decode(), tuple(v)


def _flat(*ops):
    return [float(v) for k in ops for v in np.asarray(k, dtype=np.complex128).reshape(-1).view(np.float64)]


def test_plan_refusals():
    I2, I4 = np.eye(2), np.eye(4)
    w = "kraus_channels_plan"
    nan = np.array([[np.nan, 0], [0, 1]])
    cases = [
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(I2), out=False), INVALID_ARG,
         w + ": NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=41, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(I2), prec=7), INVALID_ARG,
         w + ": NULL out4, bad precision or n_qubits not in 1..40"),
        (dict(n=4, arity=None, qubits=[0], n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL arity, qubits, n_kraus or kraus"),
        (dict(n=4, arity=[1], qubits=None, n_kraus=[1], kraus=_flat(I2)), INVALID_ARG,
         w + ": NULL arity, qubits, n_kraus or kraus"),
        (dict(n=4, arity=[1], qubits=[0], n_kraus=None, kraus=_flat(I2)), INVALID_ARG,
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
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[2], kraus=_flat(I2, nan)), INVALID_ARG,
         w + ": channel 0, operator 1: an entry is not finite"),
        (dict(n=4, arity=[1, 1], qubits=[0, 1], n_kraus=[1, 2], kraus=_flat(I2, I2, np.zeros((2, 2)))), INVALID_ARG,
         w + ": channel 1, operator 1: the zero matrix"),
        (dict(n=4, arity=[1], qubits=[0], n_kraus=[1], kraus=_flat(np.array([[1, 0.5], [0, 1]]))), INVALID_ARG,
         w + ": channel 0: the operators are not complete (entry (0, 1) of sum K^dagger K - I is 0.5+0i)"),
        (dict(n=4, arity=[2], qubits=[0, 1], n_kraus=[1], kraus=_flat(CX * np.sqrt(1 + 1e-11))), INVALID_ARG,
         w + ": channel 0: the operators are not complete (entry (0, 0) of sum K^dagger K - I is 1e-11+0i)"),
    ]
    for kw, status, msg in cases:
        st, err, _ = _plan_call(**kw)
        assert (st, err) == (status, msg), kw


def test_plan_counts():
    rng = np.random.default_rng(11)
    c128 = np.complex128
    xd = x_damping(0.1)
    assert kraus_channels_plan(30, c128, xd, [[q] for q in range(30)]) == (8, 1, 8, 17)
    s2 = [kr.stinespring(2, 4, rng) for _ in range(15)]
    assert kraus_channels_plan(30, c128, s2, [[2 * i, 2 * i + 1] for i in range(15)]) == (8, 1, 8, 17)
    ncx = ch.KrausChannel([CX]).compose(ch.two_qubit_depolarizing(0.02))
    assert kraus_channels_plan(30, c128, ncx, [[2 * i, 2 * i + 1] for i in range(15)]) == (0, 0, 0, 0)
    assert kraus_channels_plan(30, c128, ch.amplitude_damping(0.1), [[q] for q in range(30)]) == (8, 1, 8, 17)
    assert kraus_channels_plan(8, c128, [], []) == (0, 0, 0, 0)
    # a Channel is accepted where a KrausChannel is
    st, _, out = _plan_call(5, [1, 1], [0, 3], [2, 1], _flat(*ch.amplitude_damping(0.2).kraus, np.eye(2)))
    assert st == 0 and out == (1, 1, 1, 3)


def test_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "use_kraus_channels.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::B200State<double> &st) {\n"
                   "  std::vector<double> k(32, 0.0);\n"
                   "  for (int i = 0; i < 4; ++i) k[2 * (4 * i + i)] = 1.0;  // the identity on two qubits\n"
                   "  auto r = st.apply_kraus_channels({2}, {0, 1}, {1}, k, {0.5});\n"
                   "  return std::get<2>(r) + std::get<1>(r).at(0) + (double)std::get<0>(r).at(0);\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
