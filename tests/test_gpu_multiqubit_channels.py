"""Channels on one to four qubits along quantum trajectories on the device (State.apply_multiqubit_channels,
qipb200_state_apply_multiqubit_channels).

The choices, the probability and the state are compared bit for bit with the numpy emulation of
tests/multiqubit_channel_ref.py (x cross-checked against State.sample with draws[0]), single-qubit layers with
State.apply_channels, unitary monomial channels with apply_op of the same MAT, a two-qubit Z measurement with
State.measure, a two-qubit reset of every pair at N = 30, windows at n = 26 and past 2^31 and 2^32, and a trajectory
average with the exact channel."""
import ctypes as C
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import multiqubit_channel_ref as mr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200 import channels as ch
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, multiqubit_channels_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
XY = ch.Channel([np.kron(ch._X, ch._Y)])  # a fixed anti-diagonal choice on two qubits
RESET2 = ch.Channel([np.outer(np.eye(4)[0], np.eye(4)[b]) for b in range(4)])


def bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def random_channel(rng, k):
    kind = int(rng.integers(0, 6))
    g = float(rng.uniform(0.05, 0.95))
    one = [ch.amplitude_damping(g), ch.phase_damping(g), ch.depolarizing(g), ch.reset(),
           ch.pauli_channel(1.0, 0.0, 0.0), ch.amplitude_damping(g).compose(ch.phase_damping(0.5))]
    if k == 1:
        return one[kind]
    if k == 2:
        return [ch.two_qubit_depolarizing(g), ch.amplitude_damping(g).tensor(ch.depolarizing(0.3)), RESET2, XY,
                ch.pauli_string_channel({"ZZ": g, "XX": 0.02}), one[kind].tensor(ch.reset())][kind]
    if k == 3:
        return [ch.pauli_string_channel({"XYZ": g / 2, "ZIZ": 0.1}), XY.tensor(ch.amplitude_damping(g)),
                ch.amplitude_damping(g).tensor(ch.two_qubit_depolarizing(0.2))][kind % 3]
    return [ch.pauli_string_channel({"XZZY": g / 3, "ZZZZ": 0.2}), XY.tensor(ch.reset().tensor(ch.phase_damping(g))),
            ch.two_qubit_depolarizing(0.1).tensor(ch.amplitude_damping(g).tensor(ch.amplitude_damping(0.3)))][kind % 3]


def random_layer(rng, n, straddles=0):
    """Disjoint groups of 1..4 qubits; the first `straddles` groups are pairs across index-byte boundaries."""
    free = [int(q) for q in rng.permutation(n)]
    groups = []
    for s in range(straddles):
        bit = 8 * (s + 1)  # bits bit and bit - 1
        g = [n - 1 - bit, n - bit]
        if g[0] < 0 or any(q not in free for q in g):
            break
        groups.append(g if rng.random() < 0.5 else g[::-1])
        free = [q for q in free if q not in g]
    while free and len(groups) < straddles + 5:
        k = min(int(rng.integers(1, 5)), len(free))
        groups.append(free[:k])
        free = free[k:]
    return groups, [random_channel(rng, len(g)) for g in groups]


def sample_x(st, groups, chans, r):
    dep = [q for g, c in zip(groups, chans) if c.state_dependent for q in g]
    return int(st.sample(dep, [r])[0]) if dep else 0


def check_call(st, psi, n, groups, chans, draws):
    st.upload(psi)
    x = sample_x(st, groups, chans, draws[0])
    chosen, prob = st.apply_multiqubit_channels(chans, groups, draws=draws)
    want_c, want_p, want = mr.emulate(psi, n, groups, [c.kraus for c in chans], x, draws)
    assert list(chosen) == want_c
    assert np.float64(prob).tobytes() == np.float64(want_p).tobytes(), (prob, want_p)
    assert bits_equal(st.download(), want)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_emulation(ctx, dtype):
    for n in (2, 3, 5, 7, 9, 12, 16, 17, 20, 23):
        rng = np.random.default_rng(900 + n)
        psi = circuits.random_state(n, 50 + n, dtype)
        psi[rng.integers(0, 1 << n, size=2)] = complex(-0.0, -0.0)
        with State(n, dtype, ctx) as st:
            for case in range(3 if n <= 20 else 1):
                groups, chans = random_layer(rng, n, straddles=(0, 1, 3)[case] if n <= 20 else 2)
                check_call(st, psi, n, groups, chans, rng.random(1 + len(groups)))
            if n >= 16:  # as many byte-straddling pairs as the qubits allow, plus gathered pairs across the state
                groups = [[n - 1 - 8 * s, n - 8 * s] for s in range(1, (n - 1) // 8 + 1)]
                used = {q for g in groups for q in g}
                rest = [q for q in range(n) if q not in used]
                groups += [[rest[i], rest[-1 - i]] for i in range(len(rest) // 2)]
                chans = [random_channel(rng, 2) for _ in groups]
                check_call(st, psi, n, groups, chans, rng.random(1 + len(groups)))


def test_bit_exact_at_26(ctx):
    """n = 26 f32, state-dependent, gathered and byte tables: windows against the emulation of their source blocks."""
    n, W = 26, 1 << 12
    rng = np.random.default_rng(26)
    psi = circuits.random_state(n, 26, C64)
    groups = [[0, 25], [1, 17, 9], [3, 4], [2], [10, 11, 12, 13]]
    chans = [XY, XY.tensor(ch.amplitude_damping(0.4)), ch.two_qubit_depolarizing(0.5), ch.reset(),
             ch.pauli_string_channel({"XZZY": 0.9})]
    draws = rng.random(1 + len(groups))
    with State(n, C64, ctx) as st:
        st.upload(psi)
        x = sample_x(st, groups, chans, draws[0])
        chosen, prob = st.apply_multiqubit_channels(chans, groups, draws=draws)
        assert list(chosen) == mr.choices(groups, [c.kraus for c in chans], x, draws)
        ops = [c.kraus[i] for c, i in zip(chans, chosen)]
        assert not any(mr.scaled_identity(k) for k in ops)
        tabs, F = mr.tables([[n - 1 - q for q in g] for g in groups], ops)
        for o in (0, (1 << 24) - W, (1 << 24) + 3 * W, (1 << n) - W):
            idx = np.arange(o, o + W, dtype=np.uint64) ^ np.uint64(F)
            want = mr.moved(psi[idx.astype(np.int64)], idx, tabs, 1.0 / np.sqrt(prob))
            assert bits_equal(st.download(offset=o, length=W), want), o


@pytest.mark.parametrize("n", [31, 32])
def test_windows_past_2_31_f32(ctx, n):
    """A gathered pair on index bits 31 (n = 32) or 30 and 3, a damped pair on bits 29 and 5, a byte pair on bits 1
    and 0: windows, downloaded with their source blocks before the call, against the emulation."""
    top_bit = n - 1
    bit_groups = [[top_bit, 3], [29, 5], [1, 0]]
    groups = [[n - 1 - b for b in g] for g in bit_groups]
    chans = [XY, ch.amplitude_damping(0.35).tensor(ch.amplitude_damping(0.6)), XY]
    W = 1 << 12
    ctx.release_pool()
    with State(n, C64, ctx) as st:
        st.set_basis(0)
        st.apply_schedule([gates.h(k) for k in range(n)] + [gates.t(k) for k in range(0, n, 2)])
        top = (1 << n) - W
        offs = sorted({min(o, top) for o in (0, (1 << 31) - W, (1 << 31) + (5 << 12), (3 << 30) + W, top)})
        draws = [0.4] + [0.5] * len(groups)
        x = sample_x(st, groups, chans, draws[0])
        ops = [c.kraus[i] for c, i in zip(chans, mr.choices(groups, [c.kraus for c in chans], x, draws))]
        F = mr.tables(bit_groups, ops)[1]
        base = {o: o ^ (F & ~(W - 1)) for o in offs}
        srcs = {o: st.download(offset=base[o], length=W) for o in offs}
        chosen, prob = st.apply_multiqubit_channels(chans, groups, draws=draws)
        tabs, F2 = mr.tables(bit_groups, [c.kraus[i] for c, i in zip(chans, chosen)])
        assert F2 == F
        for o in offs:
            idx = np.arange(o, o + W, dtype=np.uint64) ^ np.uint64(F)
            want = mr.moved(srcs[o][(idx - np.uint64(base[o])).astype(np.int64)], idx, tabs, 1.0 / np.sqrt(prob))
            assert bits_equal(st.download(offset=o, length=W), want), (n, o)
    ctx.release_pool()


@pytest.mark.parametrize("dtype", [C128, C64])
def test_single_qubit_layer_is_apply_channels(ctx, dtype):
    n = 18
    rng = np.random.default_rng(18)
    psi = circuits.random_state(n, 18, dtype)
    with State(n, dtype, ctx) as a, State(n, dtype, ctx) as b:
        for _ in range(3):
            qubits = [int(q) for q in rng.permutation(n)[:int(rng.integers(1, n + 1))]]
            chans = [random_channel(rng, 1) for _ in qubits]
            draws = rng.random(1 + len(qubits))
            a.upload(psi)
            b.upload(psi)
            ca, pa = a.apply_channels(chans, qubits, draws=draws)
            cb, pb = b.apply_multiqubit_channels(chans, [[q] for q in qubits], draws=draws)
            assert list(ca) == list(cb) and np.float64(pa).tobytes() == np.float64(pb).tobytes()
            assert bits_equal(a.download(), b.download())


def test_matrix_convention_matches_apply_op(ctx):
    n = 12
    psi = circuits.random_state(n, 12, C128)
    cz = np.diag([1.0, 1.0, 1.0, -1.0]).astype(C128)
    xy = np.kron(ch._X, ch._Y)
    phase = np.diag(np.exp(1j * np.arange(16) * 0.37))
    for qubits, K in (([3, 9], cz), ([9, 3], xy), ([1, 11], xy), ([7, 2, 10, 4], phase), ([0, 8], xy)):
        with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
            a.upload(psi)
            b.upload(psi)
            chosen, prob = a.apply_multiqubit_channels([ch.Channel([K])], [qubits], draws=[0.5, 0.5])
            assert list(chosen) == [0] and abs(prob - 1.0) <= 1e-15
            b.apply_op(gates.mat(qubits, list(K.reshape(-1))))
            assert np.max(np.abs(a.download() - b.download())) <= 1e-14


def test_two_qubit_reset_closed_form_n30(ctx):
    """Reset every pair of 30 qubits: the state becomes e^{i phi}|0...0> and prob = |psi_x|^2 for the sampled x."""
    n = 30
    ctx.release_pool()
    with State(n, C128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule([gates.h(k) for k in range(n)] + [gates.t(k) for k in range(0, n, 3)])
        groups = [[2 * i, 2 * i + 1] for i in range(15)]
        draws = np.random.default_rng(30).random(16)
        x = int(st.sample(list(range(n)), [draws[0]])[0])
        j = sum(((x >> q) & 1) << (n - 1 - q) for q in range(n))  # the sampled basis index
        amp = st.download(offset=j, length=1)[0]
        chosen, prob = st.apply_multiqubit_channels(RESET2, groups, draws=draws)
        assert abs(prob - abs(amp) ** 2) <= 1e-9 * prob  # the weight sweep's bound at N = 30 is far below 1e-9
        W = 1 << 26
        for off in range(0, 1 << n, W):
            v = st.download(offset=off, length=W)
            if off == 0:
                assert abs(abs(v[0]) - 1.0) <= 1e-12
                v = v[1:]
            assert not np.any(v), off
    ctx.release_pool()


def test_two_qubit_z_measurement_matches_measure(ctx):
    z2 = ch.Channel([np.diag(np.eye(4)[b]) for b in range(4)])
    n = 14
    psi = circuits.random_state(n, 14, C128)
    for r, pair in ((0.3, [2, 9]), (0.71, [13, 0])):
        with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
            a.upload(psi)
            b.upload(psi)
            chosen, prob = a.apply_multiqubit_channels(z2, [pair], draws=[r, 0.5])
            m, p = b.measure(pair, r)
            # chosen is b in the matrix convention (pair[0] the top bit); measure's m has pair[0] at bit 0
            assert int(chosen[0]) == ((m & 1) << 1) | (m >> 1)
            assert abs(prob - p) <= 1e-12 * p
            assert np.max(np.abs(a.download() - b.download())) <= 1e-13


def test_trajectory_average_matches_the_channel(ctx):
    n, T = 4, 2000
    psi0 = circuits.random_state(n, 4, C128)
    groups = [[0, 2], [3, 1]]
    chans = [ch.two_qubit_depolarizing(0.3), ch.amplitude_damping(0.4).tensor(ch.amplitude_damping(0.2))]
    rng = np.random.default_rng(2000)
    acc = np.zeros((1 << n, 1 << n), dtype=np.complex128)
    acc2 = np.zeros((1 << n, 1 << n))
    with State(n, C128, ctx) as st:
        for _ in range(T):
            st.upload(psi0)
            st.apply_multiqubit_channels(chans, groups, rng=rng)
            v = st.download()
            r = np.outer(v, v.conj())
            acc += r
            acc2 += np.abs(r) ** 2
    mean = acc / T
    sigma = np.sqrt(np.maximum(acc2 / T - np.abs(mean) ** 2, 0.0) / T)
    rho = np.outer(psi0, psi0.conj())
    exact = np.zeros_like(rho)
    for tup in itertools.product(*[range(len(c)) for c in chans]):
        K = mr.full_op(n, groups, [c.kraus[i] for c, i in zip(chans, tup)])
        exact += K @ rho @ K.conj().T
    # each entry is a mean of T bounded samples: 5 standard errors (and an absolute floor for entries of no spread)
    assert np.all(np.abs(mean - exact) <= 5 * sigma + 1e-12)


def test_determinism_and_launch_counts(ctx):
    n = 20
    psi = circuits.random_state(n, 20, C128)
    groups = [[2 * i, 2 * i + 1] for i in range(10)]
    mixed = [ch.two_qubit_depolarizing(0.01)] * 5 + [ch.amplitude_damping(0.01).tensor(ch.amplitude_damping(0.02))] * 5
    with State(n, C128, ctx) as st:
        outs = []
        for _ in range(2):
            st.upload(psi)
            l0 = ctx.kernel_launches()
            c, p = st.apply_multiqubit_channels(mixed, groups, draws=np.linspace(0.1, 0.9, 11))
            assert ctx.kernel_launches() - l0 == multiqubit_channels_plan(n, C128, mixed, groups)[3] == 12
            outs.append((list(c), p, st.download()))
        assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1] and bits_equal(outs[0][2], outs[1][2])
        dep = ch.two_qubit_depolarizing(0.01)
        st.upload(psi)
        l0 = ctx.kernel_launches()
        c, p = st.apply_multiqubit_channels(dep, groups, draws=[0.5] * 10 + [0.999])  # the last pair takes an error
        assert ctx.kernel_launches() - l0 == multiqubit_channels_plan(n, C128, dep, groups)[3] == 1
        assert c[-1] > 0 and all(v == 0 for v in c[:-1])
        st.upload(psi)
        l0 = ctx.kernel_launches()
        c, p = st.apply_multiqubit_channels(dep, groups, draws=[0.5] * 11)  # every choice the scaled identity
        assert ctx.kernel_launches() == l0 and bits_equal(st.download(), psi)
        assert p == pytest.approx(0.99 ** 10, rel=1e-13)


def test_pending_collapse_and_pending_basis(ctx):
    n = 14
    psi = circuits.random_state(n, 41, C128)
    chans, groups = [ch.amplitude_damping(0.5).tensor(ch.reset()), XY, RESET2], [[1, 9], [13, 2], [6, 7]]
    draws = [0.37, 0.2, 0.5, 0.8]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 6], 0.61)
        b.collapse([0, 6], m, p)
        l0 = ctx.kernel_launches()
        ra = a.apply_multiqubit_channels(chans, groups, draws=draws)
        la = ctx.kernel_launches() - l0
        l0 = ctx.kernel_launches()
        rb = b.apply_multiqubit_channels(chans, groups, draws=draws)
        assert la == ctx.kernel_launches() - l0 + 1
        assert list(ra[0]) == list(rb[0]) and ra[1] == rb[1] and bits_equal(a.download(), b.download())
        a.set_basis(77)
        basis = np.zeros(1 << n, dtype=C128)
        basis[77] = 1.0
        b.upload(basis)
        ra, rb = (a.apply_multiqubit_channels(chans, groups, draws=draws),
                  b.apply_multiqubit_channels(chans, groups, draws=draws))
        assert list(ra[0]) == list(rb[0]) and ra[1] == rb[1] and bits_equal(a.download(), b.download())


_ROTATE_WORKER = r"""
import numpy as np
import multiqubit_channel_ref as mr
from rustqip_b200 import channels as ch, circuits
from rustqip_b200.state import Context, State

n = 18
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
xy = ch.Channel([np.kron(ch._X, ch._Y)])
cases = [([[17, 3], [0, 9, 5]], [xy, ch.pauli_string_channel({"XYZ": 0.5, "ZZX": 0.4})]),
         ([[0, 17], [4, 8]], [ch.amplitude_damping(0.3).tensor(ch.reset()), xy])]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for groups, chans in cases:
            for st in (a, b):
                st.set_basis(3)
                st.apply_schedule(ops)
            qmap = b.qubit_map().copy()
            assert not np.array_equal(qmap, np.arange(n)[::-1]), "the schedule left the canonical layout"
            psi = a.download()
            draws = [0.3] + [0.9] * len(groups)
            dep = [q for g, c in zip(groups, chans) if c.state_dependent for q in g]
            x = int(b.sample(dep, [0.3])[0]) if dep else 0
            if dep:  # the sample restored the layout
                qmap = b.qubit_map().copy()
            chosen, prob = b.apply_multiqubit_channels(chans, groups, draws=draws)
            assert np.array_equal(b.qubit_map(), qmap), "apply_multiqubit_channels changed the layout"
            idx = np.arange(1 << n, dtype=np.uint64)
            phys = np.zeros(1 << n, dtype=np.uint64)
            for q in range(n):
                phys |= ((idx >> np.uint64(n - 1 - q)) & np.uint64(1)) << np.uint64(qmap[q])
            ps = np.empty_like(psi)
            ps[phys.astype(np.int64)] = psi
            c, p, out = mr.emulate(ps, n, groups, [k.kraus for k in chans], x, draws, phys=lambda q: int(qmap[q]))
            assert list(chosen) == c and prob == p
            got = b.download()
            want = out[phys.astype(np.int64)]
            assert np.array_equal(got, want), int(np.sum(got != want))
print("ROTATE bit-exact ok")
"""


def test_permuted_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout


def test_refusals_leave_state_and_pending_collapse(ctx):
    n = 12
    psi = circuits.random_state(n, 12, C128)
    L = _lib.lib()
    I4 = np.eye(4)
    w = "apply_multiqubit_channels"

    def flat(*ops):
        return np.ascontiguousarray(np.concatenate([np.asarray(k, dtype=C128).reshape(-1) for k in ops])).view(
            np.float64)

    def arr(v, t):
        return np.ascontiguousarray(np.asarray(v, dtype=t)) if v is not None else None

    def call(st, arity, qubits, n_kraus, kraus, draws, chosen=True, prob=True):
        aa, qa, na, da = arr(arity, np.uint32), arr(qubits, np.uint64), arr(n_kraus, np.uint32), arr(draws, np.float64)
        out = np.zeros(8, dtype=np.uint32)
        p = C.c_double()
        nc = len(n_kraus) if n_kraus is not None else len(arity)
        ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
        return L.qipb200_state_apply_multiqubit_channels(st._h, nc, ptr(aa), ptr(qa), ptr(na), ptr(kraus), ptr(da),
                                                         out.ctypes.data if chosen else None,
                                                         C.byref(p) if prob else None)

    ok = flat(*RESET2.kraus)
    form = "not of the form K|b> = d(b)|b ^ f> (one nonzero entry per column, one f)"
    cases = [
        (([2], [1, 2], [4], ok, [0.1, 0.2]), dict(prob=False), INVALID_ARG, w + ": NULL prob"),
        (([2], [1, 2], [4], ok, None), {}, INVALID_ARG, w + ": NULL draws or chosen"),
        ((None, [1, 2], [4], ok, [0.1, 0.2]), {}, INVALID_ARG, w + ": NULL arity, qubits, n_kraus or kraus"),
        (([2], None, [4], ok, [0.1, 0.2]), {}, INVALID_ARG, w + ": NULL arity, qubits, n_kraus or kraus"),
        (([5], [1, 2, 3, 4, 5], [1], ok, [0.1, 0.2]), {}, INVALID_ARG, w + ": channel 0: arity must be 1..4, got 5"),
        (([2], [1, 12], [4], ok, [0.1, 0.2]), {}, BAD_INDEX, w + ": channel 0: qubit 12 out of range for 12 qubits"),
        (([1, 2], [3, 4, 3], [1, 4], flat(np.eye(2), *RESET2.kraus), [0.1, 0.2, 0.3]), {}, BAD_INDEX,
         w + ": channel 1: qubit 3 repeated"),
        (([2], [1, 2], [0], ok, [0.1, 0.2]), {}, INVALID_ARG, w + ": channel 0: n_kraus must be 1..256, got 0"),
        (([2], [1, 2], [1], flat(np.ones((4, 4)) / 2), [0.1, 0.2]), {}, INVALID_ARG,
         w + ": channel 0, operator 0: " + form),
        (([2], [1, 2], [1], flat(2 * I4), [0.1, 0.2]), {}, INVALID_ARG,
         w + ": channel 0: the operators are not complete (sum of |d_i(0)|^2 - 1 = 3)"),
        (([2], [1, 2], [4], ok, [0.1, 1.0]), {}, INVALID_ARG, w + ": draw 1 is not in [0, 1)"),
    ]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 6], 0.37)
        l0 = ctx.kernel_launches()
        for args, kw, code, msg in cases:
            assert call(a, *args, **kw) == code, msg
            assert L.qipb200_last_error(ctx.handle).decode() == msg
        assert L.qipb200_state_apply_multiqubit_channels(None, 0, None, None, None, None, None, None, None) == \
            INVALID_ARG
        assert ctx.kernel_launches() == l0
        c0, p0 = a.apply_multiqubit_channels([], [])
        assert p0 == 1.0 and ctx.kernel_launches() == l0
        with pytest.raises(ValueError):
            a.apply_multiqubit_channels(RESET2, [[0]])
        with pytest.raises(ValueError):
            a.apply_channels(RESET2, [0])
        # the collapse is still pending: one kernel for it, then the call's own
        l0 = ctx.kernel_launches()
        a.apply_multiqubit_channels(XY, [[4, 9]], draws=[0.5, 0.5])
        assert ctx.kernel_launches() - l0 == 2
        b.collapse([0, 6], m, p)
        b.apply_multiqubit_channels(XY, [[4, 9]], draws=[0.5, 0.5])
        assert bits_equal(a.download(), b.download())
    with State(n, C128, ctx, rank=0, world_size=2) as sh:
        with pytest.raises(CircuitError) as e:
            sh.apply_multiqubit_channels(RESET2, [[0, 1]])
        assert e.value.status == UNSUPPORTED and str(e.value) == w + ": sharded states are not supported"
