"""Single-qubit channels along quantum trajectories on the device (State.apply_channels,
qipb200_state_apply_channels).

The choices, the probability and the state are compared bit for bit with the numpy emulation of tests/channel_ref.py
(x cross-checked against State.sample with draws[0]), q with the long-double reference within the bound of
channel.cu, Z-measurement channels with State.measure, closed forms at N = 30 and windows past 2^31 and 2^32, and a
trajectory average with the exact channel."""
import ctypes as C
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import channel_ref as cr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200 import channels as ch
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, channels_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
FLIP = ch.pauli_channel(1.0, 0.0, 0.0)  # X always: an anti-diagonal choice on its qubit


def bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def random_channel(rng):
    kind = int(rng.integers(0, 7))
    g = float(rng.uniform(0.05, 0.95))
    return [ch.amplitude_damping(g), ch.generalized_amplitude_damping(g, 0.3), ch.phase_damping(g),
            ch.depolarizing(g), ch.reset(), FLIP, ch.amplitude_damping(g).compose(ch.phase_damping(0.5))][kind]


def sample_x(st, qubits, chans, r):
    dep = [q for q, c in zip(qubits, chans) if c.state_dependent]
    return int(st.sample(dep, [r])[0]) if dep else 0


def check_call(st, psi, n, qubits, chans, draws):
    """One call against the emulation, bit for bit, and q against the long-double reference."""
    st.upload(psi)
    x = sample_x(st, qubits, chans, draws[0])
    chosen, prob = st.apply_channels(chans, qubits, draws=draws)
    want_c, want_p, want = cr.emulate(psi, n, qubits, [c.kraus for c in chans], x, draws)
    assert list(chosen) == want_c
    assert np.float64(prob).tobytes() == np.float64(want_p).tobytes(), (prob, want_p)
    assert bits_equal(st.download(), want)
    rest = [(n - 1 - q, c.kraus[i]) for q, c, i in zip(qubits, chans, chosen) if not cr.scaled_identity(c.kraus[i])]
    if any(cr.weights(k)[0] != cr.weights(k)[1] for _, k in rest):
        S, N = cr.weight_reference(psi, n, [p for p, _ in rest], [k for _, k in rest])
        q_ref = float(S / N)
        dropped = np.prod([cr.weights(c.kraus[i])[0] for c, i in zip(chans, chosen)
                           if cr.scaled_identity(c.kraus[i])])
        assert abs(prob / dropped - q_ref) <= (cr.q_bound(n, len(rest)) + 4 * cr.U) * q_ref
    return chosen, prob


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_emulation(ctx, dtype):
    for n in (2, 3, 5, 6, 7, 9, 12, 16, 20, 23):
        rng = np.random.default_rng(700 + n)
        psi = circuits.random_state(n, 30 + n, dtype)
        psi[rng.integers(0, 1 << n, size=2)] = complex(-0.0, -0.0)
        with State(n, dtype, ctx) as st:
            for case in range(3 if n <= 20 else 1):
                nc = int(rng.integers(1, n + 1))
                qubits = [int(q) for q in rng.permutation(n)[:nc]]
                if case == 0:  # F with low bits and the top bit: flips on qubits n - 1, n - 2 and 0
                    qubits = sorted(set([n - 1, 0] + ([n - 2] if n > 2 else []) + qubits), key=lambda q: -q)
                chans = [random_channel(rng) for _ in qubits]
                if case == 0:
                    chans[0] = FLIP
                    chans[-1] = FLIP
                check_call(st, psi, n, qubits, chans, rng.random(1 + len(qubits)))


def test_bit_exact_at_26(ctx):
    """n = 26 f32 with the weight sweep: windows at both ends and on both sides of index bit 24, each against the
    emulation of its source block.  No chosen operator is a multiple of the identity, so q is the returned prob."""
    n, W = 26, 1 << 12
    rng = np.random.default_rng(26)
    psi = circuits.random_state(n, 26, C64)
    qubits = [25, 24, 17, 9, 3, 0]
    chans = [FLIP, ch.amplitude_damping(0.4), ch.pauli_channel(0.0, 0.5, 0.5), ch.reset(), FLIP,
             ch.phase_damping(0.3)]
    draws = rng.random(1 + len(qubits))
    with State(n, C64, ctx) as st:
        st.upload(psi)
        x = sample_x(st, qubits, chans, draws[0])
        chosen, prob = st.apply_channels(chans, qubits, draws=draws)
        kd, want_c = 0, []
        for q, c, u in zip(qubits, chans, draws[1:]):
            b = (x >> kd) & 1 if c.state_dependent else 0
            kd += c.state_dependent
            want_c.append(cr.choose(c.kraus, b, float(u)))
        assert list(chosen) == want_c
        ops = [c.kraus[i] for c, i in zip(chans, chosen)]
        assert not any(cr.scaled_identity(k) for k in ops)
        tabs, F = cr.tables([n - 1 - q for q in qubits], ops)
        for o in (0, (1 << 24) - W, (1 << 24) + 3 * W, (1 << n) - W):
            idx = np.arange(o, o + W, dtype=np.uint64) ^ np.uint64(F)
            want = cr.moved(psi[idx.astype(np.int64)], idx, tabs, 1.0 / np.sqrt(prob))
            assert bits_equal(st.download(offset=o, length=W), want), o


def test_z_measurement_matches_measure(ctx):
    z = ch.Channel([np.diag([1.0, 0.0]), np.diag([0.0, 1.0])])
    n = 14
    psi = circuits.random_state(n, 14, C128)
    for r, qubits in ((0.3, [2, 9]), (0.71, [13, 0, 5])):
        with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
            a.upload(psi)
            b.upload(psi)
            chosen, prob = a.apply_channels(z, qubits, draws=[r] + [0.5] * len(qubits))
            m, p = b.measure(qubits, r)
            assert sum(int(c) << k for k, c in enumerate(chosen)) == m
            assert abs(prob - p) <= 1e-12 * p
            assert np.max(np.abs(a.download() - b.download())) <= 1e-13


def test_full_damping_closed_form_n30(ctx):
    n = 30
    ctx.release_pool()
    with State(n, C128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule([gates.h(k) for k in range(n)] + [gates.t(k) for k in range(0, n, 3)])
        chosen, prob = st.apply_channels(ch.amplitude_damping(1.0), range(n), rng=np.random.default_rng(30))
        assert abs(prob - 2.0 ** -n) <= 1e-9 * prob
        W = 1 << 26
        for off in range(0, 1 << n, W):
            v = st.download(offset=off, length=W)
            if off == 0:
                assert abs(abs(v[0]) - 1.0) <= 1e-12
                v = v[1:]
            assert not np.any(v), off
    ctx.release_pool()


@pytest.mark.parametrize("n", [31, 32])
def test_windows_past_2_31_f32(ctx, n):
    """Flips on index bits 31 (n = 32), 30, 3 and 0, damping on bits 29 and 5: every window, downloaded with its source
    block before the call, against the emulation."""
    def q(bit):
        return n - 1 - bit

    bits = [b for b in (31, 30, 29, 5, 3, 0) if b < n]
    chans = [ch.amplitude_damping(0.35) if b in (29, 5) else FLIP for b in bits]
    qubits = [q(b) for b in bits]
    W = 1 << 12
    ctx.release_pool()
    with State(n, C64, ctx) as st:
        st.set_basis(0)
        st.apply_schedule([gates.h(k) for k in range(n)] + [gates.t(k) for k in range(0, n, 2)])
        top = (1 << n) - W
        offs = sorted({min(o, top) for o in (0, (1 << 31) - W, (1 << 31) + (5 << 12), (3 << 30) + W, top)})
        draws = [0.4] + [0.5] * len(bits)
        # the choices follow from x, so F (and each window's source block) is known before the call
        x, kd, ops = sample_x(st, qubits, chans, draws[0]), 0, []
        for c in chans:
            b = (x >> kd) & 1 if c.state_dependent else 0
            kd += c.state_dependent
            ops.append(c.kraus[cr.choose(c.kraus, b, 0.5)])
        F = cr.tables(bits, ops)[1]
        base = {o: o ^ (F & ~(W - 1)) for o in offs}
        srcs = {o: st.download(offset=base[o], length=W) for o in offs}
        chosen, prob = st.apply_channels(chans, qubits, draws=draws)
        tabs, F2 = cr.tables(bits, [c.kraus[i] for c, i in zip(chans, chosen)])
        assert F2 == F
        for o in offs:
            idx = np.arange(o, o + W, dtype=np.uint64) ^ np.uint64(F)  # the sources of the window
            want = cr.moved(srcs[o][(idx - np.uint64(base[o])).astype(np.int64)], idx, tabs, 1.0 / np.sqrt(prob))
            assert bits_equal(st.download(offset=o, length=W), want), (n, o)
    ctx.release_pool()


def test_trajectory_average_matches_the_channel(ctx):
    n, T = 6, 2000
    psi0 = circuits.random_state(n, 6, C128)
    qubits = [0, 2, 3, 5]
    chans = [ch.amplitude_damping(0.3), ch.depolarizing(0.2), ch.phase_damping(0.4), ch.reset()]
    rng = np.random.default_rng(2000)
    acc = np.zeros((1 << n, 1 << n), dtype=np.complex128)
    acc2 = np.zeros((1 << n, 1 << n))
    with State(n, C128, ctx) as st:
        for _ in range(T):
            st.upload(psi0)
            st.apply_channels(chans, qubits, rng=rng)
            v = st.download()
            r = np.outer(v, v.conj())
            acc += r
            acc2 += np.abs(r) ** 2
    mean = acc / T
    sigma = np.sqrt(np.maximum(acc2 / T - np.abs(mean) ** 2, 0.0) / T)
    rho = np.outer(psi0, psi0.conj())
    exact = np.zeros_like(rho)
    for tup in itertools.product(*[range(len(c)) for c in chans]):
        K = cr.full_op(n, qubits, [c.kraus[i] for c, i in zip(chans, tup)])
        exact += K @ rho @ K.conj().T
    assert np.all(np.abs(mean - exact) <= 5 * sigma + 1e-12)


def test_determinism_and_launch_counts(ctx):
    n = 20
    psi = circuits.random_state(n, 20, C128)
    with State(n, C128, ctx) as st:
        outs = []
        for _ in range(2):
            st.upload(psi)
            l0 = ctx.kernel_launches()
            c, p = st.apply_channels(ch.amplitude_damping(0.01), range(n), draws=np.linspace(0.1, 0.9, n + 1))
            assert ctx.kernel_launches() - l0 == channels_plan(n, C128, ch.amplitude_damping(0.01), range(n))[3] == 12
            outs.append((list(c), p, st.download()))
        assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1] and bits_equal(outs[0][2], outs[1][2])
        dep = ch.depolarizing(0.01)
        st.upload(psi)
        l0 = ctx.kernel_launches()
        c, p = st.apply_channels(dep, range(n), draws=[0.5] * n + [0.999])  # the last qubit takes a Pauli error
        assert ctx.kernel_launches() - l0 == channels_plan(n, C128, dep, range(n))[3] == 1
        assert c[-1] > 0 and all(v == 0 for v in c[:-1])
        st.upload(psi)
        l0 = ctx.kernel_launches()
        c, p = st.apply_channels(dep, range(n), draws=[0.5] * (n + 1))  # every choice the scaled identity
        assert ctx.kernel_launches() == l0 and bits_equal(st.download(), psi)
        assert p == pytest.approx(0.99 ** n, rel=1e-13)


def test_pending_collapse_and_pending_basis(ctx):
    n = 14
    psi = circuits.random_state(n, 41, C128)
    chans, qubits = [ch.amplitude_damping(0.5), FLIP, ch.reset()], [1, 13, 6]
    draws = [0.37, 0.2, 0.5, 0.8]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 6], 0.61)
        b.collapse([0, 6], m, p)
        l0 = ctx.kernel_launches()
        ra = a.apply_channels(chans, qubits, draws=draws)
        la = ctx.kernel_launches() - l0
        l0 = ctx.kernel_launches()
        rb = b.apply_channels(chans, qubits, draws=draws)
        assert la == ctx.kernel_launches() - l0 + 1
        assert list(ra[0]) == list(rb[0]) and ra[1] == rb[1] and bits_equal(a.download(), b.download())
        a.set_basis(77)
        basis = np.zeros(1 << n, dtype=C128)
        basis[77] = 1.0
        b.upload(basis)
        ra, rb = a.apply_channels(chans, qubits, draws=draws), b.apply_channels(chans, qubits, draws=draws)
        assert list(ra[0]) == list(rb[0]) and ra[1] == rb[1] and bits_equal(a.download(), b.download())


_ROTATE_WORKER = r"""
import numpy as np
import channel_ref as cr
from rustqip_b200 import channels as ch, circuits
from rustqip_b200.state import Context, State

n = 18
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
flip = ch.pauli_channel(1.0, 0.0, 0.0)
cases = [([17, 3, 0, 9], [flip, ch.depolarizing(0.4), flip, ch.pauli_channel(0.2, 0.3, 0.1)]),
         ([0, 17, 4], [ch.amplitude_damping(0.3), flip, ch.reset()])]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for qubits, chans in cases:
            for st in (a, b):
                st.set_basis(3)
                st.apply_schedule(ops)
            qmap = b.qubit_map().copy()
            assert not np.array_equal(qmap, np.arange(n)[::-1]), "the schedule left the canonical layout"
            psi = a.download()
            draws = [0.3] + [0.9] * len(qubits)
            dep = any(c.state_dependent for c in chans)
            x = int(b.sample([q for q, c in zip(qubits, chans) if c.state_dependent], [0.3])[0]) if dep else 0
            if dep:  # the sample restored the layout
                qmap = b.qubit_map().copy()
            chosen, prob = b.apply_channels(chans, qubits, draws=draws)
            assert np.array_equal(b.qubit_map(), qmap), "apply_channels changed the layout"
            # the emulation on the physical vector: canonical bit n-1-q lives at qmap[q]
            idx = np.arange(1 << n, dtype=np.uint64)
            phys = np.zeros(1 << n, dtype=np.uint64)
            for q in range(n):
                phys |= ((idx >> np.uint64(n - 1 - q)) & np.uint64(1)) << np.uint64(qmap[q])
            ps = np.empty_like(psi)
            ps[phys.astype(np.int64)] = psi
            c, p, out = cr.emulate(ps, n, qubits, [k.kraus for k in chans], x, draws, phys=lambda q: int(qmap[q]))
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
    I = np.eye(2)

    def flat(*ops):
        return np.ascontiguousarray(np.concatenate([np.asarray(k, dtype=C128).reshape(-1) for k in ops])).view(
            np.float64)

    def call(st, qubits, n_kraus, kraus, draws, chosen=True, prob=True):
        qa = np.ascontiguousarray(np.asarray(qubits, dtype=np.uint64)) if qubits is not None else None
        na = np.ascontiguousarray(np.asarray(n_kraus, dtype=np.uint32)) if n_kraus is not None else None
        da = np.ascontiguousarray(np.asarray(draws, dtype=np.float64)) if draws is not None else None
        out = np.zeros(8, dtype=np.uint32)
        p = C.c_double()
        nc = len(qubits) if qubits is not None else len(n_kraus)
        return L.qipb200_state_apply_channels(st._h, nc, qa.ctypes.data if qa is not None else None,
                                              na.ctypes.data if na is not None else None,
                                              kraus.ctypes.data if kraus is not None else None,
                                              da.ctypes.data if da is not None else None,
                                              out.ctypes.data if chosen else None, C.byref(p) if prob else None)

    ad = ch.amplitude_damping(0.2).kraus
    ok = flat(ad[0], ad[1])
    cases = [
        (([1], [2], ok, [0.1, 0.2]), dict(prob=False), INVALID_ARG, "apply_channels: NULL prob"),
        (([1], [2], ok, None), {}, INVALID_ARG, "apply_channels: NULL draws or chosen"),
        (([1], [2], ok, [0.1, 0.2]), dict(chosen=False), INVALID_ARG, "apply_channels: NULL draws or chosen"),
        ((None, [2], ok, [0.1, 0.2]), {}, INVALID_ARG, "apply_channels: NULL qubits, n_kraus or kraus"),
        (([1], [2], None, [0.1, 0.2]), {}, INVALID_ARG, "apply_channels: NULL qubits, n_kraus or kraus"),
        (([12], [2], ok, [0.1, 0.2]), {}, BAD_INDEX, "apply_channels: channel 0: qubit 12 out of range for 12 qubits"),
        (([3, 3], [1, 1], flat(I, I), [0.1, 0.2, 0.3]), {}, BAD_INDEX, "apply_channels: channel 1: qubit 3 repeated"),
        (([3], [0], ok, [0.1, 0.2]), {}, INVALID_ARG, "apply_channels: channel 0: n_kraus must be 1..16, got 0"),
        (([3], [2], flat(I, np.diag([np.nan, 0])), [0.1, 0.2]), {}, INVALID_ARG,
         "apply_channels: channel 0, operator 1: an entry is not finite"),
        (([3], [2], flat(I, np.zeros((2, 2))), [0.1, 0.2]), {}, INVALID_ARG,
         "apply_channels: channel 0, operator 1: the zero matrix"),
        (([3], [1], flat(np.ones((2, 2)) / np.sqrt(2)), [0.1, 0.2]), {}, INVALID_ARG,
         "apply_channels: channel 0, operator 0: neither diagonal nor anti-diagonal"),
        (([3], [1], flat(2 * I), [0.1, 0.2]), {}, INVALID_ARG,
         "apply_channels: channel 0: the operators are not complete (sum of |d_i(0)|^2 - 1 = 3)"),
        (([3], [2], ok, [0.1, 1.0]), {}, INVALID_ARG, "apply_channels: draw 1 is not in [0, 1)"),
        (([3], [2], ok, [-0.1, 0.5]), {}, INVALID_ARG, "apply_channels: draw 0 is not in [0, 1)"),
        (([3], [2], ok, [0.1, np.nan]), {}, INVALID_ARG, "apply_channels: draw 1 is not in [0, 1)"),
    ]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 6], 0.37)
        l0 = ctx.kernel_launches()
        for args, kw, code, msg in cases:
            assert call(a, *args, **kw) == code, msg
            assert L.qipb200_last_error(ctx.handle).decode() == msg
        assert L.qipb200_state_apply_channels(None, 0, None, None, None, None, None, None) == INVALID_ARG
        assert ctx.kernel_launches() == l0
        c0, p0 = a.apply_channels([], [])
        assert p0 == 1.0 and ctx.kernel_launches() == l0
        with pytest.raises(ValueError):
            a.apply_channels([ch.reset()], [0, 1])
        # the collapse is still pending: one kernel for it, then the call's own
        l0 = ctx.kernel_launches()
        a.apply_channels(FLIP, [4], draws=[0.5, 0.5])
        assert ctx.kernel_launches() - l0 == 2
        b.collapse([0, 6], m, p)
        b.apply_channels(FLIP, [4], draws=[0.5, 0.5])
        assert bits_equal(a.download(), b.download())
    with State(n, C128, ctx, rank=0, world_size=2) as sh:
        with pytest.raises(CircuitError) as e:
            sh.apply_channels(ch.reset(), [0])
        assert e.value.status == UNSUPPORTED and str(e.value) == "apply_channels: sharded states are not supported"
