"""General Kraus channels along quantum trajectories on the device (State.apply_kraus_channels,
qipb200_state_apply_kraus_channels).

The state is compared bit for bit with the emulation of tests/kraus_channel_ref.py given the returned chosen and cond;
cond with a long-double reference within its bound, and chosen with the reference's choice wherever the draw lies
farther than that bound from a cumulative boundary.  Also: a mixed layer against its state-dependent part plus
apply_schedule, X-axis damping of |->^30 at N = 30 and of windows past 2^31 and 2^32 against the product-state closed
form, a trajectory average against the exact channel, determinism, launch counts, pending work, a permuted layout and
the refusals."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import kraus_channel_ref as kr
from rustqip_b200 import _lib, circuits
from rustqip_b200 import channels as ch
from rustqip_b200.ops import make_matrix_op
from rustqip_b200.state import State, kraus_channels_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX = 1, 3
CX = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]], dtype=np.complex128)
H = np.array([[1, 1], [1, -1]], dtype=np.complex128) / np.sqrt(2)


def bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def x_damping(g):
    return ch.KrausChannel([H @ k @ H for k in ch.amplitude_damping(g).kraus])


def random_layer(rng, n, kmax=4):
    """Disjoint qubit groups of 1..min(3, n) qubits with random Stinespring channels, holding qubits n - 1 .. n - 4 (the
    low tile bits) and n - 8, n - 9 (across the first index byte) where the state has them."""
    pref = [q for q in (n - 1, n - 9, n - 2, n - 8, n - 3) if 0 <= q < n]
    rest = [int(q) for q in rng.permutation(n) if int(q) not in pref]
    free = pref + rest
    groups, chans = [], []
    while free and len(groups) < 6:
        k = int(rng.integers(1, min(kmax, 3, len(free)) + 1))
        groups.append([free.pop(0) for _ in range(k)])
        chans.append(kr.stinespring(k, int(rng.integers(2, 4)), rng))
    return groups, chans


def check_call(st, psi, n, groups, chans, draws):
    chosen, cond, prob = st.apply_kraus_channels(chans, groups, draws=draws)
    got = st.download()
    want = kr.emulate_groups(psi, n, groups, chans, chosen, cond)
    assert bits_equal(got, want), (n, int(np.sum(got != want)))
    p = 1.0
    for v in cond:
        p *= v
    assert prob == p
    for c, cl, ref_choice, dist, bound in kr.reference_conds(psi, n, groups, chans, chosen, cond, draws):
        assert abs(cond[c] - cl) <= bound, (n, c, cond[c], cl, bound)
        if dist > bound:
            assert int(chosen[c]) == ref_choice, (n, c)
    return chosen, cond, prob


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_emulation(ctx, dtype):
    rng = np.random.default_rng(5 if dtype == C128 else 6)
    for n in (2, 3, 4, 5, 7, 9, 12, 13, 16, 20, 23):
        groups, chans = random_layer(rng, n)
        psi = circuits.random_state(n, 100 + n, dtype)
        draws = rng.random(len(chans))
        with State(n, dtype, ctx) as st:
            st.upload(psi)
            check_call(st, psi, n, groups, chans, draws)


def test_bit_exact_at_26(ctx):
    rng = np.random.default_rng(26)
    n = 26
    groups = [[25, 17], [3], [24, 0], [10, 11, 12], [21]]
    chans = [kr.stinespring(len(g), 2, rng) for g in groups]
    ctx.release_pool()
    psi = circuits.random_state(n, 260, C64)
    with State(n, C64, ctx) as st:
        st.upload(psi)
        check_call(st, psi, n, groups, chans, rng.random(len(chans)))
    ctx.release_pool()


def test_mixed_layer_is_dependent_part_then_schedule(ctx):
    rng = np.random.default_rng(9)
    n = 16
    ncx = ch.KrausChannel([CX]).compose(ch.two_qubit_depolarizing(0.3))
    pz = ch.KrausChannel(ch.pauli_channel(0.2, 0.1, 0.3))
    dep = [kr.stinespring(2, 3, rng), x_damping(0.4), kr.stinespring(1, 2, rng)]
    chans = [dep[0], ncx, dep[1], pz, dep[2], ch.KrausChannel(ch.depolarizing(0.5))]
    groups = [[3, 9], [0, 15], [4], [7], [12], [1]]
    draws = [0.31, 0.77, 0.52, 0.93, 0.18, 0.64]
    for dtype in (C128, C64):
        psi = circuits.random_state(n, 7, dtype)
        with State(n, dtype, ctx) as a, State(n, dtype, ctx) as b:
            a.upload(psi)
            b.upload(psi)
            chosen, cond, prob = a.apply_kraus_channels(chans, groups, draws=draws)
            di = [0, 2, 4]
            cb, condb, _ = b.apply_kraus_channels([chans[i] for i in di], [groups[i] for i in di],
                                                  draws=[draws[i] for i in di])
            assert list(cb) == [chosen[i] for i in di] and list(condb) == [cond[i] for i in di]
            ops = []
            for i in (1, 3, 5):
                w = chans[i].weights[chosen[i]]
                assert cond[i] == w
                K = chans[i].kraus[chosen[i]]
                if np.array_equal(K, K[0, 0].real * np.eye(K.shape[0])) and K[0, 0].real > 0:
                    continue
                ops.append(make_matrix_op(groups[i], kr.scaled(K, w, dtype)))
            b.apply_schedule(ops)
            assert bits_equal(a.download(), b.download())


def _x_damped_amps(n, idx, flips):
    """Amplitudes at idx of the product state with qubit q in |+> where flips[q] else |->."""
    amp = np.full(idx.shape, 2.0 ** (-n / 2))
    for q in range(n):
        if not flips[q]:
            bit = (idx >> np.uint64(n - 1 - q)) & np.uint64(1)
            amp = np.where(bit == 1, -amp, amp)
    return amp


@pytest.mark.parametrize("n,dtype", [(30, C128), (31, C64), (32, C64)])
def test_x_damping_closed_form(ctx, n, dtype):
    g = 0.35
    chan = x_damping(g)
    draws = np.random.default_rng(n).random(n)
    ctx.release_pool()
    with State(n, dtype, ctx) as st:
        st.set_basis((1 << n) - 1)
        st.apply_schedule([make_matrix_op([q], H.astype(dtype)) for q in range(n)])  # |->^n
        l0 = ctx.kernel_launches()
        chosen, cond, prob = st.apply_kraus_channels(chan, [[q] for q in range(n)], draws=draws)
        assert ctx.kernel_launches() - l0 == kraus_channels_plan(n, dtype, chan, [[q] for q in range(n)])[3]
        flips = [int(c) == 1 for c in chosen]
        ctol = 1e-10 if dtype == C128 else 64 * n * 2.0 ** -24  # the amplitudes' rounding, relative
        for q in range(n):
            assert flips[q] == (draws[q] >= 1 - g) or abs(draws[q] - (1 - g)) < ctol, q
            assert abs(cond[q] - (g if flips[q] else 1 - g)) <= ctol
        u = 2.0 ** -53 if dtype == C128 else 2.0 ** -24
        N = 1 << n
        for off in ((0, N // 2 - (1 << 19), N - (1 << 20)) if n == 30 else (N // 2, N - (1 << 20))):
            got = st.download(offset=off, length=1 << 20)
            idx = np.arange(off, off + (1 << 20), dtype=np.uint64)
            want = _x_damped_amps(n, idx, flips)
            err = float(np.max(np.abs(got.astype(C128) - want)))
            assert err <= 16 * n * u * 2.0 ** (-n / 2) * 4, (off, err)
    ctx.release_pool()


def test_trajectory_average_matches_the_channel(ctx):
    rng = np.random.default_rng(17)
    n = 5
    groups = [[0, 3], [1], [4, 2]]
    chans = [kr.stinespring(2, 3, rng), x_damping(0.3), ch.KrausChannel([CX]).compose(
        ch.amplitude_damping(0.2).tensor(ch.amplitude_damping(0.4)))]
    psi = circuits.random_state(n, 3, C128)
    rho = np.zeros((1 << n, 1 << n), dtype=C128)
    T = 2000
    with State(n, C128, ctx) as st:
        for _ in range(T):
            st.upload(psi)
            st.apply_kraus_channels(chans, groups, rng=rng)
            v = st.download()
            rho += np.outer(v, v.conj()) / T
    want = np.outer(psi, psi.conj())
    for g, c in zip(groups, chans):
        out = np.zeros_like(want)
        for K in c.kraus:
            Kf = np.stack([kr.apply_dense(e, n, [g], [K]) for e in np.eye(1 << n, dtype=C128)], axis=1)
            out += Kf @ want @ Kf.conj().T
        want = out
    assert np.max(np.abs(rho - want)) <= 0.05


def test_determinism_and_launch_counts(ctx):
    rng = np.random.default_rng(23)
    n = 20
    groups, chans = random_layer(rng, n)
    psi = circuits.random_state(n, 23, C128)
    draws = rng.random(len(chans))
    outs = []
    with State(n, C128, ctx) as st:
        for _ in range(2):
            st.upload(psi)
            l0 = ctx.kernel_launches()
            outs.append(st.apply_kraus_channels(chans, groups, draws=draws) + (st.download(),))
            assert ctx.kernel_launches() - l0 == kraus_channels_plan(n, C128, chans, groups)[3]
        assert list(outs[0][0]) == list(outs[1][0]) and list(outs[0][1]) == list(outs[1][1])
        assert outs[0][2] == outs[1][2] and bits_equal(outs[0][3], outs[1][3])
        # a zero state is left untouched, prob 0
        z = np.zeros(1 << n, dtype=C128)
        st.upload(z)
        chosen, cond, prob = st.apply_kraus_channels(chans, groups, draws=draws)
        assert prob == 0.0 and not np.any(cond) and bits_equal(st.download(), z)


def test_pending_collapse_and_pending_basis(ctx):
    rng = np.random.default_rng(41)
    n = 14
    psi = circuits.random_state(n, 41, C128)
    chans = [kr.stinespring(2, 2, rng), x_damping(0.5), kr.stinespring(1, 3, rng)]
    groups = [[1, 9], [13], [6]]
    draws = [0.37, 0.2, 0.8]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 5], 0.61)
        b.collapse([0, 5], m, p)
        ra = a.apply_kraus_channels(chans, groups, draws=draws)
        rb = b.apply_kraus_channels(chans, groups, draws=draws)
        assert list(ra[0]) == list(rb[0]) and list(ra[1]) == list(rb[1]) and ra[2] == rb[2]
        assert bits_equal(a.download(), b.download())
        a.set_basis(77)
        basis = np.zeros(1 << n, dtype=C128)
        basis[77] = 1.0
        b.upload(basis)
        ra, rb = (a.apply_kraus_channels(chans, groups, draws=draws),
                  b.apply_kraus_channels(chans, groups, draws=draws))
        assert list(ra[0]) == list(rb[0]) and ra[2] == rb[2] and bits_equal(a.download(), b.download())


_ROTATE_WORKER = r"""
import numpy as np
import kraus_channel_ref as kr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 18
rng = np.random.default_rng(5)
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
groups = [[17, 3], [0], [9, 5, 11], [2]]
chans = [kr.stinespring(len(g), 2, rng) for g in groups]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for st in (a, b):
            st.set_basis(3)
            st.apply_schedule(ops)
        qmap = b.qubit_map().copy()
        assert not np.array_equal(qmap, np.arange(n)[::-1]), "the schedule left the canonical layout"
        psi = a.download()
        chosen, cond, prob = b.apply_kraus_channels(chans, groups, draws=[0.3, 0.9, 0.5, 0.1])
        assert np.array_equal(b.qubit_map(), qmap), "apply_kraus_channels changed the layout"
        idx = np.arange(1 << n, dtype=np.uint64)
        phys = np.zeros(1 << n, dtype=np.uint64)
        for q in range(n):
            phys |= ((idx >> np.uint64(n - 1 - q)) & np.uint64(1)) << np.uint64(qmap[q])
        ps = np.empty_like(psi)
        ps[phys.astype(np.int64)] = psi
        out = kr.emulate_groups(ps, n, groups, chans, chosen, cond, phys=lambda q: int(qmap[q]))
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
    L = _lib.lib()
    psi = circuits.random_state(n, 12, C128)

    def flat(*ops):
        return np.ascontiguousarray(np.concatenate([np.asarray(k, dtype=C128).reshape(-1) for k in ops])).view(
            np.float64)

    def arr(v, t):
        return np.ascontiguousarray(np.asarray(v, dtype=t))

    def call(st, arity, qubits, n_kraus, kraus, draws, chosen=True, prob=True):
        a, q, nk, d = arr(arity, np.uint32), arr(qubits, np.uint64), arr(n_kraus, np.uint32), arr(draws, np.float64)
        out = np.zeros(max(1, len(arity)), dtype=np.uint32)
        cond = np.zeros(max(1, len(arity)))
        p = C.c_double()
        s = L.qipb200_state_apply_kraus_channels(st._h, len(arity), a.ctypes.data, q.ctypes.data, nk.ctypes.data,
                                                 kraus.ctypes.data, d.ctypes.data if len(d) else None,
                                                 out.ctypes.data if chosen else None, cond.ctypes.data,
                                                 C.byref(p) if prob else None)
        return s, L.qipb200_last_error(ctx.handle).decode()

    I2 = np.eye(2)
    ad = ch.amplitude_damping(0.3).kraus
    cases = [
        (([1], [0], [2], flat(*ad), [0.5]), dict(prob=False), INVALID_ARG, "apply_kraus_channels: NULL prob"),
        (([1], [0], [2], flat(*ad), [0.5]), dict(chosen=False), INVALID_ARG,
         "apply_kraus_channels: NULL draws or chosen"),
        (([1], [12], [2], flat(*ad), [0.5]), {}, BAD_INDEX,
         "apply_kraus_channels: channel 0: qubit 12 out of range for 12 qubits"),
        (([1, 1], [3, 3], [2, 1], flat(*ad, I2), [0.5, 0.5]), {}, BAD_INDEX,
         "apply_kraus_channels: channel 1: qubit 3 repeated"),
        (([1], [0], [1], flat(np.array([[1, 0.5], [0, 1]])), [0.5]), {}, INVALID_ARG,
         "apply_kraus_channels: channel 0: the operators are not complete (entry (0, 1) of sum K^dagger K - I is "
         "0.5+0i)"),
        (([1], [0], [2], flat(*ad), [1.0]), {}, INVALID_ARG, "apply_kraus_channels: draw 0 is not in [0, 1)"),
    ]
    with State(n, C128, ctx) as a:
        a.upload(psi)
        m, p = a.measure([0, 6], 0.37)
        l0 = ctx.kernel_launches()
        for args, kw, status, msg in cases:
            assert call(a, *args, **kw) == (status, msg)
        assert ctx.kernel_launches() == l0  # nothing ran, the collapse is still pending
        with State(n, C128, ctx) as b:
            b.upload(psi)
            b.collapse([0, 6], m, p)
            assert bits_equal(a.download(), b.download())
        with pytest.raises(ValueError):
            a.apply_kraus_channels(ch.amplitude_damping(0.1), [[0]], draws=[0.1, 0.2])
        chosen, cond, p0 = a.apply_kraus_channels([], [], draws=[])
        assert p0 == 1.0 and len(chosen) == 0
