"""Purity and Renyi-2 entropy of a bipartition on the device (State.purity, qipb200_state_purity).

Every result is checked against |got - want| <= device bound + reference bound (tests/purity_ref.py derives both from
the summation orders); on states of Gaussian integers, and at full size on integer states, out2 must equal the exact
integers bit for bit.  The worst |got - want| / bound per group is printed (run with -s to see it)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import purity_ref as pu
from exact_circuits import exact_state
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, purity_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[purity] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-44s %.3e" % (k, WORST[k]))


def out2(st, qs):
    return st._purity2(qs)


def check_against_ref(group, psi, n, qs, got):
    s = min(len(qs), n - len(qs))
    P, T, bp_ref, bt_ref, G, W = pu.purity_ref(psi, n, qs)
    bp, bt = pu.device_bound(n, s, G, W, P, T)
    bp, bt = bp + bp_ref, bt + bt_ref
    ep, et = abs(got[0] - P), abs(got[1] - T)
    assert ep <= bp and et <= bt, (group, n, qs, got, (P, T), (bp, bt))
    note(group, max(ep / bp if bp > 0 else 0.0, et / bt if bt > 0 else 0.0))


def side_lists(n, s, rng):
    """Prefix (qubits 0..s-1: the high index bits), suffix (the low bits), scattered, and the complements of the first
    and the last (k = n - s, so that the complement is the smaller side)."""
    pre = list(range(s))
    suf = list(range(n - s, n))[::-1]
    sc = [int(q) for q in rng.permutation(n)[:s]]
    lists = [pre, suf, sc]
    if 2 * s < n:
        lists += [[q for q in range(n) if q not in pre], [q for q in range(n) if q not in sc]]
    return lists


@pytest.mark.parametrize("dtype", [C128, C64])
def test_against_reference(ctx, dtype):
    name = np.dtype(dtype).name
    for n in list(range(2, 17)) + [18, 20, 22, 24]:
        rng = np.random.default_rng(700 + n)
        sides = range(0, n // 2 + 1) if n <= 16 else [11, 12] if n == 24 else [1, 10, 11]
        with State(n, dtype, ctx) as st:
            for kind in ("random", "circuit"):
                if kind == "random":
                    st.upload(circuits.random_state(n, 180 + n, dtype))
                else:
                    st.set_basis(1)
                    st.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0500 + n, "H,T,CNOT"))
                psi = st.download()
                for s in sides:
                    lists = [list(range(n))] if s == 0 else side_lists(n, s, rng)
                    if n == 24:  # a 4096^3 reference product per list: the prefix, then the scattered side
                        lists = lists[:1] if kind == "random" else lists[2:3]
                    for qs in lists:
                        r = pu.route(min(len(qs), n - len(qs)))
                        check_against_ref("%s %s route %d" % (name, kind, r), psi, n, qs, out2(st, qs))


@pytest.mark.parametrize("n,cases", [(22, ((11, 0), (11, 1), (11, 2))), (24, ((12, 0), (11, 2), (11, 3)))])
def test_exact_on_dyadic_states(ctx, n, cases):
    """Gaussian integers times 2^-2, small enough that every entry of G and every partial sum of P is an integer (times
    a power of two) below 2^53: the device must return the exact values, in f64 and f32.  Cases are (s, list) with
    lists prefix, suffix, scattered and the prefix's complement."""
    shift = 2
    psi = exact_state(n, 910 + n, 3, shift=shift)
    rng = np.random.default_rng(n)
    want = {}
    for s, i in cases:
        qs = side_lists(n, s, rng)[i]
        P, T = pu.purity_int(psi * 2.0 ** shift, n, qs)
        want[tuple(qs)] = (np.ldexp(float(P), -4 * shift), np.ldexp(float(T), -2 * shift))
    for dtype in (C128, C64):
        with State(n, dtype, ctx) as st:
            st.upload(psi.astype(dtype))
            for qs, w in want.items():
                got = out2(st, list(qs))
                assert got == w, (n, np.dtype(dtype).name, qs, got, w)


def test_deterministic_and_launch_count(ctx):
    n = 22
    with State(n, C128, ctx) as st:
        st.upload(circuits.random_state(n, 43, C128))
        for qs in ([0], [21, 3, 9], list(range(10)), list(range(11)), [q for q in range(n) if q % 2],
                   list(range(n)), list(range(3, n))):
            a = out2(st, qs)
            l0 = ctx.kernel_launches()
            b = out2(st, qs)
            plan = purity_plan(n, C128, qs)
            assert ctx.kernel_launches() - l0 == plan[2], (qs, plan)
            assert plan == pu.plan(n, qs)
            assert np.array_equal(np.array(a).view(np.uint64), np.array(b).view(np.uint64)), qs
        p = st.purity(list(range(11)))
        assert p == out2(st, list(range(11)))[0]
        nrm = st.norm2()
        assert abs(st.renyi2_entropy(list(range(11))) + np.log(p / nrm ** 2)) <= 1e-12


def test_sees_pending_collapse(ctx):
    n = 22
    psi = circuits.random_state(n, 22, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 5], 0.37)
        assert p > 0
        l0 = ctx.kernel_launches()
        qs = list(range(11, 22))
        got = out2(a, qs)  # applies the collapse measure left pending (one more kernel)
        assert ctx.kernel_launches() - l0 == 1 + pu.plan(n, qs)[2]
        assert out2(a, qs) == got
        b.collapse([0, 5], m, p)
        check_against_ref("after measure f64", b.download(), n, qs, got)
        check_against_ref("after measure f64 rdm route", b.download(), n, [3, 7], out2(a, [3, 7]))


def test_validation_leaves_state_and_collapse(ctx):
    n = 14
    psi = circuits.random_state(n, 3, C128)
    lib = _lib.lib()
    with State(n, C128, ctx) as st, State(n, C128, ctx) as ref:
        st.upload(psi)
        ref.upload(psi)
        m, p = st.measure([2], 0.5)
        o = np.zeros(2)
        qs = np.array([0, 1, 2], dtype=np.uint64)
        l0 = ctx.kernel_launches()
        assert lib.qipb200_state_purity(None, qs.ctypes.data, 3, o.ctypes.data) == INVALID_ARG
        assert lib.qipb200_state_purity(st._h, None, 1, o.ctypes.data) == INVALID_ARG
        assert lib.qipb200_state_purity(st._h, qs.ctypes.data, 0, o.ctypes.data) == INVALID_ARG
        assert lib.qipb200_state_purity(st._h, qs.ctypes.data, 3, None) == INVALID_ARG
        for bad, code, word in ((list(range(n)) + [0], INVALID_ARG, ""), ([0, n], BAD_INDEX, "out of range"),
                                ([4, 1, 4], BAD_INDEX, "repeated"), ([], INVALID_ARG, "")):
            with pytest.raises(CircuitError) as e:
                st.purity(bad)
            assert e.value.status == code and word in str(e.value), bad
        assert ctx.kernel_launches() == l0  # nothing ran, the collapse is still pending
        ref.collapse([2], m, p)
        assert np.array_equal(st.download().view(np.uint64), ref.download().view(np.uint64))
    with State(12, C128, ctx, rank=0, world_size=2) as st:
        with pytest.raises(CircuitError) as e:
            st.purity([0])
        assert e.value.status == UNSUPPORTED and "sharded" in str(e.value)


_ROTATE_WORKER = r"""
import numpy as np
import purity_ref as pu
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 22
lists = [[0, 5, 9], list(range(11)), list(range(11, 22)), [1, 3, 5, 7, 9, 11, 13, 15, 17, 19, 21], list(range(1, 22))]
worst = 0.0
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as st:
        st.set_basis(3)
        st.apply_schedule(circuits.random_circuit(n, 10, 12, "H,T,CNOT") + circuits.qft(n)[:60])
        before = st.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        got = [st._purity2(qs) for qs in lists]
        assert np.array_equal(st.qubit_map(), before), "purity restored the layout"
        psi = st.download()
    for qs, g in zip(lists, got):
        s = min(len(qs), n - len(qs))
        P, T, bp_ref, bt_ref, G, W = pu.purity_ref(psi, n, qs)
        bp, bt = pu.device_bound(n, s, G, W, P, T)
        bp, bt = 2 * bp + bp_ref, 2 * bt + bt_ref
        assert abs(g[0] - P) <= bp and abs(g[1] - T) <= bt, (qs, g, P, T, bp, bt)
        worst = max(worst, abs(g[0] - P) / bp, abs(g[1] - T) / bt)
print("ROTATE worst ratio %.3e" % worst)
"""


def test_permuted_layout_is_read_in_place():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    note("rotate f64 n=22", float(p.stdout.split("worst ratio")[1].split()[0]))


# ---- full size -------------------------------------------------------------------------------------------------

class Holder:
    """One full-size state at a time; freeing it returns its buffer to the device."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.st = None
        ctx.release_pool()

    def take(self, n, dtype):
        self.release()
        self.st = State(n, dtype, self.ctx)
        return self.st

    def release(self):
        if self.st is not None:
            self.st.free()
            self.st = None
        self.ctx.release_pool()


@pytest.fixture(scope="module")
def holder(ctx):
    h = Holder(ctx)
    yield h
    h.release()


def upload_integer_state(st, n, dtype, pairs, plus):
    """Amplitude 1 where every pair (p, q) of qubits agrees and every qubit outside the pairs and `plus` is 0, else 0:
    Bell pairs |00> + |11>, unnormalised |0> + |1> on `plus`, |0> elsewhere.  Uploaded in chunks of 2^24 amplitudes;
    the low 24 index bits vary inside a chunk, the high bits are fixed by its offset."""
    L = 24
    j = np.arange(1 << L, dtype=np.uint64)
    bit = {q: ((j >> np.uint64(n - 1 - q)) & np.uint64(1)).astype(bool) for q in range(n - L, n)}
    zero = [q for q in range(n) if q not in plus and all(q not in pq for pq in pairs)]
    base = np.ones(1 << L, dtype=bool)
    for p, q in pairs:
        if p >= n - L:
            base &= bit[p] == bit[q]
    for q in zero:
        if q >= n - L:
            base &= ~bit[q]
    for c in range(1 << (n - L)):
        hb = lambda q: (c >> (n - 1 - q - L)) & 1  # noqa: E731  (qubit q < n - L)
        ok = base.copy()
        if any(q < n - L and hb(q) for q in zero):
            ok[:] = False
        for p, q in pairs:
            if p < n - L:
                ok &= bit[q] if hb(p) else ~bit[q]
        st.upload(ok.astype(dtype), c << L)


@pytest.mark.parametrize("n,dtype", [(30, C128), (31, C64)], ids=["n30_f64", "n31_f32"])
def test_full_size_closed_forms(holder, n, dtype):
    half = n // 2
    side = list(range(half))  # qubits 0..half-1: the high index bits
    st = holder.take(n, dtype)
    for m in range(11, half + 1) if n == 30 else (12, 15):
        pairs = [(i, half + i) for i in range(m)]
        plus = [q for q in range(m, n) if q not in [p for pq in pairs for p in pq] and q % 3 == 0]
        upload_integer_state(st, n, dtype, pairs, plus)
        P = (1 << m) * 4 ** len(plus)
        T = (1 << m) * 2 ** len(plus)
        got = out2(st, side)
        assert got == (float(P), float(T)), (m, got, P, T)
        assert got[0] / got[1] ** 2 == 2.0 ** -m
        assert purity_plan(n, dtype, side)[0] == 2
    # a product state: |0> + |1> on every qubit, all amplitudes 1
    for off in range(0, 1 << n, 1 << 24):
        st.upload(np.ones(1 << 24, dtype=dtype), off)
    T = 2 ** n
    assert out2(st, side) == (float(T) ** 2, float(T))
    # GHZ: |0..0> + |1..1>
    st.set_basis(0)
    st.upload(np.ones(1, dtype=dtype), (1 << n) - 1)
    assert out2(st, side) == (2.0, 2.0)
    assert out2(st, list(range(n - half, n))) == (2.0, 2.0)
    holder.release()


def test_full_size_prefix_and_suffix_agree(holder):
    """A random-circuit state at N=30 f64: the purity of qubits 0..s-1 (high bits, prefix loader), then a swap network
    that moves them onto qubits n-s..n-1 and the purity there (low bits, suffix loader); swaps move amplitudes exactly,
    so both see the same M.  The call leaves the state as it was: its fixed-order squared norm (the k = n route) and a
    downloaded window are bit-identical before and after."""
    n = 30
    st = holder.take(n, C128)
    st.set_basis(0)
    st.apply_schedule(circuits.random_circuit(n, 20, 0x5EED0600, "H,T,CNOT"))
    for s in (11, 15):
        nrm = out2(st, list(range(n)))
        win = st.download(offset=(1 << n) - (1 << 20) - 12345, length=1 << 16)
        a = out2(st, list(range(s)))
        assert out2(st, list(range(n))) == nrm
        assert np.array_equal(st.download(offset=(1 << n) - (1 << 20) - 12345, length=1 << 16).view(np.uint64),
                              win.view(np.uint64))
        st.apply_schedule([gates.swap(list(range(s)), list(range(n - s, n)))])
        b = out2(st, list(range(n - s, n)))
        st.apply_schedule([gates.swap(list(range(s)), list(range(n - s, n)))])
        bp, bt = pu.bound_cs(n, s, a[0], a[1])
        assert abs(a[0] - b[0]) <= 2 * bp and abs(a[1] - b[1]) <= 2 * bt, (s, a, b, bp, bt)
        note("n30 prefix vs suffix", max(abs(a[0] - b[0]) / (2 * bp), abs(a[1] - b[1]) / (2 * bt)))
        assert abs(a[1] - 1.0) < 1e-9 and 0 < a[0] <= 1.0 + 1e-9
    holder.release()
