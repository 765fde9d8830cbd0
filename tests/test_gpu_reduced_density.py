"""Reduced density matrices on the device (State.reduced_density, qipb200_state_reduced_density).

Every element is checked against |got - want| <= bound(n, k) * W_ab with W_ab = sum_r |psi_ra| |psi_rb|; tests/rdm_ref.py
derives the bound from the kernel's summation depth (and tests/test_reduced_density_cpu.py pins its references).  On
states of Gaussian integers the result must equal the integer reference bit for bit.  The worst |got - want| / bound per
group of checks is printed (run with -s to see it)."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import pauli_ref as pr
import rdm_ref as rr
from exact_circuits import exact_state
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
PRODUCT_V = [(1, 0.5), (0.5, 1j), (0.5j, 0.5), (-0.5, 1), (1, -0.25j), (0.25, -1)]
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[reduced_density] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def launches_for(k):
    """One sweep kernel and one reduction per block pair I <= J of nB = 2^max(0, k-6) blocks."""
    nb = 1 << max(0, k - 6)
    return nb * (nb + 1)


def check_against_ref(group, psi, n, qubits, got):
    k = len(qubits)
    assert got.shape == (1 << k, 1 << k) and got.dtype == np.complex128
    want = rr.rdm_ref(psi, n, qubits)
    b = rr.bound(n, k, rr.abs_weight(psi, n, qubits))
    err = np.abs(got.astype(np.clongdouble) - want).astype(np.float64)
    bad = np.argwhere(err > b)
    assert bad.size == 0, (group, n, qubits, bad[:4], err[tuple(bad[0])], b[tuple(bad[0])])
    pos = b > 0
    note(group, float(np.max(err[pos] / b[pos])) if np.any(pos) else 0.0)
    assert np.all(err[~pos] == 0)


def qubit_lists(n, k, rng):
    """The bottom and top index bits (qubits n-1 and 0) in reversed order, the lowest index bits unsorted, and a random
    choice: bits inside and outside the tile, and for k > 6 low bits that must be tile columns."""
    lists = [list(range(n - 1, n - 1 - k, -1))[::-1]]  # the k lowest index bits, from the highest of them down
    if k >= 2:
        mid = [int(q) for q in rng.permutation(np.arange(1, n - 1))[: k - 2]]
        lists.append([n - 1] + mid + [0])
    lists.append([int(q) for q in rng.permutation(n)[:k]])
    return lists


@pytest.mark.parametrize("dtype", [C128, C64])
def test_small_states_against_reference(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 17):
        rng = np.random.default_rng(500 + n)
        states = [("random", circuits.random_state(n, 170 + n, dtype))]
        if n >= 3:
            states.append(("circuit", None))
        with State(n, dtype, ctx) as st:
            for kind, psi in states:
                if psi is None:
                    st.set_basis(1)
                    st.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0300 + n, "H,T,CNOT"))
                else:
                    st.upload(psi)
                psi = st.download()
                for k in range(1, min(n, 10) + 1):
                    lists = qubit_lists(n, k, rng)
                    if n >= 14 and k >= 8:
                        lists = lists[1:2]
                    for qs in lists:
                        check_against_ref("small %s %s k%s" % (name, kind, "<=6" if k <= 6 else ">6"), psi, n, qs,
                                          st.reduced_density(qs))


@pytest.mark.parametrize("dtype", [C128, C64])
@pytest.mark.parametrize("n", [5, 12, 16, 20])
def test_exact_on_dyadic_states(ctx, n, dtype):
    """Gaussian-integer amplitudes: every product and partial sum is exact, so the device must reproduce the integer
    reference bit for bit, through the in-tile path (k <= 6) and the block path (k >= 7)."""
    bits = min(16, (52 - (n - 1)) // 2)
    psi = exact_state(n, 900 + n, bits, dtype=dtype)
    rng = np.random.default_rng(n)
    with State(n, dtype, ctx) as st:
        st.upload(psi)
        for k in range(1, min(n, 10) + 1):
            for qs in qubit_lists(n, k, rng):
                assert rr.budget_ok(psi, n, k)
                got = st.reduced_density(qs)
                want = rr.rdm_exact(psi, n, qs)
                assert np.array_equal(got, want), (n, qs, np.argwhere(got != want)[:4])


def test_hermitian_and_deterministic(ctx):
    n = 14
    with State(n, C128, ctx) as st:
        st.upload(circuits.random_state(n, 41, C128))
        for qs in ([3, 0, 13], [13, 12, 11, 10, 9, 8, 0, 1]):
            a = st.reduced_density(qs)
            b = st.reduced_density(qs)
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
            # off the diagonal, bit for bit (the conjugate of +0.0 is -0.0, so the diagonal is checked on its own)
            off = ~np.eye(a.shape[0], dtype=bool)
            h = np.conj(a.T)
            assert np.array_equal(a[off].view(np.uint64), h[off].view(np.uint64))
            assert np.all(np.diag(a).imag.view(np.uint64) == 0)  # +0.0 exactly
            assert np.all(np.diag(a).real > 0)


def test_launch_count(ctx):
    n = 16
    with State(n, C128, ctx) as st:
        st.upload(circuits.random_state(n, 5, C128))
        for qs in ([0], [15, 2, 9, 0, 4, 11], [15, 2, 9, 0, 4, 11, 7], list(range(10))):
            l0 = ctx.kernel_launches()
            st.reduced_density(qs)
            assert ctx.kernel_launches() - l0 == launches_for(len(qs)), qs
    assert [launches_for(k) for k in (1, 6, 7, 8, 9, 10)] == [2, 2, 6, 20, 72, 272]


def test_cross_checks_at_n20(ctx):
    """diag(rho) against measure_probs (bound widened by gamma_{2^n} for the histogram's unordered sums) and
    Tr(rho P) against expect_paulis for all 4^k strings on the kept qubits."""
    n = 20
    u = pr.U_DOUBLE
    with State(n, C128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule(circuits.random_circuit(n, 12, 0x5EED0400, "H,T,CNOT"))
        psi = st.download()
        for qs in ([0, 19], [7, 19, 0], [19, 18, 17, 16, 0], [3, 11]):
            rho = st.reduced_density(qs)
            b = rr.bound(n, len(qs), rr.abs_weight(psi, n, qs))
            probs = st.measure_probs(qs)
            tol = np.diag(b) + pr.gamma(1 << n, u) * probs + 1e-300
            err = np.abs(np.diag(rho).real - probs)
            assert np.all(err <= tol), (qs, np.max(err / tol))
            note("n20 diag vs measure_probs", float(np.max(err / tol)))
            if len(qs) > 3:
                continue
            terms = [[(l, q) for l, q in zip(ls, qs) if l != "I"] for ls in itertools.product("IXYZ", repeat=len(qs))]
            ev = st.expect_paulis(terms)
            tol = float(np.sum(b)) + pr.bound(n, 1.0)
            for t, e in zip(terms, ev):
                v = np.trace(rho @ rr.pauli_matrix(t, qs))
                assert abs(v.imag) <= tol and abs(v.real - e) <= tol, (qs, t, v, e, tol)
                note("n20 Tr(rho P) vs expect_paulis", abs(v.real - e) / tol)


def test_validation_on_state(ctx):
    with State(12, C128, ctx) as st:
        st.set_basis(0)
        lib = _lib.lib()
        out = np.zeros(2 * 4 ** 3)
        qs = np.array([0, 1, 2], dtype=np.uint64)
        assert lib.qipb200_state_reduced_density(st._h, None, 1, out.ctypes.data) == INVALID_ARG
        assert lib.qipb200_state_reduced_density(st._h, qs.ctypes.data, 0, out.ctypes.data) == INVALID_ARG
        assert lib.qipb200_state_reduced_density(st._h, qs.ctypes.data, 3, None) == INVALID_ARG
        with pytest.raises(CircuitError) as e:
            st.reduced_density(list(range(12)) + [0])
        assert e.value.status == INVALID_ARG  # k > n
        with pytest.raises(CircuitError) as e:
            st.reduced_density([0, 12])
        assert e.value.status == BAD_INDEX and "out of range" in str(e.value)
        with pytest.raises(CircuitError) as e:
            st.reduced_density([4, 1, 4])
        assert e.value.status == BAD_INDEX and "repeated" in str(e.value)
        with pytest.raises(CircuitError) as e:
            st.reduced_density(list(range(11)))
        assert e.value.status == UNSUPPORTED and "10" in str(e.value)
        with pytest.raises(CircuitError) as e:
            st.reduced_density([])
        assert e.value.status == INVALID_ARG
    with State(12, C128, ctx, rank=0, world_size=2) as st:
        with pytest.raises(CircuitError) as e:
            st.reduced_density([0])
        assert e.value.status == UNSUPPORTED and "sharded" in str(e.value)


def test_sees_pending_collapse(ctx):
    n = 16
    psi = circuits.random_state(n, 21, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 5], 0.37)
        assert p > 0
        got = a.reduced_density([5, 2, 15])  # applies the collapse measure left pending
        b.collapse([0, 5], m, p)
        want = b.reduced_density([5, 2, 15])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
        check_against_ref("after measure f64", b.download(), n, [5, 2, 15], got)


_ROTATE_WORKER = r"""
import numpy as np
import rdm_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 18
lists = [[0], [17, 0], [3, 9, 14], [17, 16, 15, 14, 0, 1], [0, 2, 4, 6, 8, 10, 12, 17]]
worst = 0.0
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as st:
        st.set_basis(3)
        st.apply_schedule(circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60])
        before = st.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        got = [st.reduced_density(qs) for qs in lists]
        assert np.array_equal(st.qubit_map(), before), "reduced_density restored the layout"
        psi = st.download()
    for qs, g in zip(lists, got):
        want = rr.rdm_ref(psi, n, qs)
        b = rr.bound(n, len(qs), rr.abs_weight(psi, n, qs))
        err = np.abs(g.astype(np.clongdouble) - want).astype(np.float64)
        assert np.all(err <= b), (qs, float(np.max(err - b)))
        worst = max(worst, float(np.max(err[b > 0] / b[b > 0])))
print("ROTATE worst ratio %.3e" % worst)
"""


def test_permuted_layout_is_read_in_place():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    note("rotate f64 n=18", float(p.stdout.split("worst ratio")[1].split()[0]))


# ---- full size: closed forms ------------------------------------------------------------------------------------

class Holder:
    """One full-size state at a time; freeing it returns its buffer to the device (at most 32 GiB alive)."""

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


def full_lists(n):
    return [[0], [n - 1, 0], [0, 1, n - 3, n - 2, n - 1, n // 2], [n - 1, 0, 2, 9, n - 6, 17, 1],
            [0, n - 1, 3, 12, n - 2, 7, 21, n - 5, 1, 26]]


def check_closed(group, n, qs, got, want):
    W = np.abs(want).astype(np.float64)  # one contributing row per entry (GHZ) or a product (product state)
    b = rr.bound(n, len(qs), W)
    err = np.abs(got.astype(np.clongdouble) - want).astype(np.float64)
    assert np.all(err <= b), (group, qs, float(np.max(err - b)))
    pos = b > 0
    note(group, float(np.max(err[pos] / b[pos])))


@pytest.mark.parametrize("n,dtype", [(30, C128), (32, C64)], ids=["n30_f64", "n32_f32"])
def test_full_size_closed_forms(holder, n, dtype):
    name = "n%d %s" % (n, np.dtype(dtype).name)
    st = holder.take(n, dtype)
    # GHZ with phases: H, CNOTs (exact), then T and S on the |1..1> branch; the two amplitudes are read back
    st.set_basis(0)
    st.apply_schedule([gates.h(0)] + [gates.cnot(0, k) for k in range(1, n)] + [gates.t(0), gates.s(n // 2)])
    alpha = complex(st.download(offset=0, length=1)[0])
    beta = complex(st.download(offset=(1 << n) - 1, length=1)[0])
    for qs in full_lists(n):
        check_closed("full %s ghz" % name, n, qs, st.reduced_density(qs), rr.ghz_rdm(n, qs, alpha, beta))
    # product state from one MAT op per qubit
    st.set_basis(0)
    vs = [PRODUCT_V[q % len(PRODUCT_V)] for q in range(n)]
    st.apply_schedule([gates.mat([q], [vs[q][0], 0, vs[q][1], 0]) for q in range(n)])
    for qs in full_lists(n):
        check_closed("full %s product" % name, n, qs, st.reduced_density(qs), rr.product_rdm(n, qs, vs))
    holder.release()


def test_headline_state(holder):
    """The N=30 f64 headline state (random {H,T,CNOT}, depth 40, seed 0x5EED0002) at k = 2 and 3: the diagonal against
    measure_probs, every Pauli component Tr(rho P) against expect_paulis."""
    n = 30
    u = pr.U_DOUBLE
    st = holder.take(n, C128)
    st.set_basis(0)
    st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
    for qs in ([0, 29], [29, 14, 0], [5, 6, 7]):
        k = len(qs)
        rho = st.reduced_density(qs)
        assert np.array_equal(rho, np.conj(rho.T))
        b = float(np.max(rr.bound(n, k, np.ones((1, 1)))))  # per element, with W_ab <= 1 for a unit state
        probs = st.measure_probs(qs)
        tol = b + pr.gamma(1 << n, u)
        err = np.abs(np.diag(rho).real - probs)
        assert np.all(err <= tol), (qs, float(np.max(err)), tol)
        note("headline n30 diag vs measure_probs", float(np.max(err)) / tol)
        terms = [[(l, q) for l, q in zip(ls, qs) if l != "I"] for ls in itertools.product("IXYZ", repeat=k)]
        ev = st.expect_paulis(terms)
        tol = (1 << k) * b + pr.bound(n, 1.0)  # a Pauli matrix has one unit entry per row
        for t, e in zip(terms, ev):
            v = np.trace(rho @ rr.pauli_matrix(t, qs))
            assert abs(v.real - e) <= tol and abs(v.imag) <= tol, (qs, t, v, e, tol)
            note("headline n30 Tr(rho P) vs expect_paulis", abs(v.real - e) / tol)
    holder.release()
