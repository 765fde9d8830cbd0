"""Pauli-string expectation values on the device (State.expect_paulis, qipb200_state_expect_paulis).

Every value is checked against |got - want| <= bound(n) * S with S = sum_j |a_j| |a_{j^x}|; tests/pauli_ref.py derives
the bound from the kernel's summation depth (and tests/test_expect_cpu.py pins its long-double reference to explicit
Kronecker products).  The worst |got - want| / bound per group of checks is printed (run with -s to see it)."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import pauli_ref as pr
from rustqip_b200 import circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, expect_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
UNSUPPORTED = 7
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[expect_paulis] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def check_against_ref(group, psi, n, terms, got):
    assert got.shape == (len(terms),)
    for t, g in zip(terms, got):
        want = pr.expect_ref(psi, n, t)
        b = pr.bound(n, pr.abs_weight(psi, n, t))
        err = float(abs(np.longdouble(g) - want))
        assert err <= b, (group, n, t, float(g), float(want), b)
        note(group, err / b if b > 0 else 0.0)


def random_terms(n, rng, count):
    terms = []
    for i in range(count):
        w = 1 + i % n
        qs = rng.choice(n, size=w, replace=False)
        terms.append([(str(rng.choice(list("XYZ"))), int(q)) for q in qs])
    return terms


def term_set(n, rng):
    """The all-X string first (so that the Z-only terms ride in its sweep, a tile pair when n > 11), the identity,
    all-Y and all-Z, every letter on every qubit, one X/Y mask with many Z patterns (the transform path), random
    terms of every weight."""
    terms = [[("X", q) for q in range(n)], [], [("Y", q) for q in range(n)], [("Z", q) for q in range(n)]]
    terms += [[(l, q)] for q in range(n) for l in "XYZ"]
    others = [q for q in range(n) if q not in (0, n - 1)][:4]
    for zs in range(1 << len(others)):
        terms.append([("Y", 0)] + ([("X", n - 1)] if n > 1 else []) + [("Z", q) for k, q in enumerate(others) if zs >> k & 1])
    return terms + random_terms(n, rng, 3 * n + 8)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_small_states_against_reference(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 17):
        rng = np.random.default_rng(1000 + n)
        terms = term_set(n, rng)
        states = [("random", circuits.random_state(n, 70 + n, dtype)),
                  ("random x0.5", (circuits.random_state(n, 90 + n, dtype) * 0.5).astype(dtype))]
        if n >= 3:
            states.append(("circuit", None))
        with State(n, dtype, ctx) as st:
            for kind, psi in states:
                if psi is None:
                    st.set_basis(1)
                    st.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0100 + n, "H,T,CNOT"))
                else:
                    st.upload(psi)
                got = st.expect_paulis(terms)
                psi = st.download()
                check_against_ref("small %s %s" % (name, kind), psi, n, terms, got)


def test_identity_is_norm2_and_empty_list(ctx):
    with State(12, C128, ctx) as st:
        st.upload(circuits.random_state(12, 5, C128) * 0.75)
        v = st.expect_paulis([[]])
        assert abs(v[0] - st.norm2()) <= 1e-14
        assert st.expect_paulis([]).shape == (0,)


def test_deterministic_and_launch_count(ctx):
    n = 20
    rng = np.random.default_rng(7)
    ising = [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]
    cases = [ising, term_set(n, rng), random_terms(n, rng, 600), [[("X", q) for q in range(n)]]]
    with State(n, C128, ctx) as st:
        st.set_basis(0)
        st.apply_schedule(circuits.random_circuit(n, 10, 0x5EED0200, "H,T,CNOT"))
        st.sync()
        for terms in cases:
            sweeps = expect_plan(n, C128, terms)
            l0 = ctx.kernel_launches()
            a = st.expect_paulis(terms)
            # one kernel per sweep plus one reduction kernel per batch of <= 16384 terms
            assert ctx.kernel_launches() - l0 == sweeps + 1
            b = st.expect_paulis(terms)
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_many_terms_run_in_batches(ctx):
    n = 10
    rng = np.random.default_rng(11)
    terms = [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.5)] for _ in range(20000)]
    with State(n, C64, ctx) as st:
        st.upload(circuits.random_state(n, 3, C64))
        sweeps = expect_plan(n, C64, terms)
        assert sweeps == 2  # a sweep and a reduction batch carry up to 16384 terms
        l0 = ctx.kernel_launches()
        got = st.expect_paulis(terms)
        assert ctx.kernel_launches() - l0 == sweeps + 2  # one reduction per batch
        psi = st.download()
    sel = np.concatenate([np.arange(0, 20000, 97), np.arange(16380, 16390)])
    check_against_ref("batches f32", psi, n, [terms[i] for i in sel], got[sel])


@pytest.mark.parametrize("dtype", [C128, C64])
def test_one_sweep_past_shared_memory(ctx, dtype):
    """One tile-pair sweep with more accumulators (1024) and more groups (256) than the kernel keeps in shared memory:
    400 masks that differ only inside the tile and share X on qubits 0 and 1 (outside it), 4 Z patterns each, plus
    500 Z strings riding along."""
    n = 16
    rng = np.random.default_rng(16)
    rs = rng.choice(np.arange(1, 1 << 11), size=400, replace=False)
    terms = []
    for r in rs:
        xy = [("Y" if (r >> b) & 2 else "X", n - 1 - b) for b in range(11) if (r >> b) & 1]
        for zs in range(4):
            terms.append([("X", 0), ("Y", 1)] + xy + [("Z", 2 + k) for k in range(2) if (zs >> k) & 1])
    terms += [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.4)] for _ in range(500)]
    assert expect_plan(n, dtype, terms) == 1
    with State(n, dtype, ctx) as st:
        st.upload(circuits.random_state(n, 33, dtype))
        l0 = ctx.kernel_launches()
        got = st.expect_paulis(terms)
        assert ctx.kernel_launches() - l0 == 2
        again = st.expect_paulis(terms)
        assert np.array_equal(got.view(np.uint64), again.view(np.uint64))
        psi = st.download()
    sel = np.concatenate([np.arange(0, len(terms), 7), np.arange(1020, 1030), np.arange(len(terms) - 8, len(terms))])
    check_against_ref("past shared memory %s" % np.dtype(dtype).name, psi, n, [terms[i] for i in sel], got[sel])


def test_validation_on_state(ctx):
    with State(4, C128, ctx) as st:
        st.set_basis(0)
        with pytest.raises(CircuitError) as e:
            st.expect_paulis([[("X", 0)], [("W", 1)]])
        assert e.value.status == 1 and "not 'X', 'Y' or 'Z'" in str(e.value)
        with pytest.raises(CircuitError) as e:
            st.expect_paulis([[("X", 4)]])
        assert e.value.status == 3 and "out of range" in str(e.value)
        with pytest.raises(CircuitError) as e:
            st.expect_paulis([[("X", 1), ("Z", 1)]])
        assert e.value.status == 3 and "repeated" in str(e.value)


def test_sees_pending_collapse(ctx):
    n = 16
    psi = circuits.random_state(n, 21, C128)
    terms = term_set(n, np.random.default_rng(3))
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 5], 0.37)
        assert p > 0
        got = a.expect_paulis(terms)  # applies the collapse measure left pending
        b.collapse([0, 5], m, p)
        want = b.expect_paulis(terms)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
        check_against_ref("after measure f64", b.download(), n, terms, got)


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st:
        with pytest.raises(CircuitError) as e:
            st.expect_paulis([[("Z", 0)]])
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import pauli_ref as pr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State
from test_gpu_expect import term_set

n = 18
terms = term_set(n, np.random.default_rng(18))
worst = 0.0
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as st:
        st.set_basis(3)
        st.apply_schedule(circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60])
        before = st.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        got = st.expect_paulis(terms)
        assert np.array_equal(st.qubit_map(), before), "expect_paulis restored the layout"
        psi = st.download()
    for t, g in zip(terms, got):
        want = pr.expect_ref(psi, n, t)
        b = pr.bound(n, pr.abs_weight(psi, n, t))
        err = float(abs(np.longdouble(g) - want))
        assert err <= b, (t, float(g), float(want), b)
        worst = max(worst, err / b if b > 0 else 0.0)
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

def full_terms(n):
    """X^n, Y^n, Y/X mixes with Z insertions, Z_iZ_j on the top and bottom bits, masks on both ends of the index
    (tile pairs), single letters and the identity."""
    return [
        [("X", q) for q in range(n)],
        [("Y", q) for q in range(n)],
        [("Y" if q % 3 == 0 else "X", q) for q in range(n)],
        [("Y", 0), ("X", n - 1)] + [("X", q) for q in range(1, n - 1)],
        [("Z", 0), ("Z", 1)], [("Z", n - 2), ("Z", n - 1)], [("Z", 0), ("Z", n - 1)], [("Z", n // 2)],
        [("X", 0), ("X", n - 1)], [("Y", 0), ("Z", 1), ("X", n - 1)], [("X", 0)], [("Y", n - 1)],
        [("X", 0), ("Y", 3), ("X", 9), ("Z", 12), ("Y", n - 6), ("X", n - 1)],
        [],
    ]


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


def ghz_expect(n, alpha, beta, term):
    """alpha|0..0> + beta|1..1>: only x == 0 and x == all-ones give non-zero terms."""
    x, z, ny = pr.masks(n, term)
    full = (1 << n) - 1
    sz = -1 if bin(z).count("1") & 1 else 1
    a, b = np.clongdouble(alpha), np.clongdouble(beta)
    if x == 0:
        return (abs(a) ** 2 + sz * abs(b) ** 2).real, float(abs(alpha) ** 2 + abs(beta) ** 2)
    if x != full:
        return np.longdouble(0), 0.0
    w = np.conj(b) * a + sz * np.conj(a) * b
    return (w.real, -w.imag, -w.real, w.imag)[ny & 3], float(2 * abs(alpha) * abs(beta))


PRODUCT_V = [(1, 0.5), (0.5, 1j), (0.5j, 0.5), (-0.5, 1), (1, -0.25j), (0.25, -1)]


def product_expect(n, term):
    """prod_q <v_q|sigma_q|v_q> for the product state of PRODUCT_V (every amplitude a power of two times 1 or i,
    exact in both precisions), and S."""
    letters = dict((q, l) for l, q in term)
    val, S = np.longdouble(1), 1.0
    for q in range(n):
        v0, v1 = (np.clongdouble(c) for c in PRODUCT_V[q % len(PRODUCT_V)])
        l = letters.get(q)
        c = np.conj(v0) * v1
        f = {"X": 2 * c.real, "Y": 2 * c.imag, "Z": abs(v0) ** 2 - abs(v1) ** 2, None: abs(v0) ** 2 + abs(v1) ** 2}[l]
        val *= np.longdouble(f)
        S *= float(2 * abs(v0) * abs(v1)) if l in ("X", "Y") else float(abs(v0) ** 2 + abs(v1) ** 2)
    return val, S


@pytest.mark.parametrize("n,dtype", [(30, C128), (32, C64)], ids=["n30_f64", "n32_f32"])
def test_full_size_closed_forms(holder, n, dtype):
    name = "n%d %s" % (n, np.dtype(dtype).name)
    st = holder.take(n, dtype)
    terms = full_terms(n)
    # GHZ with phases: H, CNOTs (exact), then T and S on the |1..1> branch; the two amplitudes are read back
    st.set_basis(0)
    st.apply_schedule([gates.h(0)] + [gates.cnot(0, k) for k in range(1, n)] + [gates.t(0), gates.s(n // 2)])
    got = st.expect_paulis(terms)
    alpha = complex(st.download(offset=0, length=1)[0])
    beta = complex(st.download(offset=(1 << n) - 1, length=1)[0])
    for t, g in zip(terms, got):
        want, S = ghz_expect(n, alpha, beta, t)
        b = pr.bound(n, S)
        err = float(abs(np.longdouble(g) - want))
        assert err <= b, (name, "ghz", t, float(g), float(want), b)
        note("full %s ghz" % name, err / b if b > 0 else 0.0)
    # product state from one MAT op per qubit
    st.set_basis(0)
    st.apply_schedule([gates.mat([q], [PRODUCT_V[q % len(PRODUCT_V)][0], 0, PRODUCT_V[q % len(PRODUCT_V)][1], 0])
                       for q in range(n)])
    assert expect_plan(n, dtype, terms) >= 2
    got = st.expect_paulis(terms)
    for t, g in zip(terms, got):
        want, S = product_expect(n, t)
        b = pr.bound(n, S)
        err = float(abs(np.longdouble(g) - want))
        assert err <= b, (name, "product", t, float(g), float(want), b)
        note("full %s product" % name, err / b if b > 0 else 0.0)
    holder.release()


# ---- headline state: against measure_probs after basis rotation ------------------------------------------------

def sdg(q):
    return gates.mat([q], [1, 0, 0, -1j])


def signed_sum(probs):
    odd = (np.bitwise_count(np.arange(probs.size, dtype=np.uint64)) & 1).astype(bool)
    return float(np.sum(np.where(odd, -probs, probs)))


def test_headline_state_against_measure_probs(holder):
    """The N=30 f64 headline state (random {H,T,CNOT}, depth 40, seed 0x5EED0002).  Each string is rotated into the
    Z basis (H for X, S^dagger then H for Y) and <P> = sum_m (-1)^popc(m) p(m) over its support.  Bound: the
    expectation kernel's (pauli_ref.bound with S <= 1), plus measure_probs' histogram sums of up to 2^30 values in an
    unspecified order (gamma_{2^30}), plus the rotation gates: one (X) or two (Y) per rotated qubit, each perturbing
    the state by at most 4u in norm, which moves <P> by at most twice that per gate."""
    n = 30
    u = pr.U_DOUBLE
    ops = circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT")
    z_terms = [[("Z", 0)], [("Z", 29)], [("Z", 0), ("Z", 29)], [("Z", q) for q in range(2, 26)],
               [("Z", q) for q in range(4, 30, 3)]]
    rotations = [
        {q: "X" for q in range(10)},
        {0: "Y", 5: "Y", 29: "Y", 14: "Y", 1: "X", 28: "X", 7: "X"},
    ]
    rot_terms = [
        [[("X", q) for q in range(10)], [("X", 0), ("X", 9), ("Z", 20)], [("X", 3), ("Z", 29), ("Z", 15)]],
        [[("Y", 0), ("Y", 29)], [("Y", 0), ("X", 1), ("Y", 5), ("Y", 14), ("X", 28), ("Y", 29), ("X", 7)],
         [("X", 28), ("Y", 14), ("Z", 22)]],
    ]
    def bound_for(rot):
        gates_applied = sum(2 if l == "Y" else 1 for l in rot.values())
        return pr.bound(n, 1.0) + pr.gamma(1 << n, u) + 2 * 4 * u * gates_applied

    bound = bound_for({})
    st = holder.take(n, C128)
    st.set_basis(0)
    st.apply_schedule(ops)
    all_terms = z_terms + [t for ts in rot_terms for t in ts]
    got = dict(zip(map(str, all_terms), st.expect_paulis(all_terms)))
    for t in z_terms:
        want = signed_sum(st.measure_probs([q for _, q in t]))
        err = abs(got[str(t)] - want)
        assert err <= bound, (t, got[str(t)], want, bound)
        note("headline n30 f64 Z strings", err / bound)
    for rot, ts in zip(rotations, rot_terms):
        st.set_basis(0)
        st.apply_schedule(ops)
        basis = []
        for q, l in sorted(rot.items()):
            basis += ([sdg(q)] if l == "Y" else []) + [gates.h(q)]
        st.apply_schedule(basis)
        bound = bound_for(rot)
        for t in ts:
            assert all(rot.get(q, "Z") == l for l, q in t), t
            want = signed_sum(st.measure_probs([q for _, q in t]))
            err = abs(got[str(t)] - want)
            assert err <= bound, (t, got[str(t)], want, bound)
            note("headline n30 f64 X/Y strings", err / bound)
    holder.release()
