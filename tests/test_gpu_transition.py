"""Transition elements <bra|P|ket> and overlaps between two device states (State.transition_paulis, State.overlap,
qipb200_state_transition_paulis).

Re and Im of every value are each checked against bound(n) * S with S = sum_j |bra_{j^x}| |ket_j|; tests/transition_ref.py
derives the bound from the kernel's summation depth (and tests/test_transition_cpu.py pins its long-double reference to
explicit Kronecker products).  The worst |got - want| / bound per group of checks is printed (run with -s to see it)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg

import evolve_ref as er
import pauli_ref as pr
import transition_ref as tr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, _marshal_paulis, _ptr, expect_plan, transition_plan
from test_gpu_expect import random_terms, term_set
from test_gradient_cpu import dense_h

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, SIZE_MISMATCH, BAD_INDEX, UNSUPPORTED = 1, 2, 3, 7
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[transition_paulis] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def check_against_ref(group, bra, ket, n, terms, got, slack=1.0):
    assert got.shape == (len(terms),) and got.dtype == C128
    for t, g in zip(terms, got):
        want = tr.transition_ref(bra, ket, n, t)
        b = slack * tr.bound(n, tr.abs_weight(bra, ket, n, t))
        e_re, e_im = tr.errors(g, want)
        assert e_re <= b and e_im <= b, (group, n, t, complex(g), complex(want), b)
        note(group, max(e_re, e_im) / b if b > 0 else 0.0)


def bits(v):
    return np.ascontiguousarray(v).view(np.uint64)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_small_states_against_reference(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 17):
        rng = np.random.default_rng(2000 + n)
        terms = term_set(n, rng)
        pairs = [("random", circuits.random_state(n, 170 + n, dtype),
                  (circuits.random_state(n, 190 + n, dtype) * 0.5).astype(dtype))]
        if n >= 3:
            pairs.append(("circuit", None, None))
        with State(n, dtype, ctx) as bra, State(n, dtype, ctx) as ket:
            for kind, b, k in pairs:
                if b is None:
                    bra.set_basis(1)
                    bra.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0300 + n, "H,T,CNOT"))
                    ket.set_basis(2)
                    ket.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0400 + n, "H,T,CNOT"))
                else:
                    bra.upload(b)
                    ket.upload(k)
                got = bra.transition_paulis(ket, terms)
                check_against_ref("small %s %s" % (name, kind), bra.download(), ket.download(), n, terms, got)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_overlaps_copies_and_swaps(ctx, dtype):
    name = np.dtype(dtype).name
    n = 13
    terms = term_set(n, np.random.default_rng(5))
    psi = (circuits.random_state(n, 6, dtype) * 0.75).astype(dtype)
    phi = circuits.random_state(n, 7, dtype)
    with State(n, dtype, ctx) as a, State(n, dtype, ctx) as a2, State(n, dtype, ctx) as b:
        a.upload(psi)
        a2.upload(psi)
        b.upload(phi)
        # overlap: the long-double vdot
        o = a.overlap(b)
        assert isinstance(o, complex)
        check_against_ref("overlap %s" % name, psi, phi, n, [[]], np.array([o]))
        want = np.vdot(psi.astype(np.clongdouble), phi.astype(np.clongdouble))
        assert abs(o - complex(want)) <= 2 * tr.bound(n, tr.abs_weight(psi, phi, n, []))
        # <psi|psi> is norm2
        S = float(np.sum(np.abs(psi.astype(C128)) ** 2))
        oo = a.overlap(a)
        lim = tr.bound(n, S) + pr.gamma(1 << n, pr.U_DOUBLE) * S
        assert abs(oo.real - a.norm2()) <= lim and abs(oo.imag) <= tr.bound(n, S)
        note("overlap vs norm2 %s" % name, abs(oo.real - a.norm2()) / lim)
        # the same handle and two copies: one value, expect_paulis' within both bounds
        same = a.transition_paulis(a, terms)
        copies = a.transition_paulis(a2, terms)
        assert np.array_equal(bits(same), bits(copies))
        check_against_ref("bra == ket %s" % name, psi, psi, n, terms, same)
        ex = a.expect_paulis(terms)
        for t, s, e in zip(terms, same, ex):
            lim = tr.bound(n, tr.abs_weight(psi, psi, n, t)) + pr.bound(n, pr.abs_weight(psi, n, t))
            assert abs(s.real - e) <= lim, (t, s, e, lim)
            note("bra == ket vs expect %s" % name, abs(s.real - e) / lim if lim > 0 else 0.0)
        # swapping bra and ket conjugates
        ab = a.transition_paulis(b, terms)
        ba = b.transition_paulis(a, terms)
        check_against_ref("swapped %s" % name, phi, psi, n, terms, ba)
        for t, x, y in zip(terms, ab, ba):
            lim = 2 * tr.bound(n, tr.abs_weight(psi, phi, n, t))
            assert abs(x.real - y.real) <= lim and abs(x.imag + y.imag) <= lim, (t, x, y, lim)
        assert a.transition_paulis(b, []).shape == (0,)


def test_launch_counts_and_determinism(ctx):
    n = 20
    rng = np.random.default_rng(8)
    ising = [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]
    cases = [ising, term_set(n, rng), random_terms(n, rng, 600), [[("X", q) for q in range(n)]], [[]]]
    with State(n, C128, ctx) as bra, State(n, C128, ctx) as ket:
        bra.set_basis(0)
        bra.apply_schedule(circuits.random_circuit(n, 10, 0x5EED0500, "H,T,CNOT"))
        ket.set_basis(3)
        ket.apply_schedule(circuits.random_circuit(n, 10, 0x5EED0600, "H,T,CNOT"))
        ket.sync()
        for terms in cases:
            sweeps, kernels = transition_plan(n, C128, terms)
            assert sweeps >= expect_plan(n, C128, terms)
            l0 = ctx.kernel_launches()
            got = bra.transition_paulis(ket, terms)
            assert ctx.kernel_launches() - l0 == kernels
            again = bra.transition_paulis(ket, terms)
            assert np.array_equal(bits(got), bits(again))
        check_against_ref("launch-count cases f64", bra.download(), ket.download(), n, cases[0] + cases[3],
                          bra.transition_paulis(ket, cases[0] + cases[3]))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_one_pair_sweep_past_shared_memory(ctx, dtype):
    """One tile-pair sweep (X on qubits 0 and 1, outside the tile) with more rows (4200) than the kernel keeps in
    shared memory (1024) and more groups (400) than it stages (256)."""
    n = 16
    rng = np.random.default_rng(17)
    rs = rng.choice(np.arange(1, 1 << 11), size=400, replace=False)
    terms = []
    for r in rs:
        xy = [("Y" if (r >> b) & 2 else "X", n - 1 - b) for b in range(11) if (r >> b) & 1]
        for zs in range(4):
            terms.append([("X", 0), ("Y", 1)] + xy + [("Z", 2 + k) for k in range(2) if (zs >> k) & 1])
    terms += [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.4)] for _ in range(500)]
    assert transition_plan(n, dtype, terms) == (1, 2)
    with State(n, dtype, ctx) as bra, State(n, dtype, ctx) as ket:
        bra.upload(circuits.random_state(n, 34, dtype))
        ket.upload(circuits.random_state(n, 35, dtype))
        l0 = ctx.kernel_launches()
        got = bra.transition_paulis(ket, terms)
        assert ctx.kernel_launches() - l0 == 2
        again = bra.transition_paulis(ket, terms)
        assert np.array_equal(bits(got), bits(again))
        b, k = bra.download(), ket.download()
    sel = np.concatenate([np.arange(0, len(terms), 7), np.arange(505, 520), np.arange(len(terms) - 8, len(terms))])
    check_against_ref("pair past shared memory %s" % np.dtype(dtype).name, b, k, n, [terms[i] for i in sel], got[sel])


def test_many_terms_run_in_batches(ctx):
    n = 10
    rng = np.random.default_rng(12)
    terms = [[("Z", int(q)) for q in np.flatnonzero(rng.random(n) < 0.5)] for _ in range(20000)]
    with State(n, C64, ctx) as bra, State(n, C64, ctx) as ket:
        bra.upload(circuits.random_state(n, 4, C64))
        ket.upload(circuits.random_state(n, 5, C64))
        sweeps, kernels = transition_plan(n, C64, terms)
        assert (sweeps, kernels) == (3, 6)  # 40000 rows: sweeps and batches of up to 16384
        l0 = ctx.kernel_launches()
        got = bra.transition_paulis(ket, terms)
        assert ctx.kernel_launches() - l0 == kernels
        b, k = bra.download(), ket.download()
    sel = np.concatenate([np.arange(0, 20000, 97), np.arange(8185, 8200), np.arange(16380, 16390)])
    check_against_ref("batches f32", b, k, n, [terms[i] for i in sel], got[sel])


def test_pending_collapse_on_either_state(ctx):
    n = 16
    psi, phi = circuits.random_state(n, 22, C128), circuits.random_state(n, 23, C128)
    terms = term_set(n, np.random.default_rng(4))
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b, State(n, C128, ctx) as c:
        for pending_on_bra in (True, False):
            a.upload(psi)
            b.upload(phi)
            m, p = a.measure([0, 5], 0.37)
            assert p > 0
            c.upload(psi)
            c.collapse([0, 5], m, p)
            if pending_on_bra:
                got, want = a.transition_paulis(b, terms), c.transition_paulis(b, terms)
            else:
                got, want = b.transition_paulis(a, terms), b.transition_paulis(c, terms)
            assert np.array_equal(bits(got), bits(want)), pending_on_bra
        check_against_ref("after measure f64", phi, c.download(), n, terms, got)


def _raw_call(bra, ket, terms, out=True):
    qs, ls, lens = _marshal_paulis(terms)
    buf = np.zeros(max(1, 2 * lens.shape[0]))
    L = _lib.lib()
    st = L.qipb200_state_transition_paulis(bra._h, ket._h, _ptr(qs), ls, _ptr(lens), lens.shape[0],
                                           _ptr(buf) if out else None)
    return st, L.qipb200_last_error(bra.ctx.handle).decode()


def test_refusals_leave_both_states_and_pending_collapse(ctx):
    n = 6
    psi, phi = circuits.random_state(n, 40, C128), circuits.random_state(n, 41, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b, State(n, C64, ctx) as f32, \
            State(n + 1, C128, ctx) as big, State(n, C128, ctx) as ref:
        a.upload(psi)
        b.upload(phi)
        f32.upload(phi.astype(C64))
        big.upload(circuits.random_state(n + 1, 42, C128))
        m, p = a.measure([1, 4], 0.61)
        ref.upload(psi)
        ref.collapse([1, 4], m, p)
        l0 = ctx.kernel_launches()
        for other in (f32, big):
            for x, y in ((a, other), (other, a)):
                with pytest.raises(CircuitError) as e:
                    x.transition_paulis(y, [[("Z", 0)]])
                assert e.value.status == SIZE_MISMATCH and "differ in context, precision or size" in str(e.value)
        with pytest.raises(CircuitError) as e:
            a.transition_paulis(b, [[("X", 0)], [("W", 1)]])
        assert e.value.status == INVALID_ARG and "not 'X', 'Y' or 'Z'" in str(e.value)
        with pytest.raises(CircuitError) as e:
            b.transition_paulis(a, [[("X", n)]])
        assert e.value.status == BAD_INDEX and "out of range" in str(e.value)
        with pytest.raises(CircuitError) as e:
            a.transition_paulis(b, [[("X", 1), ("Z", 1)]])
        assert e.value.status == BAD_INDEX and "repeated" in str(e.value)
        st, msg = _raw_call(a, b, [[("Z", 0)]], out=False)
        assert st == INVALID_ARG and "NULL out" in msg
        st, _ = _raw_call(a, b, [], out=False)  # n_terms == 0: a no-op
        assert st == 0
        assert a.transition_paulis(b, []).shape == (0,)
        assert ctx.kernel_launches() == l0, "a refused call or a no-op did device work"
        # the collapse is still pending (the download applies it) and the other states are untouched
        assert np.array_equal(bits(a.download()), bits(ref.download()))
        assert np.array_equal(bits(b.download()), bits(phi))
        assert np.array_equal(bits(f32.download()), bits(phi.astype(C64)))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as sh, State(12, C128, ctx) as st:
        st.set_basis(0)
        for x, y in ((sh, st), (st, sh)):
            with pytest.raises(CircuitError) as e:
                x.transition_paulis(y, [[("Z", 0)]])
            assert e.value.status == UNSUPPORTED and "sharded" in str(e.value)
        assert np.array_equal(st.download(), np.eye(1, 1 << 12, 0, dtype=C128)[0])


_ROTATE_WORKER = r"""
import numpy as np
import transition_ref as tr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State
from test_gpu_expect import term_set

n = 18
terms = term_set(n, np.random.default_rng(19))
canonical = np.arange(n)[::-1]
worst = 0.0

def check(b, k, got):
    global worst
    for t, g in zip(terms, got):
        want = tr.transition_ref(b, k, n, t)
        lim = tr.bound(n, tr.abs_weight(b, k, n, t))
        e = max(tr.errors(g, want))
        assert e <= lim, (t, complex(g), complex(want), lim)
        worst = max(worst, e / lim if lim > 0 else 0.0)

ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as bra, State(n, np.complex128, ctx) as ket, \
            State(n, np.complex128, ctx) as plain:
        bra.set_basis(3)
        bra.apply_schedule(ops)
        ket.set_basis(5)
        ket.apply_schedule(ops)
        before = bra.qubit_map().copy()
        assert not np.array_equal(before, canonical), "the schedule left the canonical layout"
        assert np.array_equal(ket.qubit_map(), before), "the same schedule gave two layouts"
        got = bra.transition_paulis(ket, terms)
        assert np.array_equal(bra.qubit_map(), before) and np.array_equal(ket.qubit_map(), before), "layout changed"
        # two layouts: the permuted bra is restored, the canonical ket read as it is
        psi = circuits.random_state(n, 77, np.complex128)
        plain.upload(psi)
        bra.set_basis(3)
        bra.apply_schedule(ops)
        assert not np.array_equal(bra.qubit_map(), canonical)
        got2 = bra.transition_paulis(plain, terms)
        assert np.array_equal(bra.qubit_map(), canonical), "the permuted state was not restored"
        assert np.array_equal(plain.qubit_map(), canonical)
        b, k = bra.download(), ket.download()
    check(b, k, got)
    check(b, psi, got2)
print("ROTATE worst ratio %.3e" % worst)
"""


def test_layouts_in_place_and_restored():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    note("rotate f64 n=18", float(p.stdout.split("worst ratio")[1].split()[0]))


# ---- full size: product states against closed forms -------------------------------------------------------------

def full_terms(n):
    """X^n, Y^n, Z^n, masks at both ends of the index (tile pairs), single letters and the empty term."""
    return [
        [("X", q) for q in range(n)], [("Y", q) for q in range(n)], [("Z", q) for q in range(n)],
        [("Y" if q % 3 == 0 else "X", q) for q in range(n)],
        [("X", 0), ("X", n - 1)], [("Y", 0), ("Z", 1), ("X", n - 1)], [("Z", 0), ("Z", n - 1)],
        [("X", 0)], [("Y", n - 1)], [("Z", n // 2)], [("X", 0), ("Y", 3), ("X", 9), ("Z", 12), ("Y", n - 6), ("X", n - 1)],
        [],
    ]


def product_factors(n, shift):
    """(cos a_q, e^{i b_q} sin a_q) per qubit, in long double."""
    out = []
    for q in range(n):
        a, b = np.longdouble(0.25 + 0.043 * ((q * 7 + shift) % 31)), np.longdouble(0.37 * q + shift)
        out.append((np.clongdouble(np.cos(a)), np.exp(np.clongdouble(1j) * b) * np.sin(a)))
    return out


SIGMA = {"X": ((0, 1), (1, 0)), "Y": ((0, -1j), (1j, 0)), "Z": ((1, 0), (0, -1))}


def product_closed_form(n, fb, fk, term):
    """prod_q <bra_q|sigma_q|ket_q> and S = prod_q sum_b |bra_q(b ^ x_q)| |ket_q(b)|."""
    letters = dict((q, l) for l, q in term)
    val, S = np.clongdouble(1), 1.0
    for q in range(n):
        b, k = fb[q], fk[q]
        l = letters.get(q)
        if l is None:
            pk = k
        else:
            m = SIGMA[l]
            pk = (np.clongdouble(m[0][0]) * k[0] + np.clongdouble(m[0][1]) * k[1],
                  np.clongdouble(m[1][0]) * k[0] + np.clongdouble(m[1][1]) * k[1])
        val *= np.conj(b[0]) * pk[0] + np.conj(b[1]) * pk[1]
        flip = l in ("X", "Y")
        S *= float(abs(b[1 if flip else 0]) * abs(k[0]) + abs(b[0 if flip else 1]) * abs(k[1]))
    return val, S


def prepare_product(st, n, factors):
    """One MAT op per qubit on |0..0>, one per-gate kernel each (no fused products of matrices)."""
    st.set_basis(0)
    st.apply_schedule([gates.mat([q], [complex(f[0]), 0, complex(f[1]), 0]) for q, f in enumerate(factors)],
                      fusion=False)


@pytest.mark.parametrize("n,dtype", [(30, C128), (31, C64)], ids=["n30_f64", "n31_f32"])
def test_full_size_product_states(ctx, n, dtype):
    """Tolerance: each amplitude is a product of n factors, each entry rounded to the state's precision (u) and each
    gate one complex product (at most 4u with or without FMA) and an exact add of zero, so every amplitude carries a
    relative error of at most eps = (1 + 6u)^n - 1 (a generous count), and a transition element of weight S moves by
    at most (2 eps + eps^2) S; the kernel's bound is added with S grown by (1 + eps)^2."""
    u = 2.0 ** -53 if dtype == C128 else 2.0 ** -24
    eps = (1 + 6 * u) ** n - 1
    ctx.release_pool()
    fb, fk = product_factors(n, 0), product_factors(n, 11)
    terms = full_terms(n)
    bra, ket = State(n, dtype, ctx), State(n, dtype, ctx)
    try:
        prepare_product(bra, n, fb)
        prepare_product(ket, n, fk)
        assert transition_plan(n, dtype, terms)[0] >= 2
        got = bra.transition_paulis(ket, terms)
        got_o = bra.overlap(ket)
    finally:
        bra.free()
        ket.free()
        ctx.release_pool()
    name = "full n%d %s" % (n, np.dtype(dtype).name)
    for t, g in zip(terms + [[]], list(got) + [got_o]):
        want, S = product_closed_form(n, fb, fk, t)
        lim = (2 * eps + eps * eps) * S + tr.bound(n, (1 + eps) ** 2 * S)
        e_re, e_im = tr.errors(np.complex128(g), want)
        assert e_re <= lim and e_im <= lim, (name, t, complex(g), complex(want), lim)
        note(name, max(e_re, e_im) / lim)


# ---- physics: Loschmidt echo, correlation functions, Trotter fidelity -------------------------------------------

def tfim(n, J=1.0, h=0.7):
    terms = [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)] + [[("X", i)] for i in range(n)]
    return terms, np.array([J] * n + [h] * n)


def _evolve(st, wa, wb, terms, coeffs, t):
    """Evolve st in place; returns the 2-norm bound of |device - exp(-iHt) start| for a start of norm 1."""
    K, _, _, tail, c = er.plan(st.n, st.dtype, terms, coeffs, t, 1e-12)
    assert st.evolve_pauli_sum(wa, wb, terms, coeffs, t)[0] == K
    return er.bound(st.n, terms, coeffs, c, st.dtype, 1.0) + tail + er.exact_allowance(terms, coeffs, t, c, 1.0) + 1e-15


def test_loschmidt_echo_and_correlations(ctx):
    n, t = 8, 0.9
    terms, coeffs = tfim(n)
    H = dense_h(n, terms, coeffs)
    U = scipy.linalg.expm(-1j * t * H)
    psi0 = circuits.random_state(n, 90, C128)
    zq = [[("Z", i)] for i in range(n)]
    with State(n, C128, ctx) as s0, State(n, C128, ctx) as st, State(n, C128, ctx) as phi, \
            State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
        s0.upload(psi0)
        st.upload(psi0)
        e_psi = _evolve(st, wa, wb, terms, coeffs, t)
        # Loschmidt echo |<psi0|e^{-iHt} psi0>|^2
        o = s0.overlap(st)
        want = np.vdot(psi0, U @ psi0)
        lim = e_psi + np.sqrt(2) * tr.bound(n, 1.0 + e_psi)
        assert abs(o - want) <= lim, (o, want, lim)
        note("loschmidt n=8", abs(o - want) / lim)
        assert abs(abs(o) ** 2 - abs(want) ** 2) <= (2 * abs(want) + lim) * lim
        # C_ij(t) = <psi(t)|Z_i|phi_j(t)>, phi_j(0) = Z_j psi0, all i in one call
        psi_t = U @ psi0
        for j in range(n):
            phi.apply_pauli_sum(s0, [[("Z", j)]], [1.0])
            e_phi = _evolve(phi, wa, wb, terms, coeffs, t)
            got = st.transition_paulis(phi, zq)
            phi_t = U @ (kron_z(n, j) * psi0)
            for i in range(n):
                want = np.vdot(psi_t, kron_z(n, i) * phi_t)
                lim = e_psi + e_phi + e_psi * e_phi + np.sqrt(2) * tr.bound(n, (1 + e_psi) * (1 + e_phi))
                assert abs(got[i] - want) <= lim, (i, j, got[i], want, lim)
                note("correlation n=8", abs(got[i] - want) / lim)


def kron_z(n, q):
    """Diagonal of Z on qubit q (index bit n-1-q)."""
    j = np.arange(1 << n)
    return np.where((j >> (n - 1 - q)) & 1, -1.0, 1.0)


def test_trotter_fidelity_n24(ctx):
    n, t, steps = 24, 0.5, 8
    terms, coeffs = tfim(n)
    dt = t / steps
    zz, xs = terms[:n], terms[n:]
    # second order: e^{-iX dt/2} e^{-iZZ dt} e^{-iX dt/2} per step, exp(-i theta/2 P) with theta = 2 c dt
    rot_terms, angles = [], []
    for _ in range(steps):
        rot_terms += xs + zz + xs
        angles += [0.7 * dt] * n + [2.0 * dt] * n + [0.7 * dt] * n
    with State(n, C128, ctx) as ex, State(n, C128, ctx) as tro, State(n, C128, ctx) as wa, \
            State(n, C128, ctx) as wb:
        for s in (ex, tro):
            s.set_basis(0)
            s.apply_pauli_rotations([[("Y", q)] for q in range(n)], np.linspace(0.3, 1.2, n))
        ex.evolve_pauli_sum(wa, wb, terms, coeffs, t)
        tro.apply_pauli_rotations(rot_terms, angles)
        o = tro.overlap(ex)
        a, b = tro.download(), ex.download()
    # the long-double vdot in chunks of 2^20 (sequential over 16 chunks: 16 more levels than transition_ref's sum)
    want, S = np.clongdouble(0), 0.0
    for i in range(0, 1 << n, 1 << 20):
        x, y = a[i:i + (1 << 20)].astype(np.clongdouble), b[i:i + (1 << 20)].astype(np.clongdouble)
        want += np.sum(np.conj(x) * y)
        S += float(np.sum(np.abs(a[i:i + (1 << 20)]) * np.abs(b[i:i + (1 << 20)])))
    lim = tr.bound(n, S) + pr.gamma(16, pr.U_LONGDOUBLE) * S
    e_re, e_im = tr.errors(np.complex128(o), want)
    assert e_re <= lim and e_im <= lim, (o, complex(want), lim)
    note("trotter n=24", max(e_re, e_im) / lim)
    f, fw = abs(o) ** 2, float(abs(want) ** 2)
    assert abs(f - fw) <= 2 * np.sqrt(2) * lim * (abs(o) + lim)
    assert 0.9 < f < 1.0, f
    print("\n[transition_paulis] n=24 TFIM fidelity(second-order Trotter, %d steps; Chebyshev) = %.15f" % (steps, f))
