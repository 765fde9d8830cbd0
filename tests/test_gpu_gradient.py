"""Pauli sums and the adjoint energy gradient on the device (State.apply_pauli_sum, State.energy_gradient).

The states are compared bit for bit (+-0 equal) with the numpy emulators of tests/gradient_ref.py, and the sum, the
energy and the gradient within their bounds of the long-double references (tests/test_gradient_cpu.py pins those to expm
of Kronecker products, finite differences and the parameter-shift rule).  The worst |got - want| / bound per group is
printed (run with -s to see it)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import gradient_ref as gr
import pauli_ref as pr
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, pauli_gradient_plan, pauli_sum_plan
from test_gpu_pauli_rotation import check_windows, families

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
    print("\n[apply_pauli_sum / energy_gradient] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def hamiltonians(n, rng):
    """Transverse-field Ising, the QAOA cost (even n >= 4) and random strings of every weight with repeats and the
    identity, each with random real coefficients."""
    out = {"ising": rr.ising_step(n)}
    if n >= 4 and n % 2 == 0:
        out["qaoa"] = rr.qaoa_layer(n)[: n + n // 2]
    rand = [[(str(rng.choice(list("XYZ"))), int(q)) for q in rng.choice(n, size=i % (n + 1), replace=False)]
            for i in range(2 * n + 3)]
    out["random"] = rand + rand[:2] + [[]]
    return {k: (v, rng.normal(size=len(v))) for k, v in out.items()}


def check_sum_accuracy(group, src, n, terms, coeffs, got, dtype):
    ref = gr.sum_ref(src, n, terms, coeffs)
    lim = gr.sum_bound(n, terms, dtype) * gr.sum_weights(src, n, terms, coeffs)
    err = np.abs(np.asarray(got).astype(np.clongdouble) - ref).astype(np.float64)
    assert np.all(err <= lim), (group, n, float(np.max(err / np.maximum(lim, 1e-300))))
    note(group, float(np.max(err / np.maximum(lim, 1e-300))))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_sum_bit_exact_within_bound_and_plan(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 19):
        rng = np.random.default_rng(700 + n)
        with State(n, dtype, ctx) as src, State(n, dtype, ctx) as dst:
            for k, (hname, (terms, coeffs)) in enumerate(sorted(hamiltonians(n, rng).items())):
                psi = circuits.random_state(n, 40 * n + k, dtype)
                src.upload(psi)
                l0 = ctx.kernel_launches()
                dst.apply_pauli_sum(src, terms, coeffs)
                assert ctx.kernel_launches() - l0 == pauli_sum_plan(n, dtype, terms) == gr.sum_sweeps(n, terms)
                got = dst.download()
                want = gr.emulate_sum(psi, n, terms, coeffs, dtype)
                assert np.array_equal(got, want), (name, n, hname, int(np.sum(got != want)))
                dst.apply_pauli_sum(src, terms, coeffs)
                assert np.array_equal(dst.download().view(np.uint8), got.view(np.uint8))
                assert np.array_equal(src.download(), psi)
                if n <= 14:
                    check_sum_accuracy("sum reference %s" % name, psi, n, terms, coeffs, got, dtype)
            l0 = ctx.kernel_launches()
            dst.apply_pauli_sum(src, [], [])
            assert ctx.kernel_launches() == l0 and not np.any(dst.download())


def check_gradient(group, psi0, n, ansatz, angles, ham, coeffs, e, g, dtype):
    er, gref = gr.adjoint_ref(psi0, n, ansatz, angles, ham, coeffs)
    b = gr.grad_bound(n, ansatz, ham, coeffs, float(np.linalg.norm(np.asarray(psi0).astype(C128))), dtype)
    worst = max([abs(float(er) - e)] + [abs(float(x) - y) for x, y in zip(gref, g)])
    assert worst <= b, (group, n, worst, b)
    note(group, worst / b)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_gradient_bit_exact_within_bound(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 19):
        rng = np.random.default_rng(900 + n)
        fam = families(n, rng)
        hams = hamiltonians(n, rng)
        hkeys = sorted(hams)
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wk:
            for k, (fname, ansatz) in enumerate(sorted(fam.items())):
                ham, coeffs = hams[hkeys[k % len(hkeys)]]
                psi0 = circuits.random_state(n, 500 + 7 * n + k, dtype)
                angles = rng.uniform(-6.5, 6.5, size=len(ansatz))
                st.upload(psi0)
                l0 = ctx.kernel_launches()
                e, g = st.energy_gradient(wk, ansatz, angles, ham, coeffs)
                f, s, b = pauli_gradient_plan(n, dtype, ansatz, ham)
                assert (f, s, b) == gr.gradient_plan_policy(n, ansatz, ham)
                assert ctx.kernel_launches() - l0 == f + s + 2 * b
                want_st, want_wk = gr.emulate_gradient(psi0, n, ansatz, angles, ham, coeffs, dtype)
                got_st, got_wk = st.download(), wk.download()
                assert np.array_equal(got_st, want_st), (name, n, fname, int(np.sum(got_st != want_st)))
                assert np.array_equal(got_wk, want_wk), (name, n, fname, int(np.sum(got_wk != want_wk)))
                st.upload(psi0)
                e2, g2 = st.energy_gradient(wk, ansatz, angles, ham, coeffs)
                assert np.array_equal(np.array([e]).view(np.uint64), np.array([e2]).view(np.uint64))
                assert np.array_equal(g.view(np.uint64), g2.view(np.uint64))
                if n <= 12 or (n <= 16 and fname != "long run"):
                    check_gradient("gradient reference %s" % name, psi0, n, ansatz, angles, ham, coeffs, e, g, dtype)


def test_gradient_with_no_ansatz_or_no_hamiltonian(ctx):
    n = 13
    psi0 = circuits.random_state(n, 3, C128)
    ham, coeffs = rr.ising_step(n), np.linspace(-1, 1, 2 * n)
    with State(n, C128, ctx) as st, State(n, C128, ctx) as wk:
        st.upload(psi0)
        e, g = st.energy_gradient(wk, [], [], ham, coeffs)
        assert g.shape == (0,)
        want = float(np.dot(coeffs, st.expect_paulis(ham)))
        assert abs(e - want) <= 1e-12
        assert np.array_equal(st.download(), psi0)
        e, g = st.energy_gradient(wk, [[("X", 2)], [("Z", 1)]], [0.3, 0.4], [], [])
        assert e == 0.0 and not np.any(g) and not np.any(wk.download())


def test_cross_check_with_parameter_shift(ctx):
    """n = 20, 22: the gradient against the parameter-shift rule through apply_pauli_rotations and expect_paulis.
    Each shifted energy lies within its rotation bound (twice: the rotations and their undoing) and the expect bound of
    the exact value, the adjoint gradient within grad_bound."""
    for n, dtype in ((20, C128), (22, C64)):
        rng = np.random.default_rng(n)
        ansatz = rr.ising_step(n) + rr.ucc_strings(n, 6, n) + [[("Y", q) for q in range(0, n, 3)]]
        angles = rng.uniform(-2, 2, size=len(ansatz))
        ham, coeffs = rr.ising_step(n), rng.normal(size=2 * n)
        psi0 = circuits.random_state(n, n + 1, dtype)
        S = float(np.sum(np.abs(coeffs)))
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wk:
            st.upload(psi0)
            e, g = st.energy_gradient(wk, ansatz, angles, ham, coeffs)

            def energy(th):
                st.upload(psi0)
                st.apply_pauli_rotations(ansatz, th)
                return float(np.dot(coeffs, st.expect_paulis(ham)))

            tol = gr.grad_bound(n, ansatz, ham, coeffs, 1.0, dtype) + \
                S * (4 * rr.bound(len(ansatz), 1.0, dtype) + pr.bound(n, 1.0))
            assert abs(e - energy(angles)) <= tol
            worst = 0.0
            for t in range(len(ansatz)):
                d = np.zeros(len(ansatz))
                d[t] = math.pi / 2
                ps = (energy(angles + d) - energy(angles - d)) / 2
                worst = max(worst, abs(ps - g[t]) / tol)
            assert worst <= 1.0, worst
            note("parameter shift n=%d" % n, worst)


def test_pending_collapse_and_refusals(ctx):
    n = 14
    rng = np.random.default_rng(14)
    psi0 = circuits.random_state(n, 15, C128)
    ansatz = families(n, rng)["mix"]
    angles = rng.uniform(-2, 2, size=len(ansatz))
    ham, coeffs = rr.ising_step(n), rng.normal(size=2 * n)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as w, State(n, C128, ctx) as b, \
            State(n - 1, C128, ctx) as small, State(n, C64, ctx) as single:
        psi1 = circuits.random_state(n, 16, C128)
        a.upload(psi0)
        b.upload(psi0)
        w.upload(psi1)
        refusals = [
            (lambda: a.energy_gradient(a, ansatz, angles, ham, coeffs), INVALID_ARG),
            (lambda: a.energy_gradient(small, ansatz, angles, ham, coeffs), SIZE_MISMATCH),
            (lambda: a.energy_gradient(single, ansatz, angles, ham, coeffs), SIZE_MISMATCH),
            (lambda: a.energy_gradient(w, ansatz + [[("W", 0)]], list(angles) + [1.0], ham, coeffs), INVALID_ARG),
            (lambda: a.energy_gradient(w, ansatz, angles, ham + [[("X", n)]], list(coeffs) + [1.0]), BAD_INDEX),
            (lambda: a.energy_gradient(w, ansatz, np.where(np.arange(len(angles)) == 3, np.nan, angles), ham,
                                       coeffs), INVALID_ARG),
            (lambda: a.energy_gradient(w, ansatz, angles, ham, np.where(np.arange(len(coeffs)) == 1, np.inf, coeffs)),
             INVALID_ARG),
            (lambda: w.apply_pauli_sum(w, ham, coeffs), INVALID_ARG),
            (lambda: w.apply_pauli_sum(small, [[("Z", 0)]], [1.0]), SIZE_MISMATCH),
            (lambda: w.apply_pauli_sum(a, ham + [[("X", 1), ("Z", 1)]], list(coeffs) + [1.0]), BAD_INDEX),
            (lambda: w.apply_pauli_sum(a, ham, np.where(np.arange(len(coeffs)) == 0, -np.inf, coeffs)), INVALID_ARG),
        ]
        for call, code in refusals:
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == code, (e.value.status, code, str(e.value))
        # NULL energy / grad / coeffs through the C entries
        from rustqip_b200 import _lib
        from rustqip_b200.state import _marshal_paulis, _ptr
        qs, ls, lens = _marshal_paulis([[("X", 0)]])
        one, out = np.ones(1), np.zeros(1)
        L = _lib.lib()
        assert L.qipb200_state_pauli_energy_gradient(a._h, w._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), _ptr(qs), ls,
                                                     _ptr(lens), 1, _ptr(one), None, _ptr(out)) == INVALID_ARG
        assert "NULL energy" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_pauli_energy_gradient(a._h, w._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), _ptr(qs), ls,
                                                     _ptr(lens), 1, _ptr(one), _ptr(out), None) == INVALID_ARG
        assert "NULL grad" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_apply_pauli_sum(w._h, a._h, _ptr(qs), ls, _ptr(lens), 1, None) == INVALID_ARG
        assert "NULL coefficients" in L.qipb200_last_error(ctx.handle).decode()
        assert np.array_equal(a.download(), psi0) and np.array_equal(w.download(), psi1)
        # a refusal keeps a pending collapse; the call applies the one on state and drops the one on work
        m, p = a.measure([0, 5], 0.41)
        w.measure([1], 0.7)
        with pytest.raises(CircuitError):
            a.energy_gradient(w, ansatz, angles, ham + [[("Q", 0)]], list(coeffs) + [1.0])
        l0 = ctx.kernel_launches()
        e, g = a.energy_gradient(w, ansatz, angles, ham, coeffs)
        f, s, bk = pauli_gradient_plan(n, C128, ansatz, ham)
        assert ctx.kernel_launches() - l0 == f + s + 2 * bk + 1
        b.collapse([0, 5], m, p)
        collapsed = b.download()
        want_st, want_wk = gr.emulate_gradient(collapsed, n, ansatz, angles, ham, coeffs, C128)
        assert np.array_equal(a.download(), want_st) and np.array_equal(w.download(), want_wk)
        e2, g2 = b.energy_gradient(w, ansatz, angles, ham, coeffs)
        assert e == e2 and np.array_equal(g, g2)
        # apply_pauli_sum applies a collapse pending on src
        b.upload(psi0)
        m, p = b.measure([2], 0.3)
        w.apply_pauli_sum(b, ham, coeffs)
        got = w.download()
        assert np.array_equal(got, gr.emulate_sum(b.download(), n, ham, coeffs, C128))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, State(12, C128, ctx, rank=0, world_size=2) as w:
        with pytest.raises(CircuitError) as e:
            st.energy_gradient(w, [[("Z", 0)]], [0.5], [[("X", 1)]], [1.0])
        assert e.value.status == UNSUPPORTED
        with pytest.raises(CircuitError) as e:
            w.apply_pauli_sum(st, [[("X", 1)]], [1.0])
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import gradient_ref as gr
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 16
rng = np.random.default_rng(16)
ansatz = rr.ising_step(n) + rr.ucc_strings(n, 10, 5)
angles = rng.uniform(-3, 3, size=len(ansatz))
ham, coeffs = rr.ising_step(n) + [[("Y", 0), ("X", 7)]], rng.normal(size=2 * n + 1)
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b, State(n, np.complex128, ctx) as w, \
            State(n, np.complex128, ctx) as d:
        for st in (a, b):
            st.set_basis(3)
            st.apply_schedule(ops)
        before = a.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        psi = b.download()  # a download restores the canonical layout: b is a's twin
        d.apply_pauli_sum(a, ham, coeffs)
        assert np.array_equal(d.qubit_map(), before), "dst did not take src's layout"
        got_sum = d.download()
        e, g = a.energy_gradient(w, ansatz, angles, ham, coeffs)
        assert np.array_equal(a.qubit_map(), before) and np.array_equal(w.qubit_map(), before)
        got_st, got_wk = a.download(), w.download()
assert np.array_equal(got_sum, gr.emulate_sum(psi, n, ham, coeffs, np.complex128, before))
want_st, want_wk = gr.emulate_gradient(psi, n, ansatz, angles, ham, coeffs, np.complex128, before)
assert np.array_equal(got_st, want_st) and np.array_equal(got_wk, want_wk)
er, gref = gr.adjoint_ref(psi, n, ansatz, angles, ham, coeffs)
b = gr.grad_bound(n, ansatz, ham, coeffs, 1.0, np.complex128)
assert max(abs(float(er) - e), float(np.max(np.abs(gref.astype(np.float64) - g)))) <= b
print("ROTATE bit-exact ok")
"""


def test_permuted_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout


# ---- full size ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,dtype", [(30, C128), (31, C64)], ids=["n30_f64", "n31_f32"])
def test_full_size_closed_form(ctx, n, dtype):
    name = "n%d %s" % (n, np.dtype(dtype).name)
    rng = np.random.default_rng(n)
    theta, phi = rng.uniform(-3, 3, size=n), rng.uniform(-3, 3, size=n)
    a, b, c = rng.normal(size=n), rng.normal(size=n), rng.normal(size=n)
    ansatz = gr.product_ansatz(n)
    angles = np.concatenate([theta, phi])
    ham, coeffs = gr.product_hamiltonian(n, a, b, c)
    ctx.release_pool()
    try:
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wk:
            st.set_basis(0)
            e, g = st.energy_gradient(wk, ansatz, angles, ham, coeffs)
            want_e, gt, gp = gr.closed_form(n, theta, phi, a, b, c)
            want = np.concatenate([gt, gp]).astype(np.float64)
            bnd = gr.grad_bound(n, ansatz, ham, coeffs, 1.0, dtype)
            worst = max(abs(e - float(want_e)), float(np.max(np.abs(g - want))))
            assert worst <= bnd, (name, worst, bnd)
            note("full %s closed form" % name, worst / bnd)

            def basis0(idx):
                w = np.zeros(idx.shape, dtype=np.clongdouble)
                w[idx == 0] = 1
                return w

            ratio = check_windows(st, n, dtype, basis0, rr.bound(2 * len(ansatz), 1.0, dtype), name + " state back")
            note("full %s state back at |0>" % name, ratio)
    finally:
        ctx.release_pool()
