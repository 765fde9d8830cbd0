"""exp(-iHt) by a Chebyshev series on the device (State.evolve_pauli_sum).

The state is compared bit for bit (+-0 equal) with the numpy emulator of tests/evolve_ref.py, and within tau_K plus the
documented rounding bound with the long-double series reference (pinned to scipy.linalg.expm of Kronecker products in
tests/test_evolve_cpu.py) and, for n <= 8, with expm itself.  At full size a diagonal H is checked against
apply_pauli_rotations and the transverse-field Ising model by evolving forward and back.  The worst
|got - want| / bound per group is printed (run with -s to see it)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg

import evolve_ref as er
import pauli_ref as pr
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, pauli_evolution_plan, pauli_sum_plan
from test_gradient_cpu import dense_h, random_terms

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, SIZE_MISMATCH, BAD_INDEX, UNSUPPORTED = 1, 2, 3, 7
TOL = {C128: 1e-12, C64: 1e-6}
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[evolve_pauli_sum] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def hamiltonians(n, rng):
    """Transverse-field Ising, the QAOA cost (even n >= 4), random strings with repeats and identities, and
    identity-only and single-term H, each with random real coefficients."""
    out = {"ising": rr.ising_step(n), "identity": [[], []], "single": [[("Y", n // 2)]]}
    if n >= 4 and n % 2 == 0:
        out["qaoa"] = rr.qaoa_layer(n)[: n + n // 2]
    rand = random_terms(n, 2 * n + 3, rng)
    out["random"] = rand + rand[:2] + [[]]
    return {k: (v, rng.normal(size=len(v))) for k, v in out.items()}


def norm2(v):
    return float(np.linalg.norm(np.asarray(v).astype(np.clongdouble).astype(C128)))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_within_bound_and_plan(ctx, dtype):
    name = np.dtype(dtype).name
    bts = (0.5, 3.0, 20.0, 100.0)
    for n in (1, 2, 3, 4, 5, 7, 9, 11, 13, 16):
        rng = np.random.default_rng(300 + n)
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
            for k, (hname, (terms, coeffs)) in enumerate(sorted(hamiltonians(n, rng).items())):
                b = max(er.split(terms, coeffs)[1], 1.0)
                bt = bts[(n + k) % len(bts)] if n < 16 else 3.0
                t = (bt / b) * (-1 if (n + k) % 2 else 1)
                psi = circuits.random_state(n, 60 * n + k, dtype)
                st.upload(psi)
                K, s, kernels, tail, c = pauli_evolution_plan(n, dtype, terms, coeffs, t, TOL[dtype])
                l0 = ctx.kernel_launches()
                got_k, got_tail = st.evolve_pauli_sum(wa, wb, terms, coeffs, t)
                assert ctx.kernel_launches() - l0 == kernels and (got_k, got_tail) == (K, tail)
                got = st.download()
                want = er.emulate(psi, n, terms, coeffs, t, TOL[dtype], dtype)
                assert np.array_equal(got, want), (name, n, hname, int(np.sum(got != want)))
                st.upload(psi)
                st.evolve_pauli_sum(wa, wb, terms, coeffs, t)
                assert np.array_equal(st.download().view(np.uint8), got.view(np.uint8))
                if n <= 12:
                    nrm = norm2(psi)
                    ref = er.cheb_ref(psi, n, terms, coeffs, t, c)
                    lim = er.bound(n, terms, coeffs, c, dtype, nrm)
                    err = norm2(got.astype(np.clongdouble) - ref)
                    assert err <= lim, (name, n, hname, err, lim)
                    note("series reference %s" % name, err / lim)
                    if n <= 8:
                        exact = scipy.linalg.expm(-1j * t * dense_h(n, terms, coeffs)) @ psi.astype(C128)
                        lim2 = lim + tail * nrm + er.exact_allowance(terms, coeffs, t, c, nrm) + 1e-15
                        err2 = norm2(got.astype(C128) - exact)
                        assert err2 <= lim2, (name, n, hname, err2, lim2)
                        note("expm %s" % name, err2 / lim2)
            # t == 0 and no terms: no kernel, the state unchanged
            st.upload(psi)
            l0 = ctx.kernel_launches()
            assert st.evolve_pauli_sum(wa, wb, terms, coeffs, 0.0) == (0, 0.0)
            assert st.evolve_pauli_sum(wa, wb, [], [], 1.0) == (0, 0.0)
            assert ctx.kernel_launches() == l0 and np.array_equal(st.download(), psi.astype(dtype))


def _prepare(st, n, seed):
    """A spread-out product state made on the device: R_Y of random angles on every qubit, then a ring of ZZ
    rotations."""
    rng = np.random.default_rng(seed)
    st.set_basis(0)
    st.apply_pauli_rotations([[("Y", q)] for q in range(n)] + [[("Z", q), ("Z", (q + 1) % n)] for q in range(n)],
                             rng.uniform(-3, 3, size=2 * n))


@pytest.mark.parametrize("n,dtype", [(26, C128), (28, C64)], ids=["n26_f64", "n28_f32"])
def test_full_size_diagonal_matches_rotations(ctx, n, dtype):
    """A diagonal H commutes term by term: exp(-iHt) = prod_h exp(-i (2 c_h t) / 2 P_h)."""
    name = "n%d %s" % (n, np.dtype(dtype).name)
    terms = rr.qaoa_layer(n)[: n + n // 2] + [[]]
    coeffs = np.random.default_rng(n).normal(size=len(terms)) * 0.2
    t = 1.3
    K, s, kernels, tail, c = pauli_evolution_plan(n, dtype, terms, coeffs, t, TOL[dtype])
    ctx.release_pool()
    try:
        with State(n, dtype, ctx) as st:
            with State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
                _prepare(st, n, 5)
                l0 = ctx.kernel_launches()
                assert st.evolve_pauli_sum(wa, wb, terms, coeffs, t) == (K, tail)
                assert ctx.kernel_launches() - l0 == kernels == K
            with State(n, dtype, ctx) as rot:
                _prepare(rot, n, 5)
                rot.apply_pauli_rotations(terms, 2 * t * coeffs)
                lim = er.bound(n, terms, coeffs, c, dtype, 1.0) + tail + 2 * rr.bound(len(terms) + 2 * n, 1.0, dtype) \
                    + er.exact_allowance(terms, coeffs, t, c, 1.0)
                err = st.max_abs_diff(rot)
                assert err <= lim, (name, err, lim)
                note("full %s vs rotations" % name, err / lim)
    finally:
        ctx.release_pool()


def test_full_size_ising_forward_and_back(ctx):
    n, dtype = 24, C128
    terms = rr.ising_step(n)
    coeffs = np.random.default_rng(24).normal(size=2 * n) * 0.5
    t = 0.9
    with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb, \
            State(n, dtype, ctx) as ref:
        _prepare(st, n, 7)
        _prepare(ref, n, 7)
        S = float(np.sum(np.abs(coeffs)))
        e0 = float(np.dot(coeffs, st.expect_paulis(terms)))
        n0 = st.norm2()
        lims = []
        for tt in (t, -t):
            K, s, kernels, tail, c = pauli_evolution_plan(n, dtype, terms, coeffs, tt, TOL[dtype])
            assert s == pauli_sum_plan(n, dtype, terms) and st.evolve_pauli_sum(wa, wb, terms, coeffs, tt) == (K, tail)
            lims.append(er.bound(n, terms, coeffs, c, dtype, 1.0) + tail + er.exact_allowance(terms, coeffs, tt, c, 1.0))
            d = sum(lims)
            assert abs(st.norm2() - n0) <= 2 * d + d * d + 1e-13
            e = float(np.dot(coeffs, st.expect_paulis(terms)))
            lim_e = 2 * S * d + 2 * S * pr.bound(n, 1.0)
            assert abs(e - e0) <= lim_e, (e, e0, lim_e)
            note("ising n24 energy drift", abs(e - e0) / lim_e)
        err = st.max_abs_diff(ref)
        assert err <= sum(lims), (err, lims)
        note("ising n24 forward and back", err / sum(lims))


def test_pending_collapse_and_refusals(ctx):
    n = 12
    rng = np.random.default_rng(12)
    terms, coeffs = rr.ising_step(n) + [[("Y", 0), ("X", 7)], []], rng.normal(size=2 * n + 2)
    t = 1.7
    psi0 = circuits.random_state(n, 21, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb, \
            State(n, C128, ctx) as b, State(n - 1, C128, ctx) as small, State(n, C64, ctx) as single:
        w1, w2 = circuits.random_state(n, 22, C128), circuits.random_state(n, 23, C128)
        a.upload(psi0)
        wa.upload(w1)
        wb.upload(w2)
        refusals = [
            (lambda: a.evolve_pauli_sum(a, wb, terms, coeffs, t), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, a, terms, coeffs, t), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wa, terms, coeffs, t), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, small, terms, coeffs, t), SIZE_MISMATCH),
            (lambda: a.evolve_pauli_sum(single, wb, terms, coeffs, t), SIZE_MISMATCH),
            (lambda: a.evolve_pauli_sum(wa, wb, terms + [[("W", 0)]], list(coeffs) + [1.0], t), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wb, terms + [[("X", n)]], list(coeffs) + [1.0], t), BAD_INDEX),
            (lambda: a.evolve_pauli_sum(wa, wb, terms + [[("X", 1), ("Z", 1)]], list(coeffs) + [1.0], t), BAD_INDEX),
            (lambda: a.evolve_pauli_sum(wa, wb, terms, np.where(np.arange(len(coeffs)) == 2, np.nan, coeffs), t),
             INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wb, terms, coeffs, np.inf), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wb, terms, coeffs, t, tol=0.0), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wb, terms, coeffs, t, tol=1.0), INVALID_ARG),
            (lambda: a.evolve_pauli_sum(wa, wb, terms, coeffs, 1e7), UNSUPPORTED),
        ]
        for call, code in refusals:
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == code, (e.value.status, code, str(e.value))
        import ctypes as C
        from rustqip_b200 import _lib
        from rustqip_b200.state import _marshal_paulis, _ptr
        qs, ls, lens = _marshal_paulis([[("X", 0)]])
        one, tl, d = np.ones(1), C.c_double(), C.c_uint32()
        L = _lib.lib()
        assert L.qipb200_state_evolve_pauli_sum(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), t, 1e-9,
                                                None, C.byref(tl)) == INVALID_ARG
        assert "NULL degree or tail" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_evolve_pauli_sum(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, None, t, 1e-9,
                                                C.byref(d), C.byref(tl)) == INVALID_ARG
        assert "NULL coefficients" in L.qipb200_last_error(ctx.handle).decode()
        for st, want in ((a, psi0), (wa, w1), (wb, w2)):
            assert np.array_equal(st.download().view(np.uint8), want.view(np.uint8))
        # a refusal keeps a pending collapse; the call applies the one on the state and drops those on the work states
        b.upload(psi0)
        m, p = a.measure([0, 5], 0.41)
        wa.measure([1], 0.7)
        wb.measure([2], 0.2)
        with pytest.raises(CircuitError):
            a.evolve_pauli_sum(wa, wb, terms, coeffs, t, tol=2.0)
        K, s, kernels, _, _ = pauli_evolution_plan(n, C128, terms, coeffs, t, TOL[C128])
        l0 = ctx.kernel_launches()
        a.evolve_pauli_sum(wa, wb, terms, coeffs, t)
        assert ctx.kernel_launches() - l0 == kernels + 1
        b.collapse([0, 5], m, p)
        collapsed = b.download()
        assert np.array_equal(a.download(), er.emulate(collapsed, n, terms, coeffs, t, TOL[C128], C128))
        # identity-only H: one kernel, the bits of the empty-term rotation by 2 RN(a t)
        b.upload(psi0)
        l0 = ctx.kernel_launches()
        assert b.evolve_pauli_sum(wa, wb, [[], []], [0.3, -1.1], t) == (0, 0.0)
        assert ctx.kernel_launches() - l0 == 1
        assert np.array_equal(b.download(), rr.emulate(psi0, n, [[]], [2.0 * ((0.3 - 1.1) * t)], C128))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, State(12, C128, ctx, rank=0, world_size=2) as wa, \
            State(12, C128, ctx, rank=0, world_size=2) as wb:
        with pytest.raises(CircuitError) as e:
            st.evolve_pauli_sum(wa, wb, [[("X", 1)]], [1.0], 0.5)
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import evolve_ref as er
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 14
rng = np.random.default_rng(14)
terms = rr.ising_step(n) + [[("Y", 0), ("X", 7)], [("X", 3), ("X", 11), ("Z", 5)], []]
coeffs = rng.normal(size=len(terms))
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b, State(n, np.complex128, ctx) as wa, \
            State(n, np.complex128, ctx) as wb:
        for st in (a, b):
            st.set_basis(3)
            st.apply_schedule(ops)
        before = a.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        psi = b.download()  # a download restores the canonical layout: b is a's twin
        a.evolve_pauli_sum(wa, wb, terms, coeffs, 2.5)
        assert np.array_equal(a.qubit_map(), before)
        assert np.array_equal(wa.qubit_map(), before) and np.array_equal(wb.qubit_map(), before)
        got = a.download()
assert np.array_equal(got, er.emulate(psi, n, terms, coeffs, 2.5, 1e-12, np.complex128, before))
print("ROTATE bit-exact ok")
"""


def test_permuted_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout
