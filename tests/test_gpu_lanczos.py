"""The lowest eigenvalue of a real Pauli sum by Lanczos on the device (State.lanczos_pauli_sum).

Given the returned alpha and beta (and |x|), the final state is compared bit for bit (+-0 equal) with the numpy
emulator of tests/lanczos_ref.py; alpha and beta lie within the documented bounds of long-double inner products of the
emulated vectors; the energy lies within the returned residual of eigh's (or eigsh's) lowest eigenvalue.  At full size
the open-chain TFIM is checked against its free-fermion closed form.  The worst |got - want| / bound per group is
printed (run with -s to see it)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse.linalg

import lanczos_ref as lr
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, pauli_lanczos_plan
from test_gradient_cpu import dense_h, random_terms

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, SIZE_MISMATCH, BAD_INDEX, UNSUPPORTED = 1, 2, 3, 7
TOL = {C128: 1e-8, C64: 1e-3}
STEPS = 600
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[lanczos_pauli_sum] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def hamiltonians(n, rng):
    out = {"tfim": lr.tfim(rng.uniform(0.2, 1.0, size=n - 1), rng.uniform(0.5, 1.5, size=n)),
           "single": ([[("Y", n // 2)]], np.array([0.7]))}
    if n >= 2:
        out["xxx"] = lr.heisenberg(n)
    rand = random_terms(n, 2 * n + 3, rng)
    rand = rand + rand[:2] + [[]]
    out["random"] = (rand, rng.normal(size=len(rand)))
    return out


def lowest(n, terms, coeffs):
    if n <= 8:
        return float(np.linalg.eigvalsh(dense_h(n, terms, coeffs))[0])
    H = lr.sparse_h(n, terms, coeffs)
    return float(scipy.sparse.linalg.eigsh(H, k=1, which="SA", tol=1e-12)[0][0])


def allowance(dtype, terms, coeffs):
    """What the stored state's rounding may add to |E - lambda| and to the residual (u per amplitude of x and Hx)."""
    a, b = lr.split(terms, coeffs)
    return 16 * rr.U[dtype] * (b + abs(a)) + 1e-12 * (b + 1)


def same_bits(x, y):
    return np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_bounds_launches_and_eigh(ctx, dtype):
    name = np.dtype(dtype).name
    for n in (1, 2, 3, 4, 5, 7, 9, 11, 13, 16):
        rng = np.random.default_rng(500 + n)
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
            for k, (hname, (terms, coeffs)) in enumerate(sorted(hamiltonians(n, rng).items())):
                tag = (name, n, hname)
                psi = circuits.random_state(n, 70 * n + k, dtype)
                plan = pauli_lanczos_plan(n, dtype, terms)
                assert plan == lr.plan_policy(n, terms)
                # energy only: the state is not written
                st.upload(psi)
                l0 = ctx.kernel_launches()
                r0 = st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=STEPS, vector=False)
                assert ctx.kernel_launches() - l0 == lr.launches(plan, r0.steps, False), tag
                assert same_bits(st.download(), psi.astype(dtype)) and r0.ritz_norm == 0.0
                # vector mode: the same recurrence, then the Ritz vector
                st.upload(psi)
                l0 = ctx.kernel_launches()
                r = st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=STEPS)
                assert ctx.kernel_launches() - l0 == lr.launches(plan, r.steps, True), tag
                assert same_bits(r.alpha, r0.alpha) and same_bits(r.beta, r0.beta) and r.steps == r0.steps
                assert r.converged == r0.converged and (r.converged or r.steps == STEPS), tag
                if n <= 11 or hname != "random":  # random strings at n >= 13: a dense, clustered low spectrum
                    assert r.converged, tag
                if n <= 3:  # the Krylov space is exhausted by 2^n steps at the latest
                    assert r.steps <= 2 ** n, tag
                got = st.download()
                keep = n <= 11
                e = lr.emulate(psi, n, terms, coeffs, dtype, r.alpha, r.beta, r.ritz_norm, keep=keep)
                assert np.array_equal(got, e["state"]), tag + (int(np.sum(got != e["state"])),)
                st.upload(psi)
                r2 = st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=STEPS)
                assert same_bits(st.download(), got) and same_bits(r2.alpha, r.alpha) and \
                    same_bits(r2.beta, r.beta) and (r2.energy, r2.residual, r2.ritz_norm) == \
                    (r.energy, r.residual, r.ritz_norm), tag
                # alpha and beta against long-double inner products of the emulated vectors (every vector is kept
                # up to n = 11)
                for j in range(r.steps if keep else 0):
                    u, w, un = (e["u"][j].astype(np.clongdouble), e["w"][j].astype(np.clongdouble),
                                e["u"][j + 1].astype(np.clongdouble))
                    la, lb = lr.alpha_beta_bound(n, e["u"][j], e["w"][j], e["u"][j + 1], r.beta[j])
                    da = abs(float(np.sum(np.conj(u) * w).real / np.longdouble(r.beta[j])) - r.alpha[j])
                    db = abs(float(np.sqrt(np.sum(np.abs(un) ** 2))) - r.beta[j + 1])
                    assert da <= la and db <= lb, tag + (j, da, la, db, lb)
                    note("alpha %s" % name, da / la)
                    note("beta %s" % name, db / lb)
                # the energy: an eigenvalue within the residual; here the lowest
                a, b = lr.split(terms, coeffs)
                lam = lowest(n, terms, coeffs)
                allow = allowance(dtype, terms, coeffs)
                err = abs(r.energy - lam)
                assert err <= r.residual + allow, tag + (r.energy, lam, r.residual)
                assert abs(r0.energy - lam) <= r0.residual + allow, tag + (r0.energy, lam, r0.residual)
                if r.converged:
                    assert r0.residual <= TOL[dtype] * b and r.residual <= 4 * TOL[dtype] * b + allow, tag
                    assert abs(r.ritz_norm - 1) <= 1e-3, tag
                note("|E - lambda| / (residual + allowance) %s" % name, err / (r.residual + allow))


def test_small_n_breakdown_b_zero_and_cap(ctx):
    for n in (1, 2, 3):
        rng = np.random.default_rng(n)
        terms, coeffs = lr.tfim(rng.uniform(0.2, 1, size=n - 1), rng.uniform(0.5, 1.5, size=n))
        with State(n, C128, ctx) as st, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
            st.upload(circuits.random_state(n, 9, C128))
            r = st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=2 ** n + 5)
            assert r.converged and r.steps <= 2 ** n
            lam = float(np.linalg.eigvalsh(dense_h(n, terms, coeffs))[0])
            assert abs(r.energy - lam) <= r.residual + 1e-12
    n = 10
    with State(n, C128, ctx) as st, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
        psi = circuits.random_state(n, 3, C128)
        # b == 0: every vector is an eigenvector; vector mode normalises
        st.upload(3.0 * psi)
        l0 = ctx.kernel_launches()
        r = st.lanczos_pauli_sum(wa, wb, [[], [("Z", 2)], []], [0.25, 0.0, -1.0])
        assert ctx.kernel_launches() - l0 == 2 and (r.energy, r.residual, r.steps, r.converged) == (-0.75, 0.0, 0, True)
        assert abs(st.norm2() - 1) <= 1e-14 and r.beta.shape == (1,) and abs(r.beta[0] - 3) <= 1e-13
        l0 = ctx.kernel_launches()
        r = st.lanczos_pauli_sum(wa, wb, [], [], vector=False)
        assert ctx.kernel_launches() - l0 == 1 and (r.energy, r.steps) == (0.0, 0)
        # the cap: not converged, the best estimate returned
        terms, coeffs = lr.heisenberg(n)
        st.upload(psi)
        r = st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=3)
        assert r.steps == 3 and not r.converged and r.residual > TOL[C128] * lr.split(terms, coeffs)[1]
        assert r.energy >= lowest(n, terms, coeffs) - 1e-12


def test_symmetry_sector_from_neel(ctx):
    n = 12
    terms, coeffs = lr.heisenberg(n)
    H = lr.sparse_h(n, terms, coeffs).tocsr()
    sec = np.array([i for i in range(1 << n) if bin(i).count("1") == n // 2])
    lam0 = float(np.linalg.eigvalsh(H[sec][:, sec].toarray())[0])
    one = np.array([i for i in range(1 << n) if bin(i).count("1") == n // 2 + 1])
    lam1 = float(np.linalg.eigvalsh(H[one][:, one].toarray())[0])
    assert lam1 > lam0 + 1e-3
    with State(n, C128, ctx) as st, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
        for basis, want in ((int("01" * (n // 2), 2), lam0), (int("11" + "01" * (n // 2 - 1), 2), lam1)):
            st.set_basis(basis)
            r = st.lanczos_pauli_sum(wa, wb, terms, coeffs)
            assert r.converged and abs(r.energy - want) <= r.residual + 1e-12, (basis, r.energy, want)
            note("sector |E - lambda| / residual", abs(r.energy - want) / (r.residual + 1e-12))


@pytest.mark.parametrize("n,dtype", [(26, C128), (28, C64)], ids=["n26_f64", "n28_f32"])
def test_full_size_tfim_closed_form(ctx, n, dtype):
    name = "n%d %s" % (n, np.dtype(dtype).name)
    rng = np.random.default_rng(1000 + n)
    J, h = rng.uniform(0.2, 0.6, size=n - 1), rng.uniform(0.9, 1.3, size=n)  # paramagnetic: h_i > J_i
    terms, coeffs = lr.tfim(J, h)
    e0 = lr.tfim_ground(J, h)
    allow = allowance(dtype, terms, coeffs)
    ctx.release_pool()
    try:
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
            st.set_basis(0)
            st.apply_pauli_rotations([[("Y", q)] for q in range(n)], rng.uniform(-0.4, 0.4, size=n))
            plan = pauli_lanczos_plan(n, dtype, terms)
            l0 = ctx.kernel_launches()
            r = st.lanczos_pauli_sum(wa, wb, terms, coeffs)
            assert ctx.kernel_launches() - l0 == lr.launches(plan, r.steps, True)
            assert r.converged, (name, r.steps, r.residual)
            err = abs(r.energy - e0)
            assert err <= r.residual + allow, (name, r.energy, e0, r.residual, allow)
            note("full %s |E - closed form| / (residual + allowance)" % name, err / (r.residual + allow))
            ev = float(np.dot(coeffs, st.expect_paulis(terms)))
            assert abs(ev - r.energy) <= allow, (name, ev, r.energy)
            assert abs(st.norm2() - 1) <= 8 * rr.U[dtype] * n + 1e-12
            print("\n[%s] steps %d energy %.15f closed form %.15f residual %.3e |x| %.15f"
                  % (name, r.steps, r.energy, e0, r.residual, r.ritz_norm))
    finally:
        ctx.release_pool()


def test_pending_collapse_and_refusals(ctx):
    n = 12
    rng = np.random.default_rng(12)
    terms, coeffs = lr.tfim(rng.uniform(0.2, 1, size=n - 1), rng.uniform(0.5, 1.5, size=n))
    terms, coeffs = terms + [[("Y", 0), ("X", 7)], []], np.append(coeffs, [0.3, -0.4])
    psi0 = circuits.random_state(n, 21, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb, \
            State(n, C128, ctx) as b, State(n - 1, C128, ctx) as small, State(n, C64, ctx) as single:
        w1, w2 = circuits.random_state(n, 22, C128), circuits.random_state(n, 23, C128)
        a.upload(psi0)
        wa.upload(w1)
        wb.upload(w2)
        refusals = [
            (lambda: a.lanczos_pauli_sum(a, wb, terms, coeffs), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, a, terms, coeffs), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wa, terms, coeffs), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, small, terms, coeffs), SIZE_MISMATCH),
            (lambda: a.lanczos_pauli_sum(single, wb, terms, coeffs), SIZE_MISMATCH),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms + [[("W", 0)]], list(coeffs) + [1.0]), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms + [[("X", n)]], list(coeffs) + [1.0]), BAD_INDEX),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms + [[("X", 1), ("Z", 1)]], list(coeffs) + [1.0]), BAD_INDEX),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms, np.where(np.arange(len(coeffs)) == 2, np.nan, coeffs)),
             INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=0), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=4097), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms, coeffs, tol=0.0), INVALID_ARG),
            (lambda: a.lanczos_pauli_sum(wa, wb, terms, coeffs, tol=1.0), INVALID_ARG),
        ]
        for call, code in refusals:
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == code, (e.value.status, code, str(e.value))
        import ctypes as C
        from rustqip_b200 import _lib
        from rustqip_b200.state import _marshal_paulis, _ptr
        qs, ls, lens = _marshal_paulis([[("X", 0)]])
        one, out3, m, cv = np.ones(1), np.zeros(3), C.c_uint32(), C.c_uint32()
        L = _lib.lib()
        for args in ((None, C.byref(cv), _ptr(out3)), (C.byref(m), None, _ptr(out3)), (C.byref(m), C.byref(cv), None)):
            assert L.qipb200_state_lanczos_pauli_sum(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), 10,
                                                     1e-8, 1, args[0], args[1], None, None, args[2]) == INVALID_ARG
            assert "NULL steps, converged or out3" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_lanczos_pauli_sum(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, None, 10, 1e-8, 1,
                                                 C.byref(m), C.byref(cv), None, None, _ptr(out3)) == INVALID_ARG
        assert "NULL coefficients" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_lanczos_pauli_sum(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), 10, 1e-8,
                                                 6, C.byref(m), C.byref(cv), None, None, _ptr(out3)) == INVALID_ARG
        assert "unknown flags" in L.qipb200_last_error(ctx.handle).decode()
        for st, want in ((a, psi0), (wa, w1), (wb, w2)):
            assert same_bits(st.download(), want)
        # a zero state is refused after the first read sweep, unchanged
        with State(n, C128, ctx) as z:
            z.upload(np.zeros(1 << n, dtype=C128))
            with pytest.raises(CircuitError) as e:
                z.lanczos_pauli_sum(wa, wb, terms, coeffs)
            assert e.value.status == INVALID_ARG and "zero" in str(e.value)
            assert not np.any(z.download())
        # a refusal keeps a pending collapse; the call applies the one on the state and drops those on the work states
        b.upload(psi0)
        mm, p = a.measure([0, 5], 0.41)
        wa.measure([1], 0.7)
        wb.measure([2], 0.2)
        with pytest.raises(CircuitError):
            a.lanczos_pauli_sum(wa, wb, terms, coeffs, tol=2.0)
        plan = pauli_lanczos_plan(n, C128, terms)
        l0 = ctx.kernel_launches()
        r = a.lanczos_pauli_sum(wa, wb, terms, coeffs)
        assert ctx.kernel_launches() - l0 == lr.launches(plan, r.steps, True) + 1
        b.collapse([0, 5], mm, p)
        collapsed = b.download()
        e = lr.emulate(collapsed, n, terms, coeffs, C128, r.alpha, r.beta, r.ritz_norm)
        assert np.array_equal(a.download(), e["state"])


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, State(12, C128, ctx, rank=0, world_size=2) as wa, \
            State(12, C128, ctx, rank=0, world_size=2) as wb:
        with pytest.raises(CircuitError) as e:
            st.lanczos_pauli_sum(wa, wb, [[("X", 1)]], [1.0])
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import lanczos_ref as lr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 14
rng = np.random.default_rng(14)
terms, coeffs = lr.tfim(rng.uniform(0.2, 1, size=n - 1), rng.uniform(0.5, 1.5, size=n))
terms, coeffs = terms + [[("Y", 0), ("X", 7)], [("X", 3), ("X", 11), ("Z", 5)], []], np.append(coeffs, [0.2, -0.3, 0.1])
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
        r = a.lanczos_pauli_sum(wa, wb, terms, coeffs)
        assert np.array_equal(a.qubit_map(), before)
        assert np.array_equal(wa.qubit_map(), before) and np.array_equal(wb.qubit_map(), before)
        got = a.download()
e = lr.emulate(psi, n, terms, coeffs, np.complex128, r.alpha, r.beta, r.ritz_norm, before)
assert np.array_equal(got, e["state"])
print("ROTATE bit-exact ok", r.steps)
"""


def test_permuted_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout
