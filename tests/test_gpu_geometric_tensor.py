"""The quantum geometric tensor on the device (State.geometric_tensor, qipb200_state_pauli_geometric_tensor).

The three end states are compared bit for bit (+-0 equal) with the emulation of tests/qgt_ref.py, and G and e within
qgt_bound of the long-double fork-and-segment reference (tests/test_geometric_tensor_cpu.py pins it to the definition,
the parameter-shift rule and the closed form).  The worst |got - want| / bound per group is printed (run with -s)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gradient_ref as gr
import pauli_rot_ref as rr
import qgt_ref as qr
from rustqip_b200 import circuits
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, pauli_geometric_tensor_plan
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
    print("\n[geometric_tensor] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def check_values(group, psi0, n, ansatz, angles, G, e, dtype):
    Gr, er = qr.qgt_ref(psi0, n, ansatz, angles)
    bg, be = qr.qgt_bound(n, len(ansatz), float(np.linalg.norm(np.asarray(psi0).astype(C128))), dtype)
    dg = float(np.max(np.abs(G.astype(np.clongdouble) - Gr))) if len(ansatz) else 0.0
    de = float(np.max(np.abs(e.astype(np.longdouble) - er))) if len(ansatz) else 0.0
    assert dg <= bg and de <= be, (group, n, dg, bg, de, be)
    note(group, max(dg / bg, de / be))


def check_end_states(st, wa, wb, psi0, n, ansatz, angles, dtype, label):
    want = qr.emulate_end_states(psi0, n, ansatz, angles, dtype)
    for got, w, name in zip((st.download(), wa.download(), wb.download()), want, ("state", "work_a", "work_b")):
        assert np.array_equal(got, w), (label, name, int(np.sum(got != w)))


def hermitian(G):
    return np.array_equal(G, np.conj(G.T))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_within_bound_and_plan(ctx, dtype):
    name = np.dtype(dtype).name
    for n in (6, 7, 9, 11, 12, 14, 16, 18, 20):
        rng = np.random.default_rng(1300 + n)
        fam = families(n, rng)
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
            for k, (fname, ansatz) in enumerate(sorted(fam.items())):
                psi0 = circuits.random_state(n, 800 + 7 * n + k, dtype)
                angles = rng.uniform(-6.5, 6.5, size=len(ansatz))
                st.upload(psi0)
                l0 = ctx.kernel_launches()
                G, e = st.geometric_tensor(wa, wb, ansatz, angles)
                plan = pauli_geometric_tensor_plan(n, dtype, ansatz)
                assert plan == qr.plan_policy(n, ansatz)
                assert ctx.kernel_launches() - l0 == plan[2], (n, fname)
                assert G.shape == (len(ansatz), len(ansatz)) and e.shape == (len(ansatz),)
                assert hermitian(G) and not np.any(np.signbit(G.diagonal().imag)) and not np.any(G.diagonal().imag)
                check_end_states(st, wa, wb, psi0, n, ansatz, angles, dtype, (name, n, fname))
                st.upload(psi0)
                G2, e2 = st.geometric_tensor(wa, wb, ansatz, angles)
                assert np.array_equal(G.view(np.uint64), G2.view(np.uint64)) and \
                    np.array_equal(e.view(np.uint64), e2.view(np.uint64)), (name, n, fname)
                if n <= 7 or (n <= 12 and fname != "long run"):
                    check_values("reference %s" % name, psi0, n, ansatz, angles, G, e, dtype)


def test_zero_and_one_term(ctx):
    n = 12
    psi0 = circuits.random_state(n, 12, C128)
    junk = circuits.random_state(n, 13, C128)
    with State(n, C128, ctx) as st, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
        st.upload(psi0)
        wa.upload(junk)
        wb.upload(junk)
        l0 = ctx.kernel_launches()
        G, e = st.geometric_tensor(wa, wb, [], [])
        assert ctx.kernel_launches() == l0 and G.shape == (0, 0) and e.shape == (0,)
        assert np.array_equal(st.download(), psi0) and np.array_equal(wa.download(), junk)
        assert np.array_equal(wb.download(), junk)
        term = [("Y", 3), ("Z", 7), ("X", 11)]
        l0 = ctx.kernel_launches()
        G, e = st.geometric_tensor(wa, wb, [term], [0.7])
        assert ctx.kernel_launches() - l0 == 2 == pauli_geometric_tensor_plan(n, C128, [term])[2]
        check_end_states(st, wa, wb, psi0, n, [term], [0.7], C128, "one term")
        ex = float(st.expect_paulis([term])[0])  # P commutes with R: <P> after R is e_0
        assert abs(e[0] - ex) <= 1e-14 and abs(G[0, 0].real - (st.norm2() - ex * ex) / 4) <= 1e-14
        assert G[0, 0].imag == 0.0 and not np.signbit(G[0, 0].imag)
        check_values("one term", psi0, n, [term], [0.7], G, e, C128)


def test_empty_string_row_is_zero(ctx):
    n = 10
    rng = np.random.default_rng(10)
    ansatz = rr.ising_step(n)[:8] + [[]] + rr.ucc_strings(n, 5, 3) + [[]]
    angles = rng.uniform(-3, 3, size=len(ansatz))
    psi0 = circuits.random_state(n, 14, C128)
    with State(n, C128, ctx) as st, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb:
        st.upload(psi0)
        G, e = st.geometric_tensor(wa, wb, ansatz, angles)
    bg, _ = qr.qgt_bound(n, len(ansatz), 1.0, C128)
    for t in (8, len(ansatz) - 1):
        assert np.max(np.abs(G[t])) <= bg and np.max(np.abs(G[:, t])) <= bg
        assert abs(e[t] - 1.0) <= 1e-14
    check_values("empty strings", psi0, n, ansatz, angles, G, e, C128)


def test_pending_collapse_and_refusals(ctx):
    n = 13
    rng = np.random.default_rng(13)
    ansatz = families(n, rng)["ucc"][:10] + rr.ising_step(n)
    angles = rng.uniform(-2, 2, size=len(ansatz))
    psi0 = circuits.random_state(n, 17, C128)
    psi1 = circuits.random_state(n, 18, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as wa, State(n, C128, ctx) as wb, State(n, C128, ctx) as b, \
            State(n - 1, C128, ctx) as small, State(n, C64, ctx) as single:
        a.upload(psi0)
        b.upload(psi0)
        wa.upload(psi1)
        wb.upload(psi1)
        nan = np.where(np.arange(len(angles)) == 4, np.nan, angles)
        refusals = [
            (lambda: a.geometric_tensor(a, wb, ansatz, angles), INVALID_ARG),
            (lambda: a.geometric_tensor(wa, wa, ansatz, angles), INVALID_ARG),
            (lambda: a.geometric_tensor(wa, small, ansatz, angles), SIZE_MISMATCH),
            (lambda: a.geometric_tensor(single, wb, ansatz, angles), SIZE_MISMATCH),
            (lambda: a.geometric_tensor(wa, wb, ansatz + [[("W", 0)]], list(angles) + [1.0]), INVALID_ARG),
            (lambda: a.geometric_tensor(wa, wb, ansatz + [[("X", n)]], list(angles) + [1.0]), BAD_INDEX),
            (lambda: a.geometric_tensor(wa, wb, ansatz + [[("X", 2), ("Z", 2)]], list(angles) + [1.0]), BAD_INDEX),
            (lambda: a.geometric_tensor(wa, wb, ansatz, nan), INVALID_ARG),
            (lambda: a.geometric_tensor(wa, wb, [[("Z", 0)]] * 2049, np.zeros(2049)), UNSUPPORTED),
        ]
        for call, code in refusals:
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == code, (e.value.status, code, str(e.value))
        from rustqip_b200 import _lib
        from rustqip_b200.state import _marshal_paulis, _ptr
        qs, ls, lens = _marshal_paulis([[("X", 0)]])
        one = np.ones(1)
        L = _lib.lib()
        assert L.qipb200_state_pauli_geometric_tensor(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, _ptr(one), None,
                                                      None) == INVALID_ARG
        assert "NULL qgt" in L.qipb200_last_error(ctx.handle).decode()
        assert L.qipb200_state_pauli_geometric_tensor(a._h, wa._h, wb._h, _ptr(qs), ls, _ptr(lens), 1, None,
                                                      _ptr(np.zeros(2)), None) == INVALID_ARG
        assert "NULL angles" in L.qipb200_last_error(ctx.handle).decode()
        assert np.array_equal(a.download(), psi0) and np.array_equal(wa.download(), psi1)
        assert np.array_equal(wb.download(), psi1)
        # a refusal keeps a pending collapse; the call applies the one on state and drops the ones on the work states
        m, p = a.measure([0, 5], 0.41)
        wa.measure([1], 0.7)
        wb.measure([2], 0.2)
        with pytest.raises(CircuitError):
            a.geometric_tensor(wa, wb, ansatz + [[("Q", 0)]], list(angles) + [1.0])
        l0 = ctx.kernel_launches()
        G, e = a.geometric_tensor(wa, wb, ansatz, angles)
        assert ctx.kernel_launches() - l0 == pauli_geometric_tensor_plan(n, C128, ansatz)[2] + 1
        b.collapse([0, 5], m, p)
        collapsed = b.download()
        check_end_states(a, wa, wb, collapsed, n, ansatz, angles, C128, "collapse")
        G2, e2 = b.geometric_tensor(wa, wb, ansatz, angles)
        assert np.array_equal(G, G2) and np.array_equal(e, e2)
        # T = 0 applies a collapse pending on state, and only that
        b.upload(psi0)
        b.measure([3], 0.5)
        l0 = ctx.kernel_launches()
        b.geometric_tensor(wa, wb, [], [])
        assert ctx.kernel_launches() - l0 == 1


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, State(12, C128, ctx, rank=0, world_size=2) as wa, \
            State(12, C128, ctx, rank=0, world_size=2) as wb:
        with pytest.raises(CircuitError) as e:
            st.geometric_tensor(wa, wb, [[("Z", 0)]], [0.5])
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import pauli_rot_ref as rr
import qgt_ref as qr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 14
rng = np.random.default_rng(16)
ansatz = rr.ising_step(n) + rr.ucc_strings(n, 6, 5) + [[("Y", 0), ("X", 9)]]
angles = rng.uniform(-3, 3, size=len(ansatz))
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
        G, e = a.geometric_tensor(wa, wb, ansatz, angles)
        for s in (a, wa, wb):
            assert np.array_equal(s.qubit_map(), before), "a state left the layout"
        got = [a.download(), wa.download(), wb.download()]
want = qr.emulate_end_states(psi, n, ansatz, angles, np.complex128)
assert all(np.array_equal(g, w) for g, w in zip(got, want))
Gr, er = qr.qgt_ref(psi, n, ansatz, angles)
bg, be = qr.qgt_bound(n, len(ansatz), 1.0, np.complex128)
assert float(np.max(np.abs(G - Gr))) <= bg and float(np.max(np.abs(e - er))) <= be
assert np.array_equal(G, np.conj(G.T))
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
    rng = np.random.default_rng(n + 5)
    theta, phi = rng.uniform(-3, 3, size=n), rng.uniform(-3, 3, size=n)
    ansatz = gr.product_ansatz(n)
    angles = np.concatenate([theta, phi])
    ctx.release_pool()
    try:
        with State(n, dtype, ctx) as st, State(n, dtype, ctx) as wa, State(n, dtype, ctx) as wb:
            st.set_basis(0)
            l0 = ctx.kernel_launches()
            G, e = st.geometric_tensor(wa, wb, ansatz, angles)
            assert ctx.kernel_launches() - l0 == pauli_geometric_tensor_plan(n, dtype, ansatz)[2]
            Gw, ew = qr.closed_form(n, theta, phi)
            bg, be = qr.qgt_bound(n, len(ansatz), 1.0, dtype)
            dg = float(np.max(np.abs(G.astype(np.clongdouble) - Gw)))
            de = float(np.max(np.abs(e.astype(np.longdouble) - ew)))
            assert dg <= bg and de <= be, (name, dg, bg, de, be)
            assert hermitian(G)
            note("full %s closed form" % name, max(dg / bg, de / be))
            assert st.max_abs_diff(wa) == 0.0

            # U|0..0>: the R_Y layer's product amplitudes times the phases of the ZZ layer
            c = np.cos(np.asarray(theta, dtype=np.longdouble) / 2)
            s = np.sin(np.asarray(theta, dtype=np.longdouble) / 2)
            ph = np.asarray(phi, dtype=np.longdouble)

            def final(idx):
                bits = [((idx >> np.uint64(n - 1 - q)) & np.uint64(1)).astype(bool) for q in range(n)]
                amp = np.ones(idx.shape, dtype=np.longdouble)
                ang = np.zeros(idx.shape, dtype=np.longdouble)
                for q in range(n):
                    amp *= np.where(bits[q], s[q], c[q])
                    zz = np.where(bits[q] == bits[(q + 1) % n], 1, -1)
                    ang -= ph[q] / 2 * zz
                return amp * (np.cos(ang) + 1j * np.sin(ang))

            ratio = check_windows(st, n, dtype, final, rr.bound(len(ansatz), 1.0, dtype), name + " U|0>")
            note("full %s state U|0>" % name, ratio)
    finally:
        ctx.release_pool()
