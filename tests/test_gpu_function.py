"""Table-defined function ops on the device (State.apply_function, qipb200_state_apply_function).

The device result is compared bit for bit with the numpy emulator of tests/function_ref.py (which
tests/test_function_cpu.py pins to the reference iterator's row rule), with gate circuits on the device at full size
(max_abs_diff == 0), with Shor's period-finding distribution at N = 30, and with closed forms past 2^31 and 2^32
amplitudes."""
import os
import subprocess
import sys

import numpy as np
import pytest

import function_ref as fr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.ops import make_control_op
from rustqip_b200.state import FUNCTION_PAIR, FUNCTION_TILE, Context, Function, State, function_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7


def bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def registers(n, rng, path, dtype):
    """Random unsorted registers that take `path` (FUNCTION_TILE or FUNCTION_PAIR) on an n-qubit state."""
    tmax = 11 if dtype == C128 else 12
    for _ in range(1000):
        perm = [int(q) for q in rng.permutation(n)]
        if path == FUNCTION_PAIR:
            k = tmax - 3 + int(rng.integers(0, 3))
            out_q = [q for q in perm if q < n - 4][:k]  # on index bits >= 4
            rest = [q for q in perm if q not in out_q]
            in_q = rest[:int(rng.integers(1, min(12, len(rest)) + 1))]
        else:
            n_out = int(rng.integers(1, min(8, n - 1) + 1))
            out_q = perm[:n_out]
            in_q = perm[n_out:n_out + int(rng.integers(1, min(12, n - n_out) + 1))]
        if len(out_q) and function_plan(n, dtype, in_q, out_q)[0] == path:
            return in_q, out_q
    raise AssertionError("no registers for path %d at n = %d" % (path, n))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_numpy(ctx, dtype):
    seen = set()
    for n in (6, 8, 11, 13, 14, 16, 18, 20):
        rng = np.random.default_rng(900 + n)
        psi0 = circuits.random_state(n, 40 + n, dtype)
        psi0[rng.integers(0, 1 << n, size=3)] = complex(-0.0, -0.0)
        paths = (FUNCTION_TILE, FUNCTION_PAIR) if n >= 14 else (FUNCTION_TILE,)
        with State(n, dtype, ctx) as st:
            for path in paths:
                in_q, out_q = registers(n, rng, path, dtype)
                f = rng.integers(0, 1 << len(out_q), size=1 << len(in_q), dtype=np.uint64)
                theta = rng.uniform(-7, 7, size=1 << len(in_q))
                seen.add(path)
                # permutation only: the numpy move exactly, and twice gives the state back
                with Function(ctx, len(in_q), len(out_q), f=f) as fn:
                    st.upload(psi0)
                    st.apply_function(fn, in_q, out_q)
                    assert bits_equal(st.download(), fr.apply(psi0, n, in_q, out_q, f)), (n, path, in_q, out_q)
                    st.apply_function(fn, in_q, out_q)
                    assert bits_equal(st.download(), psi0), (n, path)
                # with theta: the emulation bit for bit
                with Function(ctx, len(in_q), len(out_q), f=f, theta=theta) as fn:
                    st.upload(psi0)
                    st.apply_function(fn, in_q, out_q)
                    assert bits_equal(st.download(), fr.apply(psi0, n, in_q, out_q, f, theta)), (n, path)
                # phase only (tile path)
                assert function_plan(n, dtype, in_q, [])[0] == FUNCTION_TILE
                with Function(ctx, len(in_q), 0, theta=theta) as fn:
                    st.upload(psi0)
                    st.apply_function(fn, in_q)
                    assert bits_equal(st.download(), fr.apply(psi0, n, in_q, (), None, theta)), (n, "phase")
    assert seen == {FUNCTION_TILE, FUNCTION_PAIR}


def test_one_function_serves_both_precisions(ctx):
    n, in_q, out_q = 12, [3, 9, 0, 5], [11, 2]
    rng = np.random.default_rng(12)
    f = rng.integers(0, 4, size=16, dtype=np.uint64)
    theta = rng.uniform(-3, 3, size=16)
    with Function(ctx, 4, 2, f=f, theta=theta) as fn:
        for dtype in (C128, C64):
            psi0 = circuits.random_state(n, 5, dtype)
            with State(n, dtype, ctx) as st:
                st.upload(psi0)
                st.apply_function(fn, in_q, out_q)
                assert bits_equal(st.download(), fr.apply(psi0, n, in_q, out_q, f, theta))


# ---- against gate circuits at full size ----------------------------------------------------------------------------

class Pair:
    """At most two full-size states at a time; freeing them returns their buffers to the device."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.sts = []
        ctx.release_pool()

    def take(self, n, dtype, count=2):
        self.release()
        self.sts = [State(n, dtype, self.ctx) for _ in range(count)]
        return self.sts

    def release(self):
        for s in self.sts:
            s.free()
        self.sts = []
        self.ctx.release_pool()


@pytest.fixture(scope="module")
def pair(ctx):
    p = Pair(ctx)
    yield p
    p.release()


@pytest.mark.parametrize("n,dtype", [(28, C128), (30, C64)], ids=["n28_f64", "n30_f32"])
def test_against_gate_circuits(ctx, pair, n, dtype):
    a, b = pair.take(n, dtype)
    prep = circuits.random_circuit(n, 2, 0x5EED0000 + n, "H,T,CNOT")
    rng = np.random.default_rng(n)
    m = n - 10  # x takes every qubit the 10-qubit y leaves: 18 at N = 28, 20 at N = 30
    A = fr.random_matrix(10, m, n)
    f = fr.linear_table(A)
    perm = [int(q) for q in rng.permutation(n)]
    cases = [(list(range(m - 1, -1, -1)), list(range(n - 1, m - 1, -1))),  # x high, y low: tile
             (perm[:m], perm[m:])]                                            # random registers
    for in_q, out_q in cases:
        for st in (a, b):
            st.set_basis(0)
            st.apply_schedule(prep)
        with Function(ctx, m, 10, f=f) as fn:
            a.apply_function(fn, in_q, out_q)
        b.apply_schedule(fr.cnot_network(A, in_q, out_q))
        assert a.max_abs_diff(b) == 0.0, (n, in_q, out_q)
    # one-bit oracle f(x) = [x == w] against one multi-controlled X between X layers on the controls whose bit of w is
    # 0; 11 controls, the most the per-gate flip kernel takes (kMaxIns = 12 positions with the target)
    k = 11
    in_q, target = perm[:k], perm[k]
    w = int(rng.integers(0, 1 << k))
    flips = [gates.x(q) for i, q in enumerate(in_q) if not (w >> i) & 1]
    mcx = make_control_op(list(in_q), gates.x(target))
    for st in (a, b):
        st.set_basis(0)
        st.apply_schedule(prep)
    oracle = np.zeros(1 << k, dtype=np.uint64)
    oracle[w] = 1
    with Function(ctx, k, 1, f=oracle) as fn:
        a.apply_function(fn, in_q, [target])
    b.apply_schedule(flips + [mcx] + flips)
    assert a.max_abs_diff(b) == 0.0
    pair.release()


def test_shor_period_finding_n30(ctx, pair):
    """x = qubits 0..19 (m = 20, qubit 0 the most significant bit), y = qubits 20..29, N = 1007 = 19 * 53, a = 2
    (r = 468): H on x, |x>|0> -> |x>|2^x mod 1007>, the MatrixOp QFT on x, then the probabilities of x."""
    n, m, N, a = 30, 20, 1007, 2
    r = fr.order(a, N)
    assert r == 468
    in_q, out_q = list(range(m - 1, -1, -1)), list(range(n - 1, m - 1, -1))
    assert function_plan(n, C128, in_q, out_q)[0] == FUNCTION_TILE
    st, = pair.take(n, C128, 1)
    st.set_basis(0)
    st.apply_schedule([gates.h(q) for q in range(m)])
    with Function(ctx, m, 10, f=fr.modexp_table(a, N, m)) as fn:
        st.apply_function(fn, in_q, out_q)
    st.apply_schedule(circuits.qft(m))
    probs = st.measure_probs(in_q)
    want = fr.shor_probs(m, r)
    err = float(np.max(np.abs(probs - want)))
    print("\n[apply_function] Shor N=1007 max |P - closed form| = %.3e" % err)
    assert err <= 1e-10
    shots = st.sample(in_q, draws=np.random.default_rng(1007).random(20))
    found = [fr.period_from_shot(int(k), m, a, N) for k in shots]
    assert sum(1 for v in found if v == r) >= 12, found
    pair.release()


@pytest.mark.parametrize("n", [31, 32])
def test_large_indices_f32(ctx, pair, n):
    """Registers on index bits 30 and 31 (qubits n-31, n-32), both paths, from the H layer: a phase function phi, then
    a permutation with theta; every window against 2^(-n/2) e^{i theta(x(j))} e^{i phi(x1(j ^ d))}."""
    def q(bit):
        return n - 1 - bit

    top = [b for b in (31, 30) if b < n]
    in1 = [q(b) for b in top + [1, 9, 17]]
    cases = {FUNCTION_TILE: ([q(b) for b in [29, 5, 17, 0]], [q(b) for b in top + [3]]),
             FUNCTION_PAIR: ([q(b) for b in [0, 2, 10, 15]], [q(b) for b in top + list(range(29, 29 - (11 - len(top)),
                                                                                          -1))])}
    rng = np.random.default_rng(n)
    phi = rng.uniform(-3, 3, size=1 << len(in1))
    st, = pair.take(n, C64, 1)
    for path, (in2, out2) in cases.items():
        assert function_plan(n, C64, in2, out2)[0] == path
        f = rng.integers(0, 1 << len(out2), size=1 << len(in2), dtype=np.uint64)
        theta = rng.uniform(-3, 3, size=1 << len(in2))
        st.set_basis(0)
        st.apply_schedule([gates.h(k) for k in range(n)])
        with Function(ctx, len(in1), 0, theta=phi) as p1, Function(ctx, len(in2), len(out2), f=f, theta=theta) as p2:
            st.apply_function(p1, in1)
            st.apply_function(p2, in2, out2)
        W = 1 << 12
        top = (1 << n) - W
        for off in sorted({min(o, top) for o in (0, (1 << 31) - W // 2, (1 << 31) + (5 << 12), (3 << 30) + W, top)}):
            idx = np.arange(off, off + W, dtype=np.uint64)
            x2 = fr.register_value(idx, n, in2)
            x1 = fr.register_value(idx ^ fr.scatter(f[x2], n, out2), n, in1)
            want = 2.0 ** (-n / 2) * np.exp(1j * (theta[x2] + phi[x1]))
            got = st.download(offset=off, length=W)
            err = float(np.max(np.abs(got.astype(C128) - want)))
            assert err <= 1e-6, (n, path, off, err)
    pair.release()


# ---- errors and side conditions ------------------------------------------------------------------------------------

def test_function_new_errors(ctx):
    f2 = np.arange(4, dtype=np.uint64) % 2
    cases = [
        (dict(n_in=0, n_out=1, f=[]), INVALID_ARG, "n_in must be at least 1"),
        (dict(n_in=27, n_out=1), UNSUPPORTED, "at most 26 input qubits"),
        (dict(n_in=2, n_out=33, f=f2), UNSUPPORTED, "at most 32 output qubits"),
        (dict(n_in=2, n_out=1), INVALID_ARG, "NULL f"),
        (dict(n_in=2, n_out=0), INVALID_ARG, "nothing to apply"),
        (dict(n_in=2, n_out=1, f=[0, 1, 2, 1]), INVALID_ARG, "f[2] = 2 does not fit in 1 output bits"),
        (dict(n_in=2, n_out=0, theta=[0.0, np.nan, np.inf, 1.0]), INVALID_ARG, "theta[1] is not finite"),
        (dict(n_in=2, n_out=1, f=f2, theta=[0.0, 1.0, -np.inf, 1.0]), INVALID_ARG, "theta[2] is not finite"),
    ]
    for kw, code, msg in cases:
        with pytest.raises(CircuitError) as e:
            Function(ctx, **kw)
        assert e.value.status == code and msg in str(e.value) and str(e.value).startswith("function_new:"), kw
    with pytest.raises(ValueError):
        Function(ctx, 3, 1, f=[0, 1])


def test_refusals_leave_state_and_pending_collapse(ctx):
    n = 14
    psi0 = circuits.random_state(n, 14, C128)
    rng = np.random.default_rng(14)
    in_q, out_q = [3, 11, 0, 7], [13, 5]
    f = rng.integers(0, 4, size=16, dtype=np.uint64)
    theta = rng.uniform(-3, 3, size=16)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b, Function(ctx, 4, 2, f=f, theta=theta) as fn, \
            Context(0) as other_ctx:
        a.upload(psi0)
        b.upload(psi0)
        m, p = a.measure([0, 6], 0.37)
        assert p > 0
        L = _lib.lib()
        ia = np.ascontiguousarray(np.asarray(in_q, dtype=np.uint64))
        oa = np.ascontiguousarray(np.asarray(out_q, dtype=np.uint64))
        bad = [
            (lambda: L.qipb200_state_apply_function(a._h, fn.handle, None, oa.ctypes.data), INVALID_ARG, "NULL qubit"),
            (lambda: L.qipb200_state_apply_function(a._h, fn.handle, ia.ctypes.data, None), INVALID_ARG, "NULL qubit"),
            (lambda: L.qipb200_state_apply_function(a._h, None, ia.ctypes.data, oa.ctypes.data), INVALID_ARG, "NULL"),
        ]
        for call, code, msg in bad:
            assert call() == code
            assert msg in L.qipb200_last_error(ctx.handle).decode()
        for iq, oq, code, msg in (([3, 11, 0, n], out_q, BAD_INDEX, "out of range"),
                                  ([3, 11, 3, 7], out_q, BAD_INDEX, "qubit 3 repeated"),
                                  (in_q, [13, 0], BAD_INDEX, "qubit 0 repeated")):
            with pytest.raises(CircuitError) as e:
                a.apply_function(fn, iq, oq)
            assert e.value.status == code and msg in str(e.value) and str(e.value).startswith("apply_function:")
        with Function(other_ctx, 4, 2, f=f) as foreign:
            with pytest.raises(CircuitError) as e:
                a.apply_function(foreign, in_q, out_q)
            assert e.value.status == INVALID_ARG and "another context" in str(e.value)
        with pytest.raises(ValueError):
            a.apply_function(fn, in_q, out_q[:1])
        # the collapse is still pending: one kernel for it, one for the function
        l0 = ctx.kernel_launches()
        a.apply_function(fn, in_q, out_q)
        assert ctx.kernel_launches() - l0 == 2
        b.collapse([0, 6], m, p)
        collapsed = b.download()
        l0 = ctx.kernel_launches()
        b.apply_function(fn, in_q, out_q)
        assert ctx.kernel_launches() - l0 == 1
        got, want = a.download(), b.download()
    assert bits_equal(got, want)
    assert bits_equal(got, fr.apply(collapsed, n, in_q, out_q, f, theta))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, Function(ctx, 2, 1, f=[0, 1, 1, 0]) as fn:
        with pytest.raises(CircuitError) as e:
            st.apply_function(fn, [0, 1], [2])
        assert e.value.status == UNSUPPORTED


def test_free_straight_after_apply(ctx):
    n = 16
    psi0 = circuits.random_state(n, 16, C64)
    rng = np.random.default_rng(16)
    want = psi0
    with State(n, C64, ctx) as st:
        st.upload(psi0)
        for k in range(8):
            in_q, out_q = registers(n, rng, FUNCTION_PAIR if k % 2 else FUNCTION_TILE, C64)
            f = rng.integers(0, 1 << len(out_q), size=1 << len(in_q), dtype=np.uint64)
            theta = rng.uniform(-3, 3, size=1 << len(in_q))
            fn = Function(ctx, len(in_q), len(out_q), f=f, theta=theta)
            st.apply_function(fn, in_q, out_q)
            fn.free()  # stream-ordered: the kernel queued before still reads the tables
            want = fr.apply(want, n, in_q, out_q, f, theta)
        assert bits_equal(st.download(), want)


def test_large_table_is_freed(ctx):
    import torch
    torch.cuda.init()
    n_in = 24
    rng = np.random.default_rng(24)
    f = rng.integers(0, 1 << 16, size=1 << n_in, dtype=np.uint64)
    theta = rng.uniform(-3, 3, size=1 << n_in)
    table = (4 + 16) << n_in  # 320 MiB
    with State(10, C128, ctx) as st:
        ctx.release_pool()
        st.sync()
        free0 = torch.cuda.mem_get_info(0)[0]
        fn = Function(ctx, n_in, 16, f=f, theta=theta)
        free1 = torch.cuda.mem_get_info(0)[0]
        fn.free()
        st.sync()
        ctx.release_pool()
        free2 = torch.cuda.mem_get_info(0)[0]
    assert free0 - free1 >= table - (16 << 20), (free0, free1)
    assert free2 >= free0 - (64 << 20), (free0, free2)


_ROTATE_WORKER = r"""
import numpy as np
import function_ref as fr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, Function, State

n = 18
rng = np.random.default_rng(18)
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
cases = [([0, 17, 4, 9, 12], [16, 15, 2]), ([17, 16, 15, 14, 13, 12], list(range(0, 10)))]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for in_q, out_q in cases:
            f = rng.integers(0, 1 << len(out_q), size=1 << len(in_q), dtype=np.uint64)
            theta = rng.uniform(-3, 3, size=1 << len(in_q))
            for st in (a, b):
                st.set_basis(3)
                st.apply_schedule(ops)
            before = b.qubit_map().copy()
            assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
            psi = a.download()
            with Function(ctx, len(in_q), len(out_q), f=f, theta=theta) as fn:
                b.apply_function(fn, in_q, out_q)
            assert np.array_equal(b.qubit_map(), before), "apply_function changed the layout"
            got = b.download()
            want = fr.apply(psi, n, in_q, out_q, f, theta)
            # value for value: the swap-only passes that restore a permuted layout before a download may turn -0 into
            # +0, so psi (restored first) and b (restored after the function) can differ in the sign of zeros
            assert np.array_equal(got, want), int(np.sum(got != want))
print("ROTATE bit-exact ok")
"""


def test_permuted_layout_is_worked_in_place():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout
