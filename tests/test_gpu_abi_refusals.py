"""Refusals of the state entry points, called through the C ABI with ctypes on 12-qubit states.

Every case has exactly one fault.  Each one pins the status and the whole qipb200_last_error text.  After a test's
refusals, no kernel has run, every state downloads bit-identical, and the collapse left pending on `a` is still pending:
every check is made on the host before any device work.  The Python wrappers are bypassed because they refuse some
faults (length mismatches) before the C checks see them."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import function_code_ref as fc
from rustqip_b200 import _lib, circuits
from rustqip_b200.state import Context, Function, State
from test_abi_refusals_cpu import no_terms, term_faults, terms

pytestmark = pytest.mark.gpu
C128, C64 = np.complex128, np.complex64
OK, INVALID_ARG, SIZE_MISMATCH, BAD_INDEX, UNSUPPORTED = 0, 1, 2, 3, 7
N = 12


def L():
    return _lib.lib()


def h(s):
    return None if s is None else s._h


def f64(*v):
    return (C.c_double * max(1, len(v)))(*v)


def u64(v):
    v = list(v)
    return (C.c_uint64 * max(1, len(v)))(*v)


def bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


@pytest.fixture(scope="module")
def fns(ctx):
    other = Context(0)
    src = fc.mix_source(0, True)
    with Function(ctx, 2, 1, f=[0, 1, 1, 0]) as table, \
            Function.from_code(ctx, 2, 0, src, theta=True, n_params=2) as code, \
            Function.from_code(ctx, 2, 1, fc.mix_source(1)) as no_theta, \
            Function(other, 2, 1, f=[0, 1, 1, 0]) as other_table, \
            Function.from_code(other, 2, 0, src, theta=True, n_params=2) as other_code:
        yield SimpleNamespace(table=table, code=code, no_theta=no_theta, other_table=other_table,
                              other_code=other_code)
    other.close()


@pytest.fixture
def w(ctx, fns):
    """States a (a collapse pending), b, c, d; f32 (complex64), big (13 qubits), sh (rank 0 of 2)."""
    psi = {k: circuits.random_state(N, 70 + i, C128) for i, k in enumerate("abcd")}
    with State(N, C128, ctx) as a, State(N, C128, ctx) as b, State(N, C128, ctx) as c, State(N, C128, ctx) as d, \
            State(N, C64, ctx) as f32, State(N + 1, C128, ctx) as big, \
            State(N, C128, ctx, rank=0, world_size=2) as sh:
        for s, k in ((a, "a"), (b, "b"), (c, "c"), (d, "d")):
            s.upload(psi[k])
        f32.upload(psi["b"].astype(C64))
        big.upload(circuits.random_state(N + 1, 75, C128))
        d.upload(psi["a"])
        m, p = d.measure([0, 5], 0.37)
        want_a = d.download()  # the download applies the pending collapse
        d.upload(psi["d"])
        assert a.measure([0, 5], 0.37) == (m, p)
        ns = SimpleNamespace(a=a, b=b, c=c, d=d, f32=f32, big=big, sh=sh, fn=fns, ctx=ctx)
        l0 = ctx.kernel_launches()
        yield ns
        assert ctx.kernel_launches() == l0, "a refused call did device work"
        assert np.array_equal(bits(a.download()), bits(want_a)), "the collapse pending on a was lost"
        for s, k in ((b, "b"), (c, "c"), (d, "d")):
            assert np.array_equal(bits(s.download()), bits(psi[k])), k
        assert np.array_equal(bits(f32.download()), bits(psi["b"].astype(C64)))


def run(w, label, call, status, msg, on_ctx=True):
    """call() refuses with status and leaves msg in the last error of the states' context (of no context when the
    refused argument is the state itself)."""
    L().qipb200_stream_handle(None, None)  # a different message in both slots before every call
    L().qipb200_launch_stats(w.ctx.handle, None)
    st = call()
    err = L().qipb200_last_error(w.ctx.handle if on_ctx else None).decode()
    assert st == status, (label, st, err)
    if status != OK:
        assert err == msg, label


def run_terms(w, call):
    for label, t, status, msg in term_faults(N):
        run(w, label, lambda: call(t), status, msg)


def run_states(w, who, call, names, count):
    """NULL, other-precision, other-size, sharded and aliased states in each state argument of call(**states)."""
    for i, name in enumerate(names):
        run(w, "NULL " + name, lambda: call(**{name: None}), INVALID_ARG, who + ": NULL state", on_ctx=False)
        for bad in ("f32", "big"):
            run(w, "%s %s" % (bad, name), lambda: call(**{name: getattr(w, bad)}), SIZE_MISMATCH,
                who + ": the states differ in context, precision or size")
        run(w, "sharded " + name, lambda: call(**{name: w.sh}), UNSUPPORTED, who + ": sharded states are not supported")
        for other in names[i + 1:]:
            run(w, "%s is %s" % (other, name), lambda: call(**{other: call.defaults[name]}), INVALID_ARG,
                "%s: the %s states must differ" % (who, "two" if count == 2 else "three"))


def index_faults():
    return [("NULL qubits", dict(null=True), INVALID_ARG, "measurement: bad index list"),
            ("k 0", dict(k=0), INVALID_ARG, "measurement: bad index list"),
            ("k > n", dict(qubits=range(N + 1)), INVALID_ARG, "measurement: bad index list"),
            ("qubit out of range", dict(qubits=(0, N)), BAD_INDEX, "measurement: qubit index out of range"),
            ("repeated qubit", dict(qubits=(3, 3)), BAD_INDEX, "measurement: repeated qubit index")]


# ---- one state -------------------------------------------------------------------------------------------------------

def test_expect_paulis(w):
    def call(s=w.a, t=None, out=True):
        buf = np.zeros(8)
        return L().qipb200_state_expect_paulis(h(s), *(t or terms()), buf.ctypes.data if out else None)

    who = "expect_paulis"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, who + ": NULL state", on_ctx=False)
    run_terms(w, lambda t: call(t=t))
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "NULL out", lambda: call(out=False), INVALID_ARG, who + ": NULL out")
    run(w, "no terms", lambda: call(t=no_terms(), out=False), OK, None)
    run(w, "bad term before sharded", lambda: call(s=w.sh, t=terms((N,), b"X", (1,))), BAD_INDEX,
        "expect: term 0: qubit 12 out of range for 12 qubits")


def test_transition_paulis(w):
    def call(bra=w.a, ket=w.b, t=None, out=True):
        buf = np.zeros(16)
        return L().qipb200_state_transition_paulis(h(bra), h(ket), *(t or terms()), buf.ctypes.data if out else None)

    who = "transition_paulis"
    for name in ("bra", "ket"):
        run(w, "NULL " + name, lambda: call(**{name: None}), INVALID_ARG, who + ": NULL state", on_ctx=False)
        for bad in ("f32", "big"):
            run(w, "%s %s" % (bad, name), lambda: call(**{name: getattr(w, bad)}), SIZE_MISMATCH,
                who + ": the states differ in context, precision or size")
        run(w, "sharded " + name, lambda: call(**{name: w.sh}), UNSUPPORTED, who + ": sharded states are not supported")
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL out", lambda: call(out=False), INVALID_ARG, who + ": NULL out")
    run(w, "no terms", lambda: call(t=no_terms(), out=False), OK, None)
    run(w, "no terms, bra is ket", lambda: call(ket=w.a, t=no_terms(), out=False), OK, None)


def test_reduced_density(w):
    def call(s=w.a, qubits=(1, 4), k=None, null=False, out=True):
        q = list(qubits)
        buf = np.zeros(2 << (2 * len(q)) if len(q) <= 10 else 2)
        return L().qipb200_state_reduced_density(h(s), None if null else u64(q), len(q) if k is None else k,
                                                 buf.ctypes.data if out else None)

    who = "reduced_density"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, who + ": NULL state", on_ctx=False)
    for label, kw, status, msg in index_faults():
        run(w, label, lambda: call(**kw), status, msg)
    run(w, "NULL out", lambda: call(out=False), INVALID_ARG, who + ": NULL out")
    run(w, "11 qubits", lambda: call(qubits=range(11)), UNSUPPORTED,
        who + ": at most 10 kept qubits (the output at 10 is already 16 MiB)")
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "qubits before out", lambda: call(qubits=(3, 3), out=False), BAD_INDEX, "measurement: repeated qubit index")


def test_purity(w):
    def call(s=w.a, qubits=(1, 4), k=None, null=False, out=True):
        q = list(qubits)
        buf = np.zeros(2)
        return L().qipb200_state_purity(h(s), None if null else u64(q), len(q) if k is None else k,
                                        buf.ctypes.data if out else None)

    who = "purity"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, who + ": NULL state", on_ctx=False)
    run(w, "NULL out2", lambda: call(out=False), INVALID_ARG, who + ": NULL out2")
    for label, kw, status, msg in index_faults():
        run(w, label, lambda: call(**kw), status, msg)
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "out2 before qubits", lambda: call(qubits=(3, 3), out=False), INVALID_ARG, who + ": NULL out2")


def test_apply_pauli_rotations(w):
    def call(s=w.a, t=None, angles=(0.3,), null=False):
        return L().qipb200_state_apply_pauli_rotations(h(s), *(t or terms()), None if null else f64(*angles))

    who = "apply_pauli_rotations"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, who + ": NULL state", on_ctx=False)
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL angles", lambda: call(null=True), INVALID_ARG, who + ": NULL angles")
    for bad in (np.nan, np.inf, -np.inf):
        run(w, "angle %r" % bad, lambda: call(angles=(bad,)), INVALID_ARG, who + ": angle 0 is not finite")
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "no terms", lambda: call(t=no_terms(), null=True), OK, None)


def test_apply_function(w):
    def call(s=w.a, fn=w.fn.table, in_q=(0, 1), out_q=(2,), null_in=False, null_out=False):
        return L().qipb200_state_apply_function(h(s), None if fn is None else fn.handle,
                                                None if null_in else u64(in_q), None if null_out else u64(out_q))

    who = "apply_function"
    msg = who + ": NULL state or function"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, msg, on_ctx=False)
    run(w, "NULL function", lambda: call(fn=None), INVALID_ARG, msg)
    run(w, "NULL in", lambda: call(null_in=True), INVALID_ARG, who + ": NULL qubit array")
    run(w, "NULL out", lambda: call(null_out=True), INVALID_ARG, who + ": NULL qubit array")
    run(w, "in qubit out of range", lambda: call(in_q=(0, N)), BAD_INDEX, who + ": qubit 12 out of range for 12 qubits")
    run(w, "out qubit repeated", lambda: call(out_q=(1,)), BAD_INDEX, who + ": qubit 1 repeated")
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "another context", lambda: call(fn=w.fn.other_table), INVALID_ARG,
        who + ": the function was made on another context")


def test_expect_function(w):
    def call(s=w.a, fn=w.fn.code, in_q=(0, 1), null_in=False, out=True):
        v = C.c_double()
        return L().qipb200_state_expect_function(h(s), None if fn is None else fn.handle,
                                                 None if null_in else u64(in_q), C.byref(v) if out else None)

    who = "expect_function"
    msg = who + ": NULL state, function or out"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, msg, on_ctx=False)
    run(w, "NULL function", lambda: call(fn=None), INVALID_ARG, msg)
    run(w, "NULL out", lambda: call(out=False), INVALID_ARG, msg)
    run(w, "table", lambda: call(fn=w.fn.table), UNSUPPORTED,
        who + ": a table function keeps cos theta and sin theta, not theta: make it from code")
    run(w, "no theta", lambda: call(fn=w.fn.no_theta), UNSUPPORTED,
        who + ": the function has no theta (QIPB200_FN_CODE_THETA)")
    run(w, "NULL in", lambda: call(null_in=True), INVALID_ARG, who + ": NULL qubit array")
    run(w, "in qubit out of range", lambda: call(in_q=(N, 0)), BAD_INDEX, who + ": qubit 12 out of range for 12 qubits")
    run(w, "in qubit repeated", lambda: call(in_q=(1, 1)), BAD_INDEX, who + ": qubit 1 repeated")
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED, who + ": sharded states are not supported")
    run(w, "another context", lambda: call(fn=w.fn.other_code), INVALID_ARG,
        who + ": the function was made on another context")


def test_measure_probs(w):
    def call(s=w.a, qubits=(1, 4), k=None, null=False, out=True):
        q = list(qubits)
        buf = np.zeros(2 << len(q))
        return L().qipb200_state_measure_probs(h(s), None if null else u64(q), len(q) if k is None else k,
                                               buf.ctypes.data if out else None)

    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, "measure_probs: NULL argument", on_ctx=False)
    run(w, "NULL out", lambda: call(out=False), INVALID_ARG, "measure_probs: NULL argument")
    for label, kw, status, msg in index_faults():
        run(w, label, lambda: call(**kw), status, msg)


def test_sample(w):
    def call(s=w.a, qubits=(1, 4), k=None, null=False, draws=(0.25, 0.5), null_draws=False, null_out=False):
        q = list(qubits)
        out = (C.c_uint64 * max(1, len(draws)))()
        return L().qipb200_state_sample(h(s), None if null else u64(q), len(q) if k is None else k,
                                        None if null_draws else f64(*draws), len(draws), None if null_out else out)

    who = "sample"
    run(w, "NULL state", lambda: call(s=None), INVALID_ARG, who + ": NULL state", on_ctx=False)
    for label, kw, status, msg in index_faults():
        run(w, label, lambda: call(**kw), status, msg)
    run(w, "sharded", lambda: call(s=w.sh), UNSUPPORTED,
        who + ": sharded states are not supported (use soft_measure per draw)")
    run(w, "no draws", lambda: call(draws=(), null_draws=True, null_out=True), OK, None)
    run(w, "NULL draws", lambda: call(null_draws=True), INVALID_ARG, who + ": NULL draws or measured")
    run(w, "NULL measured", lambda: call(null_out=True), INVALID_ARG, who + ": NULL draws or measured")


# ---- two and three states --------------------------------------------------------------------------------------------

def with_defaults(f, **defaults):
    def call(**kw):
        return f(**{**defaults, **kw})
    call.defaults = defaults
    return call


def test_apply_pauli_sum(w):
    def f(dst, src, t=None, coeffs=(0.5,), null=False):
        return L().qipb200_state_apply_pauli_sum(h(dst), h(src), *(t or terms()), None if null else f64(*coeffs))

    who = "apply_pauli_sum"
    call = with_defaults(f, dst=w.b, src=w.a)
    run_states(w, who, call, ("dst", "src"), 2)
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL coefficients", lambda: call(null=True), INVALID_ARG, who + ": NULL coefficients")
    for bad in (np.nan, np.inf):
        run(w, "coefficient %r" % bad, lambda: call(coeffs=(bad,)), INVALID_ARG, who + ": coefficient 0 is not finite")


def test_pauli_energy_gradient(w):
    def f(state, work, ansatz=None, angles=(0.3,), null_angles=False, ham=None, coeffs=(0.5,), null_coeffs=False,
          energy=True, grad=True):
        e, g = C.c_double(), f64(0.0, 0.0)
        return L().qipb200_state_pauli_energy_gradient(
            h(state), h(work), *(ansatz or terms()), None if null_angles else f64(*angles), *(ham or terms()),
            None if null_coeffs else f64(*coeffs), C.byref(e) if energy else None, g if grad else None)

    who = "pauli_energy_gradient"
    call = with_defaults(f, state=w.a, work=w.b)
    run_states(w, who, call, ("state", "work"), 2)
    for label, t, status, msg in term_faults(N):
        run(w, "ansatz " + label, lambda: call(ansatz=t), status, msg)
        run(w, "hamiltonian " + label, lambda: call(ham=t), status, msg)
    run(w, "NULL angles", lambda: call(null_angles=True), INVALID_ARG, who + ": NULL angles")
    run(w, "angle nan", lambda: call(angles=(np.nan,)), INVALID_ARG, who + ": angle 0 is not finite")
    run(w, "NULL coefficients", lambda: call(null_coeffs=True), INVALID_ARG, who + ": NULL coefficients")
    run(w, "coefficient inf", lambda: call(coeffs=(np.inf,)), INVALID_ARG, who + ": coefficient 0 is not finite")
    run(w, "NULL energy", lambda: call(energy=False), INVALID_ARG, who + ": NULL energy")
    run(w, "NULL grad", lambda: call(grad=False), INVALID_ARG, who + ": NULL grad")


def test_pauli_geometric_tensor(w):
    def f(state, work_a, work_b, t=None, angles=(0.3,), null=False, qgt=True):
        T = (t or terms())[3]
        g, e = np.zeros(max(2, 2 * T * T)), np.zeros(max(1, T))
        return L().qipb200_state_pauli_geometric_tensor(h(state), h(work_a), h(work_b), *(t or terms()),
                                                        None if null else f64(*angles),
                                                        g.ctypes.data if qgt else None, e.ctypes.data)

    who = "pauli_geometric_tensor"
    call = with_defaults(f, state=w.a, work_a=w.b, work_b=w.c)
    run_states(w, who, call, ("state", "work_a", "work_b"), 3)
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL angles", lambda: call(null=True), INVALID_ARG, who + ": NULL angles")
    run(w, "angle inf", lambda: call(angles=(np.inf,)), INVALID_ARG, who + ": angle 0 is not finite")
    run(w, "NULL qgt", lambda: call(qgt=False), INVALID_ARG, who + ": NULL qgt")
    run(w, "2049 terms", lambda: call(t=terms([0] * 2049, b"X" * 2049, [1] * 2049), angles=[0.1] * 2049),
        UNSUPPORTED, who + ": 2049 terms, at most 2048")


def test_evolve_pauli_sum(w):
    def f(state, work_a, work_b, t=None, coeffs=(0.5,), null=False, time=1.0, tol=1e-9, degree=True, tail=True):
        d, tl = C.c_uint32(), C.c_double()
        return L().qipb200_state_evolve_pauli_sum(h(state), h(work_a), h(work_b), *(t or terms()),
                                                  None if null else f64(*coeffs), time, tol,
                                                  C.byref(d) if degree else None, C.byref(tl) if tail else None)

    who = "evolve_pauli_sum"
    call = with_defaults(f, state=w.a, work_a=w.b, work_b=w.c)
    run_states(w, who, call, ("state", "work_a", "work_b"), 3)
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL coefficients", lambda: call(null=True), INVALID_ARG, who + ": NULL coefficients")
    run(w, "coefficient nan", lambda: call(coeffs=(np.nan,)), INVALID_ARG, who + ": coefficient 0 is not finite")
    run(w, "time inf", lambda: call(time=np.inf), INVALID_ARG, who + ": time is not finite")
    for tol in (0.0, 1.0, np.nan):
        run(w, "tol %r" % tol, lambda: call(tol=tol), INVALID_ARG, who + ": tol must be in (0, 1)")
    run(w, "NULL degree", lambda: call(degree=False), INVALID_ARG, who + ": NULL degree or tail")
    run(w, "NULL tail", lambda: call(tail=False), INVALID_ARG, who + ": NULL degree or tail")


def test_lanczos_pauli_sum(w):
    def f(state, work_a, work_b, t=None, coeffs=(0.5,), null=False, max_steps=8, tol=1e-6, flags=0, nulls=()):
        steps, conv = C.c_uint32(), C.c_uint32()
        alpha, beta, out3 = np.zeros(8), np.zeros(9), np.zeros(3)
        outs = dict(steps=C.byref(steps), converged=C.byref(conv), out3=out3.ctypes.data)
        for k in nulls:
            outs[k] = None
        return L().qipb200_state_lanczos_pauli_sum(
            h(state), h(work_a), h(work_b), *(t or terms()), None if null else f64(*coeffs), max_steps, tol, flags,
            outs["steps"], outs["converged"], alpha.ctypes.data, beta.ctypes.data, outs["out3"])

    who = "lanczos_pauli_sum"
    call = with_defaults(f, state=w.a, work_a=w.b, work_b=w.c)
    run_states(w, who, call, ("state", "work_a", "work_b"), 3)
    run_terms(w, lambda t: call(t=t))
    run(w, "NULL coefficients", lambda: call(null=True), INVALID_ARG, who + ": NULL coefficients")
    run(w, "coefficient inf", lambda: call(coeffs=(-np.inf,)), INVALID_ARG, who + ": coefficient 0 is not finite")
    for m in (0, 4097):
        run(w, "max_steps %d" % m, lambda: call(max_steps=m), INVALID_ARG, who + ": max_steps must be in 1..4096")
    for tol in (0.0, 1.0, np.nan):
        run(w, "tol %r" % tol, lambda: call(tol=tol), INVALID_ARG, who + ": tol must be in (0, 1)")
    run(w, "flags 2", lambda: call(flags=2), INVALID_ARG, who + ": unknown flags")
    for k in ("steps", "converged", "out3"):
        run(w, "NULL " + k, lambda: call(nulls=(k,)), INVALID_ARG, who + ": NULL steps, converged or out3")
