"""Refusals of the host-only entry points, called through the C ABI with ctypes (no GPU).

Every case has exactly one fault.  Each one pins the status and the whole qipb200_last_error text, so that the checks
the entries share stay the same checks with the same words wherever they are made."""
import ctypes as C

import numpy as np
import pytest

from rustqip_b200 import _lib

OK, INVALID_ARG, BAD_INDEX, UNSUPPORTED = 0, 1, 3, 7
N = 4  # qubits of every plan below


def L():
    return _lib.lib()


def terms(qubits=(0, 2), letters=b"XZ", lens=(2,), n_terms=None):
    """(qubits, letters, term lengths, n_terms) C arrays of a Pauli term list."""
    return [(C.c_uint64 * max(1, len(qubits)))(*qubits), C.create_string_buffer(bytes(letters), max(1, len(letters))),
            (C.c_uint32 * max(1, len(lens)))(*lens), len(lens) if n_terms is None else n_terms]


def term_faults(n):
    """(label, term arrays, status, message) of the faults parse_pauli_terms refuses in an n-qubit term list."""
    cases = []
    for i, name in enumerate(("qubits", "paulis", "term_len")):
        t = terms()
        t[i] = None
        cases.append(("NULL " + name, t, INVALID_ARG, "expect: NULL qubits, paulis or term_len"))
    cases += [
        ("bad letter", terms((0, 1), b"ZW", (1, 1)), INVALID_ARG,
         "expect: term 1: Pauli letter 0x57 is not 'X', 'Y' or 'Z'"),
        ("qubit out of range", terms((n,), b"X", (1,)), BAD_INDEX,
         "expect: term 0: qubit %d out of range for %d qubits" % (n, n)),
        ("repeated qubit", terms((0, 2, 2), b"XYZ", (3,)), BAD_INDEX, "expect: term 0: qubit 2 repeated"),
    ]
    return cases


def no_terms():
    return [None, None, None, 0]


def last_error():
    return L().qipb200_last_error(None).decode()


def check(label, st, status, msg):
    assert st == status, (label, st, last_error())
    if status != OK:
        assert last_error() == msg, label


def run(label, call, status, msg):
    L().qipb200_stream_handle(None, None)  # a different message in the slot before every call
    check(label, call(), status, msg)


def plan_args_faults(who, outs):
    """The plan preconditions: a NULL output, a bad precision, n_qubits outside 1..40."""
    msg = "%s: NULL %s, bad precision or n_qubits not in 1..40" % (who, outs)
    return [("precision 7", dict(prec=7), INVALID_ARG, msg), ("n_qubits 0", dict(n=0), INVALID_ARG, msg),
            ("n_qubits 41", dict(n=41), INVALID_ARG, msg)]


# ---- the plans of one term list and a uint32 result ----------------------------------------------------------------

U32_PLANS = {  # entry: (result length, result name)
    "expect_plan": (1, "sweeps"),
    "transition_plan": (2, "out2"),
    "pauli_rotation_plan": (1, "sweeps"),
    "pauli_sum_plan": (1, "sweeps"),
    "pauli_geometric_tensor_plan": (3, "out3"),
    "pauli_lanczos_plan": (4, "out4"),
}


def u32_plan(who, prec=1, n=N, t=None, out=True):
    v = (C.c_uint32 * U32_PLANS[who][0])()
    return getattr(L(), "qipb200_" + who)(prec, n, *(t or terms()), v if out else None)


@pytest.mark.parametrize("who", sorted(U32_PLANS))
def test_u32_plan_refusals(who):
    run("good", lambda: u32_plan(who), OK, None)
    run("no terms", lambda: u32_plan(who, t=no_terms()), OK, None)
    for label, kw, status, msg in plan_args_faults(who, U32_PLANS[who][1]):
        run(label, lambda: u32_plan(who, **kw), status, msg)
    run("NULL out", lambda: u32_plan(who, out=False), INVALID_ARG,
        "%s: NULL %s, bad precision or n_qubits not in 1..40" % (who, U32_PLANS[who][1]))
    for label, t, status, msg in term_faults(N):
        run(label, lambda: u32_plan(who, t=t), status, msg)


def test_geometric_tensor_plan_term_limit():
    t = terms([0] * 2049, b"X" * 2049, [1] * 2049)
    run("2049 terms", lambda: u32_plan("pauli_geometric_tensor_plan", t=t), UNSUPPORTED,
        "pauli_geometric_tensor_plan: 2049 terms, at most 2048")
    t = terms([0] * 2048, b"X" * 2048, [1] * 2048)
    run("2048 terms", lambda: u32_plan("pauli_geometric_tensor_plan", t=t), OK, None)


# ---- the other plans -------------------------------------------------------------------------------------------------

def gradient_plan(prec=1, n=N, ansatz=None, ham=None, out=True):
    v = (C.c_uint32 * 3)()
    return L().qipb200_pauli_gradient_plan(prec, n, *(ansatz or terms()), *(ham or terms()), v if out else None)


def test_gradient_plan_refusals():
    run("good", gradient_plan, OK, None)
    run("no terms", lambda: gradient_plan(ansatz=no_terms(), ham=no_terms()), OK, None)
    for label, kw, status, msg in plan_args_faults("pauli_gradient_plan", "out3"):
        run(label, lambda: gradient_plan(**kw), status, msg)
    run("NULL out3", lambda: gradient_plan(out=False), INVALID_ARG,
        "pauli_gradient_plan: NULL out3, bad precision or n_qubits not in 1..40")
    for label, t, status, msg in term_faults(N):
        run("ansatz " + label, lambda: gradient_plan(ansatz=t), status, msg)
        run("hamiltonian " + label, lambda: gradient_plan(ham=t), status, msg)


def evolution_plan(prec=1, n=N, t=None, coeffs=(0.5,), time=1.0, tol=1e-9, out3=True, tail=True):
    c = np.ascontiguousarray(coeffs, dtype=np.float64)
    v, tl = (C.c_uint32 * 3)(), C.c_double()
    return L().qipb200_pauli_evolution_plan(prec, n, *(t or terms()), c.ctypes.data if coeffs is not None else None,
                                            time, tol, v if out3 else None, C.byref(tl) if tail else None, None, 0)


def test_evolution_plan_refusals():
    who = "pauli_evolution_plan"
    run("good", evolution_plan, OK, None)
    run("no terms", lambda: evolution_plan(t=no_terms(), coeffs=None), OK, None)
    for label, kw, status, msg in plan_args_faults(who, "out3 or tail"):
        run(label, lambda: evolution_plan(**kw), status, msg)
    msg = who + ": NULL out3 or tail, bad precision or n_qubits not in 1..40"
    run("NULL out3", lambda: evolution_plan(out3=False), INVALID_ARG, msg)
    run("NULL tail", lambda: evolution_plan(tail=False), INVALID_ARG, msg)
    for label, t, status, msg in term_faults(N):
        run(label, lambda: evolution_plan(t=t), status, msg)
    run("NULL coeffs", lambda: evolution_plan(coeffs=None), INVALID_ARG, who + ": NULL coefficients")
    for bad in (np.nan, np.inf):
        run("coefficient %r" % bad, lambda: evolution_plan(coeffs=(bad,)), INVALID_ARG,
            who + ": coefficient 0 is not finite")
        run("time %r" % bad, lambda: evolution_plan(time=bad), INVALID_ARG, who + ": time is not finite")
    for tol in (0.0, 1.0, np.nan):
        run("tol %r" % tol, lambda: evolution_plan(tol=tol), INVALID_ARG, who + ": tol must be in (0, 1)")


def purity_plan(prec=1, n=N, qubits=(0, 2), k=None, null=False, out=True):
    q = (C.c_uint64 * max(1, len(qubits)))(*qubits)
    v = (C.c_uint32 * 4)()
    return L().qipb200_purity_plan(prec, n, None if null else q, len(qubits) if k is None else k, v if out else None)


def test_purity_plan_refusals():
    run("good", purity_plan, OK, None)
    for label, kw, status, msg in plan_args_faults("purity_plan", "out4"):
        run(label, lambda: purity_plan(**kw), status, msg)
    run("NULL out4", lambda: purity_plan(out=False), INVALID_ARG,
        "purity_plan: NULL out4, bad precision or n_qubits not in 1..40")
    for label, kw in (("NULL qubits", dict(null=True)), ("k 0", dict(k=0)), ("k > n", dict(qubits=range(5)))):
        run(label, lambda: purity_plan(**kw), INVALID_ARG, "purity_plan: bad qubit list")
    run("qubit out of range", lambda: purity_plan(qubits=(0, 4)), BAD_INDEX, "purity_plan: qubit index out of range")
    run("repeated qubit", lambda: purity_plan(qubits=(2, 2)), BAD_INDEX, "purity_plan: repeated qubit index")


def function_plan(prec=1, n=N, in_q=(0, 1), out_q=(2,), n_in=None, n_out=None, null_in=False, null_out=False,
                  out=True):
    ia = (C.c_uint64 * max(1, len(in_q)))(*in_q)
    oa = (C.c_uint64 * max(1, len(out_q)))(*out_q)
    v = (C.c_uint32 * 2)()
    return L().qipb200_function_plan(prec, n, None if null_in else ia, len(in_q) if n_in is None else n_in,
                                     None if null_out else oa, len(out_q) if n_out is None else n_out,
                                     v if out else None)


def test_function_plan_refusals():
    who = "function_plan"
    run("good", function_plan, OK, None)
    run("no out register", lambda: function_plan(out_q=(), null_out=True), OK, None)
    for label, kw, status, msg in plan_args_faults(who, "out2"):
        run(label, lambda: function_plan(**kw), status, msg)
    run("NULL out2", lambda: function_plan(out=False), INVALID_ARG,
        who + ": NULL out2, bad precision or n_qubits not in 1..40")
    run("n_in 0", lambda: function_plan(in_q=()), INVALID_ARG, who + ": n_in must be at least 1")
    run("n_in 27", lambda: function_plan(n=40, in_q=range(27), out_q=()), UNSUPPORTED,
        who + ": at most 26 input qubits (the table of 2^n_in entries would exceed 1.25 GiB)")
    run("n_out 33", lambda: function_plan(n=40, in_q=(0,), out_q=range(1, 34)), UNSUPPORTED,
        who + ": at most 32 output qubits")
    run("NULL in", lambda: function_plan(null_in=True), INVALID_ARG, who + ": NULL qubit array")
    run("NULL out", lambda: function_plan(null_out=True), INVALID_ARG, who + ": NULL qubit array")
    run("in qubit out of range", lambda: function_plan(in_q=(0, 4)), BAD_INDEX,
        who + ": qubit 4 out of range for 4 qubits")
    run("out qubit repeated", lambda: function_plan(out_q=(1,)), BAD_INDEX, who + ": qubit 1 repeated")


def lanczos_ritz(alpha=(1.0, 2.0), beta=(1.0, 0.5, 0.25), m=None, null=()):
    a = np.ascontiguousarray(alpha, dtype=np.float64)
    b = np.ascontiguousarray(beta, dtype=np.float64)
    theta, est, y = C.c_double(), C.c_double(), np.zeros(4)
    args = dict(alpha=a.ctypes.data, beta=b.ctypes.data, theta=C.byref(theta), estimate=C.byref(est))
    for k in null:
        args[k] = None
    return L().qipb200_lanczos_ritz(args["alpha"], args["beta"], len(alpha) if m is None else m, args["theta"],
                                    y.ctypes.data, args["estimate"])


def test_lanczos_ritz_refusals():
    who = "lanczos_ritz"
    run("good", lanczos_ritz, OK, None)
    msg = who + ": NULL alpha, beta, theta or estimate, or m == 0"
    for k in ("alpha", "beta", "theta", "estimate"):
        run("NULL " + k, lambda: lanczos_ritz(null=(k,)), INVALID_ARG, msg)
    run("m 0", lambda: lanczos_ritz(m=0), INVALID_ARG, msg)
    for bad in (np.nan, np.inf):
        run("alpha %r" % bad, lambda: lanczos_ritz(alpha=(1.0, bad)), INVALID_ARG, who + ": alpha 1 is not finite")
        run("beta %r" % bad, lambda: lanczos_ritz(beta=(1.0, 0.5, bad)), INVALID_ARG, who + ": beta 2 is not finite")
