"""Functions given as CUDA source on the device (Function.from_code, qipb200_function_new_code).

The apply is compared bit for bit with the numpy emulator fed with the function's own device table
(Function.tabulate), and with the table handle of the same f; the tabulated f and (cos, sin) with host evaluations;
whole-register functions at N = 30 with Grover's closed form and with Pauli rotations and expectation values of the
same cost; closed forms past 2^31 and 2^32 amplitudes; the expectation value against numpy within its documented
bound."""
import math

import numpy as np
import pytest

import function_code_ref as fc
import function_ref as fr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import FUNCTION_PAIR, FUNCTION_TILE, Function, State, function_plan

pytestmark = pytest.mark.gpu
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7


def bits_equal(a, b):
    return np.array_equal(np.atleast_1d(a).view(np.uint8), np.atleast_1d(b).view(np.uint8))


def registers(n, rng, path, dtype):
    """Random unsorted registers (in register of up to 12 qubits) that take `path` on an n-qubit state."""
    tmax = 11 if dtype == C128 else 12
    for _ in range(1000):
        perm = [int(q) for q in rng.permutation(n)]
        if path == FUNCTION_PAIR:
            out_q = [q for q in perm if q < n - 4][:tmax - 3 + int(rng.integers(0, 3))]
            rest = [q for q in perm if q not in out_q]
            in_q = rest[:int(rng.integers(1, min(12, len(rest)) + 1))]
        else:
            n_out = int(rng.integers(1, min(8, n - 1) + 1))
            out_q = perm[:n_out]
            in_q = perm[n_out:n_out + int(rng.integers(1, min(12, n - n_out) + 1))]
        if function_plan(n, dtype, in_q, out_q)[0] == path:
            return in_q, out_q
    raise AssertionError("no registers for path %d at n = %d" % (path, n))


def ulps(got, want):
    return np.abs(got - want) / np.spacing(np.maximum(np.abs(got), np.abs(want)))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_tabulated_emulation(ctx, dtype):
    seen = set()
    for n in (6, 8, 11, 13, 14, 16, 18, 20):
        rng = np.random.default_rng(700 + n)
        psi0 = circuits.random_state(n, 70 + n, dtype)
        psi0[rng.integers(0, 1 << n, size=3)] = complex(-0.0, -0.0)
        paths = (FUNCTION_TILE, FUNCTION_PAIR) if n >= 14 else (FUNCTION_TILE,)
        params = rng.uniform(-2, 2, size=2)
        with State(n, dtype, ctx) as st:
            for path in paths:
                in_q, out_q = registers(n, rng, path, dtype)
                n_in, n_out = len(in_q), len(out_q)
                seen.add(path)
                for theta in (False, True):
                    with Function.from_code(ctx, n_in, n_out, fc.mix_source(n_out, theta), theta=theta,
                                            n_params=2 if theta else 0) as fn:
                        if theta:
                            fn.set_params(params)
                        f, cs = fn.tabulate()
                        st.upload(psi0)
                        st.apply_function(fn, in_q, out_q)
                        want = fc.apply_cs(psi0, n, in_q, out_q, f, cs if theta else None)
                        assert bits_equal(st.download(), want), (n, path, theta, in_q, out_q)
            # phase only over the whole register (tile path)
            with Function.from_code(ctx, n, 0, fc.mix_source(0, True), theta=True, n_params=2) as fn:
                fn.set_params(params)
                _, cs = fn.tabulate()
                in_q = [int(q) for q in rng.permutation(n)]
                st.upload(psi0)
                st.apply_function(fn, in_q)
                assert bits_equal(st.download(), fc.apply_cs(psi0, n, in_q, (), None, cs)), (n, "phase")
    assert seen == {FUNCTION_TILE, FUNCTION_PAIR}


@pytest.mark.parametrize("dtype", [C128, C64])
def test_permutation_code_equals_its_table(ctx, dtype):
    n = 20
    prep = circuits.random_circuit(n, 2, 0x5EED0020, "H,T,CNOT")
    for path in (FUNCTION_TILE, FUNCTION_PAIR):
        in_q, out_q = registers(n, np.random.default_rng(20 + path), path, dtype)
        x = np.arange(1 << len(in_q), dtype=np.uint64)
        with Function.from_code(ctx, len(in_q), len(out_q), fc.mix_source(len(out_q))) as code, \
                Function(ctx, len(in_q), len(out_q), f=fc.mix_f(x, len(out_q))) as table, \
                State(n, dtype, ctx) as a, State(n, dtype, ctx) as b:
            for s in (a, b):
                s.set_basis(0)
                s.apply_schedule(prep)
            a.apply_function(code, in_q, out_q)
            b.apply_function(table, in_q, out_q)
            assert a.max_abs_diff(b) == 0.0, path


def test_tabulate_against_host_evaluation(ctx):
    p = [0.37, -1.25]
    for n_in, n_out in ((20, 10), (30, 4)):
        with Function.from_code(ctx, n_in, n_out, fc.mix_source(n_out, True), theta=True, n_params=2) as fn:
            fn.set_params(p)
            for x0, count in ((0, 4096), ((1 << n_in) - 3000, 3000), (123457, 1 << 16)):
                f, cs = fn.tabulate(x0, count)
                x = np.arange(x0, x0 + count, dtype=np.uint64)
                assert np.array_equal(f, fc.mix_f(x, n_out))
                th = fc.mix_theta(x, p)
                assert float(np.max(ulps(cs[:, 0], np.cos(th)))) <= 3 and float(np.max(ulps(cs[:, 1], np.sin(th)))) <= 3
    with Function.from_code(ctx, 6, 3, fc.mix_source(3)) as fn:  # no phase: (1, 0)
        f, cs = fn.tabulate(5, 7)
        assert np.array_equal(f, fc.mix_f(np.arange(5, 12, dtype=np.uint64), 3))
        assert np.array_equal(cs, np.tile([1.0, 0.0], (7, 1)))
    with Function(ctx, 3, 1, f=[0, 1, 1, 0, 1, 0, 0, 1], theta=np.arange(8) * 0.5) as fn:  # a table: its entries
        f, cs = fn.tabulate()
        assert f.tolist() == [0, 1, 1, 0, 1, 0, 0, 1]
        assert np.array_equal(cs[:, 0], np.cos(np.arange(8) * 0.5)) and np.array_equal(cs[:, 1], np.sin(np.arange(8) * 0.5))
        with pytest.raises(CircuitError) as e:
            fn.tabulate(4, 5)
        assert e.value.status == INVALID_ARG and "exceeds 2^n_in" in str(e.value)


# ---- whole registers at N = 30 -------------------------------------------------------------------------------------

GROVER_BITS, GROVER_MARKED_LOG2 = 29, 21
# h is a bijection of 29-bit values (an odd multiplier mod 2^29, then an xorshift), so exactly 2^21 x have h(x) < 2^21
GROVER_H = ("__device__ uint64_t grover_h(uint64_t x) {\n"
            "  x = (x * 0x1F3D5B79ull) & 0x1FFFFFFFull;\n"
            "  return x ^ (x >> 13);\n}\n")
GROVER_ORACLE = GROVER_H + "__device__ uint64_t qip_f(uint64_t x) { return grover_h(x) < (1ull << 21); }\n"
GROVER_ZERO = "__device__ uint64_t qip_f(uint64_t x) { return x == 0; }\n"
GROVER_HIT = GROVER_H + ("__device__ double qip_theta(uint64_t x, const double *p) {\n"
                         "  return grover_h(x) < (1ull << 21) ? 1.0 : 0.0;\n}\n")


def test_grover_full_register_n30(ctx):
    """x = qubits 0..28 (29 > 26 in-qubits), ancilla qubit 29 in |->: the oracle and the reflection about |0> are
    code functions with one out qubit.  After k iterations the success probability, read by expect_function of the
    marked set's indicator, is sin^2((2k + 1) asin sqrt(M / 2^29)) with M = 2^21.  Every op is exact or rounds at the
    f64 unit (H layers), so 1e-9 bounds the difference with room to spare."""
    n, m = 30, GROVER_BITS
    xq = list(range(m))
    hx = [gates.h(q) for q in xq]
    w = math.asin(math.sqrt(2.0 ** (GROVER_MARKED_LOG2 - m)))
    with State(n, C128, ctx) as st, Function.from_code(ctx, m, 1, GROVER_ORACLE) as oracle, \
            Function.from_code(ctx, m, 1, GROVER_ZERO) as zero, \
            Function.from_code(ctx, m, 0, GROVER_HIT, theta=True) as hit:
        st.set_basis(0)
        st.apply_schedule(hx + [gates.x(m), gates.h(m)])
        p0 = st.expect_function(hit, xq)
        assert abs(p0 - math.sin(w) ** 2) <= 1e-12, p0
        for k in range(1, 5):
            st.apply_function(oracle, xq, [m])
            st.apply_schedule(hx)
            st.apply_function(zero, xq, [m])
            st.apply_schedule(hx)
            got = st.expect_function(hit, xq)
            assert abs(got - math.sin((2 * k + 1) * w) ** 2) <= 1e-9, (k, got)
        assert abs(st.norm2() - 1.0) <= 1e-9


def test_ring_maxcut_against_pauli_rotations_n30(ctx):
    """exp(-i gamma C) for the cut count C of the 30-ring: the code phase theta = -gamma C against
    apply_pauli_rotations of the 30 ZZ terms with angle -gamma, exp(i gamma/2 ZZ) per edge, equal up to the global
    phase e^{-i 15 gamma}.  Each side rounds at most a few units of 2^-53 per amplitude (the rotations: 30 updates of
    4 roundings each, the code phase: 4 roundings, plus cos and sin within 2 ulp), so |<a|b> e^{-i 15 gamma} - 1|
    <= 1e-12 and window differences <= 1e-13 on amplitudes of size 2^-15."""
    n, gamma = 30, 0.61
    prep = [gates.h(q) for q in range(n)] + [gates.rz(q, 0.1 * (q + 1)) for q in range(n)] + \
        [gates.cnot(q, q + 1) for q in range(0, n - 1, 3)]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b, \
            Function.from_code(ctx, n, 0, fc.ring_source(n), theta=True, n_params=1) as cut:
        for s in (a, b):
            s.set_basis(0)
            s.apply_schedule(prep)
        # the energies before the phase: expect_function against expect_paulis, both within their bounds
        cut.set_params([1.0])
        e_code = a.expect_function(cut, list(range(n)))
        zz = a.expect_paulis(fc.ring_terms(n))
        e_pauli = float(np.sum((1.0 - zz) / 2.0))
        bound = fc.expect_bound(n, n * a.norm2()) + 64 * n * 2.0 ** -53 * n
        assert abs(e_code - e_pauli) <= bound, (e_code, e_pauli, bound)
        cut.set_params([-gamma])
        a.apply_function(cut, list(range(n)))
        b.apply_pauli_rotations(fc.ring_terms(n), [-gamma] * n)
        ov = a.overlap(b) * np.exp(-1j * 15 * gamma)
        assert abs(ov - 1.0) <= 1e-12, ov
        for off in (0, (1 << 29) + 12345, (1 << n) - 4096):
            ga, gb = a.download(offset=off, length=4096), b.download(offset=off, length=4096)
            assert float(np.max(np.abs(ga - gb * np.exp(-1j * 15 * gamma)))) <= 1e-13, off


# ---- past 2^31 and 2^32 amplitudes ----------------------------------------------------------------------------------

LARGE_PHASE = "__device__ double qip_theta(uint64_t x, const double *p) { return p[0] * (double)(x % 1009); }\n"


@pytest.mark.parametrize("n", [31, 32])
def test_large_indices_f32(ctx, n):
    """From the H layer: a phase over the whole register (x up to 32 bits), then a permutation with a phase whose out
    register holds index bits 30 and 31 (both paths); windows around 2^31 and 2^32 against
    2^(-n/2) e^{i theta2(x2(j))} e^{i theta1(x1(j ^ d))}."""
    def q(bit):
        return n - 1 - bit

    top = [b for b in (31, 30) if b < n]
    in1 = [int(v) for v in np.random.default_rng(n).permutation(n)]
    cases = {FUNCTION_TILE: ([q(b) for b in [29, 5, 17, 0]], [q(b) for b in top + [3]]),
             FUNCTION_PAIR: ([q(b) for b in [0, 2, 10, 15]], [q(b) for b in top + list(range(29, 29 - (11 - len(top)),
                                                                                          -1))])}
    p1, p2 = [0.173], [0.61, -0.4]
    with State(n, C64, ctx) as st, \
            Function.from_code(ctx, n, 0, LARGE_PHASE, theta=True, n_params=1) as f1:
        f1.set_params(p1)
        for path, (in2, out2) in cases.items():
            assert function_plan(n, C64, in2, out2)[0] == path
            st.set_basis(0)
            st.apply_schedule([gates.h(k) for k in range(n)])
            with Function.from_code(ctx, len(in2), len(out2), fc.mix_source(len(out2), True), theta=True,
                                    n_params=2) as f2:
                f2.set_params(p2)
                st.apply_function(f1, in1)
                st.apply_function(f2, in2, out2)
            W = 1 << 12
            last = (1 << n) - W
            for off in sorted({min(o, last) for o in (0, (1 << 31) - W // 2, (1 << 31) + (5 << 12), (3 << 30) + W,
                                                      last)}):
                idx = np.arange(off, off + W, dtype=np.uint64)
                x2 = fr.register_value(idx, n, in2)
                x1 = fr.register_value(idx ^ fr.scatter(fc.mix_f(x2, len(out2)), n, out2), n, in1)
                th1 = p1[0] * (x1 % np.uint64(1009)).astype(np.float64)
                want = 2.0 ** (-n / 2) * np.exp(1j * (fc.mix_theta(x2, p2) + th1))
                got = st.download(offset=off, length=W)
                err = float(np.max(np.abs(got.astype(C128) - want)))
                assert err <= 2.0 ** (-n / 2) * 1e-5, (n, path, off, err)


# ---- the expectation value ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [C128, C64])
def test_expect_against_numpy(ctx, dtype):
    for n in (1, 5, 11, 12, 16, 20):
        rng = np.random.default_rng(300 + n)
        psi = circuits.random_state(n, 30 + n, dtype) * dtype(1.3)  # not normalised: read as it is
        in_q = [int(q) for q in rng.permutation(n)][:max(1, n - 2)]
        p = rng.uniform(-3, 3, size=2)
        with State(n, dtype, ctx) as st, Function.from_code(ctx, len(in_q), 0, fc.mix_source(0, True), theta=True,
                                                            n_params=2) as fn:
            fn.set_params(p)
            st.upload(psi)
            got = st.expect_function(fn, in_q)
            assert bits_equal(np.float64(st.expect_function(fn, in_q)), np.float64(got))
            x = fr.register_value(np.arange(1 << n, dtype=np.uint64), n, in_q)
            th = fc.mix_theta(x, p)
            w = np.abs(psi.astype(C128)) ** 2
            want = float(np.sum(w * th, dtype=np.longdouble))
            bound = fc.expect_bound(n, float(np.sum(w * np.abs(th)))) + 1e-300
            assert abs(got - want) <= 2 * bound, (n, got, want, bound)


# ---- refusals and lifetime ----------------------------------------------------------------------------------------

def test_new_code_refusals(ctx):
    with pytest.raises(CircuitError) as e:
        Function.from_code(ctx, 4, 2, "__device__ uint64_t qip_f(uint64_t x) { return x; }")
    assert e.value.status == INVALID_ARG and "f(4) = 4 does not fit in 2 output bits" in str(e.value)
    with pytest.raises(CircuitError) as e:
        Function.from_code(ctx, 6, 0, "__device__ double qip_theta(uint64_t x, const double *p) "
                                      "{ return x >= 9 ? 0.0 / (p[0] * x) : 1.0; }", theta=True, n_params=1)
    assert e.value.status == INVALID_ARG and "theta(9) is not finite" in str(e.value)
    with pytest.raises(CircuitError) as e:
        Function.from_code(ctx, 6, 1, "__device__ uint64_t qip_f(uint64_t x) { return x +; }")
    assert e.value.status == INVALID_ARG and "expected an expression" in str(e.value)
    with pytest.raises(CircuitError) as e:
        Function.from_code(ctx, 30, 5, fc.mix_source(5))
    assert e.value.status == UNSUPPORTED


def test_set_params_refusal_keeps_the_previous_parameters(ctx):
    src = ("__device__ double qip_theta(uint64_t x, const double *p) {\n"
           "  return (x >= 5 && x % 4 == 1) ? p[0] * 1e308 * 10.0 : p[0] * (double)x;\n}\n")
    with Function.from_code(ctx, 8, 0, src, theta=True, n_params=1) as fn:
        fn.set_params([1e-300])
        _, before = fn.tabulate()
        with pytest.raises(CircuitError) as e:
            fn.set_params([1.0])
        assert e.value.status == INVALID_ARG and "theta(5) is not finite" in str(e.value)
        _, after = fn.tabulate()
        assert bits_equal(before, after)
        with pytest.raises(CircuitError) as e:
            fn.set_params([1.0, 2.0])
        assert e.value.status == INVALID_ARG and "takes 1 parameters, got 2" in str(e.value)
    with Function(ctx, 2, 1, f=[0, 1, 1, 0]) as table:
        with pytest.raises(CircuitError) as e:
            table.set_params([])
        assert e.value.status == UNSUPPORTED


def test_refused_apply_and_expect_leave_state_and_pending_collapse(ctx):
    n = 14
    psi0 = circuits.random_state(n, 14, C128)
    in_q, out_q = [3, 11, 0, 7], [13, 5]
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b, \
            Function.from_code(ctx, 4, 2, fc.mix_source(2, True), theta=True, n_params=2) as fn, \
            Function.from_code(ctx, 4, 2, fc.mix_source(2)) as no_theta, \
            Function(ctx, 4, 0, theta=np.arange(16) * 0.1) as table:
        fn.set_params([0.3, -0.2])
        a.upload(psi0)
        b.upload(psi0)
        m, p = a.measure([0, 6], 0.37)
        for call, code, msg in (
                (lambda: a.apply_function(fn, [3, 11, 0, n], out_q), BAD_INDEX, "out of range"),
                (lambda: a.apply_function(fn, in_q, [13, 3]), BAD_INDEX, "qubit 3 repeated"),
                (lambda: a.expect_function(fn, [3, 11, 3, 7]), BAD_INDEX, "qubit 3 repeated"),
                (lambda: a.expect_function(table, in_q), UNSUPPORTED, "not theta"),
                (lambda: a.expect_function(no_theta, in_q), UNSUPPORTED, "no theta")):
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == code and msg in str(e.value), msg
        L = _lib.lib()
        ia = np.ascontiguousarray(np.asarray(in_q, dtype=np.uint64))
        assert L.qipb200_state_expect_function(a._h, fn.handle, ia.ctypes.data, None) == INVALID_ARG
        # the collapse is still pending: one kernel for it, one for the function
        l0 = ctx.kernel_launches()
        a.apply_function(fn, in_q, out_q)
        assert ctx.kernel_launches() - l0 == 2
        b.collapse([0, 6], m, p)
        collapsed = b.download()
        b.apply_function(fn, in_q, out_q)
        got, want = a.download(), b.download()
        f, cs = fn.tabulate()
    assert bits_equal(got, want)
    assert bits_equal(got, fc.apply_cs(collapsed, n, in_q, out_q, f, cs))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st, \
            Function.from_code(ctx, 2, 0, fc.mix_source(0, True), theta=True, n_params=2) as fn:
        for call in (lambda: st.apply_function(fn, [0, 1]), lambda: st.expect_function(fn, [0, 1])):
            with pytest.raises(CircuitError) as e:
                call()
            assert e.value.status == UNSUPPORTED


def test_free_straight_after_apply(ctx):
    n = 22
    psi0 = circuits.random_state(n, 22, C64)
    in_q, out_q = list(range(4, 20)), [1, 21, 0]
    with State(n, C64, ctx) as st:
        st.upload(psi0)
        fn = Function.from_code(ctx, len(in_q), len(out_q), fc.mix_source(len(out_q), True), theta=True, n_params=2)
        fn.set_params([0.5, 0.25])
        f, cs = fn.tabulate()
        st.apply_function(fn, in_q, out_q)
        fn.free()
        got = st.download()
    assert bits_equal(got, fc.apply_cs(psi0, n, in_q, out_q, f, cs))
