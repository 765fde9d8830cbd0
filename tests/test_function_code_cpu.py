"""Functions given as CUDA source (qipb200_function_new_code) without a GPU: the host-only NVRTC compile of the
program (qipb200_function_code_compile), its argument checks, the C++ mirror and the path plan."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import function_code_ref as fc
from rustqip_b200 import _lib
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import FUNCTION_PAIR, FUNCTION_TILE, function_code_compile, function_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG, UNSUPPORTED = 1, 7
THETA = "__device__ double qip_theta(uint64_t x, const double *p) { return p[0] * (double)(x & 7); }\n"


def _compile_raw(n_in, n_out, source, flags=0, n_params=0):
    log = C.create_string_buffer(1 << 16)
    st = _lib.lib().qipb200_function_code_compile(n_in, n_out, source, flags, n_params, log, len(log))
    return st, log.value.decode(), _lib.lib().qipb200_last_error(None).decode()


@pytest.mark.parametrize("n_in,n_out,theta", [(1, 1, False), (20, 10, True), (26, 8, False), (30, 4, True),
                                               (34, 0, True), (2, 32, False), (2, 32, True)])
def test_valid_sources_compile(n_in, n_out, theta):
    function_code_compile(n_in, n_out, fc.mix_source(n_out, theta), theta=theta, n_params=2 if theta else 0)


def test_ring_source_compiles_with_sixteen_parameters():
    function_code_compile(30, 0, fc.ring_source(30), theta=True, n_params=16)


def test_compile_errors_carry_the_nvrtc_log():
    st, log, err = _compile_raw(8, 2, b"__device__ uint64_t qip_f(uint64_t x) { return x +; }")
    assert st == INVALID_ARG and "expected an expression" in log and "qip_function(1)" in log
    assert err.startswith("function_code_compile: the source does not compile") and "expected an expression" in err
    # qip_f is required with n_out > 0, qip_theta with THETA
    st, log, _ = _compile_raw(8, 2, THETA.encode(), 1)
    assert st == INVALID_ARG and "qip_f" in log and "undefined" in log
    st, log, _ = _compile_raw(8, 2, fc.mix_source(2).encode(), 1)
    assert st == INVALID_ARG and "qip_theta" in log
    with pytest.raises(CircuitError) as e:
        function_code_compile(8, 0, "__device__ double qip_theta(uint64_t x, const double *p) { return y; }",
                              theta=True)
    assert e.value.status == INVALID_ARG and '"y" is undefined' in str(e.value)


def test_user_warnings_are_reported_and_library_ones_are_not():
    src = b"__device__ uint64_t qip_f(uint64_t x) { int unused; return x & 1; }"
    st, log, _ = _compile_raw(4, 1, src)
    assert st == 0 and '"unused" was declared but never referenced' in log
    assert "qipb200" not in log
    st, log, _ = _compile_raw(4, 1, fc.mix_source(1).encode())
    assert st == 0 and "warning" not in log


def test_sizes_and_flags_are_refused():
    good = fc.mix_source(4, True).encode()
    for args, code, msg in [
        ((0, 4, good, 1), INVALID_ARG, "n_in must be at least 1"),
        ((8, 0, fc.mix_source(0).encode() or b" ", 0), INVALID_ARG, "nothing to apply"),
        ((8, 4, good, 1, 17), INVALID_ARG, "at most 16 parameters"),
        ((8, 4, good, 3), INVALID_ARG, "unknown flags 3"),
        ((8, 4, b"", 1), INVALID_ARG, "NULL or empty source"),
        ((8, 4, None, 1), INVALID_ARG, "NULL or empty source"),
        ((2, 33, good, 1), UNSUPPORTED, "at most 32 output qubits"),
        ((31, 4, good, 1), UNSUPPORTED, "n_in + n_out = 35 exceeds 34"),
        ((35, 0, good, 1), UNSUPPORTED, "exceeds 34"),
    ]:
        st, _, err = _compile_raw(*args)
        assert st == code and msg in err and err.startswith("function_code_compile:"), (args, err)


def test_new_code_refuses_a_null_context():
    out = C.c_void_p()
    st = _lib.lib().qipb200_function_new_code(None, 4, 1, fc.mix_source(1).encode(), 0, 0, None, 0, C.byref(out))
    assert st == INVALID_ARG and not out.value
    assert _lib.lib().qipb200_function_set_params(None, None, 0) == INVALID_ARG
    assert _lib.lib().qipb200_function_tabulate(None, 0, 1, None, None) == INVALID_ARG
    d = C.c_double()
    assert _lib.lib().qipb200_state_expect_function(None, None, None, C.byref(d)) == INVALID_ARG


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_plan_depends_on_the_out_register_only(dtype):
    """A code handle takes the table path's plan: it depends on the out register, not on n_in."""
    rng = np.random.default_rng(5)
    seen = set()
    for n in (12, 20, 30, 34):
        for _ in range(20):
            perm = [int(q) for q in rng.permutation(n)]
            n_out = int(rng.integers(1, 12))
            out_q = perm[:n_out]
            plans = {function_plan(n, dtype, perm[n_out:n_out + k], out_q) for k in (1, 5, min(26, n - n_out))}
            assert len(plans) == 1, (n, out_q, plans)
            seen.add(plans.pop()[0])
    assert seen == {FUNCTION_TILE, FUNCTION_PAIR}


def test_cpp_mirror_code_function_compiles(tmp_path):
    src = tmp_path / "use_code_function.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "double run(qip::Context &ctx, qip::B200State<double> &a, qip::B200State<float> &b) {\n"
                   "  auto f = qip::B200Function::from_code(ctx, 4, 2, \"__device__ uint64_t qip_f(uint64_t x) "
                   "{ return x & 3; }\");\n"
                   "  auto g = qip::B200Function::from_code(ctx, 3, 0, \"__device__ double qip_theta(uint64_t x, "
                   "const double *p) { return p[0] * x; }\", true, 1);\n"
                   "  g.set_params({0.25});\n"
                   "  std::vector<uint64_t> fx;\n"
                   "  std::vector<double> cs;\n"
                   "  f.tabulate(0, 16, &fx, nullptr);\n"
                   "  g.tabulate(2, 6, nullptr, &cs);\n"
                   "  a.apply_function(f, {0, 1, 2, 3}, {4, 5});\n"
                   "  b.apply_function(g, {2, 0, 1});\n"
                   "  return a.expect_function(g, {5, 4, 3});\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I" + os.path.join(ROOT, "include"),
                        str(src)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
