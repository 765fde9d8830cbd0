"""Sources and host models of code functions (Function.from_code, qipb200_function_new_code) for the tests.

``apply_cs`` is the device apply taken from the function's own (f, c, s): the arithmetic of tests/function_ref.py's
emulator, fed with the table of ``Function.tabulate`` instead of host cos/sin."""
import numpy as np

from function_ref import register_value, scatter

MIX = 0x9E3779B97F4A7C15


def mix_source(n_out, theta=False):
    """f(x) = the top n_out bits of x * MIX (mod 2^64); theta(x, p) = p[0] (x mod 97) + p[1] (x mod 5)."""
    s = ""
    if n_out:
        s += ("__device__ uint64_t qip_f(uint64_t x) { return (x * 0x%016xull) >> %d; }\n" % (MIX, 64 - n_out))
    if theta:
        s += ("__device__ double qip_theta(uint64_t x, const double *p) {\n"
              "  return p[0] * (double)(x % 97) + p[1] * (double)(x % 5);\n}\n")
    return s


def mix_f(x, n_out):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return (x * np.uint64(MIX)) >> np.uint64(64 - n_out)


def mix_theta(x, p):
    x = np.asarray(x, dtype=np.uint64)
    return p[0] * (x % np.uint64(97)).astype(np.float64) + p[1] * (x % np.uint64(5)).astype(np.float64)


def ring_source(n):
    """theta(x, p) = p[0] * (the number of cut edges of the n-ring), bit i of x = vertex i."""
    mask = (1 << n) - 1
    return ("__device__ double qip_theta(uint64_t x, const double *p) {\n"
            "  const uint64_t r = ((x << 1) | (x >> %d)) & 0x%xull;\n"
            "  return p[0] * (double)__popcll(x ^ r);\n}\n" % (n - 1, mask))


def ring_terms(n):
    return [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]


def apply_cs(psi, n, in_q, out_q, f, cs):
    """The device apply with f[x] and cs[x] = (cos, sin) in double from Function.tabulate (cs None: no phase)."""
    psi = np.asarray(psi)
    R = np.float64 if psi.dtype == np.complex128 else np.float32
    j = np.arange(1 << n, dtype=np.uint64)
    x = register_value(j, n, in_q)
    src = j ^ scatter(np.asarray(f, dtype=np.uint64)[x], n, out_q) if len(out_q) else j
    moved = psi[src]
    if cs is None:
        return moved.copy()
    c, s = cs[x, 0].astype(R), cs[x, 1].astype(R)
    a, b = moved.real.astype(R), moved.imag.astype(R)
    out = np.empty(1 << n, dtype=psi.dtype)
    out.real = c * a - s * b
    out.imag = c * b + s * a
    return out


def expect_bound(n, abs_sum):
    """The first-order bound of rustqip_b200/csrc/function.cu on |got - sum_j |psi_j|^2 theta_j|."""
    G, C = 264, min(1 << n, 2048)
    V = (1 << n) // C
    D = 8 * -(-V // G) + 5 + 7 + (G - 1)
    return (3 + D) * 2.0 ** -53 * abs_sum
