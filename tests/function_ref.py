"""References for table-defined function ops (State.apply_function, qipb200_state_apply_function).

U|x>|y> = e^{i theta(x)} |x>|y XOR f(x)>, with bit i of x the value of qubit in_q[i] and bit i of f(x) XORed into
qubit out_q[i]; qubit q is index bit n-1-q.  So (U psi)_j = e^{i theta(x(j))} psi_{j ^ d(x(j))}, d(x) = f(x) scattered
to the out qubits' index bits.

  - apply: the device arithmetic in numpy float64 / float32, bit for bit.  c and s are cos and sin of theta(x) from
    Python's math module (the C library the host side calls), rounded once to the state's precision; then
    (RN(RN(c a) - RN(s b)), RN(RN(c b) + RN(s a))) for the partner (a, b), one numpy operation per rounding.  Without
    theta the partner is copied (-0 stays -0).
  - oracle_apply: tests/native/function_oracle.c, the reference iterator's row rule (flip_bits on both registers)
    over a whole state.
  - linear functions over GF(2) and their CNOT networks; Shor's modular exponentiation and the closed form of the
    period-finding distribution."""
import ctypes as C
import math
import os

import numpy as np

from rustqip_b200 import gates

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "tests", "native", "_build", "libfunction_oracle.so")


def register_value(idx, n, qubits):
    """Value of the register `qubits` (bit i = qubit qubits[i]) at each index of `idx` (uint64 array)."""
    idx = np.asarray(idx, dtype=np.uint64)
    v = np.zeros(idx.shape, dtype=np.uint64)
    for i, q in enumerate(qubits):
        v |= ((idx >> np.uint64(n - 1 - int(q))) & np.uint64(1)) << np.uint64(i)
    return v


def scatter(vals, n, qubits):
    """Index bits of register values `vals` put on `qubits` (the inverse of register_value)."""
    vals = np.asarray(vals, dtype=np.uint64)
    d = np.zeros(vals.shape, dtype=np.uint64)
    for i, q in enumerate(qubits):
        d |= ((vals >> np.uint64(i)) & np.uint64(1)) << np.uint64(n - 1 - int(q))
    return d


def cos_sin(theta, R):
    """cos and sin of every theta in double through the C library, rounded once to R."""
    c = np.array([math.cos(float(t)) for t in theta], dtype=np.float64).astype(R)
    s = np.array([math.sin(float(t)) for t in theta], dtype=np.float64).astype(R)
    return c, s


def apply(psi, n, in_q, out_q=(), f=None, theta=None, dtype=None):
    """The device result, bit for bit, as an array of dtype (default: psi's)."""
    dtype = np.dtype(dtype or np.asarray(psi).dtype)
    R = np.float64 if dtype == np.complex128 else np.float32
    psi = np.asarray(psi).astype(dtype)
    j = np.arange(1 << n, dtype=np.uint64)
    x = register_value(j, n, in_q)
    src = j
    if len(out_q):
        src = j ^ scatter(np.asarray(f, dtype=np.uint64)[x], n, out_q)
    moved = psi[src]
    if theta is None:
        return moved.copy()
    c, s = cos_sin(theta, R)
    c, s = c[x], s[x]
    a, b = moved.real.astype(R), moved.imag.astype(R)
    out = np.empty(1 << n, dtype=dtype)
    out.real = c * a - s * b
    out.imag = c * b + s * a
    return out


_oracle = None


def oracle_apply(psi, n, in_q, out_q=(), f=None, theta=None):
    """The reference iterator's row rule (tests/native/function_oracle.c) applied to psi."""
    global _oracle
    if _oracle is None:
        _oracle = C.CDLL(ORACLE_SO)
        for name in ("fo_apply_function_f64", "fo_apply_function_f32"):
            getattr(_oracle, name).restype = None
            getattr(_oracle, name).argtypes = [C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
    psi = np.ascontiguousarray(psi)
    out = np.empty_like(psi)
    ia = np.ascontiguousarray(np.asarray(list(in_q) or [0], dtype=np.uint64))
    oa = np.ascontiguousarray(np.asarray(list(out_q) or [0], dtype=np.uint64))
    fa = None if f is None else np.ascontiguousarray(np.asarray(f, dtype=np.uint64))
    ta = None if theta is None else np.ascontiguousarray(np.asarray(theta, dtype=np.float64))
    fn = _oracle.fo_apply_function_f64 if psi.dtype == np.complex128 else _oracle.fo_apply_function_f32
    fn(n, ia.ctypes.data, len(in_q), oa.ctypes.data, len(out_q), None if fa is None else fa.ctypes.data,
       None if ta is None else ta.ctypes.data, psi.ctypes.data, out.ctypes.data)
    return out


# ---- linear functions over GF(2) -----------------------------------------------------------------------------------

def random_matrix(rows, cols, seed):
    return np.random.default_rng(seed).integers(0, 2, size=(rows, cols)).astype(np.uint64)


def linear_table(A):
    """f(x) = A x over GF(2) for every x < 2^cols: bit r of f(x) is the parity of row r of A and the bits of x."""
    rows, cols = A.shape
    x = np.arange(1 << cols, dtype=np.uint64)
    f = np.zeros(1 << cols, dtype=np.uint64)
    for r in range(rows):
        mask = np.uint64(sum(1 << i for i in range(cols) if A[r, i]))
        f |= (np.bitwise_count(x & mask).astype(np.uint64) & np.uint64(1)) << np.uint64(r)
    return f


def cnot_network(A, in_q, out_q):
    """The CNOT network of y ^= A x: one CNOT(in_q[i] -> out_q[r]) per 1 in A."""
    rows, cols = A.shape
    return [gates.cnot(int(in_q[i]), int(out_q[r])) for r in range(rows) for i in range(cols) if A[r, i]]


# ---- Shor's period finding -----------------------------------------------------------------------------------------

def modexp_table(a, N, m):
    """f(x) = a^x mod N for x < 2^m."""
    f = np.empty(1 << m, dtype=np.uint64)
    v = 1
    for x in range(1 << m):
        f[x] = v
        v = (v * a) % N
    return f


def order(a, N):
    v, r = a % N, 1
    while v != 1:
        v, r = (v * a) % N, r + 1
    return r


def shor_probs(m, r, ks=None):
    """P(k) = 2^-2m sum_{s<r} |sin(pi k r M_s / 2^m) / sin(pi k r / 2^m)|^2, M_s = #{j < 2^m : j = s mod r} (the
    ratio is M_s where the denominator vanishes): the distribution of the QFT of the x register after
    H^m and |x>|0> -> |x>|a^x mod N> for a of order r."""
    M = 1 << m
    k = np.arange(M, dtype=np.int64) if ks is None else np.asarray(ks, dtype=np.int64)
    base, extra = divmod(M, r)
    out = np.zeros(k.shape, dtype=np.float64)

    def sin_pi_over_M(q):  # sin(pi q / M) with q reduced exactly mod 2M first
        return np.sin(np.pi * ((q % (2 * M)).astype(np.float64) / M))

    den = sin_pi_over_M(k * r)
    exact = (k * r) % M == 0
    for Ms, count in ((base + 1, extra), (base, r - extra)):
        if count == 0:
            continue
        num = sin_pi_over_M(k * r % (2 * M) * Ms)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(exact, float(Ms), num / np.where(exact, 1.0, den))
        out += count * ratio ** 2
    return out / float(M) ** 2


def period_from_shot(k, m, a, N):
    """r from one measured k by continued fractions of k / 2^m: the first convergent denominator q < N with a small
    multiple t q (t <= 20) such that a^(t q) = 1 mod N, or None."""
    num, den = int(k), 1 << m
    q0, q1 = 1, 0
    while den:
        c, rem = divmod(num, den)
        q0, q1 = q1, c * q1 + q0
        num, den = den, rem
        if q1 >= N:
            break
        for t in range(1, 21):
            if pow(a, t * q1, N) == 1:
                return t * q1
    return None
