"""References and rounding bound for reduced density matrices (State.reduced_density).

Qubit q is index bit n-1-q.  For kept qubits A = qubits[0..k-1], bit i of the row / column index a is the value of
qubit qubits[i] (the convention of measure_probs), and

    rho[a, b] = sum_r psi(r, a) * conj(psi(r, b))      (r: every other index bit).

rdm_ref evaluates this in long double; tests/test_reduced_density_cpu.py pins it against np.einsum over the reshaped
state and against tests/pauli_ref.expect_ref (Tr(rho P_A) = <P>).  rdm_int is the exact reference for states of
Gaussian integers (tests/exact_circuits.exact_state): int64 sums, exact while 2 bits + (n - k) + 1 <= 53.

Rounding bound of the device kernel (rustqip_b200/csrc/rdm.cu), per entry, in units of W_ab = sum_r |psi_ra||psi_rb|:
  - f32 amplitudes are exact in double, and so are their products;
  - each thread accumulates its rows with two fma per component and row: 2 m sequential roundings, where m is the
    number of rows a thread visits: ceil(rows per tile / S) per tile times ceil(V / G) tiles (V tiles or tile pairs
    per sweep over G = 264 CTAs; S threads split a tile's rows);
  - the S row splits are summed sequentially, then the G per-CTA partials;
  - each real component sums terms whose moduli add to at most W_ab (|xr yr| + |xi yi| <= |x| |y|), and the complex
    error is at most sqrt(2) times the componentwise one.
So the depth is D = 2 m + S + G, and |got - want| <= 2 (gamma_D(2^-53) + gamma_ref) W_ab, where gamma_ref covers the
long-double reference (a product and a sequential sum over the 2^(n-k) rows)."""
import math

import numpy as np

import pauli_ref as pr

U_DOUBLE = 2.0 ** -53
U_LONGDOUBLE = pr.U_LONGDOUBLE
TILE_BITS = 11
COLS_LOG2 = 6
THREADS = 256
GRID = 264
MAX_KEPT = 10


def split_index(n, qubits):
    """(a, r) for every index j: a from the kept bits (bit i <-> qubits[i]), r from the others in index order."""
    j = np.arange(1 << n, dtype=np.uint64)
    a = np.zeros(1 << n, dtype=np.int64)
    for i, q in enumerate(qubits):
        a |= ((j >> np.uint64(n - 1 - int(q))) & np.uint64(1)).astype(np.int64) << i
    kept = set(n - 1 - int(q) for q in qubits)
    r = np.zeros(1 << n, dtype=np.int64)
    pos = 0
    for b in range(n):
        if b not in kept:
            r |= ((j >> np.uint64(b)) & np.uint64(1)).astype(np.int64) << pos
            pos += 1
    return a, r


def blocks(psi, n, qubits, dtype):
    """X[r, a] = psi(r, a)."""
    a, r = split_index(n, qubits)
    X = np.zeros((1 << (n - len(qubits)), 1 << len(qubits)), dtype=dtype)
    X[r, a] = np.asarray(psi).astype(dtype)
    return X


def rdm_ref(psi, n, qubits):
    """rho in complex long double."""
    X = blocks(psi, n, qubits, np.clongdouble)
    return X.T @ np.conj(X)


def abs_weight(psi, n, qubits):
    """W[a, b] = sum_r |psi_ra| |psi_rb| (in double; it scales the bound only)."""
    A = np.abs(blocks(psi, n, qubits, np.complex128))
    return A.T @ A


def kernel_depth(n, k):
    k_in = min(k, COLS_LOG2)
    blk = k - k_in
    tb = min(TILE_BITS, n - blk)
    C = 1 << k_in
    rb = min(4, C)
    S = THREADS // ((C // rb) ** 2)
    rows = (1 << tb) // C
    visits = 1 << (n - tb - blk)
    m = math.ceil(rows / S) * math.ceil(visits / GRID)
    return 2 * m + S + GRID


def bound(n, k, W):
    return 2 * (pr.gamma(kernel_depth(n, k), U_DOUBLE) + pr.gamma((1 << (n - k)) + 2, U_LONGDOUBLE)) * W


def int_parts(psi):
    """Integer real and imaginary parts of a state of Gaussian integers (asserts that they are integers)."""
    p = np.asarray(psi).astype(np.complex128)
    re, im = p.real, p.imag
    assert np.array_equal(re, np.round(re)) and np.array_equal(im, np.round(im)), "not a state of Gaussian integers"
    return re.astype(np.int64), im.astype(np.int64)


def mantissa_bits(psi):
    re, im = int_parts(psi)
    m = int(max(np.max(np.abs(re)), np.max(np.abs(im)), 1))
    return m.bit_length()


def budget_ok(psi, n, k):
    """Every product (2 bits) and every partial sum of 2 (n - k) + ... terms fits 53 bits."""
    return 2 * mantissa_bits(psi) + (n - k) + 1 <= 53


def rdm_int(psi, n, qubits):
    """The exact rho of a state of Gaussian integers, from int64 sums (complex128 result, exact by the budget)."""
    assert budget_ok(psi, n, len(qubits))
    re, im = int_parts(psi)
    Xr = blocks(re, n, qubits, np.int64)
    Xi = blocks(im, n, qubits, np.int64)
    real = Xr.T @ Xr + Xi.T @ Xi
    imag = Xi.T @ Xr - Xr.T @ Xi
    out = real.astype(np.float64) + 1j * imag.astype(np.float64)
    assert np.array_equal(out.real.astype(np.int64), real) and np.array_equal(out.imag.astype(np.int64), imag)
    return out


def rdm_exact(psi, n, qubits):
    """rdm_int through double matrix products: every product and partial sum is an integer below 2^53, so exact in any
    summation order (fast enough for 2^20-amplitude states); pinned to rdm_int by the CPU tests."""
    assert budget_ok(psi, n, len(qubits))
    re, im = int_parts(psi)
    Xr = blocks(re, n, qubits, np.float64)
    Xi = blocks(im, n, qubits, np.float64)
    return (Xr.T @ Xr + Xi.T @ Xi) + 1j * (Xi.T @ Xr - Xr.T @ Xi)


# ---- closed forms -------------------------------------------------------------------------------------------------

def product_rdm(n, qubits, vs):
    """The product state of the 2-vectors vs[q]: rho = kron over the kept qubits of v v^dagger (qubits[0] the least
    significant factor), times the squared norms of the traced-out vectors."""
    scale = np.longdouble(1)
    for q in range(n):
        if q not in qubits:
            v = np.asarray(vs[q], dtype=np.clongdouble)
            scale *= np.sum(np.abs(v) ** 2)
    rho = np.array([[np.clongdouble(1)]])
    for q in qubits:
        v = np.asarray(vs[q], dtype=np.clongdouble)
        rho = np.kron(np.outer(v, np.conj(v)), rho)
    return rho * scale


def product_state(n, vs):
    psi = np.array([1.0 + 0j])
    for q in range(n):  # qubit 0 is the most significant index bit
        psi = np.kron(psi, np.asarray(vs[q], dtype=np.complex128))
    return psi


def ghz_rdm(n, qubits, alpha, beta):
    """alpha |0..0> + beta |1..1>: a proper subset has |alpha|^2 and |beta|^2 on the first and last diagonal entries,
    all n qubits add the two corners alpha conj(beta) and beta conj(alpha)."""
    K = 1 << len(qubits)
    a, b = np.clongdouble(alpha), np.clongdouble(beta)
    rho = np.zeros((K, K), dtype=np.clongdouble)
    rho[0, 0] = abs(a) ** 2
    rho[K - 1, K - 1] = abs(b) ** 2
    if len(qubits) == n:
        rho[0, K - 1] = a * np.conj(b)
        rho[K - 1, 0] = b * np.conj(a)
    return rho


def pauli_matrix(term, qubits):
    """The matrix of a Pauli string on the kept qubits in rho's index convention (bit i <-> qubits[i])."""
    P1 = {"I": np.eye(2), "X": np.array([[0, 1], [1, 0]]), "Y": np.array([[0, -1j], [1j, 0]]), "Z": np.diag([1, -1])}
    letters = dict((q, l) for l, q in term)
    m = np.array([[1.0 + 0j]])
    for q in qubits:
        m = np.kron(np.asarray(P1[letters.get(q, "I")], dtype=complex), m)
    return m
