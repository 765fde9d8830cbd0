"""References and rounding bounds for the purity of a bipartition (State.purity, qipb200_state_purity).

Qubit q is index bit n-1-q.  For kept qubits A and s = min(k, n - k), the side is A when k <= n - k and its complement
otherwise; M[a][r] = psi(side bits a, other bits r), G = M M^dagger and

    P = sum_{a,b} |G_ab|^2 = Tr rho_A^2 = Tr rho_B^2,      T = sum_a G_aa = sum_j |psi_j|^2.

purity_ld evaluates P and T in long double (small states); purity_ref forms G with a complex128 matrix product and
returns its own first-order bound next to P and T (states up to 2^24 amplitudes); purity_int is exact for states of
Gaussian integers while every sum stays below 2^53.

Device bounds, first order in u = 2^-53 (the orders are documented in rustqip_b200/csrc/purity.cu and rdm.cu):
  - Gram route (s >= 11): |dG_ab| <= delta_ab = sqrt(2) gamma_D W_ab with D = 2 * 2^(n-s) and W = |M| |M|^T; the final
    sum is a chain of E = 64 + 8 + ceil(B / 256) + 8 roundings over non-negative terms (B Gram blocks), so
        |dP| <= sum (2 |G| delta + delta^2) (1 + gamma_E) + gamma_E P,   |dT| <= gamma_{D+E} T.
  - reduced_density route (1 <= s <= 10): |d rho_ab| <= 2 gamma_{D_rdm} W_ab (tests/rdm_ref.kernel_depth), then the host
    sums each row (2 * 2^s roundings) and the rows (2^s): E = 3 * 2^s, same propagation.
  - norm2 route (s = 0): gamma_{2^n} T for the norm2 sweep in any order, then the square.
By Cauchy-Schwarz sum_{a,b} |G_ab| W_ab <= T^2, so bound_cs needs only the outputs (used at full size)."""
import math

import numpy as np

import pauli_ref as pr
import rdm_ref as rr

U_DOUBLE = 2.0 ** -53
U_LONGDOUBLE = pr.U_LONGDOUBLE
GRAM_MIN_SIDE = 11
RDM_MAX = 10
THREADS = 256


def gamma(m, u=U_DOUBLE):
    return pr.gamma(m, u)


def side_of(n, qubits):
    """The side the device works on: the kept qubits, or their complement when that is smaller."""
    qubits = [int(q) for q in qubits]
    if len(qubits) <= n - len(qubits):
        return qubits
    return [q for q in range(n) if q not in qubits]


def route(s):
    return 0 if s == 0 else 1 if s < GRAM_MIN_SIDE else 2


def gram_blocks(s):
    nr = 1 << (s - 7)
    return nr * (nr + 1)


def launches(s):
    """Kernels of the call for a side of s qubits: norm2, reduced_density's nB (nB + 1), or Gram + reduction."""
    if route(s) == 0:
        return 1
    if route(s) == 1:
        nb = 1 << max(0, s - 6)
        return nb * (nb + 1)
    return 2


def plan(n, qubits):
    s = min(len(qubits), n - len(qubits))
    return (route(s), s, launches(s), gram_blocks(s) if route(s) == 2 else 0)


def side_matrix(psi, n, qubits, dtype):
    """M[a, r] over the side of the cut (a: side bits, bit i <-> side[i]; r: the other qubits, qubit order).  P, T, |G|
    and W are invariant under permutations of rows and columns, so only the split matters."""
    side = side_of(n, qubits)
    rest = [q for q in range(n) if q not in side]
    t = np.asarray(psi).astype(dtype).reshape((2,) * n)
    return np.ascontiguousarray(np.transpose(t, side[::-1] + rest).reshape(1 << len(side), 1 << len(rest)))


def purity_ld(psi, n, qubits):
    """(P, T) in long double."""
    M = side_matrix(psi, n, qubits, np.clongdouble)
    G = M @ np.conj(M.T)
    return np.sum(np.abs(G) ** 2), np.sum(np.abs(M) ** 2)


def purity_ref(psi, n, qubits):
    """(P, T, bound of this reference, G, W): G from a complex128 matrix product, the squares in double, their sums in long double."""
    M = side_matrix(psi, n, qubits, np.complex128)
    K = M.shape[1]
    G = M @ np.conj(M.T)
    A = np.abs(M)
    W = A @ A.T
    P = np.sum(G.real ** 2 + G.imag ** 2, dtype=np.longdouble)
    T = np.sum(M.real ** 2 + M.imag ** 2, dtype=np.longdouble)
    delta = 2 * gamma(K + 2) * W
    aG = np.abs(G)
    # the squares round once in double (u each, relative), the sums in long double
    b = float(np.sum(2 * aG * delta + delta * delta)) + float((2 * U_DOUBLE + gamma(G.size + 2, U_LONGDOUBLE)) * P)
    bt = float((2 * U_DOUBLE + gamma(M.size + 2, U_LONGDOUBLE)) * T)
    return float(P), float(T), b, bt, G, W


def _propagate(sum_gw, sum_w2, P, E):
    return (2 * sum_gw + sum_w2) * (1 + gamma(E)) + gamma(E) * P


def gram_depths(n, s):
    D = 2 * (1 << (n - s))
    E = 64 + 8 + math.ceil(gram_blocks(s) / THREADS) + 8
    return D, E


def device_bound(n, s, G, W, P, T):
    """(bound on |P_got - P|, bound on |T_got - T|) of the device route for a side of s qubits, from |G| and W."""
    aG = np.abs(G)
    if route(s) == 0:
        b = gamma(1 << n) * T  # norm2 in any order
        return 2 * T * b + b * b + U_DOUBLE * T * T, b
    if route(s) == 1:
        d = 2 * gamma(rr.kernel_depth(n, s)) * W
        E = 3 * (1 << s)
        return (_propagate(float(np.sum(aG * d)), float(np.sum(d * d)), P, E),
                gamma(rr.kernel_depth(n, s) + (1 << s)) * T)
    D, E = gram_depths(n, s)
    d = math.sqrt(2) * gamma(D) * W
    return _propagate(float(np.sum(aG * d)), float(np.sum(d * d)), P, E), gamma(D + E) * T


def bound_cs(n, s, P, T):
    """device_bound with sum |G| W <= T^2 and sum W^2 <= T^2 (Cauchy-Schwarz): needs only the outputs."""
    if route(s) == 0:
        b = gamma(1 << n) * T  # norm2 in any order
        return 2 * T * b + b * b + U_DOUBLE * T * T, b
    if route(s) == 1:
        g = 2 * gamma(rr.kernel_depth(n, s))
        E = 3 * (1 << s)
        return _propagate(g * T * T, g * g * T * T, P, E), gamma(rr.kernel_depth(n, s) + (1 << s)) * T
    D, E = gram_depths(n, s)
    g = math.sqrt(2) * gamma(D)
    return _propagate(g * T * T, g * g * T * T, P, E), gamma(D + E) * T


def purity_int(psi, n, qubits):
    """Exact (P, T) of a state of Gaussian integers as Python ints; asserts that every device partial sum (entries of
    G, and P itself) stays below 2^53, so that the device result is exact too."""
    re, im = rr.int_parts(psi)
    Mr = side_matrix(re, n, qubits, np.float64)
    Mi = side_matrix(im, n, qubits, np.float64)
    m = int(max(np.max(np.abs(re)), np.max(np.abs(im)), 1))
    assert 2 * m * m * Mr.shape[1] < 2 ** 53, "entries of G may round"
    Gr = (Mr @ Mr.T + Mi @ Mi.T).astype(np.int64)
    Gi = (Mi @ Mr.T - Mr @ Mi.T).astype(np.int64)
    P = int(np.sum(Gr * Gr + Gi * Gi, dtype=np.int64))
    T = int(np.sum(re * re + im * im, dtype=np.int64))
    assert P < 2 ** 53 and T < 2 ** 53, "P or T may round"
    return P, T
