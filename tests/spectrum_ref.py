"""References and rounding bounds for the entanglement spectrum of a bipartition (State.entanglement_spectrum,
qipb200_state_entanglement_spectrum).

Qubit q is index bit n-1-q.  The side is taken as by purity (tests/purity_ref.side_of): the kept qubits when
k <= n - k, else their complement; s is its size, M[a][r] = psi(side bits a, other bits r) and G = M M^dagger, whose
eigenvalues are the squared singular values of M (the squared Schmidt coefficients times the norm).

References:
  - schmidt_ref: numpy svd of M in complex128, squared, descending (states up to 2^24 amplitudes);
  - gram_exact: G of a dyadic state (entries +-2^-e, or 0) from a float64 product of the integer-scaled M: exact while
    every sum stays below 2^53 (asserted), so it is also what the device must return bit for bit;
  - closed forms: product states, Bell pairs, GHZ and Schmidt-form states with a chosen spectrum.

Bounds (first order in u = 2^-53; gamma_m = m u / (1 - m u)):
  - the device's G: the Gram route stores entries with |dG_ab| <= sqrt(2) gamma_D W_ab, D = 2 * 2^(n-s) and
    W = |M| |M|^T (rustqip_b200/csrc/purity.cu); ||W||_F <= || |M| ||_F^2 = T, so ||dG||_F <= sqrt(2) gamma_D T.  The
    reduced_density route has |d rho_ab| <= 2 gamma_{D_rdm} W_ab (tests/rdm_ref.kernel_depth), so ||dG||_F <=
    2 gamma_{D_rdm} T.  The norm2 route (s = 0) returns one value within gamma_{2^n} T.
  - the solver: cusolverDnZheevd reduces G to tridiagonal form with Householder reflections and solves that by divide
    and conquer; both are backward stable, so the computed eigenvalues are exact for G + E with ||E||_2 <= p(K) u ||G||_2.
    We take p(K) = c K with c = SOLVER_C = 16: the classical analyses of Householder tridiagonalisation and of the
    tridiagonal solvers give a small multiple of K (Wilkinson; Higham, Accuracy and Stability, sections 19.3 and 19.7;
    Demmel, Applied Numerical Linear Algebra, section 5.3.3), and 16 covers the reduction, the back transformation of
    nothing (values only) and the tridiagonal solve with a margin.  ||G||_2 = lambda_max <= T.
  - Weyl's inequality: |lambda_hat_i - lambda_i| <= ||dG||_2 + ||E||_2 <= ||dG||_F + c K u ||G||_2 for every i (both
    sorted the same way).
  - the svd reference: numpy's LAPACK gesdd is backward stable in the same sense, |dsigma| <= c max(K, L) u sigma_max
    (L = 2^(n-s)), so |dsigma^2| <= (2 c max(K, L) u + (c max(K, L) u)^2) lambda_max.
  - entropy: with p = lambda / T, Fannes-Audenaert gives |S(p_hat) - S(p)| <= t ln(d - 1) + H(t), t = 1/2 ||dp||_1,
    H the binary entropy, d = 2^s.  ||dp||_1 <= (d e + |dT|) / (T - |dT|) (e the per-eigenvalue bound; clipping
    rounded negative values at 0 moves them by less than e), plus the rounding of the host's sum of d terms p ln p
    (gamma_{d + 8} (S + 1): each term is within a few u of p ln p, and d u p |ln p| summed is d u S)."""
import math

import numpy as np

import purity_ref as pu
import rdm_ref as rr

U_DOUBLE = 2.0 ** -53
SOLVER_C = 16
MAX_SIDE = 13


def gamma(m, u=U_DOUBLE):
    return m * u / (1.0 - m * u)


side_of = pu.side_of
route = pu.route


def launches(s):
    """Kernels of the call: norm2 (1), reduced_density's nB (nB + 1), or the Gram kernel with the store (1)."""
    return 1 if route(s) == 2 else pu.launches(s)


def plan(n, qubits, solver_loads=1):
    s = min(len(qubits), n - len(qubits))
    return (route(s), s, launches(s), 0 if s == 0 else 16 * 4 ** s, solver_loads)


def side_matrix(psi, n, qubits, dtype=np.complex128):
    """M over the side in the convention of reduced_density: row bit i <-> side qubit i."""
    return pu.side_matrix(psi, n, qubits, dtype)


def schmidt_ref(psi, n, qubits):
    """(eigenvalues of G descending, 2^s of them, T) from numpy's svd of M (complex128)."""
    M = side_matrix(psi, n, qubits)
    sv = np.linalg.svd(M, compute_uv=False)
    lam = np.zeros(M.shape[0])
    lam[: sv.size] = sv.astype(np.float64) ** 2
    T = float(np.sum(M.real ** 2 + M.imag ** 2, dtype=np.longdouble))
    return lam, T


def gram_exact(psi, n, qubits, scale_log2):
    """G (complex128, the side's convention) of a dyadic state: M * 2^scale_log2 is a matrix of Gaussian integers,
    its Gram product in float64 is exact (asserted: every sum below 2^53), and the result is scaled back exactly."""
    M = side_matrix(psi, n, qubits) * 2.0 ** scale_log2
    re, im = M.real, M.imag
    assert np.array_equal(re, np.round(re)) and np.array_equal(im, np.round(im)), "not dyadic at this scale"
    m = max(float(np.max(np.abs(re))), float(np.max(np.abs(im))), 1.0)
    assert 2 * m * m * M.shape[1] < 2 ** 53, "entries of G may round"
    Gr = re @ re.T + im @ im.T
    Gi = im @ re.T - re @ im.T
    return (Gr + 1j * Gi) * 2.0 ** (-2 * scale_log2)


def entropy(lam, T):
    """-sum p ln p over lambda > 0 in ascending order, p = lambda / T (0 if T == 0), as the device call sums it."""
    if T == 0:
        return 0.0
    h = 0.0
    for x in np.sort(np.asarray(lam, dtype=np.float64)):
        if x > 0:
            p = x / T
            h -= p * math.log(p)
    return h


def renyi(lam, T, alpha):
    p = np.asarray(lam)[np.asarray(lam) > 0] / T
    if np.isinf(alpha):
        return -math.log(p.max())
    return math.log(np.sum(p ** alpha)) / (1.0 - alpha)


def gram_error_frobenius(n, s, T):
    """Bound on ||G_device - G||_F for a side of s qubits (see the module docstring)."""
    if route(s) == 0:
        return gamma(1 << n) * T
    if route(s) == 1:
        return 2 * gamma(rr.kernel_depth(n, s)) * T
    return math.sqrt(2) * gamma(2 * (1 << (n - s))) * T


def trace_bound(n, s, T):
    """Bound on |out2[0] - T|: the diagonal entries' errors (relative to G_aa = W_aa) and the host's sum of 2^s."""
    if route(s) == 0:
        return gamma(1 << n) * T
    if route(s) == 1:
        return (2 * gamma(rr.kernel_depth(n, s)) + gamma(1 << s)) * T
    return (math.sqrt(2) * gamma(2 * (1 << (n - s))) + gamma(1 << s)) * T


def solver_bound(s, lam_max):
    return SOLVER_C * (1 << s) * U_DOUBLE * lam_max


def svd_ref_bound(n, s, lam_max):
    e = SOLVER_C * max(1 << s, 1 << (n - s)) * U_DOUBLE
    return (2 * e + e * e) * lam_max


def eig_bound(n, s, T, lam_max, with_ref=True):
    """Per-eigenvalue bound |lambda_device_i - lambda_ref_i| (Weyl), device plus (optionally) the svd reference."""
    b = gram_error_frobenius(n, s, T) + (solver_bound(s, lam_max) if s > 0 else 0.0)
    return b + (svd_ref_bound(n, s, lam_max) if with_ref else 0.0)


def binary_entropy(t):
    if t <= 0:
        return 0.0
    if t >= 1:
        return 0.0
    return -t * math.log(t) - (1 - t) * math.log(1 - t)


def entropy_bound(s, T, e, dT, S):
    """Fannes-Audenaert with t = 1/2 ||dp||_1 bounded from the per-eigenvalue bound e and the trace bound dT, plus
    the rounding of both entropy sums (device and reference)."""
    d = 1 << s
    rnd = 2 * gamma(d + 8) * (S + 1)
    if T - dT <= 0:
        return math.log(max(d, 2)) + rnd
    t = 0.5 * (d * e + 2 * dT) / (T - dT)
    if d == 1:  # S = 0 exactly; a reference p = lambda / T within 2 t of 1 has -p ln p <= 2 t (1 + 2 t)
        return 2 * t * (1 + 2 * t) + rnd
    if t >= 1 - 1 / d:
        return math.log(d) + rnd
    return t * math.log(d - 1) + binary_entropy(t) + rnd


def sum_sq_bound(s, T, e):
    """|sum lambda_hat^2 - sum lambda^2| for per-eigenvalue errors e (sum |lambda| <= T + d e), plus the sum's rounding."""
    d = 1 << s
    return 2 * (T + d * e) * e + d * e * e + gamma(d) * (T + d * e) ** 2


# ---- closed forms ---------------------------------------------------------------------------------------------------

def geometric_spectrum(d, r):
    """lambda_i = r^i / sum_j r^j, i < d: descending, summing to 1."""
    lam = r ** np.arange(d, dtype=np.float64)
    return lam / lam.sum()


def schmidt_state(n, side, lam, seed):
    """sum_i sqrt(lambda_i) |u_i>_A |v_i>_B with random unitaries on each side (side: qubit list of A; |u_i>, |v_i>
    the columns of Haar-random unitaries restricted to len(lam) vectors).  Returns psi (complex128) with spectrum lam
    on A (zeros padding to 2^|A|)."""
    rng = np.random.default_rng(seed)
    rest = [q for q in range(n) if q not in side]
    dA, dB = 1 << len(side), 1 << len(rest)

    def haar(d):
        z = (rng.normal(size=(d, d)) + 1j * rng.normal(size=(d, d))) / math.sqrt(2)
        q, r = np.linalg.qr(z)
        return q * (np.diag(r) / np.abs(np.diag(r)))

    m = len(lam)
    U, V = haar(dA)[:, :m], haar(dB)[:, :m]
    M = (U * np.sqrt(np.asarray(lam))) @ V.T  # M[a, r] in the side's convention: a bit i <-> side[i]
    t = M.reshape((2,) * (len(side) + len(rest)))  # axes: side[::-1] then rest, both most significant first
    axes = side[::-1] + rest
    psi = np.transpose(t, np.argsort(axes)).reshape(-1)
    return np.ascontiguousarray(psi)
