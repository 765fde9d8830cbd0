"""References for exp(-iHt) by a Chebyshev series (State.evolve_pauli_sum, qipb200_state_evolve_pauli_sum).  Built on
tests/gradient_ref.py and tests/pauli_rot_ref.py: terms, masks and the sum sweep policy are those of those modules.

  - split: the identity sum a, the half-width b = sum |c_h| of the other terms, and those terms.
  - degree_policy: the smallest k >= 2 whose tail bound tau_k = 2 sum_(j > k) |J_j(bt)| is <= tol, from scipy.
  - cheb_ref: the series sum_k C_k T_k(H~) psi in long double with the library's coefficients C_k.
  - emulate: the device arithmetic in numpy, bit for bit (rustqip_b200/csrc/gradient.cu, "evolution mode").
  - bound: the documented forward rounding-error bound of the device result from cheb_ref, in 2-norm."""
import math

import numpy as np
import scipy.special

import gradient_ref as gr
import pauli_rot_ref as rr
from rustqip_b200.state import pauli_evolution_plan

U53 = 2.0 ** -53


def split(terms, coeffs):
    """(a, b, non-identity terms, their coefficients), a and b added in list order from +0.0 in double."""
    a = b = 0.0
    nt, nc = [], []
    for t, c in zip(terms, coeffs):
        if len(t) == 0:
            a += float(c)
        else:
            nt.append(t)
            nc.append(float(c))
            b += abs(float(c))
    return a, b, nt, nc


def tails(x, kmax):
    """tau_k = 2 sum_(j > k) |J_j(x)| for k = 0..kmax, from scipy.special.jv (summed far past kmax)."""
    top = int(kmax + 60 + 4 * abs(x) ** (1 / 3.0))
    j = np.abs(scipy.special.jv(np.arange(top + 1), abs(x)))
    suffix = np.cumsum(j[::-1])[::-1]  # suffix[k] = sum_(j >= k)
    return 2 * np.append(suffix[1:], 0.0)[: kmax + 1]


def degree_policy(x, tol):
    tau = tails(x, int(abs(x) + 200 + 20 * abs(x) ** (1 / 3.0)))
    k = 2
    while tau[k] > tol:
        k += 1
    return k, tau


def series_coeffs(a, b, t, K):
    """C_k = (2 - delta_k0) (-i)^k J_k(RN(b t)) e^{-i RN(a t)} from scipy."""
    k = np.arange(K + 1)
    x = b * t
    return np.where(k == 0, 1, 2) * (-1j) ** k * scipy.special.jv(k, x) * np.exp(-1j * (a * t))


def plan(n, dtype, terms, coeffs, t, tol):
    return pauli_evolution_plan(n, dtype, terms, coeffs, t, tol)


def cheb_ref(psi, n, terms, coeffs, t, C):
    """sum_k C_k T_k(H~) psi in long double, H~ = (H - a) / b, for the library's C (complex128 array)."""
    a, b, nt, nc = split(terms, coeffs)
    p = np.asarray(psi).astype(np.clongdouble)
    K = len(C) - 1
    if K == 0:
        return np.clongdouble(C[0]) * p
    bl = np.longdouble(b)

    def ht(v):
        return gr.sum_ref(v, n, nt, nc) / bl

    prev, cur = p, ht(p)
    out = np.clongdouble(C[0]) * prev + np.clongdouble(C[1]) * cur
    for k in range(2, K + 1):
        prev, cur = cur, 2 * ht(cur) - prev
        out = out + np.clongdouble(C[k]) * cur
    return out


def _cmul(cr, ci, xr, xi):
    return cr * xr - ci * xi, cr * xi + ci * xr


def emulate(psi, n, terms, coeffs, t, tol, dtype, qubit_map=None):
    """The state the device leaves, bit for bit (up to the sign of zero), for a state in the layout qubit_map (None:
    canonical).  Per step k and sweep of the sum plan, in double with every operation rounded: the accumulator starts
    at 0 (step 1), -state (step 2) or -T_(k-2) (k >= 3) in the first sweep and at the stored partial in later ones,
    adds each group's (a p.x - b p.y, a p.y + b p.x) in sweep order and is stored rounded to the state's precision;
    the last sweep then sets S <- (C_0 S + C_1 T_1) + C_2 T_2 (step 2) or S <- S + C_k T_k (k >= 3)."""
    R = gr._real_dtype(dtype)
    K, _, _, _, C = plan(n, dtype, terms, coeffs, t, tol)
    psi = np.asarray(psi).astype(dtype)
    sr, si = psi.real.astype(np.float64), psi.imag.astype(np.float64)

    def rnd(v):
        return v.astype(R).astype(np.float64)

    def out(re, im):
        o = np.empty(1 << n, dtype=dtype)
        o.real, o.imag = re, im
        return o

    if K == 0:
        a, b, _, _ = split(terms, coeffs)
        if t == 0 or not terms:
            return psi.copy()
        return rr.emulate(psi, n, [[]], [2.0 * (a * t)], dtype)  # identity only: the empty-term rotation
    a, b, nt, nc = split(terms, coeffs)
    groups, sweeps = gr.sum_plan_policy(n, nt, qubit_map)
    j = np.arange(1 << n, dtype=np.uint64)
    tables = []  # per scale: per sweep, per group (partner index, a, b)
    for scale in (1.0 / b, 2.0 / b):
        tab = []
        for sw in sweeps:
            row = []
            for g in sw:
                x, ts = groups[g]
                k = j ^ np.uint64(x)
                ca = np.zeros(1 << n)
                cb = np.zeros(1 << n)
                for h in ts:
                    _, z, ny = rr.masks(n, nt[h])
                    c = scale * nc[h]
                    c = c if (ny & 3) < 2 else -c
                    cv = np.where(rr._parity(k & np.uint64(z)), -c, c)
                    if ny & 1:
                        cb = cb + cv
                    else:
                        ca = ca + cv
                row.append((k, ca, cb))
            tab.append(row)
        tables.append(tab)
    Cr, Ci = C.real, C.imag
    T = {0: (sr, si)}
    for step in range(1, K + 1):
        src = T[step - 1]
        tab = tables[0 if step == 1 else 1]
        for s, row in enumerate(tab):
            if s > 0:
                ar, ai = dr, di
            elif step == 1:
                ar, ai = np.zeros(1 << n), np.zeros(1 << n)
            else:
                pr_, pi_ = T[step - 2]
                ar, ai = -pr_, -pi_
            for k, ca, cb in row:
                px, py = src[0][k], src[1][k]
                ar = ar + (ca * px - cb * py)
                ai = ai + (ca * py + cb * px)
            dr, di = rnd(ar), rnd(ai)
        T[step] = (dr, di)
        T.pop(step - 2, None)
        if step == 2:
            r0 = _cmul(Cr[0], Ci[0], sr, si)
            r1 = _cmul(Cr[1], Ci[1], T[1][0], T[1][1])
            r2 = _cmul(Cr[2], Ci[2], dr, di)
            sr, si = rnd((r0[0] + r1[0]) + r2[0]), rnd((r0[1] + r1[1]) + r2[1])
        elif step >= 3:
            r = _cmul(Cr[step], Ci[step], dr, di)
            sr, si = rnd(sr + r[0]), rnd(si + r[1])
    return out(sr, si)


def bound(n, terms, coeffs, C, dtype, norm):
    """The forward bound of rustqip_b200/csrc/gradient.cu: |device - cheb_ref| (2-norm) for a start state of 2-norm
    norm, plus cheb_ref's own long-double rounding."""
    K = len(C) - 1
    if K == 0:
        return rr.bound(1, norm, dtype)
    _, _, nt, _ = split(terms, coeffs)
    groups, sweeps = gr.sum_plan_policy(n, nt)
    u = rr.U[dtype]
    delta = 2 * (rr.gamma(len(nt) + len(groups) + 4, U53) + rr.gamma(len(sweeps), u))
    ab = np.abs(np.asarray(C))
    k = np.arange(K + 1)
    csum = float(np.sum(ab))
    rec = 3 * delta * float(np.sum(ab * k * (k + 1) / 2))
    acc = math.sqrt(2) * (2 * rr.gamma(4, U53) + u) * K * csum
    grow = 1 + 3 * delta * K * (K + 1) / 2
    ld = rr.gamma((K + 1) * (len(nt) + 4), rr.U_LONGDOUBLE) * K * K * csum
    return (rec + acc) * grow * norm + ld * norm


def exact_allowance(terms, coeffs, t, C, norm):
    """What separates cheb_ref from exp(-iHt) psi besides the tail: the coefficients' rounding (~1e-16 each, counted
    as 1e-15) and the rounding of b t and a t."""
    a, b, _, _ = split(terms, coeffs)
    csum = float(np.sum(np.abs(np.asarray(C))))
    return (len(C) * 1e-15 + 4 * U53 * (abs(a * t) + abs(b * t)) * csum) * norm
