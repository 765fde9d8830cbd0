"""References for the lowest eigenvalue of a real Pauli sum by Lanczos (State.lanczos_pauli_sum,
qipb200_state_lanczos_pauli_sum).  Built on tests/gradient_ref.py and tests/pauli_rot_ref.py: terms, masks and the sum
sweep policy are those of those modules.

  - split: the identity sum a and the scale b = sum |c_h| of the other terms.
  - plan_policy: the kernel counts of rustqip_b200/csrc/lanczos.h restated.
  - emulate: the device arithmetic in numpy, bit for bit, given alpha, beta (and |x| for the normalisation): every
    u_j, every stored w_j, the accumulated x and the state the call leaves (rustqip_b200/csrc/lanczos.cu).
  - lanczos: the whole call with the emulator's vectors and numpy reductions in place of the device's.
  - alpha_beta_bound: the documented first-order bounds of alpha_j and beta_(j+1) given the stored vectors.
  - tfim / tfim_ground: the open transverse-field Ising chain H = -sum J_i Z_iZ_i+1 - sum h_i X_i and its ground
    energy -sum_k sigma_k(M), M bidiagonal with M_ii = h_i, M_i,i+1 = J_i (free fermions).
  - heisenberg: the open XXX chain sum X_iX_i+1 + Y_iY_i+1 + Z_iZ_i+1 (scaled).
  - sparse_h: H as a scipy.sparse matrix, for eigsh."""
import numpy as np
import scipy.sparse

import gradient_ref as gr
import pauli_rot_ref as rr
from rustqip_b200.state import lanczos_ritz

U53 = 2.0 ** -53


def split(terms, coeffs):
    a = b = 0.0
    for t, c in zip(terms, coeffs):
        if len(t) == 0:
            a += float(c)
        else:
            b += abs(float(c))
    return a, b


def plan_policy(n, terms):
    if all(len(t) == 0 for t in terms):
        return 0, 0, 0, 2
    s = gr.sum_sweeps(n, terms)
    return s, s + 1, s + 1, s + 4


def launches(plan, m, vector):
    s, k1, k2, k0 = plan
    return m * k1 + (m - 1) * k2 + k0 if vector else 1 + m * k1


# ---- Hamiltonians ---------------------------------------------------------------------------------------------------

def tfim(J, h):
    n = len(h)
    terms = [[("Z", i), ("Z", i + 1)] for i in range(n - 1)] + [[("X", i)] for i in range(n)]
    return terms, -np.concatenate([np.asarray(J, dtype=np.float64), np.asarray(h, dtype=np.float64)])


def tfim_ground(J, h):
    n = len(h)
    M = np.diag(np.asarray(h, dtype=np.float64)) + np.diag(np.asarray(J, dtype=np.float64), 1) if n > 1 else \
        np.array([[float(h[0])]])
    return -float(np.sum(np.linalg.svd(M, compute_uv=False)))


def heisenberg(n, scale=0.25):
    terms = []
    for i in range(n - 1):
        terms += [[("X", i), ("X", i + 1)], [("Y", i), ("Y", i + 1)], [("Z", i), ("Z", i + 1)]]
    return terms, np.full(len(terms), scale)


def sparse_h(n, terms, coeffs):
    N = 1 << n
    j = np.arange(N, dtype=np.uint64)
    H = scipy.sparse.csr_matrix((N, N), dtype=np.complex128)
    for t, c in zip(terms, coeffs):
        x, z, ny = rr.masks(n, t)
        k = j ^ np.uint64(x)
        val = np.where(rr._parity(k & np.uint64(z)), -1.0, 1.0) * (1j ** (ny & 3)) * float(c)
        H = H + scipy.sparse.csr_matrix((val, (j.astype(np.int64), k.astype(np.int64))), shape=(N, N))
    return H


# ---- the device arithmetic ----------------------------------------------------------------------------------------

class _Tables:
    """Per sweep of the sum plan, per group: (partner index k, [(sign parity of term, nY, coefficient)])."""

    def __init__(self, n, terms, coeffs, qubit_map=None):
        groups, sweeps = gr.sum_plan_policy(n, terms, qubit_map)
        j = np.arange(1 << n, dtype=np.uint64)
        self.rows = []
        for sw in sweeps:
            row = []
            for g in sw:
                x, ts = groups[g]
                k = j ^ np.uint64(x)
                mem = []
                for h in ts:
                    _, z, ny = rr.masks(n, terms[h])
                    mem.append((rr._parity(k & np.uint64(z)), ny, float(coeffs[h])))
                row.append((k, mem))
            self.rows.append(row)


def _sum_step(tab, src, frm, start, scale, R):
    """w = sum_h RN(c_h scale) P_h src + RN(start frm), sweep by sweep, rounded to R at the end of each."""
    n_amp = src[0].shape[0]
    dr = di = None
    for s, row in enumerate(tab.rows):
        if s > 0:
            ar, ai = dr, di
        elif frm is None:
            ar, ai = np.zeros(n_amp), np.zeros(n_amp)
        else:
            ar, ai = start * frm[0], start * frm[1]
        for k, mem in row:
            ca, cb = np.zeros(n_amp), np.zeros(n_amp)
            for par, ny, c in mem:
                cc = scale * c
                cc = cc if (ny & 3) < 2 else -cc
                cv = np.where(par, -cc, cc)
                if ny & 1:
                    cb = cb + cv
                else:
                    ca = ca + cv
            px, py = src[0][k], src[1][k]
            ar = ar + (ca * px - cb * py)
            ai = ai + (ca * py + cb * px)
        dr, di = ar.astype(R).astype(np.float64), ai.astype(R).astype(np.float64)
    return dr, di


def _pair(v, dtype):
    v = np.asarray(v).astype(dtype)
    return v.real.astype(np.float64), v.imag.astype(np.float64)


def _array(p, dtype):
    o = np.empty(p[0].shape[0], dtype=dtype)
    o.real, o.imag = p
    return o


def _step(tab, u, j, alpha, beta, R):
    """(w_j, u_(j+1)) from u = [.., u_(j-1), u_j]."""
    start = 1.0 if j == 0 else -(beta[j] / beta[j - 1])
    w = _sum_step(tab, u[j], u[j - 1] if j else None, start, 1.0 / beta[j], R)
    mu = alpha[j] / beta[j]
    un = ((w[0] - mu * u[j][0]).astype(R).astype(np.float64), (w[1] - mu * u[j][1]).astype(R).astype(np.float64))
    return w, un


def emulate(psi, n, terms, coeffs, dtype, alpha, beta, xnorm=None, qubit_map=None, keep=True):
    """dict(u=[u_0..u_m], w=[w_0..w_(m-1)] (when keep), x=the accumulated x before normalisation, state=the state the
    vector call leaves) for m = len(alpha); needs xnorm (out3[2]) for the state.  Arrays of dtype, bit for bit (up to
    the sign of zero)."""
    R = gr._real_dtype(dtype)
    tab = _Tables(n, terms, coeffs, qubit_map)
    m = len(alpha)
    u, w = [_pair(psi, dtype)], []
    out = {}
    c = []
    if m:
        _, y, _ = lanczos_ritz(alpha, beta[: m + 1])
        c = [y[j] / beta[j] for j in range(m)]
    S = u[0]
    for j in range(m):
        wj, un = _step(tab, u, j, alpha, beta, R)
        if keep:
            w.append(wj)
        # the second pass's accumulation, in the update sweep of step j <= m - 2
        if j <= m - 2 and not (j == 0 and m > 2):
            w0 = 1.0 if j >= 2 else c[0]
            w1 = c[1] if j == 1 else 0.0
            w2 = c[j + 1]
            S = tuple(((w0 * S[q] + w1 * u[j][q]) + w2 * un[q]).astype(R).astype(np.float64) for q in (0, 1))
        u.append(un)
        if not keep and j >= 1:
            u[j - 1] = None
    if keep:
        out["u"] = [_array(p, dtype) for p in u]
        out["w"] = [_array(p, dtype) for p in w]
    if m == 0:
        return out
    out["x"] = _array(S, dtype)
    if xnorm is not None:
        nx = beta[0] if m == 1 else xnorm
        s = 1.0 / nx
        out["state"] = _array(tuple((s * S[q]).astype(R).astype(np.float64) for q in (0, 1)), dtype)
    return out


def lanczos(psi, n, terms, coeffs, dtype, tol, max_steps=300):
    """The call with the emulated vectors and numpy reductions: dict(alpha, beta, steps, converged, theta, estimate,
    state = the normalised x, energy and residual of it in long double)."""
    R = gr._real_dtype(dtype)
    a, b = split(terms, coeffs)
    tab = _Tables(n, terms, coeffs)
    u = [_pair(psi, dtype)]
    beta = [float(np.sqrt(np.sum(u[0][0] ** 2 + u[0][1] ** 2)))]
    alpha = []
    conv, theta, est = False, 0.0, 0.0
    for j in range(max_steps):
        start = 1.0 if j == 0 else -(beta[j] / beta[j - 1])
        w = _sum_step(tab, u[j], u[j - 1] if j else None, start, 1.0 / beta[j], R)
        alpha.append(float(np.sum(u[j][0] * w[0] + u[j][1] * w[1])) / beta[j])
        mu = alpha[j] / beta[j]
        un = ((w[0] - mu * u[j][0]).astype(R).astype(np.float64), (w[1] - mu * u[j][1]).astype(R).astype(np.float64))
        u.append(un)
        beta.append(float(np.sqrt(np.sum(un[0] ** 2 + un[1] ** 2))))
        theta, _, est = lanczos_ritz(alpha, beta)
        if est <= tol * b:
            conv = True
            break
    m = len(alpha)
    xs = emulate(psi, n, terms, coeffs, dtype, np.array(alpha), np.array(beta))
    x = xs["x"].astype(np.clongdouble)
    x = x / np.sqrt(np.sum(np.abs(x) ** 2))
    hx = gr.sum_ref(x, n, terms, coeffs)
    E = np.sum(np.conj(x) * hx).real
    res = float(np.sqrt(np.sum(np.abs(hx - E * x) ** 2)))
    return {"alpha": np.array(alpha), "beta": np.array(beta), "steps": m, "converged": conv, "theta": theta,
            "estimate": est, "energy": float(E), "residual": res}


def depth(n):
    """D of rustqip_b200/csrc/lanczos.cu: the depth of every reduction."""
    return 2 * (((1 << n) + 255) // 256) + 1069


def alpha_beta_bound(n, u_j, w_j, u_next, beta_j):
    """(bound on |alpha_j - Re<u_j|w_j> / beta_j|, bound on |beta_(j+1) - |u_(j+1)||) for stored vectors."""
    g = rr.gamma(depth(n) + 2, U53)
    nu, nw, nn = (float(np.linalg.norm(np.asarray(v).astype(np.complex128))) for v in (u_j, w_j, u_next))
    ld = rr.gamma(8, rr.U_LONGDOUBLE)
    return g * nu * nw / beta_j + ld * nu * nw / beta_j, g * nn + ld * nn
