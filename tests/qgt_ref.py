"""References for the quantum geometric tensor of a Pauli-rotation circuit (State.geometric_tensor,
qipb200_state_pauli_geometric_tensor).  Built on tests/pauli_rot_ref.py (terms, masks, the rotation emulator) and
tests/gradient_ref.py (the walk planner's policy, P psi).

  - plan_policy: (forks, segment sweeps, kernels) by the documented policy of rustqip_b200/csrc/gradient.h.
  - emulate_end_states: the three states the call leaves, bit for bit: state = work_a = the rotation emulator's
    result, work_b = P_(T-1) of it (exact).
  - qgt_ref (long double): the fork and segment algorithm of the call, G and e.
  - qgt_bound: the forward error bound of rustqip_b200/csrc/gradient.cu for G and e, plus the reference's own rounding.
  - closed_form: G and e of gradient_ref.product_ansatz at |0..0>."""
import math

import numpy as np

import gradient_ref as gr
import pauli_rot_ref as rr

U53 = 2.0 ** -53


# ---- the plan ------------------------------------------------------------------------------------------------------

def segment_sweeps(n, terms):
    """Sweeps of one segment: the rotation planner with 6 high tile bits over the terms in order, cut every 256."""
    return gr.adjoint_sweeps(n, list(terms)[::-1]) if terms else 0


def plan_policy(n, ansatz):
    T = len(ansatz)
    S = sum(segment_sweeps(n, ansatz[i + 1:]) for i in range(T))
    return T, S, (T + 2 * S + 1) if T else 0


# ---- the end states ------------------------------------------------------------------------------------------------

def emulate_end_states(psi0, n, ansatz, angles, dtype):
    """(state, work_a, work_b) as the call leaves them (T >= 1), bit for bit up to the sign of zero."""
    st = rr.emulate(psi0, n, ansatz, angles, dtype)
    return st, st.copy(), gr.apply_pauli(st, n, ansatz[-1]).astype(dtype)


# ---- the long-double reference -------------------------------------------------------------------------------------

class _Rotor:
    """exp(-i theta/2 P) and P on clongdouble vectors (several at once, as rows), masks computed once."""

    def __init__(self, n, term):
        x, z, ny = rr.masks(n, term)
        j = np.arange(1 << n, dtype=np.uint64)
        self.p = j ^ np.uint64(x)
        self.sign = np.where(rr._parity(self.p & np.uint64(z)), -1, 1).astype(np.longdouble)
        self.phase = np.clongdouble(1j ** (ny & 3))

    def pauli(self, a):
        return a[..., self.p] * self.sign * self.phase

    def rotate(self, a, theta):
        h = np.longdouble(float(theta)) / 2
        return np.cos(h) * a - 1j * np.sin(h) * self.pauli(a)


def qgt_ref(psi0, n, ansatz, angles):
    """(G, e) in long double (clongdouble (T, T), longdouble (T,)) by the call's algorithm: G_tt = (|psi_t|^2 - e_t^2)/4,
    G_ij = (M_ij - e_i e_j) / 4 for i < j with M_ij = <mu|P_j|phi> after carrying phi = psi_i and mu = P_i psi_i through
    R_(i+1) .. R_(j-1), and G_ji = conj(G_ij)."""
    T = len(ansatz)
    rot = [_Rotor(n, t) for t in ansatz]
    psi = np.asarray(psi0).astype(np.clongdouble)
    G = np.zeros((T, T), dtype=np.clongdouble)
    e = np.zeros(T, dtype=np.longdouble)
    nrm = np.zeros(T, dtype=np.longdouble)
    M = np.zeros((T, T), dtype=np.clongdouble)
    for i in range(T):
        psi = rot[i].rotate(psi, angles[i])
        mu = rot[i].pauli(psi)
        nrm[i] = np.sum(np.abs(psi) ** 2)
        e[i] = np.sum(np.conj(psi) * mu).real
        pair = np.stack([psi, mu])
        for j in range(i + 1, T):
            M[i, j] = np.sum(np.conj(pair[1]) * rot[j].pauli(pair[0]))
            pair = rot[j].rotate(pair, angles[j])
    for i in range(T):
        G[i, i] = (nrm[i] - e[i] * e[i]) / 4
        for j in range(i + 1, T):
            G[i, j] = (M[i, j] - e[i] * e[j]) / 4
            G[j, i] = np.conj(G[i, j])
    return G, e


def qgt_bound(n, T, norm, dtype):
    """(bound on |G_device - G_ref| per entry, bound on |e_device - e_ref|) for psi0 of 2-norm `norm`, to first order.
    After k rotations a device state is within sqrt(2) gamma_(5k)(u) |psi0| of exact (pauli_rot_ref.bound), k <= T for
    psi_t, phi and mu (P is exact).  M_ij, e_t and |psi_t|^2 are inner products of two such states: each errs by
    2 sqrt(2) gamma_(5T)(u) |psi0|^2 plus the double accumulation gamma_D(2^-53) |psi0|^2 (D the summation depth:
    elements per thread, warp, slots over visits, warps, CTAs).  G = (M - e_i e_j) / 4 then errs by at most
    delta (1 + 2 |psi0|^2) / 4 plus the host's three roundings of |psi0|^4-sized values."""
    T = max(1, T)
    N2 = norm * norm
    depth = (1 << n) // 256 + 300
    delta = (2 * math.sqrt(2) * rr.gamma(5 * T, rr.U[dtype]) + rr.gamma(depth, U53)) * N2
    own = rr.gamma(20 * T + 64 * n, rr.U_LONGDOUBLE) * N2 * (1 + N2)
    return delta * (1 + 2 * N2) / 4 + rr.gamma(3, U53) * N2 * N2 + own, delta + own


# ---- closed form ---------------------------------------------------------------------------------------------------

def closed_form(n, theta, phi):
    """(G, e) in long double for psi0 = |0..0> and gradient_ref.product_ansatz(n) (n >= 3): terms 0..n-1 are R_Y(theta_q),
    terms n..2n-1 exp(-i phi_b/2 Z_b Z_(b+1)), indices mod n.  With <Z_q> = cos theta_q on the R_Y layer:
      G_(theta p, theta q) = delta_pq / 4,  e_theta = 0;
      G_(theta b, phi b) = (i/4) sin theta_b cos theta_(b+1),  G_(theta b+1, phi b) = (i/4) cos theta_b sin theta_(b+1),
      other mixed entries 0;
      G_(phi a, phi a) = (1 - cos^2 theta_a cos^2 theta_(a+1)) / 4,
      G_(phi a, phi a+1) = cos theta_a sin^2 theta_(a+1) cos theta_(a+2) / 4, bonds sharing no qubit 0;
      e_(phi b) = cos theta_b cos theta_(b+1)."""
    th = np.asarray(theta, dtype=np.longdouble)
    ct, st = np.cos(th), np.sin(th)
    G = np.zeros((2 * n, 2 * n), dtype=np.clongdouble)
    e = np.zeros(2 * n, dtype=np.longdouble)
    for q in range(n):
        G[q, q] = np.longdouble(0.25)
    for b in range(n):
        b1, b2 = (b + 1) % n, (b + 2) % n
        G[b, n + b] += 0.25j * st[b] * ct[b1]
        G[b1, n + b] += 0.25j * ct[b] * st[b1]
        G[n + b, n + b] = (1 - ct[b] ** 2 * ct[b1] ** 2) / 4
        G[n + b, n + b1] = ct[b] * st[b1] ** 2 * ct[b2] / 4
        e[n + b] = ct[b] * ct[b1]
    for i in range(2 * n):  # the lower triangle (and the adjacent-bond entries of the last bond with the first)
        for j in range(i + 1, 2 * n):
            if G[j, i] != 0 and G[i, j] == 0:
                G[i, j] = np.conj(G[j, i])
            else:
                G[j, i] = np.conj(G[i, j])
    return G, e
