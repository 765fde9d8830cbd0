"""References for Pauli sums and the adjoint energy gradient (State.apply_pauli_sum, State.energy_gradient;
qipb200_state_apply_pauli_sum, qipb200_state_pauli_energy_gradient).  Built on tests/pauli_rot_ref.py: terms, masks and
the rotation emulator are those of that module.

  - sum_plan_policy: the documented sweep policy of rustqip_b200/csrc/gradient.h, independently of the library.
  - emulate_sum: the device arithmetic of apply_pauli_sum in numpy, bit for bit (it follows the plan: per amplitude the
    groups in sweep order, a double sum per sweep, rounded to the state's precision at the end of each sweep).
  - sum_ref (long double) and sum_bound: per amplitude |dst_j - (H src)_j| <= 2 (gamma_(T+G+2)(2^-53) + gamma_S(u)) A_j
    with A_j = sum_h |c_h| |src_(j^x_h)| (T terms, G groups, S sweeps), plus the reference's own rounding.
  - emulate_gradient: the states the gradient call leaves, bit for bit: the rotation emulator forward, emulate_sum,
    then per term, last first, the rotation update with the host-rounded c and the negated s on both states.
  - adjoint_ref: energy and gradient in long double, and grad_bound: their distance from the device, to first order.
  - closed_form: the product ansatz of the full-size tests (R_Y on every qubit, then Z_iZ_i+1 rotations on the ring)
    with H = sum a_i X_i + b_i Z_i + c_i Z_iZ_i+1: energy and analytic gradient."""
import math

import numpy as np

import pauli_rot_ref as rr

U53 = 2.0 ** -53


# ---- the sweep policy of apply_pauli_sum ---------------------------------------------------------------------------

def _phys(n, x, qubit_map):
    """A logical index-bit mask on the physical bits of a layout (qubit_map[q] = physical bit of qubit q)."""
    if qubit_map is None:
        return x
    return sum(1 << int(qubit_map[q]) for q in range(n) if (x >> (n - 1 - q)) & 1)


def sum_plan_policy(n, terms, qubit_map=None):
    """(groups, sweeps): groups[g] = (x mask, [term indices]) in order of first appearance, sweeps = [[group indices]].
    The library plans on physical index bits, so a permuted layout (qubit_map, as State.qubit_map) may split the groups
    differently."""
    L = min(4, n)
    m = min(6, n - L)
    low = (1 << L) - 1
    groups, where = [], {}
    for t, term in enumerate(terms):
        x, _, _ = rr.masks(n, term)
        if x not in where:
            where[x] = len(groups)
            groups.append((x, []))
        groups[where[x]][1].append(t)
    used = [False] * len(groups)
    sweeps = []
    while not all(used):
        hi = x_out = 0
        taken = []
        for g, (x, _) in enumerate(groups):
            if used[g]:
                continue
            r = _phys(n, x, qubit_map) & ~(low | hi)
            if r == 0 or r == x_out:
                pass
            elif not (r & x_out) and bin(hi).count("1") + bin(r).count("1") <= m:
                hi |= r
            elif x_out == 0:
                x_out = r
            else:
                continue
            used[g] = True
            taken.append(g)
        sweeps.append(taken)
    return groups, sweeps


def sum_sweeps(n, terms):
    return len(sum_plan_policy(n, terms)[1])


def adjoint_sweeps(n, ansatz):
    """Backward sweeps: the rotation planner with 6 high tile bits over the reversed list, cut every 256 terms."""
    L = min(4, n)
    m = min(6, n - L)
    low = (1 << L) - 1
    if not ansatz:
        return 1
    count, size = 0, 0
    hi = x_out = 0
    for term in ansatz[::-1]:
        x, _, _ = rr.masks(n, term)
        r = x & ~(low | hi)
        joins = count > 0
        if joins and not (r == 0 or r == x_out):
            if not (r & x_out) and bin(hi).count("1") + bin(r).count("1") <= m:
                hi |= r
            elif x_out == 0:
                x_out = r
            else:
                joins = False
        if not joins:
            count += 1
            size = 0
            hi = x_out = 0
            r = x & ~low
            if bin(r).count("1") <= m:
                hi = r
            else:
                x_out = r
        if size == 256:
            count += 1
            size = 0
        size += 1
    return count


def gradient_plan_policy(n, ansatz, ham):
    return rr.plan_policy(n, ansatz), sum_sweeps(n, ham), adjoint_sweeps(n, ansatz)


# ---- apply_pauli_sum -----------------------------------------------------------------------------------------------

def _real_dtype(dtype):
    return np.float64 if np.dtype(dtype) == np.complex128 else np.float32


def emulate_sum(src, n, terms, coeffs, dtype, qubit_map=None):
    """The device's dst, bit for bit (up to the sign of zero), as an array of dtype, for a source in the layout
    qubit_map (None: canonical)."""
    R = _real_dtype(dtype)
    src = np.asarray(src).astype(dtype)
    pr, pi = src.real.astype(np.float64), src.imag.astype(np.float64)
    j = np.arange(1 << n, dtype=np.uint64)
    groups, sweeps = sum_plan_policy(n, terms, qubit_map)
    acc_r = np.zeros(1 << n)
    acc_i = np.zeros(1 << n)
    for sw in sweeps:
        for g in sw:
            x, ts = groups[g]
            k = j ^ np.uint64(x)
            a = np.zeros(1 << n)
            b = np.zeros(1 << n)
            for t in ts:
                _, z, ny = rr.masks(n, terms[t])
                c = float(coeffs[t]) if (ny & 3) < 2 else -float(coeffs[t])
                cv = np.where(rr._parity(k & np.uint64(z)), -c, c)
                if ny & 1:
                    b = b + cv
                else:
                    a = a + cv
            px, py = pr[k], pi[k]
            acc_r = acc_r + (a * px - b * py)
            acc_i = acc_i + (a * py + b * px)
        acc_r = acc_r.astype(R).astype(np.float64)
        acc_i = acc_i.astype(R).astype(np.float64)
    out = np.empty(1 << n, dtype=dtype)
    out.real, out.imag = acc_r, acc_i
    return out


def apply_pauli(a, n, term):
    """P a for one Pauli string, in the precision of a."""
    x, z, ny = rr.masks(n, term)
    j = np.arange(1 << n, dtype=np.uint64)
    p = j ^ np.uint64(x)
    pa = np.where(rr._parity(p & np.uint64(z)), -a[p], a[p])
    return pa * a.dtype.type(1j ** (ny & 3))


def sum_ref(src, n, terms, coeffs):
    """H src in long double (clongdouble array)."""
    a = np.asarray(src).astype(np.clongdouble)
    out = np.zeros(1 << n, dtype=np.clongdouble)
    for t, c in zip(terms, coeffs):
        out += np.longdouble(float(c)) * apply_pauli(a, n, t)
    return out


def sum_weights(src, n, terms, coeffs):
    """A_j = sum_h |c_h| |src_(j^x_h)| (float64)."""
    a = np.abs(np.asarray(src).astype(np.complex128))
    j = np.arange(1 << n, dtype=np.uint64)
    w = np.zeros(1 << n)
    for t, c in zip(terms, coeffs):
        x, _, _ = rr.masks(n, t)
        w += abs(float(c)) * a[j ^ np.uint64(x)]
    return w


def sum_bound(n, terms, dtype):
    """The factor K of |dst_j - sum_ref_j| <= K A_j."""
    groups, sweeps = sum_plan_policy(n, terms)
    T = len(terms)
    return 2 * (rr.gamma(T + len(groups) + 2, U53) + rr.gamma(max(1, len(sweeps)), rr.U[dtype])) + \
        2 * rr.gamma(4 * T + 4, rr.U_LONGDOUBLE)


# ---- the gradient --------------------------------------------------------------------------------------------------

def undo_step(re, im, n, term, th, R):
    """One R_t^dagger on (re, im) as the device does it: c and -s from the host's cos and sin, rounded to R."""
    x, z, ny = rr.masks(n, term)
    c, s = R(math.cos(float(th) / 2)), -R(math.sin(float(th) / 2))
    j = np.arange(1 << n, dtype=np.uint64)
    p = j ^ np.uint64(x)
    neg = rr._parity(p & np.uint64(z))
    wr, wi = rr._times_i_power(ny + 3, re[p], im[p])
    wr, wi = np.where(neg, -wr, wr), np.where(neg, -wi, wi)
    return c * re + s * wr, c * im + s * wi


def emulate_gradient(psi0, n, ansatz, angles, ham, coeffs, dtype, qubit_map=None):
    """(state, work) as the gradient call leaves them, bit for bit (up to the sign of zero), for a state in the layout
    qubit_map (None: canonical)."""
    R = _real_dtype(dtype)
    fwd = rr.emulate(psi0, n, ansatz, angles, dtype)
    lam = emulate_sum(fwd, n, ham, coeffs, dtype, qubit_map)
    pr, pi = fwd.real.astype(R), fwd.imag.astype(R)
    lr, li = lam.real.astype(R), lam.imag.astype(R)
    for t in range(len(ansatz) - 1, -1, -1):
        pr, pi = undo_step(pr, pi, n, ansatz[t], angles[t], R)
        lr, li = undo_step(lr, li, n, ansatz[t], angles[t], R)
        assert pr.dtype == R and lr.dtype == R
    st, wk = np.empty(1 << n, dtype=dtype), np.empty(1 << n, dtype=dtype)
    st.real, st.imag = pr, pi
    wk.real, wk.imag = lr, li
    return st, wk


def adjoint_ref(psi0, n, ansatz, angles, ham, coeffs):
    """(E, grad) in long double by the adjoint method: grad[t] = Im <lambda|P_t|phi> before term t is undone."""
    phi = rr.rotate_ref(psi0, n, ansatz, angles)
    lam = sum_ref(phi, n, ham, coeffs)
    energy = np.sum(np.conj(lam) * phi).real
    grad = np.zeros(len(ansatz), dtype=np.longdouble)
    for t in range(len(ansatz) - 1, -1, -1):
        grad[t] = np.sum(np.conj(lam) * apply_pauli(phi, n, ansatz[t])).imag
        phi = rr.rotate_ref(phi, n, [ansatz[t]], [-float(angles[t])])
        lam = rr.rotate_ref(lam, n, [ansatz[t]], [-float(angles[t])])
    return energy, grad


def grad_bound(n, ansatz, ham, coeffs, norm, dtype):
    """|device - adjoint_ref| for the energy and every grad[t], to first order.  phi carries at most
    sqrt(2) gamma_(5k)(u) |psi0| after k rotations (pauli_rot_ref.bound, a 2-norm bound), k <= 2T; lambda = H phi adds
    sum_bound's factor times S |psi0| (S = sum |c_h| >= |H|) and, through H, S times phi's error; the undo adds
    sqrt(2) gamma_(5T) S |psi0| to lambda.  Each inner product then errs by |d lambda| |psi0| + S |psi0| |d phi| plus its
    own double rounding, gamma_D(2^-53) S |psi0|^2 with D the summation depth (elements per thread, warp, CTA, grid)."""
    T = max(1, len(ansatz))
    S = sum(abs(float(c)) for c in coeffs)
    u = rr.U[dtype]
    depth = (1 << n) // 256 + 300
    k = 3 * math.sqrt(2) * rr.gamma(10 * T, u) + sum_bound(n, ham, dtype) + rr.gamma(depth, U53)
    k += rr.gamma(20 * T + 8 * len(ham) + 64 * n, rr.U_LONGDOUBLE)
    return k * S * norm * norm


# ---- closed form ---------------------------------------------------------------------------------------------------

def product_ansatz(n):
    """R_Y(theta_i) on every qubit, then exp(-i phi_i/2 Z_i Z_i+1) for the ring bonds (i, i+1 mod n); n >= 3."""
    return [[("Y", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]


def product_hamiltonian(n, a, b, c):
    terms = [[("X", i)] for i in range(n)] + [[("Z", i)] for i in range(n)]
    terms += [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]
    return terms, np.concatenate([a, b, c]).astype(np.float64)


def closed_form(n, theta, phi, a, b, c):
    """(E, dE/dtheta, dE/dphi) in long double for psi0 = |0..0>, the product ansatz and H = sum a_i X_i + b_i Z_i +
    c_i Z_iZ_i+1:  <Z_i> = cos theta_i, <Z_iZ_i+1> = cos theta_i cos theta_i+1 and
    <X_i> = sin theta_i (cos phi_i-1 cos phi_i - sin phi_i-1 sin phi_i cos theta_i-1 cos theta_i+1)."""
    th = np.asarray(theta, dtype=np.longdouble)
    ph = np.asarray(phi, dtype=np.longdouble)
    a, b, c = (np.asarray(v, dtype=np.longdouble) for v in (a, b, c))
    ct, st = np.cos(th), np.sin(th)
    cp, sp = np.cos(ph), np.sin(ph)
    m, p = np.roll(np.arange(n), 1), np.roll(np.arange(n), -1)  # i - 1, i + 1
    A = cp[m] * cp  # cos phi_i-1 cos phi_i
    B = sp[m] * sp
    X = st * (A - B * ct[m] * ct[p])
    E = np.sum(a * X) + np.sum(b * ct) + np.sum(c * ct * ct[p])
    # d/dtheta_k: X_k through sin theta_k; X_k+1 and X_k-1 through cos theta_k; the Z and ZZ terms
    gt = a * ct * (A - B * ct[m] * ct[p])
    gt += a[p] * st[p] * B[p] * ct[np.roll(np.arange(n), -2)] * st
    gt += a[m] * st[m] * B[m] * ct[np.roll(np.arange(n), 2)] * st
    gt += -b * st - c * st * ct[p] - c[m] * ct[m] * st
    # d/dphi_k: phi_k is the second bond of qubit k and the first of qubit k + 1
    gp = a * st * (-cp[m] * sp - sp[m] * cp * ct[m] * ct[p])
    gp += a[p] * st[p] * (-sp * cp[p] - cp * sp[p] * ct * ct[np.roll(np.arange(n), -2)])
    return E, gt, gp
