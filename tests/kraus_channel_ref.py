"""Numpy reference of qipb200_state_apply_kraus_channels (include/qipb200.h): the grouping rule, the grouped sequential
choice, a bit-for-bit emulation of the group sweeps' apply given chosen and cond, a long-double reference of the
conditional probabilities with a bound on the library's error, and dense references.

Operators follow the qip_op MAT convention (the channel's first qubit is the most significant bit of the index);
qubit q is index bit n - 1 - q unless a ``phys`` map says otherwise."""
import numpy as np

from rustqip_b200.channels import KrausChannel

U = 2.0 ** -53
LD = np.clongdouble


def as_kraus(c):
    return c if isinstance(c, KrausChannel) else KrausChannel(c)


def groups(chans):
    """The groups of the state-dependent channels (lists of channel indices): runs of consecutive ones, at most four
    qubits each."""
    out, bits = [], 0
    for c, ch in enumerate(chans):
        ch = as_kraus(ch)
        if ch.state_independent:
            continue
        if not out or bits + ch.n_qubits > 4:
            out.append([])
            bits = 0
        out[-1].append(c)
        bits += ch.n_qubits
    return out


def plan(chans):
    r = len(groups(chans))
    return (r, 1 if r else 0, r, 2 * r + 1 if r else 0)


def choose(e, u):
    """The rule of kraus_choose: the smallest i with u S < cumulative sum, else the last i with e_i > 0."""
    S = 0.0
    for v in e:
        S += v
    t = u * S
    acc = 0.0
    for i, v in enumerate(e):
        acc += v
        if t < acc:
            return i
    pos = [i for i, v in enumerate(e) if v > 0]
    return pos[-1] if pos else 0


def group_rho(psi, n, qubits, dtype=np.complex128):
    """The reduced density matrix of qubits (in order, the first the most significant bit), in dtype's precision."""
    t = np.asarray(psi).astype(dtype).reshape([2] * n)
    t = np.moveaxis(t, list(qubits), list(range(len(qubits)))).reshape(1 << len(qubits), -1)
    return t @ t.conj().T


def numerators(rho, grams, prev, ks_arity, later_bits, dtype=np.complex128):
    """numerator_i = Re Tr[(L (x) M_i (x) I) rho] for every M_i in grams, L = the Kronecker product of prev (the chosen
    M of the group's earlier channels) and I on later_bits low bits.  Negative values clamped to 0."""
    L = np.ones((1, 1), dtype=dtype)
    for m in prev:
        L = np.kron(L, np.asarray(m, dtype=dtype))
    Dx = L.shape[0] << ks_arity
    r = np.asarray(rho, dtype=dtype).reshape(Dx, 1 << later_bits, Dx, 1 << later_bits)
    rp = np.einsum("atbt->ab", r)
    out = []
    for m in grams:
        A = np.kron(L, np.asarray(m, dtype=dtype))
        v = np.sum(A * rp.T).real
        out.append(v if v > 0 else 0 * v)
    return out


def grams_of(ch, dtype=np.complex128):
    ks = np.asarray(as_kraus(ch).kraus).astype(dtype)
    return [k.conj().T @ k for k in ks]


def draw_group(rho, chans, g, draws, dtype=np.complex128):
    """(chosen, cond) of group g's channels from rho by the library's rule, with arithmetic in dtype."""
    arity = [as_kraus(chans[c]).n_qubits for c in g]
    m = sum(arity)
    chosen, cond, prev, s = {}, {}, [], 0
    for c, k in zip(g, arity):
        M = grams_of(chans[c], dtype)
        num = numerators(rho, M, prev, k, m - s - k, dtype)
        S = sum(num)
        if not S > 0:
            return None
        i = choose([float(v) for v in num], float(draws[c]))
        chosen[c], cond[c] = i, num[i] / S
        prev.append(M[i])
        s += k
    return chosen, cond


def scaled(K, p, dtype):
    """K * (1 / sqrt(p)) in double, rounded once to dtype."""
    inv = 1.0 / np.sqrt(np.float64(p))
    K = np.asarray(K, dtype=np.complex128)
    R = np.float32 if dtype == np.complex64 else np.float64
    out = np.empty(K.shape, dtype=dtype)
    out.real = np.multiply(K.real, inv).astype(R)
    out.imag = np.multiply(K.imag, inv).astype(R)
    return out


def apply_op_emulated(psi, n, pos, Kp):
    """The group sweep's matvec of one channel on physical bits pos (the first the most significant), bit for bit:
    products and sums in the state's precision without FMA, columns ascending."""
    k = len(pos)
    D = 1 << k
    idx = np.arange(1 << n, dtype=np.int64)
    mask = sum(1 << p for p in pos)
    base = idx[(idx & mask) == 0]
    offs = [sum(((b >> (k - 1 - i)) & 1) << p for i, p in enumerate(pos)) for b in range(D)]
    x = [psi[base | o] for o in offs]
    out = psi.copy()
    for r in range(D):
        yr = yi = None
        for b in range(D):
            kr, ki = Kp[r, b].real, Kp[r, b].imag
            xr, xi = x[b].real, x[b].imag
            tr = np.subtract(np.multiply(kr, xr), np.multiply(ki, xi))
            ti = np.add(np.multiply(kr, xi), np.multiply(ki, xr))
            if b == 0:
                yr, yi = tr, ti
            else:
                yr, yi = np.add(yr, tr), np.add(yi, ti)
        v = np.empty(base.shape, dtype=psi.dtype)
        v.real, v.imag = yr, yi
        out[base | offs[r]] = v
    return out


def emulate_groups(psi, n, qubit_groups, chans, chosen, cond, phys=None):
    """The state after the group sweeps, given the call's chosen and cond (state-dependent channels only: the
    state-independent ones run through apply_schedule)."""
    phys = phys or (lambda q: n - 1 - q)
    out = np.array(psi, copy=True)
    for g in groups(chans):
        for c in g:
            ch = as_kraus(chans[c])
            Kp = scaled(ch.kraus[chosen[c]], cond[c], out.dtype)
            out = apply_op_emulated(out, n, [phys(q) for q in qubit_groups[c]], Kp)
    return out


def reference_conds(psi, n, qubit_groups, chans, chosen, cond, draws):
    """[(c, cond_ld, choice_ld, dist, bound)] for every state-dependent channel c, from the emulated states in long
    double: the conditional probability of the call's choice, the choice the long-double numerators give, the distance
    of the draw from the nearest cumulative boundary, and the bound on the library's error in cond."""
    out, cur = [], np.array(psi, copy=True)
    for g in groups(chans):
        qs = [q for c in g for q in qubit_groups[c]]
        rho = group_rho(cur, n, qs, LD)
        tr = float(np.trace(rho).real)
        arity = [as_kraus(chans[c]).n_qubits for c in g]
        m, prev, s = sum(arity), [], 0
        rows = 1 << (n - m)
        for c, k in zip(g, arity):
            M = grams_of(chans[c], LD)
            num = numerators(rho, M, prev, k, m - s - k, LD)
            S = sum(num)
            i = int(chosen[c])
            cum = np.cumsum(np.array(num, dtype=np.longdouble)) / S
            u = np.longdouble(draws[c])
            dist = float(np.min(np.abs(cum - u)))
            ref_choice = int(np.searchsorted(cum, u, side="right"))
            # |d rho_ab| <= gamma_T sqrt(2) Tr rho (T: the longest chain of the device sums), the host's sums of at most
            # 4^(s + k) + 2^rest products of three factors a few more u; a numerator moves by at most ||L (x) M_i||_1
            # times that, S by the sum over i, and cond = num / S by (|d num| + cond |d S|) / S.
            L = np.ones((1, 1), dtype=LD)
            for mm in prev:
                L = np.kron(L, mm)
            norm1 = [float(np.sum(np.abs(np.kron(L, mi)))) for mi in M]
            chain = rows + 4096 + 264 + (1 << (2 * m)) + 16
            e_entry = 2.0 * chain * U * tr
            d_num = [v * e_entry for v in norm1]
            bound = 2.0 * (d_num[i] + float(num[i] / S) * sum(d_num)) / float(S)
            out.append((c, float(num[i] / S), ref_choice, dist, bound))
            prev.append(M[i])
            s += k
        for c in g:
            Kp = scaled(as_kraus(chans[c]).kraus[chosen[c]], cond[c], cur.dtype)
            cur = apply_op_emulated(cur, n, [n - 1 - q for q in qubit_groups[c]], Kp)
    return out


# ---- exact channel action (dense, for the enumeration checks) ------------------------------------------------------

def apply_dense(psi, n, qubit_groups, ops):
    """(x)_c K_c psi with qubit q on index bit n - 1 - q."""
    t = np.asarray(psi, dtype=np.complex128).reshape([2] * n)
    for g, k in zip(qubit_groups, ops):
        m = len(g)
        K = np.asarray(k, dtype=np.complex128).reshape([2] * (2 * m))
        t = np.tensordot(K, t, axes=(list(range(m, 2 * m)), list(g)))
        t = np.moveaxis(t, list(range(m)), list(g))
    return t.reshape(-1)


def stinespring(k, m, rng):
    """m Kraus operators of a random channel on k qubits: blocks of a random isometry C^(2^k) -> C^(m 2^k)."""
    D = 1 << k
    a = rng.normal(size=(m * D, D)) + 1j * rng.normal(size=(m * D, D))
    q, _ = np.linalg.qr(a)
    return KrausChannel([q[i * D:(i + 1) * D, :] for i in range(m)])


def trajectory_step(psi, n, qubit_groups, chans, tup):
    """(probability by the grouped sequential rule, post-state) of the outcome tuple tup, exactly as the library draws
    it (state-independent channels from their weights), in double from dense states."""
    cur = np.array(psi, dtype=np.complex128)
    p = 1.0
    for g in groups(chans):
        qs = [q for c in g for q in qubit_groups[c]]
        rho = group_rho(cur, n, qs)
        arity = [as_kraus(chans[c]).n_qubits for c in g]
        m, prev, s = sum(arity), [], 0
        for c, k in zip(g, arity):
            M = grams_of(chans[c])
            num = numerators(rho, M, prev, k, m - s - k)
            cnd = num[tup[c]] / sum(num)
            p *= cnd
            if cnd == 0:
                return 0.0, None
            prev.append(M[tup[c]])
            s += k
        ops = [as_kraus(chans[c]).kraus[tup[c]] for c in g]
        cur = apply_dense(cur, n, [qubit_groups[c] for c in g], ops)
        cur = cur / np.sqrt(np.vdot(cur, cur).real) * np.sqrt(np.vdot(psi, psi).real)
    for c, ch in enumerate(chans):
        ch = as_kraus(ch)
        if ch.state_independent:
            w = ch.weights[tup[c]]
            p *= w
            cur = apply_dense(cur, n, [qubit_groups[c]], [ch.kraus[tup[c]] / np.sqrt(w)])
    return p, cur
