"""Numpy emulation of qipb200_state_apply_channels (include/qipb200.h), bit for bit, and a long-double reference of its
weight sweep with the first-order bound of rustqip_b200/csrc/channel.cu.

`emulate` takes the state, the channels, x (what State.sample returns for draws[0] over the state-dependent qubits)
and the draws, and reproduces the choices, q (the weight kernel's summation order included), prob and the new state.
"""
import numpy as np

U = 2.0 ** -53
GRID, THREADS, PER = 264, 256, 8
CHUNK = THREADS * PER


def monomial(k):
    """(flip, d) of a diagonal or anti-diagonal operator: K|b> = d[b] |b ^ flip>."""
    k = np.asarray(k, dtype=np.complex128)
    flip = not (k[0, 1] == 0 and k[1, 0] == 0)
    return flip, ((complex(k[1, 0]), complex(k[0, 1])) if flip else (complex(k[0, 0]), complex(k[1, 1])))


def weight(d):
    """|d|^2 = re^2 + im^2 in double, as the library computes it."""
    return d.real * d.real + d.imag * d.imag


def weights(k):
    return [weight(d) for d in monomial(k)[1]]


def state_dependent(ks):
    return any(e[0] != e[1] for e in map(weights, ks))


def choose(ks, b, u):
    e = [weights(k)[b] for k in ks]
    S = 0.0
    for v in e:
        S += v
    t = u * S
    acc = 0.0
    for i, v in enumerate(e):
        acc += v
        if t < acc:
            return i
    return max(i for i, v in enumerate(e) if v > 0)


def scaled_identity(k):
    flip, d = monomial(k)
    return (not flip) and d[0] == d[1] and d[0].imag == 0 and d[0].real > 0


def plan(chans):
    sd = sum(1 for ks in chans if state_dependent(ks))
    rw = any(not scaled_identity(k) for ks in chans for k in ks)
    return (sd, 3 if sd else 0, int(rw), (11 if sd else 0) + int(rw))


def cmul(ar, ai, br, bi):
    """Complex product in double, each product and sum rounded once (scalars or arrays)."""
    return np.subtract(np.multiply(ar, br), np.multiply(ai, bi)), np.add(np.multiply(ar, bi), np.multiply(ai, br))


def tables(pos, ops):
    """[(byte, d re[256], d im[256], e[256])] of the chosen operators ops on physical bits pos, and F."""
    F = 0
    for p, k in zip(pos, ops):
        if monomial(k)[0]:
            F |= 1 << p
    out = []
    for byte in range(5):
        bits = sorted((p, i) for i, p in enumerate(pos) if p // 8 == byte)  # ascending bit order
        if not bits:
            continue
        dr, di, ee = np.zeros(256), np.zeros(256), np.zeros(256)
        for v in range(256):
            r = i_ = e = None
            for m, (p, i) in enumerate(bits):
                b = (v >> (p % 8)) & 1
                d = monomial(ops[i])[1][b]
                w = weight(d)
                if m == 0:
                    r, i_, e = d.real, d.imag, w
                else:
                    r, i_ = (r * d.real - i_ * d.imag, r * d.imag + i_ * d.real)
                    e = e * w
            dr[v], di[v], ee[v] = r, i_, e
        out.append((byte, dr, di, ee))
    return out, F


def _byte(idx, byte):
    return ((idx >> np.uint64(8 * byte)) & np.uint64(255)).astype(np.int64)


def weight_sums(psi, n, tabs):
    """(S, N) of the weight kernel, in its order of summation."""
    N = 1 << n
    idx = np.arange(N, dtype=np.uint64)
    w = tabs[0][3][_byte(idx, tabs[0][0])]
    for byte, _, _, e in tabs[1:]:
        w = np.multiply(w, e[_byte(idx, byte)])
    a = psi.astype(np.complex128)
    p = np.add(np.multiply(a.real, a.real), np.multiply(a.imag, a.imag))
    term = np.multiply(p, w)
    C = min(N, CHUNK)
    V = N // C
    res = []
    for vals in (term, p):
        acc = np.zeros((GRID, THREADS))
        for r in range((V + GRID - 1) // GRID):
            chunks = r * GRID + np.arange(GRID)
            for k in range(PER):
                e = np.arange(THREADS) + THREADS * k
                ok = (chunks[:, None] < V) & (e[None, :] < C)
                j = np.where(ok, chunks[:, None] * C + e[None, :], 0)
                acc = np.where(ok, np.add(acc, vals[j]), acc)
        acc = acc.reshape(GRID, THREADS // 32, 32)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            acc = np.add(acc, acc[:, :, lane ^ o])
        s = acc[:, 0, 0].copy()
        for wp in range(1, THREADS // 32):
            s = np.add(s, acc[:, wp, 0])
        tot = 0.0
        for g in range(GRID):
            tot += float(s[g])
        res.append(tot)
    return res[0], res[1]


def emulate(psi, n, qubits, chans, x, draws, phys=None):
    """(chosen, prob, new state) of the call.  phys(q) is the physical bit of qubit q (n - 1 - q by default); x holds
    the state-dependent qubits' values in channel order (bit k for the k-th)."""
    phys = phys or (lambda q: n - 1 - q)
    chosen, rest_pos, rest_ops = [], [], []
    dropped, uniform, nonuniform, kd = 1.0, 1.0, False, 0
    for c, (q, ks) in enumerate(zip(qubits, chans)):
        if state_dependent(ks):
            b = (int(x) >> kd) & 1
            kd += 1
        else:
            b = 0
        i = choose(ks, b, float(draws[1 + c]))
        chosen.append(i)
        k = ks[i]
        e = weights(k)
        if scaled_identity(k):
            dropped *= e[0]
            continue
        rest_pos.append(phys(q))
        rest_ops.append(k)
        if e[0] != e[1]:
            nonuniform = True
        else:
            uniform *= e[0]
    if not rest_ops:
        return chosen, dropped, psi.copy()
    tabs, F = tables(rest_pos, rest_ops)
    q = uniform
    if nonuniform:
        S, N = weight_sums(psi, n, tabs)
        q = S / N if N > 0 else 0.0
    prob = q * dropped
    if not q > 0:
        return chosen, prob, psi.copy()
    idx = np.arange(1 << n, dtype=np.uint64)
    out = np.empty_like(psi)
    out[(idx ^ np.uint64(F)).astype(np.int64)] = moved(psi, idx, tabs, 1.0 / np.sqrt(q))
    return chosen, prob, out


def moved(src, idx, tabs, inv):
    """W(j) psi_j for the amplitudes src at indices idx: the value the apply writes to j ^ F."""
    wr, wi = tabs[0][1][_byte(idx, tabs[0][0])], tabs[0][2][_byte(idx, tabs[0][0])]
    for byte, dr, di, _ in tabs[1:]:
        b = _byte(idx, byte)
        wr, wi = cmul(wr, wi, dr[b], di[b])
    wr, wi = np.multiply(wr, inv), np.multiply(wi, inv)
    R = np.float32 if src.dtype == np.complex64 else np.float64
    wr, wi = wr.astype(R), wi.astype(R)
    a, b = src.real.astype(R), src.imag.astype(R)
    out = np.empty_like(src)
    out.real = np.subtract(np.multiply(wr, a), np.multiply(wi, b))
    out.imag = np.add(np.multiply(wr, b), np.multiply(wi, a))
    return out


# ---- long-double reference of the weight sweep and its bound ------------------------------------------------------

def chain(n):
    """D: the longest chain of additions of the weight kernel's sums."""
    N = 1 << n
    C = min(N, CHUNK)
    V = N // C
    return 8 * -(-V // GRID) + 5 + 7 + (GRID - 1)


def weight_reference(psi, n, pos, ops):
    """(S, N) in long double from the state's amplitudes and the per-bit weights |d|^2 (doubles)."""
    idx = np.arange(1 << n, dtype=np.uint64)
    w = np.ones(1 << n, dtype=np.longdouble)
    for p, k in zip(pos, ops):
        e = np.array(weights(k), dtype=np.longdouble)
        w = w * e[((idx >> np.uint64(p)) & np.uint64(1)).astype(np.int64)]
    a = psi.astype(np.complex128)
    p2 = a.real.astype(np.longdouble) ** 2 + a.imag.astype(np.longdouble) ** 2
    return np.sum(p2 * w), np.sum(p2)


def q_bound(n, k):
    """Relative first-order bound on q = S / N for k weight factors (channel.cu)."""
    D = chain(n)
    return (k + 5 + 2 * D) * U


# ---- exact channel action (dense, for the enumeration checks) ------------------------------------------------------

def full_op(n, qubits, ops):
    """The 2^n x 2^n matrix of (x)_c K_c with qubit q on index bit n - 1 - q."""
    M = np.ones((1, 1), dtype=np.complex128)
    per = {q: k for q, k in zip(qubits, ops)}
    for q in range(n):  # qubit 0 is the most significant index bit
        M = np.kron(M, np.asarray(per.get(q, np.eye(2)), dtype=np.complex128))
    return M
