"""Numpy emulation of qipb200_state_apply_multiqubit_channels (include/qipb200.h), bit for bit, extending
tests/channel_ref.py to channels on k = 1..4 qubits: byte tables that fold the operators whose physical bits share an
index byte, gathered tables for the others, the weight kernel's summation order, and dense references.

Operators follow the qip_op MAT convention (the channel's first qubit is the most significant bit of b), x holds the
state-dependent channels' qubits in channel order, then qubit order (bit i for the i-th)."""
import numpy as np

import channel_ref as cr

U = cr.U


def form(k):
    """(f, d) of an operator K|b> = d[b] |b ^ f>."""
    k = np.asarray(k, dtype=np.complex128)
    D = k.shape[0]
    f = next(int(r) ^ c for c in range(D) for r in np.flatnonzero(k[:, c] != 0))
    return f, [complex(k[b ^ f, b]) for b in range(D)]


def arity(k):
    return np.asarray(k).shape[0].bit_length() - 1


def weights(k):
    return [cr.weight(d) for d in form(k)[1]]


def state_dependent(ks):
    return any(len(set(weights(k))) > 1 for k in ks)


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
    f, d = form(k)
    return f == 0 and d[0].real > 0 and all(v.real == d[0].real and v.imag == 0 for v in d)


def plan(chans):
    sd = sum(1 for ks in chans if state_dependent(ks))
    rw = any(not scaled_identity(k) for ks in chans for k in ks)
    return (sd, 3 if sd else 0, int(rw), (11 if sd else 0) + int(rw))


def channel_value(bits):
    """b in the matrix convention from the channel's qubit values, first qubit first."""
    b = 0
    for v in bits:
        b = (b << 1) | int(v)
    return b


def tables(groups, ops):
    """([table], F) of the chosen operators ops on the physical bit groups (first qubit first).  A table is
    ("byte", byte, dr, di, e) or ("gat", positions, dr, di, e); byte tables come first, ascending, then the gathered
    ones in operator order."""
    F = 0
    for g, k in zip(groups, ops):
        f = form(k)[0]
        for i, p in enumerate(g):
            if (f >> (len(g) - 1 - i)) & 1:
                F |= 1 << p
    byte_of = [g[0] // 8 if all(p // 8 == g[0] // 8 for p in g) else None for g in groups]
    out = []
    for byte in range(5):
        members = sorted((min(g), i) for i, g in enumerate(groups) if byte_of[i] == byte)
        if not members:
            continue
        dr, di, ee = np.zeros(256), np.zeros(256), np.zeros(256)
        for v in range(256):
            r = i_ = e = None
            for m, (_, i) in enumerate(members):
                b = channel_value((v >> (p % 8)) & 1 for p in groups[i])
                d = form(ops[i])[1][b]
                w = cr.weight(d)
                if m == 0:
                    r, i_, e = d.real, d.imag, w
                else:
                    r, i_ = (r * d.real - i_ * d.imag, r * d.imag + i_ * d.real)
                    e = e * w
            dr[v], di[v], ee[v] = r, i_, e
        out.append(("byte", byte, dr, di, ee))
    for i, g in enumerate(groups):
        if byte_of[i] is None:
            d = form(ops[i])[1]
            out.append(("gat", list(g), np.array([v.real for v in d]), np.array([v.imag for v in d]),
                        np.array([cr.weight(v) for v in d])))
    return out, F


def index(tab, idx):
    """The entry of tab each physical index in idx reads."""
    if tab[0] == "byte":
        return cr._byte(idx, tab[1])
    b = np.zeros(idx.shape, dtype=np.int64)
    for p in tab[1]:
        b = (b << 1) | ((idx >> np.uint64(p)) & np.uint64(1)).astype(np.int64)
    return b


def weight_sums(psi, n, tabs):
    """(S, N) of the weight kernel, in its order of summation (channel_ref.weight_sums for any tables)."""
    N = 1 << n
    idx = np.arange(N, dtype=np.uint64)
    w = tabs[0][4][index(tabs[0], idx)]
    for t in tabs[1:]:
        w = np.multiply(w, t[4][index(t, idx)])
    a = psi.astype(np.complex128)
    p = np.add(np.multiply(a.real, a.real), np.multiply(a.imag, a.imag))
    term = np.multiply(p, w)
    C = min(N, cr.CHUNK)
    V = N // C
    res = []
    for vals in (term, p):
        acc = np.zeros((cr.GRID, cr.THREADS))
        for r in range((V + cr.GRID - 1) // cr.GRID):
            chunks = r * cr.GRID + np.arange(cr.GRID)
            for k in range(cr.PER):
                e = np.arange(cr.THREADS) + cr.THREADS * k
                ok = (chunks[:, None] < V) & (e[None, :] < C)
                j = np.where(ok, chunks[:, None] * C + e[None, :], 0)
                acc = np.where(ok, np.add(acc, vals[j]), acc)
        acc = acc.reshape(cr.GRID, cr.THREADS // 32, 32)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            acc = np.add(acc, acc[:, :, lane ^ o])
        s = acc[:, 0, 0].copy()
        for wp in range(1, cr.THREADS // 32):
            s = np.add(s, acc[:, wp, 0])
        tot = 0.0
        for g in range(cr.GRID):
            tot += float(s[g])
        res.append(tot)
    return res[0], res[1]


def choices(groups, chans, x, draws):
    """The chosen operator of every channel for the sample x."""
    chosen, kd = [], 0
    for c, (g, ks) in enumerate(zip(groups, chans)):
        b = 0
        if state_dependent(ks):
            b = channel_value((int(x) >> (kd + i)) & 1 for i in range(len(g)))
            kd += len(g)
        chosen.append(choose(ks, b, float(draws[1 + c])))
    return chosen


def emulate(psi, n, groups, chans, x, draws, phys=None):
    """(chosen, prob, new state) of the call.  phys(q) is the physical bit of qubit q (n - 1 - q by default)."""
    phys = phys or (lambda q: n - 1 - q)
    chosen = choices(groups, chans, x, draws)
    rest_pos, rest_ops = [], []
    dropped, uniform, nonuniform = 1.0, 1.0, False
    for g, ks, i in zip(groups, chans, chosen):
        k = ks[i]
        e = weights(k)
        if scaled_identity(k):
            dropped *= e[0]
            continue
        rest_pos.append([phys(q) for q in g])
        rest_ops.append(k)
        if len(set(e)) > 1:
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
    b = index(tabs[0], idx)
    wr, wi = tabs[0][2][b], tabs[0][3][b]
    for t in tabs[1:]:
        b = index(t, idx)
        wr, wi = cr.cmul(wr, wi, t[2][b], t[3][b])
    wr, wi = np.multiply(wr, inv), np.multiply(wi, inv)
    R = np.float32 if src.dtype == np.complex64 else np.float64
    wr, wi = wr.astype(R), wi.astype(R)
    a, b = src.real.astype(R), src.imag.astype(R)
    out = np.empty_like(src)
    out.real = np.subtract(np.multiply(wr, a), np.multiply(wi, b))
    out.imag = np.add(np.multiply(wr, b), np.multiply(wi, a))
    return out


def weight_reference(psi, n, groups, ops):
    """(S, N) in long double from the amplitudes and the per-operator weights |d(b)|^2 (doubles)."""
    idx = np.arange(1 << n, dtype=np.uint64)
    w = np.ones(1 << n, dtype=np.longdouble)
    for g, k in zip(groups, ops):
        e = np.array(weights(k), dtype=np.longdouble)
        w = w * e[index(("gat", g), idx)]
    a = psi.astype(np.complex128)
    p2 = a.real.astype(np.longdouble) ** 2 + a.imag.astype(np.longdouble) ** 2
    return np.sum(p2 * w), np.sum(p2)


# ---- exact channel action (dense, for the enumeration checks) ------------------------------------------------------

def apply_dense(psi, n, groups, ops):
    """(x)_c K_c psi with qubit q on index bit n - 1 - q (axis q of the reshaped vector)."""
    t = np.asarray(psi, dtype=np.complex128).reshape([2] * n)
    for g, k in zip(groups, ops):
        m = len(g)
        K = np.asarray(k, dtype=np.complex128).reshape([2] * (2 * m))
        t = np.tensordot(K, t, axes=(list(range(m, 2 * m)), list(g)))
        t = np.moveaxis(t, list(range(m)), list(g))
    return t.reshape(-1)


def full_op(n, groups, ops):
    """The 2^n x 2^n matrix of (x)_c K_c."""
    return np.stack([apply_dense(e, n, groups, ops) for e in np.eye(1 << n, dtype=np.complex128)], axis=1)
