"""Extended-precision references for states too large for the host: windows, closed forms, per-element bounds.

A state of 2^30..2^32 amplitudes cannot be held by the oracle, so the full-size checks work on windows: aligned runs
of 2^w amplitudes downloaded with ``State.download(offset=, length=)``.

* ``op_window_reference`` computes one op's output on a window in ``np.clongdouble`` (x86 80-bit, u ~ 5.4e-20) from
  the device's own input values, downloaded before the op, so the check bounds the kernel's arithmetic alone.  The
  op's matrix comes from the oracle (``qo.make_op_matrix`` on the op relabelled to its own qubits); an op on more
  than ``MAX_MATRIX_QUBITS`` qubits is split into its controls and the inner op's matrix.
* ``check_window`` applies the per-element bound |got_i - want_i| <= c * u * sum_j |m_ij| |x_j| with
  c = 4 * (non-zero entries of row i): 2^(k+2) for a dense k-qubit block, 4 for a diagonal.  That is Higham's
  gamma bound for a 2 * 2^k-term real dot product with or without FMA, doubled, in any summation order.  Rows with a
  single entry equal to 1 (permutations, the rows a controlled or promoted-diagonal op leaves alone) must be
  bit-identical to their input (==, +-0 equal).
* ``ProductPhaseState`` is a state whose every amplitude, marginal and ``soft_measure`` outcome has a closed form.
* ``qft_basis_amp`` is the closed form of ``circuits.qft(n)`` applied to a basis state.

Qubit q lives at index bit n-1-q throughout, as in the library and the oracle.
"""
from __future__ import annotations

import cmath
import math

import numpy as np

from oracle import qip_oracle as qo
from rustqip_b200 import gates
from rustqip_b200.ops import MatrixOp, make_control_op, make_swap_op

LD = np.clongdouble
U_ROUND = {np.complex128: 2.0 ** -53, np.complex64: 2.0 ** -24}
MAX_MATRIX_QUBITS = 10


def unit_roundoff(dtype) -> float:
    return U_ROUND[np.dtype(dtype).type]


def _qubit_bit(n, q):
    return n - 1 - int(q)


# ---------------------------------------------------------------------------------------------------------------
# one op on one window
# ---------------------------------------------------------------------------------------------------------------
def relabel(op: MatrixOp, mapping) -> MatrixOp:
    """The same op with qubit q renamed mapping[q] (nested controls included)."""
    inner = relabel(op.inner, mapping) if op.inner is not None else None
    return MatrixOp(op.kind, [mapping[q] for q in op.indices()], data=op.data, rows=op.rows,
                    n_control=op.n_control, inner=inner, swap_n=op.swap_n)


class OpModel:
    """An op on an n-qubit state as (control mask, qubits, matrix on those qubits)."""

    def __init__(self, n: int, op: MatrixOp, dtype):
        self.n = n
        ctrls = []
        while len(op.indices()) > MAX_MATRIX_QUBITS and op.kind == "control":
            ctrls += op.indices()[: op.n_control]
            op = op.inner
        self.qubits = list(dict.fromkeys(op.indices()))
        k = len(self.qubits)
        if k > MAX_MATRIX_QUBITS:
            raise ValueError("op on %d qubits besides its controls" % k)
        local = relabel(op, {q: i for i, q in enumerate(self.qubits)})
        self.k = k
        self.mat = qo.make_op_matrix(k, local, dtype).astype(LD)  # entries rounded to the state's precision
        self.ctrl_mask = 0
        for q in ctrls:
            self.ctrl_mask |= 1 << _qubit_bit(n, q)
        self.full_bits = [_qubit_bit(n, q) for q in self.qubits]       # local qubit i <-> full index bit
        self.local_bits = [k - 1 - i for i in range(k)]                 # local qubit i <-> local index bit
        nz = self.mat != 0
        rows, cols = np.nonzero(nz)
        coupled = 0
        for r, c in zip(rows, cols):
            coupled |= int(r) ^ int(c)
        self.coupled = [i for i in range(k) if (coupled >> self.local_bits[i]) & 1]  # local qubits that mix
        self.row_nnz = nz.sum(axis=1)
        self.row_exact = (self.row_nnz == 1) & (self.mat == 1).any(axis=1)
        self.abs_row_sum = float(np.abs(self.mat).sum(axis=1).max())

    def coupled_full_bits(self):
        return [self.full_bits[i] for i in self.coupled]

    def local_index(self, g: np.ndarray) -> np.ndarray:
        l = np.zeros_like(g)
        for fb, lb in zip(self.full_bits, self.local_bits):
            l |= ((g >> np.uint64(fb)) & np.uint64(1)) << np.uint64(lb)
        return l


def span_offsets(bits):
    """Every XOR combination of 1 << b for b in bits."""
    out = [0]
    for b in bits:
        out += [o | (1 << b) for o in out]
    return out


def input_offsets(model: OpModel, w: int):
    """Window translations whose inputs one output window of 2^w amplitudes needs (coupled bits >= w)."""
    return span_offsets([b for b in model.coupled_full_bits() if b >= w])


def op_window_reference(n, op, inputs, window, dtype, model=None):
    """Expected output of `op` on the window [window, window + 2^w) in extended precision.

    inputs: {s: device values of the window at offset window ^ s, downloaded before the op} for every s of
    ``input_offsets``.  Returns (want, absacc, c, exact): want (clongdouble), absacc = sum_j |m_ij| |x_j|
    (longdouble), the bound constant c per element and the rows that must equal their input exactly."""
    model = model or OpModel(n, op, dtype)
    x0 = np.asarray(inputs[0])
    length = x0.shape[0]
    w = length.bit_length() - 1
    assert length == 1 << w and window % length == 0
    low = np.uint64(length - 1)
    g = np.arange(window, window + length, dtype=np.uint64)
    xin = {s: np.asarray(v).astype(LD) for s, v in inputs.items()}
    ctrl_ok = (g & np.uint64(model.ctrl_mask)) == np.uint64(model.ctrl_mask)
    lrow = model.local_index(g)
    cmask_full = 0
    cmask_local = 0
    for i in model.coupled:
        cmask_full |= 1 << model.full_bits[i]
        cmask_local |= 1 << model.local_bits[i]
    want = np.zeros(length, dtype=LD)
    absacc = np.zeros(length, dtype=np.longdouble)
    for t in range(1 << len(model.coupled)):
        sf = sl = 0
        for j, i in enumerate(model.coupled):
            if (t >> j) & 1:
                sf |= 1 << model.full_bits[i]
                sl |= 1 << model.local_bits[i]
        src = (g & ~np.uint64(cmask_full)) | np.uint64(sf)
        lcol = (lrow & ~np.uint64(cmask_local)) | np.uint64(sl)
        m = model.mat[lrow.astype(np.int64), lcol.astype(np.int64)]
        shift = (src ^ g) & ~low
        x = np.empty(length, dtype=LD)
        for s in np.unique(shift):
            sel = shift == s
            x[sel] = xin[int(s)][(src[sel] & low).astype(np.int64)]
        want += m * x
        absacc += np.abs(m) * np.abs(x)
    # rows whose controls are not all set are untouched
    want = np.where(ctrl_ok, want, xin[0])
    absacc = np.where(ctrl_ok, absacc, np.abs(xin[0]))
    li = lrow.astype(np.int64)
    exact = ~ctrl_ok | model.row_exact[li]
    c = 4.0 * model.row_nnz[li].astype(np.float64)
    return want, absacc, c, exact


class WindowCheckError(AssertionError):
    pass


def check_window(got, want, absacc, c, exact, u, label="", offset=0):
    """Assert the per-element bound on one window; returns the worst |got - want| / bound over the bounded rows."""
    got_ld = np.asarray(got).astype(LD)
    bad_exact = exact & ~((got_ld.real == want.real) & (got_ld.imag == want.imag))
    if bad_exact.any():
        i = int(np.nonzero(bad_exact)[0][0])
        raise WindowCheckError("%s: offset %d index %d must be exact: got %r want %r (%d rows differ)" % (
            label, offset, offset + i, complex(got[i]), complex(want[i]), int(bad_exact.sum())))
    err = np.abs(got_ld - want)
    bound = np.asarray(c, dtype=np.longdouble) * np.longdouble(u) * absacc
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0))
    ratio = np.where(exact, 0, ratio)
    worst = int(np.argmax(ratio))
    if ratio[worst] > 1:
        raise WindowCheckError("%s: offset %d index %d: got %r want %r |diff| %.3e > bound %.3e (%d elements over)" % (
            label, offset, offset + worst, complex(got[worst]), complex(want[worst]), float(err[worst]),
            float(bound[worst]), int((ratio > 1).sum())))
    return float(ratio[worst])


# ---------------------------------------------------------------------------------------------------------------
# an analytic state: product of 1-qubit states times a phase polynomial
# ---------------------------------------------------------------------------------------------------------------
class ProductPhaseState:
    """a(i) = prod_q v_q[bit_q(i)] * prod_{(a,b) in E, bit_a(i) = bit_b(i) = 1} ph_ab.

    v_q = U_q |0> for a 1-qubit unitary at an angle near pi/4 (small dynamic range); ph_ab = e^(i theta_ab) is the
    constant of ``gates.cphase(a, b, theta_ab)``.  Both are taken as rounded to the state's precision, the values the
    device multiplies by, so the closed form carries no constant-rounding error.  bit_q(i) is qubit q's bit, index bit
    n-1-q.  Prepared on the device from |0> by ``prep_ops()``: n 1-qubit gates and |E| cphase gates."""

    def __init__(self, n: int, dtype, seed: int, n_edges=None, spread=0.05):
        self.n = n
        self.dtype = np.dtype(dtype).type
        rng = np.random.default_rng(seed)
        phi = math.pi / 4 + rng.uniform(-spread, spread, n)
        beta = rng.uniform(-math.pi, math.pi, n)
        self.u = []
        for q in range(n):
            c, s, e = math.cos(phi[q]), math.sin(phi[q]), cmath.exp(1j * beta[q])
            self.u.append(np.array([[c, -s * e.conjugate()], [s * e, c]], dtype=np.complex128))
        rounded = [uq.astype(self.dtype).astype(np.complex128) for uq in self.u]
        self.v = np.array([[LD(r[0, 0]), LD(r[1, 0])] for r in rounded], dtype=LD)  # v[q, bit]
        n_edges = n if n_edges is None else n_edges
        self.edges = []
        seen = set()
        while len(self.edges) < n_edges:
            a, b = (int(x) for x in rng.choice(n, 2, replace=False))
            if (min(a, b), max(a, b)) in seen:
                continue
            seen.add((min(a, b), max(a, b)))
            self.edges.append((a, b, float(rng.uniform(-math.pi, math.pi))))
        self.ph = [LD(complex(np.complex128(cmath.rect(1.0, th)).astype(self.dtype))) for _, _, th in self.edges]

    def prep_ops(self):
        return ([gates.mat([q], self.u[q].reshape(-1)) for q in range(self.n)] +
                [gates.cphase(a, b, th) for a, b, th in self.edges])

    def prep_rel_error(self) -> float:
        """(n + |E|) * 4u: relative bound of the prepared amplitudes (each gate rounds a product at most twice)."""
        return (self.n + len(self.edges)) * 4 * unit_roundoff(self.dtype)

    def bit(self, idx, q):
        return (np.asarray(idx, dtype=np.uint64) >> np.uint64(self.n - 1 - q)) & np.uint64(1)

    def amp(self, idx) -> np.ndarray:
        idx = np.asarray(idx, dtype=np.uint64)
        a = np.ones(idx.shape, dtype=LD)
        for q in range(self.n):
            a *= np.where(self.bit(idx, q) == 1, self.v[q, 1], self.v[q, 0])
        for (qa, qb, _), ph in zip(self.edges, self.ph):
            a *= np.where((self.bit(idx, qa) & self.bit(idx, qb)) == 1, ph, LD(1))
        return a

    def max_abs(self) -> float:
        return float(np.prod(np.abs(self.v).max(axis=1)))

    def qubit_probs(self) -> np.ndarray:
        """|v_q[b]|^2 (the phases do not enter the marginals), float64 [q, b]."""
        return (np.abs(self.v) ** 2).astype(np.float64)

    def marginal(self, indices) -> np.ndarray:
        """Closed form of measure_probs(indices): out[m], bit i of m = qubit indices[i]."""
        p = self.qubit_probs()
        rest = 1.0
        for q in range(self.n):
            if q not in indices:
                rest *= p[q, 0] + p[q, 1]
        out = np.full(1 << len(indices), rest)
        for m in range(1 << len(indices)):
            for i, q in enumerate(indices):
                out[m] *= p[q, (m >> i) & 1]
        return out

    def descend(self, r: float):
        """soft_measure over the whole index for draw r: the smallest index whose cumulative |a|^2 reaches r, by a
        bitwise descent of the product CDF from index bit n-1 (qubit 0).  Returns (index, margins): margins[q] is the
        distance of r from the boundary decided at qubit q (the qubit's bit is certain while it exceeds the error of
        the cumulative sums).  A draw beyond the total mass gives index 0, as the reference's scan does."""
        p = self.qubit_probs()
        total = float(np.prod(p.sum(axis=1)))
        margins = np.zeros(self.n)
        if r > total:
            margins[:] = r - total
            return 0, margins
        mass, idx, rem = total, 0, float(r)
        edge = total - rem
        for q in range(self.n):
            m0 = mass * p[q, 0] / (p[q, 0] + p[q, 1])
            margins[q] = min(abs(rem - m0), edge)
            if rem <= m0:
                mass = m0
            else:
                rem -= m0
                mass -= m0
                idx |= 1 << (self.n - 1 - q)
        return idx, margins


# ---------------------------------------------------------------------------------------------------------------
# QFT of a basis state
# ---------------------------------------------------------------------------------------------------------------
def bit_reverse(v, n):
    v = np.asarray(v, dtype=np.uint64)
    r = np.zeros_like(v)
    for b in range(n):
        r |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(n - 1 - b)
    return r


def qft_basis_amp(n: int, x: int, idx) -> np.ndarray:
    """circuits.qft(n) applied to |x>: 2^(-n/2) * exp(2 pi i * x * y / 2^n) at output index y.

    (The library's QFT puts qubit 0, index bit n-1, first and ends with the bit-reversing swaps, so in index order
    it is the textbook DFT with the + sign; ``tests/test_fullsize_ref_cpu.py`` pins this against the oracle.)"""
    y = np.asarray(idx, dtype=np.uint64)
    # x * y mod 2^n without overflow: multiply bit by bit
    prod = np.zeros_like(y)
    mask = np.uint64((1 << n) - 1) if n < 64 else np.uint64(~0)
    for b in range(n):
        if (x >> b) & 1:
            prod = (prod + (y << np.uint64(b))) & mask
    frac = prod.astype(np.longdouble) / np.longdouble(2.0) ** n
    ang = np.longdouble(8) * np.arctan(np.longdouble(1)) * frac  # 2 pi in long double
    return (np.cos(ang) + 1j * np.sin(ang)).astype(LD) * LD(np.longdouble(2.0) ** (-n / 2))


def qft_bound(n: int, dtype) -> float:
    """Per-element bound of the fused QFT of a basis state: (n^2/2 + 2n) * 4u * 2^(-n/2), plus for f32 the rounding
    of each gate constant the amplitude passes (n H gates and up to n(n-1)/2 phases, |delta| <= sqrt(2) u each)."""
    u = unit_roundoff(dtype)
    b = (n * n / 2 + 2 * n) * 4 * u
    if np.dtype(dtype).type == np.complex64:
        b += (n + n * (n - 1) / 2) * math.sqrt(2) * u
    return b * 2.0 ** (-n / 2)


# ---------------------------------------------------------------------------------------------------------------
# permutation circuits with a host-side index map
# ---------------------------------------------------------------------------------------------------------------
def random_permutation_circuit(n: int, count: int, seed: int):
    """`count` seeded permutation ops over all qubits: X, CNOT, Toffoli, multi-controlled X, Swap (1-3 pairs) and
    controlled Swap.  Each entry is (ctrls, flip_target or None, swap_a, swap_b)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        kind = int(rng.integers(6))
        qs = [int(x) for x in rng.choice(n, 8, replace=False)]
        if kind == 0:
            out.append(([], qs[0], [], []))
        elif kind == 1:
            out.append((qs[1:2], qs[0], [], []))
        elif kind == 2:
            out.append((qs[1:3], qs[0], [], []))
        elif kind == 3:
            out.append((qs[1:1 + int(rng.integers(3, 7))], qs[0], [], []))
        elif kind == 4:
            m = int(rng.integers(1, 4))
            out.append(([], None, qs[:m], qs[m:2 * m]))
        else:
            out.append((qs[6:8][: int(rng.integers(1, 3))], None, qs[:1], qs[1:2]))
    return out


def perm_op(entry) -> MatrixOp:
    ctrls, flip, a, b = entry
    base = gates.x(flip) if flip is not None else make_swap_op(a, b)
    return make_control_op(ctrls, base) if ctrls else base


def perm_apply_index(n: int, entry, idx: np.ndarray) -> np.ndarray:
    """The index map of one permutation op (an involution): the op moves old[f(i)] to new[i]."""
    ctrls, flip, a, b = entry
    idx = np.asarray(idx, dtype=np.uint64)
    cm = 0
    for q in ctrls:
        cm |= 1 << _qubit_bit(n, q)
    on = (idx & np.uint64(cm)) == np.uint64(cm)
    out = idx.copy()
    if flip is not None:
        out = np.where(on, idx ^ np.uint64(1 << _qubit_bit(n, flip)), idx)
    else:
        for qa, qb in zip(a, b):
            ba, bb = np.uint64(_qubit_bit(n, qa)), np.uint64(_qubit_bit(n, qb))
            diff = ((out >> ba) ^ (out >> bb)) & np.uint64(1)
            out = np.where(on & (diff == 1), out ^ ((np.uint64(1) << ba) | (np.uint64(1) << bb)), out)
    return out


def perm_source(n: int, circuit, idx: np.ndarray) -> np.ndarray:
    """pi^-1 of the whole circuit: after it, new[i] = old[perm_source(i)]."""
    src = np.asarray(idx, dtype=np.uint64)
    for entry in reversed(circuit):
        src = perm_apply_index(n, entry, src)
    return src


# ---------------------------------------------------------------------------------------------------------------
# the per-gate zoo and its windows
# ---------------------------------------------------------------------------------------------------------------
def _rand_unitary(k, rng):
    a = rng.standard_normal((1 << k, 1 << k)) + 1j * rng.standard_normal((1 << k, 1 << k))
    q, r = np.linalg.qr(a)
    return q * (np.diag(r) / np.abs(np.diag(r)))


def _rand_diag(k, rng):
    return np.diag(np.exp(1j * rng.uniform(-math.pi, math.pi, 1 << k))).reshape(-1)


def fullsize_zoo(n: int, seed: int, in_place: bool = True):
    """(name, op, launches) for every per-gate kernel class, on low bits (bit 0 included), top bits and scattered
    unordered sets.  Ops are written by index bit: bit b is qubit n-1-b.  in_place=False gives the ops that take the
    out-of-place row kernel (k_gather): a 7-qubit CSR sparse op and a 9-control, 4-target dense op."""
    rng = np.random.default_rng(seed)
    Q = lambda bits: [n - 1 - b for b in bits]  # noqa: E731
    top = lambda k: list(range(n - 1, n - 1 - k, -1))  # noqa: E731
    scattered = lambda k, excl=(): [int(b) for b in rng.choice([b for b in range(n) if b not in excl], k, replace=False)]  # noqa: E731
    zoo = []
    if not in_place:
        k = 7
        perm = rng.permutation(1 << k)
        phases = np.exp(1j * rng.uniform(-math.pi, math.pi, 1 << k))
        rows = [[(int(perm[r]), complex(phases[r]))] for r in range(1 << k)]
        rows[0] = [(int(perm[0]), complex(phases[0]) * 0.6), (int(perm[1]), 0.8j * complex(phases[0]))]
        rows[1] = [(int(perm[0]), 0.8j * complex(phases[1])), (int(perm[1]), complex(phases[1]) * 0.6)]
        fixed = [0, n - 1, 3, n - 2]
        zoo.append(("sparse7_gather", MatrixOp.new_sparse(Q(fixed + scattered(3, fixed)), rows), 1))
        bits = [n - 1, 0] + scattered(11, (n - 1, 0))
        zoo.append(("c9dense4_gather", make_control_op(Q(bits[:9]), gates.mat(Q(bits[9:]), _rand_unitary(4, rng).reshape(-1))), 1))
        return zoo
    for k in (1, 2, 3, 4):
        u = _rand_unitary(k, rng).reshape(-1)
        zoo.append(("dense%d_low0" % k, gates.mat(Q(range(k))[::-1], u), 1))
        zoo.append(("dense%d_low1" % k, gates.mat(Q(range(1, k + 1)), u), 1))
        zoo.append(("dense%d_top" % k, gates.mat(Q(top(k)), u), 1))
        zoo.append(("dense%d_scat" % k, gates.mat(Q(scattered(k)), u), 1))
        b = scattered(k + 8)
        zoo.append(("c1dense%d" % k, make_control_op(Q([n - 1]), gates.mat(Q(scattered(k, (n - 1,))), u)), 1))
        zoo.append(("c2dense%d" % k, make_control_op(Q([0, n - 2]), gates.mat(Q(range(1, k + 1)), u)), 1))
        zoo.append(("c8dense%d" % k, make_control_op(Q(b[k:k + 8]), gates.mat(Q(b[:k]), u)), 1))
    for k in (1, 2, 3, 4):
        zoo.append(("diag%d_low0" % k, gates.mat(Q(range(k)), _rand_diag(k, rng)), 1))
        zoo.append(("diag%d_top" % k, gates.mat(Q(top(k)), _rand_diag(k, rng)), 1))
    zoo.append(("t_bit0", gates.t(n - 1), 1))
    zoo.append(("t_top", gates.t(0), 1))
    zoo.append(("cz_top_low", gates.cz(0, n - 1), 1))
    zoo.append(("cphase_low_top", gates.cphase(n - 2, 1, 0.7123), 1))
    zoo.append(("c8phase", make_control_op(Q(scattered(8, (5,))), gates.mat(Q([5]), [1, 0, 0, cmath.rect(1.0, 0.3)])), 1))
    for k in (5, 7, 10):
        zoo.append(("diag%d" % k, gates.mat(Q([n - 1] + scattered(k - 1, (n - 1,))), _rand_diag(k, rng)), 1))
    zoo.append(("x_bit0", gates.x(n - 1), 1))
    zoo.append(("x_top", gates.x(0), 1))
    zoo.append(("cnot_high_low", gates.cnot(0, n - 1), 1))
    zoo.append(("cnot_low_high", gates.cnot(n - 1, 1), 1))
    zoo.append(("toffoli", gates.toffoli(0, n - 1, n // 2), 1))
    zoo.append(("toffoli_low", gates.toffoli(n - 1, n - 2, 0), 1))
    zoo.append(("swap1", make_swap_op(Q([0]), Q([n - 1])), 1))
    s = scattered(2, (n - 2, 0, 1, n - 1))
    zoo.append(("swap3", make_swap_op(Q([n - 2, 0, s[0]]), Q([1, n - 1, s[1]])), 3))
    zoo.append(("cswap", make_control_op(Q([n // 2]), make_swap_op(Q([n - 1]), Q([0]))), 1))
    for k in (5, 6):
        u = _rand_unitary(k, rng).reshape(-1)
        zoo.append(("dense%d_low0" % k, gates.mat(Q(range(k)), u), 1))
        zoo.append(("dense%d_top" % k, gates.mat(Q(top(k)), u), 1))
        zoo.append(("dense%d_scat" % k, gates.mat(Q(scattered(k)), u), 1))
        zoo.append(("c1dense%d" % k, make_control_op(Q([n - 1]), gates.mat(Q(range(k)), u)), 1))
    for k in (7, 10):
        zoo.append(("dense%d" % k, gates.mat(Q([n - 1] + scattered(k - 1, (n - 1,))), _rand_unitary(k, rng).reshape(-1)), 1))
    return zoo


def window_plan(n: int, model: OpModel, seed: int, extra=()):
    """(w, bases) for one op: w = 12 less the op's coupled bits (at least 2), so that one window and its translated
    inputs hold about 4096 amplitudes; bases are aligned window offsets: index 0, the top window, the windows either
    side of every bit of the op at or above w, `extra` offsets, and two seeded random ones."""
    w = min(n, max(2, 12 - len(model.coupled)))
    size = 1 << w
    total = 1 << n
    bases = [0, total - size]
    for b in sorted(set(model.full_bits) | {i for i in range(n) if (model.ctrl_mask >> i) & 1}):
        if b >= w:
            bases += [(1 << b) - size, 1 << b]
    for e in extra:
        bases += [(e // size) * size]
    rng = np.random.default_rng(seed)
    bases += [int(rng.integers(0, total >> w)) << w for _ in range(2)]
    return w, list(dict.fromkeys(int(b) for b in bases if 0 <= b < total))


# ---------------------------------------------------------------------------------------------------------------
# inverses of zoo ops
# ---------------------------------------------------------------------------------------------------------------
def inverse_op(op: MatrixOp) -> MatrixOp:
    if op.kind == "control":
        return MatrixOp("control", op.indices(), n_control=op.n_control, inner=inverse_op(op.inner))
    if op.kind == "swap":
        return op
    if op.kind == "matrix":
        d = 1 << len(op.indices())
        return MatrixOp.new_matrix(op.indices(), np.asarray(op.data).reshape(d, d).conj().T.reshape(-1))
    d = 1 << len(op.indices())
    dense = np.zeros((d, d), dtype=np.complex128)
    for r, row in enumerate(op.rows):
        for c, v in row:
            dense[r, c] += v
    inv = dense.conj().T
    return MatrixOp.new_sparse(op.indices(), [[(int(c), complex(inv[r, c])) for c in np.nonzero(inv[r])[0]]
                                              for r in range(d)])
