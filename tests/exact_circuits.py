"""Exactly representable circuits: generator, mantissa budget and reference (host only).

Every amplitude is a Gaussian integer times a power of two, and so is every matrix entry of every op.  As long as
no intermediate needs more than 53 (f64) or 24 (f32) mantissa bits, every product and partial sum is exact -- in any
order, with or without FMA contraction, on the DMMA pipe, and in the planner's host-side compositions (peephole folds,
conditional-phase factor tables, the deferred Hadamard scale, CTA-uniform store phases).  The fused passes must then
reproduce the reference bit for bit, on every amplitude however small.

Budget: let 2^e be the smallest power of two that makes all entries of an op Gaussian integers N.  The op costs
``op_bits(op) = ceil(log2(max_row sum_j |Re N_ij| + |Im N_ij|))`` bits.  The l1 complex row norm is submultiplicative,
so the sum of the costs bounds the integer mantissa of every partial sum of any product of ops the planner may
compose.  A circuit is refused when ``bits0 + 1 + sum(op_bits) > 52`` (f64) or ``> 23`` (f32), where every input
amplitude has ``|Re|, |Im| < 2^bits0``.

Entries are kept at or above 2^-40 in magnitude: the planner drops a folded op within 1e-15 of the identity on
purpose (planner.cpp), so no non-identity op may come that close to it.
"""
import itertools
import math

import numpy as np

from oracle import qip_oracle as qo
from rustqip_b200 import gates
from rustqip_b200.ops import MatrixOp, make_control_op, make_matrix_op, make_swap_op  # noqa: F401 (re-exported)

LIMIT = {np.dtype(np.complex128): 52, np.dtype(np.complex64): 23}
MIN_EXP = -40


class BudgetError(ValueError):
    """The circuit may need more mantissa bits than the precision has: its result is not exact."""


# ---- states ----------------------------------------------------------------------------------------------------
def exact_state(n, seed, bits, shift=0, dtype=np.complex128):
    """Gaussian integers with |Re|, |Im| < 2^bits, times 2^-shift (not normalised: the gate path never assumes it)."""
    rng = np.random.default_rng(seed)
    lim = 1 << bits
    re = rng.integers(-lim + 1, lim, size=1 << n).astype(np.float64)
    im = rng.integers(-lim + 1, lim, size=1 << n).astype(np.float64)
    return (np.ldexp(re, -shift) + 1j * np.ldexp(im, -shift)).astype(dtype)


def exact_window(block, k):
    """Window k of a large state generated window by window from one block of Gaussian integers (an exact_state):
    the block rotated by k and multiplied by i^k, so that windows differ while each costs only a roll to regenerate.
    Large states are uploaded and compared window by window without ever being held on the host."""
    return np.roll(block, 977 * k) * block.dtype.type((1, 1j, -1, -1j)[k % 4])


# ---- op matrices and their cost -------------------------------------------------------------------------------
def op_matrix(op):
    """(qubits, dense matrix) of a whole op, controls included; qubits[0] is the most significant sub-index bit."""
    if op.kind == "matrix":
        k = len(op.indices())
        return list(op.indices()), np.asarray(op.data, dtype=np.complex128).reshape(1 << k, 1 << k)
    if op.kind == "sparse":
        k = len(op.indices())
        m = np.zeros((1 << k, 1 << k), dtype=np.complex128)
        for r, row in enumerate(op.rows):
            for c, v in row:
                m[r, c] += v
        return list(op.indices()), m
    if op.kind == "swap":
        h = op.swap_n
        m = np.zeros((1 << 2 * h, 1 << 2 * h), dtype=np.complex128)
        lo = (1 << h) - 1
        for c in range(1 << 2 * h):
            m[((c & lo) << h) | (c >> h), c] = 1
        return list(op.indices()), m
    q, inner = op_matrix(op.inner)
    nc = op.n_control
    k = len(q)
    m = np.eye(1 << (nc + k), dtype=np.complex128)
    at = ((1 << nc) - 1) << k
    m[at:, at:] = inner
    return list(op.indices()[:nc]) + q, m


def dyadic_exponent(values):
    """Smallest e >= 0 such that every Re/Im of values * 2^e is an integer (raises if there is none above 2^-40)."""
    v = np.concatenate([np.real(values).ravel(), np.imag(values).ravel()])
    for e in range(0, -MIN_EXP + 1):
        s = np.ldexp(v, e)
        if np.all(s == np.round(s)):
            return e
    raise BudgetError("entries are not dyadic with denominators >= 2^%d" % MIN_EXP)


def op_bits(op):
    q, m = op_matrix(op)
    e = dyadic_exponent(m)
    N = np.ldexp(m.real, e), np.ldexp(m.imag, e)
    l1 = float(np.max(np.sum(np.abs(N[0]) + np.abs(N[1]), axis=1)))
    return max(0, int(math.ceil(math.log2(l1))))


def circuit_bits(ops):
    return sum(op_bits(op) for op in ops)


def check_budget(ops, bits0, dtype):
    need = bits0 + 1 + circuit_bits(ops)
    if need > LIMIT[np.dtype(dtype)]:
        raise BudgetError("circuit needs %d mantissa bits, %s has %d" % (need, np.dtype(dtype).name, LIMIT[np.dtype(dtype)]))
    return need


# ---- gate shapes --------------------------------------------------------------------------------------------------
_I = 1j
BFLY = np.array([1, 1, 1, -1], dtype=np.complex128)        # s*[[1,1],[1,-1]]: the un-normalised Hadamard, 1 bit
IBFLY = 0.5 * np.array([1, _I, _I, 1])                        # 1/2*[[1,i],[i,1]], 1 bit
REAL2 = [0.5 * np.array([1, -1, 1, 1]), np.array([1, 1, -1, 1]), 0.25 * np.array([2, 2, -2, 2])]
CPLX2 = [0.5 * np.array([1, _I, 1, -_I]), np.array([1 + _I, 0, 0, 1]), 0.5 * np.array([_I, 1, 1, _I])]
PHASES = [1, -1, _I, -_I]


def bfly(q, s=1.0):
    return make_matrix_op([q], s * BFLY)


def diag_op(qs, entries):
    return make_matrix_op(list(qs), np.diag(np.asarray(entries, dtype=np.complex128)).reshape(-1))


def phased_perm(k, rng):
    """Random permutation matrix with +-1 / +-i entries on k qubits (0 bits)."""
    p = rng.permutation(1 << k)
    m = np.zeros((1 << k, 1 << k), dtype=np.complex128)
    m[p, np.arange(1 << k)] = np.array(PHASES)[rng.integers(4, size=1 << k)]
    return m


def dense_block(qs, rng, mix=True):
    """Dense dyadic block: phased permutation, optionally times a butterfly on one sub-bit (then 1 bit)."""
    k = len(qs)
    m = phased_perm(k, rng)
    if mix:
        j = int(rng.integers(k))
        b = np.kron(np.kron(np.eye(1 << j), BFLY.reshape(2, 2) * (0.5 if rng.integers(2) else 1.0)), np.eye(1 << (k - 1 - j)))
        m = phased_perm(k, rng) @ b @ m
    return make_matrix_op(list(qs), m.reshape(-1))


def dense_kron(qs, rng):
    """Dense 2- or 3-qubit block, a product of 1-bit factors between phased permutations: len(qs) bits."""
    m = np.ones((1, 1), dtype=np.complex128)
    for _ in qs:
        f = [BFLY, IBFLY * 2, REAL2[1], CPLX2[0] * 2][int(rng.integers(4))].reshape(2, 2) * (0.5 if rng.integers(2) else 1.0)
        m = np.kron(m, f)
    m = phased_perm(len(qs), rng) @ m @ phased_perm(len(qs), rng)
    return make_matrix_op(list(qs), m.reshape(-1))


def sparse_perm(qs, rng):
    """Sparse CSR op: a phased permutation with one row pair mixed as (x+y)/2, (x-y)/2 (1 bit)."""
    k = len(qs)
    p = rng.permutation(1 << k)
    ph = np.array(PHASES)[rng.integers(4, size=1 << k)]
    rows = [[(int(p[r]), complex(ph[r]))] for r in range(1 << k)]
    rows[0] = [(int(p[0]), 0.5 + 0j), (int(p[1]), 0.5 + 0j)]
    rows[1] = [(int(p[0]), 0.5 + 0j), (int(p[1]), -0.5 + 0j)]
    return MatrixOp.new_sparse(list(qs), rows)


def fredkin(c, a, b):
    return make_control_op([c], make_swap_op([a], [b]))


def x4(cs, t):
    """4-control Toffoli: wider than any elementary record, so its pass runs on the interpreter kernel."""
    return make_control_op(list(cs), gates.x(t))


# ---- the generator ------------------------------------------------------------------------------------------------
def _pick(rng, pool, k):
    return [int(x) for x in rng.choice(pool, k, replace=False)]


def random_exact_circuit(n, count, seed, dtype=np.complex128, bits0=8, growing=None, wide=False, qubits=None):
    """`count` ops of every cheap and growing shape on random qubits (low, high and middle index bits alike).

    Growing ops are drawn while the budget lasts (`growing` caps their total cost); `wide` adds the ops that leave
    the tile path: 4-control Toffolis (interpreter passes) and, for n >= 8, dense 4..min(10, n) qubit blocks, wide
    diagonals and a sparse op on 7 qubits (per-gate kernels).  `qubits`: the qubits to draw from (default all)."""
    rng = np.random.default_rng(seed)
    pool = list(range(n)) if qubits is None else list(qubits)
    limit = LIMIT[np.dtype(dtype)] - bits0 - 1
    budget = limit if growing is None else min(limit, growing)
    ops, spent = [], 0
    cheap = [
        lambda q: gates.x(q[0]), lambda q: gates.cnot(q[0], q[1]), lambda q: gates.toffoli(q[0], q[1], q[2]),
        lambda q: make_swap_op([q[0]], [q[1]]), lambda q: fredkin(q[0], q[1], q[2]),
        lambda q: make_control_op([q[0]], make_control_op([q[1]], gates.cnot(q[2], q[3]))),
        lambda q: gates.z(q[0]), lambda q: gates.s(q[0]), lambda q: gates.cz(q[0], q[1]), lambda q: gates.y(q[0]),
        lambda q: make_control_op([q[0]], gates.s(q[1])), lambda q: diag_op([q[0]], [1, -_I]),
        lambda q: diag_op([q[0], q[1]], np.array(PHASES)[rng.integers(4, size=4)]),
        lambda q: diag_op([q[0], q[1], q[2]], np.array(PHASES)[rng.integers(4, size=8)]),
        lambda q: make_matrix_op([q[0], q[1]], phased_perm(2, rng).reshape(-1)),
        lambda q: make_matrix_op([q[0], q[1], q[2]], phased_perm(3, rng).reshape(-1)),
        lambda q: make_control_op([q[0], q[1]], make_swap_op([q[2]], [q[3]])),
        lambda q: make_matrix_op([q[0]], np.array([0, _I, -_I, 0])),
        # wider than an elementary record inside a pass: the interpreter's wide dense / diagonal micro-ops
        lambda q: make_control_op([q[2], q[3]], make_matrix_op([q[0], q[1]], phased_perm(2, rng).reshape(-1))),
        lambda q: diag_op(q[:4], np.array(PHASES)[rng.integers(4, size=16)]),
        lambda q: make_control_op(q[1:4], gates.z(q[0])),
    ]
    grow = [
        lambda q: bfly(q[0], 1.0), lambda q: bfly(q[0], 0.5), lambda q: make_matrix_op([q[0]], IBFLY),
        lambda q: make_control_op([q[1]], make_matrix_op([q[0]], IBFLY)),
        lambda q: make_control_op([q[1], q[2]], make_matrix_op([q[0]], IBFLY)),
        lambda q: make_matrix_op([q[0]], REAL2[int(rng.integers(3))]), lambda q: make_matrix_op([q[0]], CPLX2[int(rng.integers(3))]),
        lambda q: make_control_op([q[1]], make_matrix_op([q[0]], REAL2[0])),
        lambda q: make_control_op([q[1], q[2]], make_matrix_op([q[0]], CPLX2[0])),
        lambda q: make_control_op([q[1]], bfly(q[0], 0.5)),
        lambda q: diag_op([q[0]], [1, 2 + _I]), lambda q: make_control_op([q[1]], diag_op([q[0]], [1, 1 - 2 * _I])),
        lambda q: dense_kron(q[:2], rng), lambda q: dense_kron(q[:3], rng),
        # cancelling pairs / foldable chains on one target, also across a commuting op
        lambda q: make_control_op(q[1:4], make_matrix_op([q[0]], IBFLY)),
        lambda q: [bfly(q[0], 0.5), bfly(q[0], 1.0)], lambda q: [bfly(q[0], 0.5), gates.z(q[1]), bfly(q[0], 0.5)],
        lambda q: [make_matrix_op([q[0]], IBFLY), gates.s(q[0]), make_matrix_op([q[0]], IBFLY)],
    ]
    cheap_runs = [
        lambda q: [gates.x(q[0]), gates.x(q[0])], lambda q: [gates.s(q[0]), gates.s(q[0]), gates.z(q[0])],
        lambda q: [gates.cnot(q[0], q[1]), gates.z(q[2]), gates.cnot(q[0], q[1])],
        # a run of controlled phases on one target whose controls are spread over the state (factor tables)
        lambda q: [make_control_op([c], diag_op([q[0]], [1, PHASES[1 + i % 3]])) for i, c in enumerate(q[1:])],
    ]
    while len(ops) < count:
        q = _pick(rng, pool, min(len(pool), 6))
        r = rng.random()
        if r < 0.3 and spent < budget:
            new = grow[int(rng.integers(len(grow)))](q)
        elif r < 0.4:
            new = cheap_runs[int(rng.integers(len(cheap_runs)))](q)
        else:
            new = cheap[int(rng.integers(len(cheap)))](q)
        new = new if isinstance(new, list) else [new]
        cost = circuit_bits(new)
        if spent + cost > budget:
            continue
        spent += cost
        ops.extend(new)
    if wide:
        ops = _with_wide_ops(n, ops, rng, budget - spent)
    check_budget(ops, bits0, dtype)
    return ops


def _with_wide_ops(n, ops, rng, left):
    """Insert the ops that leave the tile path at random places."""
    extra = []
    if n >= 5:
        for _ in range(2):
            q = _pick(rng, range(n), 5)
            extra.append(x4(q[:4], q[4]))
    if n >= 8:
        for k in (4, 6, min(10, n)):
            extra.append(dense_block(_pick(rng, range(n), k), rng, mix=left > 0))
            left -= 1 if left > 0 else 0
        k = min(8, n)
        extra.append(diag_op(_pick(rng, range(n), k), np.array(PHASES)[rng.integers(4, size=1 << k)]))
        extra.append(sparse_perm(_pick(rng, range(n), 7), rng) if left > 0 else
                     MatrixOp.new_sparse(_pick(rng, range(n), 7), [[(int(c), 1j)] for c in rng.permutation(128)]))
    out = list(ops)
    for op in extra:
        out.insert(int(rng.integers(len(out) + 1)), op)
    return out


def narrow(ops):
    """The ops on at most three qubits, controls included: every pass of their plan fits the generated kernels (wider ops
    send their pass to the interpreter kernel, or run as per-gate kernels)."""
    return [op for op in ops if len(op_matrix(op)[0]) <= 3]


def condition_overflow_block(n, outside, seed):
    """Ops on the three lowest index bits (qubits n-1..n-3: always inside the tile) under every 1-, 2- and 3-subset
    of the `outside` qubits as controls: 92 distinct CTA-uniform conditions for 8 qubits, more than the 63 slots of
    a pass's condition table.  Cheap non-diagonal ops only (0 bits): a diagonal under outside controls would become a
    CTA-uniform phase term instead of a conditional op."""
    rng = np.random.default_rng(seed)
    ops = []
    for k in (1, 2, 3):
        for ctrls in itertools.combinations(outside, k):
            t = n - 1 - int(rng.integers(3))
            inner = [gates.x(t), gates.y(t), make_matrix_op([t], np.array([0, _I, _I, 0]))][int(rng.integers(3))]
            ops.append(make_control_op(list(ctrls), inner))
    return ops


# ---- the circuits of tests/test_gpu_exact.py (also planned on the CPU by tests/test_exact_circuits_cpu.py) ------------
DEVICE_BITS0 = {np.dtype(np.complex128): 8, np.dtype(np.complex64): 3}
DEVICE_GEOMETRIES = [(n, d) for n in (5, 9, 12, 13, 16, 17, 20, 22, 24) for d in (np.complex128, np.complex64)] + [(26, np.complex128)]
OVERFLOW_N = 22


def device_case(n, dtype, seed, wide=True):
    """One device circuit and input state.  wide=False: ops on at most three qubits only (every pass of the plan fits
    the generated kernels)."""
    bits0 = DEVICE_BITS0[np.dtype(dtype)]
    count = 150 if n <= 20 else (60 if n <= 24 else 30)
    ops = random_exact_circuit(n, count, 9000 + 37 * n + seed, dtype, bits0, wide=wide)
    ops = ops if wide else narrow(ops)
    psi = exact_state(n, 100 + n + seed, bits0, shift=seed % 3, dtype=dtype)
    return ops, psi


def device_overflow_block():
    """92 conditions on the OVERFLOW_N-qubit state whose default plan (f64 and f32, generated kernels or not) is one pass
    with more than 63 distinct CTA-uniform conditions: controls on qubits 8..15, which the planner leaves outside the
    tile (tests/test_exact_circuits_cpu.py::test_device_overflow_block_overflows checks the plan)."""
    return condition_overflow_block(OVERFLOW_N, list(range(8, 16)), 5)


def inverse_circuit(ops):
    """Exact inverse of a circuit of phased permutations, butterflies and diagonal phases: the butterfly's inverse is
    1/2*[[1,1],[1,-1]], phases are conjugated, permutations inverted -- each from the op's own matrix (M^-1 = M^H / d
    with the op's row norm d, a power of four for these shapes)."""
    out = []
    for op in reversed(ops):
        q, m = op_matrix(op)
        g = m.conj().T @ m
        d = g[0, 0].real
        if not np.allclose(g, d * np.eye(len(g))) or d <= 0 or math.log2(d) != round(math.log2(d)):
            raise ValueError("op is not a scaled unitary with a power-of-two norm: %r" % op)
        out.append(make_matrix_op(q, (m.conj().T / d).reshape(-1)))
    return out


def reversible_circuit(n, count, seed, growing=12, qubits=None):
    """Phased permutations, diagonal phases and butterflies only (ops with an exact dyadic inverse)."""
    rng = np.random.default_rng(seed)
    pool = list(range(n)) if qubits is None else list(qubits)
    ops, spent = [], 0
    while len(ops) < count:
        q = _pick(rng, pool, 4)
        r = rng.random()
        if r < 0.2 and spent < growing:
            ops.append(bfly(q[0], 1.0))
            spent += 1
        else:
            ops.append([gates.x(q[0]), gates.cnot(q[0], q[1]), gates.toffoli(q[0], q[1], q[2]), make_swap_op([q[0]], [q[1]]),
                        gates.s(q[0]), gates.cz(q[0], q[1]), make_control_op([q[1]], gates.s(q[0])),
                        make_matrix_op([q[0], q[1]], phased_perm(2, rng).reshape(-1))][int(rng.integers(8))])
    return ops


# ---- references ---------------------------------------------------------------------------------------------------
def reference(n, ops, psi):
    """The oracle's f64 fold.  For an f32 input the fold runs in f64 on the f32 values and the result must be
    representable in f32 (it is, within the budget): returned in the input's precision."""
    dtype = np.dtype(psi.dtype)
    want = qo.run_pipeline(n, ops, state=psi.astype(np.complex128), dtype=np.complex128)
    if dtype == np.complex64:
        narrow = want.astype(np.complex64)
        if not np.array_equal(narrow.astype(np.complex128), want):
            raise BudgetError("the f64 fold is not representable in f32")
        return narrow
    return want


def integer_fold(n, ops, psi):
    """Independent reference: int64 Gaussian-integer mantissas with one common exponent, op by op."""
    v = np.asarray(psi, dtype=np.complex128)
    E = dyadic_exponent(v)
    xr = np.ldexp(v.real, E).astype(np.int64).reshape((2,) * n)
    xi = np.ldexp(v.imag, E).astype(np.int64).reshape((2,) * n)
    for op in ops:
        q, m = op_matrix(op)
        e = dyadic_exponent(m)
        Nr = np.ldexp(m.real, e).astype(np.int64)
        Ni = np.ldexp(m.imag, e).astype(np.int64)
        k = len(q)

        def lift(x):
            return np.moveaxis(x, q, list(range(k))).reshape(1 << k, -1)

        def drop(y):
            return np.moveaxis(y.reshape((2,) * n), list(range(k)), q)

        ar, ai = lift(xr), lift(xi)
        xr, xi = drop(Nr @ ar - Ni @ ai), drop(Nr @ ai + Ni @ ar)
        E += e
        if max(int(np.max(np.abs(xr))), int(np.max(np.abs(xi)))) >= 1 << 53:
            raise BudgetError("integer mantissa exceeds 53 bits")
    return np.ldexp(xr.reshape(-1).astype(np.float64), -E) + 1j * np.ldexp(xi.reshape(-1).astype(np.float64), -E)


def first_mismatch(got, want):
    """'' when equal value for value, else where and by how much (for assertion messages)."""
    got = np.asarray(got)
    want = np.asarray(want)
    if got.shape == want.shape and np.array_equal(got, want):
        return ""
    if got.shape != want.shape:
        return "shape %s vs %s" % (got.shape, want.shape)
    bad = np.flatnonzero(got != want)
    i = int(bad[0])
    return "%d amplitudes differ, first at %d: %r vs %r" % (len(bad), i, complex(got[i]), complex(want[i]))
