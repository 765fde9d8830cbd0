"""The full-size window reference (tests/fullsize_ref.py) against the oracle, on states the oracle can hold.

The GPU checks at N = 30..32 (tests/test_gpu_full_size.py) rest on these helpers, so each one is pinned here: the
window reference equals the oracle's apply_op_overwrite on windows of random states for every op of the zoo, the
analytic state and the QFT closed form equal the oracle's pipeline, the CDF descent equals soft_measure, the host
permutation map equals the oracle, and the per-element bound fails on errors the max-relative check lets through."""
import math

import numpy as np
import pytest

import fullsize_ref as fr
from oracle import qip_oracle as qo
from rustqip_b200 import circuits, gates

DTYPES = [np.complex128, np.complex64]


def rand_state(n, dtype, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(1 << n) + 1j * rng.standard_normal(1 << n)
    return np.ascontiguousarray((v / np.linalg.norm(v)).astype(dtype))


def window_inputs(psi, base, w, model):
    return {s: psi[base ^ s: (base ^ s) + (1 << w)] for s in fr.input_offsets(model, w)}


def check_op_against_oracle(n, op, psi, dtype, seed):
    want_full = np.zeros_like(psi)
    qo.apply_op_overwrite(n, op, psi, want_full)
    model = fr.OpModel(n, op, dtype)
    w, bases = fr.window_plan(n, model, seed)
    worst = 0.0
    for base in bases:
        want, acc, c, exact = fr.op_window_reference(n, op, window_inputs(psi, base, w, model), base, dtype, model)
        got = want_full[base: base + (1 << w)]
        worst = max(worst, fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(dtype), repr(op), base))
    return worst


@pytest.mark.parametrize("dtype", DTYPES)
def test_window_reference_equals_oracle_on_zoo(dtype):
    """Every in-place op of the zoo at n = 12 (8 controls + 4 targets fill it), and the row-kernel ops at n = 14."""
    for n, in_place in ((12, True), (14, False)):
        psi = rand_state(n, dtype, 3 + n)
        for i, (name, op, _) in enumerate(fr.fullsize_zoo(n, 40 + n, in_place)):
            check_op_against_oracle(n, op, psi, dtype, i)


@pytest.mark.parametrize("dtype", DTYPES)
def test_window_reference_small_states(dtype):
    """n = 10 and 11, where the windows cover most of the state, with nested controls and a sparse op."""
    from rustqip_b200.ops import MatrixOp, make_control_op, make_swap_op
    for n in (10, 11):
        rng = np.random.default_rng(n)
        psi = rand_state(n, dtype, n)
        ops = [gates.h(0), gates.cnot(n - 1, 2), make_swap_op([0, 3], [n - 1, 4]),
               MatrixOp.new_control([0], [1, 2], MatrixOp.new_control([1], [2], gates.x(2))),
               MatrixOp.new_sparse([0, n - 1], [[(0, 0.6), (3, 0.8j)], [(1, 1.0)], [(2, -1.0)], [(0, 0.8j), (3, 0.6)]]),
               make_control_op([n - 1], gates.mat([0, 5, 2], fr._rand_unitary(3, rng).reshape(-1)))]
        for i, op in enumerate(ops):
            check_op_against_oracle(n, op, psi, dtype, i)


def test_window_reference_uses_translated_inputs():
    """A dense op on a bit above the window reads the partner window: dropping it must change the answer."""
    n = 12
    psi = rand_state(n, np.complex128, 1)
    op = gates.h(0)  # index bit 11
    model = fr.OpModel(n, op, np.complex128)
    assert fr.input_offsets(model, 8) == [0, 1 << 11]
    inputs = window_inputs(psi, 256, 8, model)
    want, *_ = fr.op_window_reference(n, op, inputs, 256, np.complex128, model)
    inputs[1 << 11] = np.zeros(256, dtype=np.complex128)
    want0, *_ = fr.op_window_reference(n, op, inputs, 256, np.complex128, model)
    assert np.max(np.abs(want - want0)) > 1e-3


# ---------------------------------------------------------------------------------------------------------------
# sensitivity of the per-element bound
# ---------------------------------------------------------------------------------------------------------------
def _naive_apply(model, psi, base, w, dtype, mat, order):
    """Outputs of one window computed in the state's precision, without FMA, summing the columns in `order`."""
    real = np.float64 if dtype == np.complex128 else np.float32
    n = model.n
    out = np.zeros(1 << w, dtype=dtype)
    for o in range(1 << w):
        g = base + o
        if (g & model.ctrl_mask) != model.ctrl_mask:
            out[o] = psi[g]
            continue
        row = int(model.local_index(np.array([g], dtype=np.uint64))[0])
        re = real(0)
        im = real(0)
        cols = range(1 << model.k)
        for col in (cols if order > 0 else reversed(cols)):
            src = g
            for fb, lb in zip(model.full_bits, model.local_bits):
                src = (src & ~(1 << fb)) | (((col >> lb) & 1) << fb)
            m, x = mat[row, col], psi[src]
            re = real(re + real(real(m.real) * x.real) - real(real(m.imag) * x.imag))
            im = real(im + real(real(m.real) * x.imag) + real(real(m.imag) * x.real))
        out[o] = re + 1j * im
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_bound_accepts_other_summation_orders(dtype):
    n, w = 10, 6
    rng = np.random.default_rng(5)
    psi = rand_state(n, dtype, 5)
    for op in (gates.mat([0, 7, 3], fr._rand_unitary(3, rng).reshape(-1)),
               gates.mat([2, 9], fr._rand_unitary(2, rng).reshape(-1))):
        model = fr.OpModel(n, op, dtype)
        mat = model.mat.astype(np.complex128).astype(dtype)
        for base in (0, 320, (1 << n) - 64):
            want, acc, c, exact = fr.op_window_reference(n, op, window_inputs(psi, base, w, model), base, dtype, model)
            for order in (1, -1):
                got = _naive_apply(model, psi, base, w, dtype, mat, order)
                assert fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(dtype)) <= 1


@pytest.mark.parametrize("dtype", DTYPES)
def test_bound_rejects_perturbed_matrix_entry(dtype):
    n, w = 10, 6
    rng = np.random.default_rng(6)
    psi = rand_state(n, dtype, 6)
    op = gates.mat([1, 8], fr._rand_unitary(2, rng).reshape(-1))
    model = fr.OpModel(n, op, dtype)
    mat = model.mat.astype(np.complex128)
    mat[2, 1] += 1e-12 if dtype == np.complex128 else 1e-6
    mat = mat.astype(dtype)
    base = 320  # index bit 8 set, bit 1 clear on half the rows: local row 2
    want, acc, c, exact = fr.op_window_reference(n, op, window_inputs(psi, base, w, model), base, dtype, model)
    got = _naive_apply(model, psi, base, w, dtype, mat, 1)
    with pytest.raises(fr.WindowCheckError):
        fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
def test_bound_rejects_error_on_a_small_amplitude(dtype):
    """One amplitude 1e-3 x the smallest of its window, off by 1 %: the per-element bound catches it; in f32 a
    tolerance relative to the largest amplitude (the oracle comparisons of the smaller tests) does not."""
    n, w = 10, 8
    psi = rand_state(n, dtype, 7)
    base = 256
    win = np.abs(psi[base: base + (1 << w)])
    psi[base + 17] = psi[base + 17] / abs(psi[base + 17]) * win.min() * 1e-3
    for op in (gates.t(n - 1), gates.mat([3, 4], fr._rand_diag(2, np.random.default_rng(1)))):
        model = fr.OpModel(n, op, dtype)
        inputs = window_inputs(psi, base, w, model)
        want, acc, c, exact = fr.op_window_reference(n, op, inputs, base, dtype, model)
        full = np.zeros_like(psi)
        qo.apply_op_overwrite(n, op, psi, full)
        got = full[base: base + (1 << w)].copy()
        assert fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(dtype)) <= 1
        got[17] *= dtype(1.01)
        if dtype == np.complex64:  # the f32 max-relative tolerance of 1e-5 does not see it
            assert np.max(np.abs(got - want.astype(np.complex128))) <= 1e-5 * np.max(np.abs(want.astype(np.complex128)))
        with pytest.raises(fr.WindowCheckError):
            fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(dtype))


def test_exact_rows_reject_any_change():
    n, w = 10, 6
    psi = rand_state(n, np.complex128, 8)
    for op in (gates.cnot(2, 7), gates.t(4)):
        model = fr.OpModel(n, op, np.complex128)
        want, acc, c, exact = fr.op_window_reference(n, op, window_inputs(psi, 0, w, model), 0, np.complex128, model)
        full = np.zeros_like(psi)
        qo.apply_op_overwrite(n, op, psi, full)
        got = full[: 1 << w].copy()
        fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(np.complex128))
        i = int(np.nonzero(exact)[0][0])
        got[i] = np.nextafter(got[i].real, 2.0) + 1j * got[i].imag
        with pytest.raises(fr.WindowCheckError):
            fr.check_window(got, want, acc, c, exact, fr.unit_roundoff(np.complex128))


# ---------------------------------------------------------------------------------------------------------------
# closed forms
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_analytic_state_equals_pipeline(dtype):
    n = 10
    a = fr.ProductPhaseState(n, dtype, 11)
    got = qo.run_pipeline(n, a.prep_ops(), 0, dtype)
    want = a.amp(np.arange(1 << n))
    err = np.abs(got.astype(fr.LD) - want)
    assert np.all(err <= a.prep_rel_error() * np.abs(want)), float(np.max(err / np.abs(want)))
    # the marginals: measure_probs of the oracle on the same state
    for idx in ([0], [n - 1], [3, 7], [9, 0, 4]):
        p = qo.measure_probs(n, idx, got).astype(np.float64)
        assert np.allclose(p, a.marginal(idx), rtol=4 * a.prep_rel_error() + 1e-6, atol=0), idx


def test_analytic_state_has_small_dynamic_range():
    a = fr.ProductPhaseState(32, np.complex64, 3)
    assert a.max_abs() < 8 * 2.0 ** -16


def test_cdf_descent_equals_soft_measure():
    n = 10
    a = fr.ProductPhaseState(n, np.complex128, 12)
    psi = np.ascontiguousarray(a.amp(np.arange(1 << n)).astype(np.complex128))
    rng = np.random.default_rng(13)
    order = list(range(n - 1, -1, -1))  # bit i of the outcome = index bit i
    checked = 0
    for r in list(rng.random(400)) + [0.0, 1e-12, 0.999999]:
        idx, margins = a.descend(r)
        if margins.min() <= 1e-12:
            continue
        assert qo.soft_measure(n, order, psi, r) == idx, r
        assert qo.soft_measure(n, [0, n - 1], psi, r) == ((idx >> (n - 1)) & 1) | ((idx & 1) << 1)
        checked += 1
    assert checked > 350


@pytest.mark.parametrize("dtype", DTYPES)
def test_qft_closed_form_equals_oracle(dtype):
    for n in (6, 7, 8, 9, 10):
        ops = circuits.qft(n)
        for x in (0, 1, (1 << n) - 1, 0b101101 & ((1 << n) - 1), (1 << n) - 3):
            got = qo.run_pipeline(n, ops, x, dtype)
            want = fr.qft_basis_amp(n, x, np.arange(1 << n))
            err = np.abs(got.astype(fr.LD) - want)
            assert np.all(err <= fr.qft_bound(n, dtype)), (n, x, float(err.max()))
    # the bound is tight enough to see a wrong convention: the conjugate phase fails it
    n = 8
    got = qo.run_pipeline(n, circuits.qft(n), 77, np.complex128)
    assert np.abs(got.astype(fr.LD) - np.conj(fr.qft_basis_amp(n, 77, np.arange(1 << n)))).max() > 1e-3


def test_permutation_map_equals_oracle():
    n = 11
    circ = fr.random_permutation_circuit(n, 120, 21)
    psi = rand_state(n, np.complex128, 21)
    got = qo.run_pipeline(n, [fr.perm_op(e) for e in circ], state=psi)
    src = fr.perm_source(n, circ, np.arange(1 << n, dtype=np.uint64))
    assert np.array_equal(got, psi[src.astype(np.int64)])


@pytest.mark.parametrize("dtype", DTYPES)
def test_inverse_ops_undo_the_zoo(dtype):
    n = 12
    psi = rand_state(n, np.complex128, 4).astype(dtype)
    for name, op, _ in fr.fullsize_zoo(n, 52, True)[::3] + fr.fullsize_zoo(14, 54, False)[:1]:
        m = 14 if name.endswith("gather") else n
        x = psi if m == n else rand_state(m, dtype, 4)
        y = qo.run_pipeline(m, [op, fr.inverse_op(op)], state=x, dtype=dtype)
        assert np.max(np.abs(y - x)) < (1e-12 if dtype == np.complex128 else 1e-5), name


def test_kernel_counts_and_release_pool_reject_null_context():
    """The two context calls the full-size GPU tests rely on: argument checks at the C boundary (no GPU needed)."""
    import ctypes as C
    from rustqip_b200 import _lib
    L = _lib.lib()
    out = (C.c_uint64 * 8)()
    assert L.qipb200_kernel_counts(None, out, 8) == 1  # QIPB200_ERR_INVALID_ARG
    assert b"kernel_counts" in L.qipb200_last_error(None)
    assert L.qipb200_release_pool(None) == 1
    assert b"release_pool" in L.qipb200_last_error(None)
