"""Every per-gate kernel, the fused passes, sampling and measure at full state size, against extended-precision
references on windows (tests/fullsize_ref.py; the helpers are pinned to the oracle by tests/test_fullsize_ref_cpu.py).

Sizes: N = 30 f64 (16 GiB, the headline size), N = 31 f32 (16 GiB: amplitude indices >= 2^31, float offsets >= 2^32),
N = 32 f32 (32 GiB: amplitude indices >= 2^32), and N = 28 f64 for the out-of-place row kernel, whose arena doubles the
memory.  N = 31/32 f64 would need 32-64 GiB per state and are not run.  One size is alive at a time: at most 32 GiB.

Each check works on windows of 2^w amplitudes: the op's inputs are downloaded before it runs, the outputs after, and
every element must satisfy |got - want| <= c u sum_j |m_ij| |x_j| (permutations and untouched rows: bit-identical).
The worst |got - want| / bound per kernel class and size is printed (run with -s to see it)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import fullsize_ref as fr
from rustqip_b200 import circuits
from rustqip_b200.state import State

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
SIZES = [(30, C128), (31, C64), (32, C64)]
SIZE_IDS = ["n30_f64", "n31_f32", "n32_f32"]


class Holder:
    """The states of one size; taking another size frees them first, so device memory stays <= 32 GiB.

    A freed state's buffer would stay with the context for the next state of its size (qipb200_state_free keeps one):
    release() hands it back to the device too, and the module starts by dropping what earlier modules left there."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.states = []
        ctx.release_pool()

    def take(self, n, dtype, count):
        self.release()
        self.states = [State(n, dtype, self.ctx) for _ in range(count)]
        return self.states

    def release(self):
        for s in self.states:
            s.free()
        self.states = []
        self.ctx.release_pool()


@pytest.fixture(scope="module")
def holder(ctx):
    h = Holder(ctx)
    yield h
    h.release()


def report(title, worst):
    print("\n[full size] %s: worst |got - want| / bound per kernel class" % title)
    for k in sorted(worst):
        print("  %-34s %.3e" % (k, worst[k]))


def kernel_class(name, dtype):
    """The kernel a zoo op must run on (api.cu: launch_local_op); run_op_case checks it against the library's
    per-kernel launch counters."""
    if name.endswith("gather"):
        return "k_gather"
    m = re.search(r"dense(\d+)", name)
    if m:
        k = int(m.group(1))
        if k <= 4:
            return "k_dense<%d>" % k
        if k in (5, 6) and dtype == C128 and os.environ.get("QIPB200_DENSE_DMMA", "1") != "0":
            return "k_dense_dmma<%d>" % k
        return "k_dense5" if k == 5 else "k_dense_big"
    m = re.search(r"diag(\d+)", name)
    if m:
        return "k_diag" if int(m.group(1)) <= 4 else "k_diag_wide"
    if name.startswith(("t_", "cz", "cphase")) or name.endswith("phase"):
        return "k_diag"
    return "k_exchange"


def prepare(st, a):
    st.set_basis(0)
    st.apply_schedule(a.prep_ops(), fusion=False)


def windows_of(st, bases, w):
    return {b: st.download(offset=b, length=1 << w) for b in bases}


def run_op_case(ctx, st, n, dtype, name, op, launches, seed, extra=()):
    """Apply one op in place and check its windows; returns the worst bound ratio."""
    model = fr.OpModel(n, op, dtype)
    w, bases = fr.window_plan(n, model, seed, extra)
    offs = fr.input_offsets(model, w)
    inputs = {b: {s: st.download(offset=b ^ s, length=1 << w) for s in offs} for b in bases}
    l0, k0 = ctx.kernel_launches(), ctx.kernel_counts()
    st.apply_op(op)
    assert ctx.kernel_launches() - l0 == launches, (name, ctx.kernel_launches() - l0)
    ran = {k: v - k0.get(k, 0) for k, v in ctx.kernel_counts().items() if v != k0.get(k, 0)}
    assert ran == {kernel_class(name, dtype).split("<")[0]: launches}, (name, ran)
    worst = 0.0
    u = fr.unit_roundoff(dtype)
    for b in bases:
        want, acc, c, exact = fr.op_window_reference(n, op, inputs[b], b, dtype, model)
        got = st.download(offset=b, length=1 << w)
        worst = max(worst, fr.check_window(got, want, acc, c, exact, u, "n=%d %s" % (n, name), b))
    return worst, model, {b: inputs[b][0] for b in bases}, w


def roundtrip_bound(model, dtype, amax):
    """|U^-1 (U x) - x| per element: both applications' bounds plus the rounding of the inverse's entries."""
    u = fr.unit_roundoff(dtype)
    c = 4.0 * float(model.row_nnz.max())
    r = model.abs_row_sum
    return 4 * c * u * r * r * amax


def extra_windows(n):
    return {30: (), 31: ((1 << 30) - 1, 1 << 30), 32: ((1 << 31) - 1, 1 << 31)}.get(n, ())


def run_zoo(ctx, holder, n, dtype, zoo, seed):
    a = fr.ProductPhaseState(n, dtype, seed)
    with_ref = n <= 31
    states = holder.take(n, dtype, 2 if with_ref else 1)
    st = states[0]
    for s in states:
        prepare(s, a)
    if with_ref:
        ref = states[1]
        assert st.max_abs_diff(ref) == 0.0
    amax = a.max_abs()
    worst = {}
    allowed = 0.0
    # permutations first: while the state is still bit-identical to the copy, each round trip must give 0
    zoo = sorted(zoo, key=lambda e: kernel_class(e[0], dtype) != "k_exchange")
    for i, (name, op, launches) in enumerate(zoo):
        r, model, before, w = run_op_case(ctx, st, n, dtype, name, op, launches, seed + i, extra_windows(n))
        cls = kernel_class(name, dtype)
        worst[cls] = max(worst.get(cls, 0.0), r)
        st.apply_op(fr.inverse_op(op))
        exact = bool(model.row_exact.all())
        rt = 0.0 if exact else roundtrip_bound(model, dtype, amax)
        if with_ref:
            allowed += rt
            d = st.max_abs_diff(ref)
            assert d <= allowed, (name, d, allowed)
        else:
            for b, x in before.items():
                y = st.download(offset=b, length=1 << w)
                if exact:
                    assert np.array_equal(y, x), (name, b)
                else:
                    assert np.max(np.abs(y.astype(C128) - x.astype(C128))) <= rt, (name, b)
    return worst


# ---------------------------------------------------------------------------------------------------------------
# QIPB200_DENSE_DMMA=0: the f64 5- and 6-qubit blocks on the FMA kernels (k_dense5 / k_dense_big) at N = 30.
# The switch is read once per process, so it runs in a child; it starts before this module holds any state.
# ---------------------------------------------------------------------------------------------------------------
_DMMA_OFF_WORKER = r"""
import sys
sys.path.insert(0, "tests")
import numpy as np
import fullsize_ref as fr
import test_gpu_full_size as t
from rustqip_b200.state import Context, State
n = 30
with Context(0) as ctx:
    a = fr.ProductPhaseState(n, np.complex128, 505)
    with State(n, np.complex128, ctx) as st:
        t.prepare(st, a)
        worst = {}
        for i, (name, op, launches) in enumerate(fr.fullsize_zoo(n, 506)):
            if not name.startswith(("dense5", "dense6", "c1dense5", "c1dense6")):
                continue
            r, *_ = t.run_op_case(ctx, st, n, np.complex128, name, op, launches, 600 + i)
            cls = t.kernel_class(name, np.complex128)
            worst[cls] = max(worst.get(cls, 0.0), r)
            st.apply_op(fr.inverse_op(op))
        t.report("n=30 f64, QIPB200_DENSE_DMMA=0", worst)
        assert set(worst) == {"k_dense5", "k_dense_big"}, worst
"""


def test_dense_f64_fma_kernels_with_dmma_off(holder):
    holder.release()
    env = dict(os.environ, QIPB200_DENSE_DMMA="0", PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-c", _DMMA_OFF_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    sys.stdout.write(p.stdout[-3000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]


# ---------------------------------------------------------------------------------------------------------------
# per-gate kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,dtype", SIZES, ids=SIZE_IDS)
def test_per_gate_kernels_full_size(ctx, holder, n, dtype):
    worst = run_zoo(ctx, holder, n, dtype, fr.fullsize_zoo(n, 1000 + n), 2000 + n)
    report("n=%d %s per-gate" % (n, np.dtype(dtype).name), worst)
    want = {"k_dense<1>", "k_dense<2>", "k_dense<3>", "k_dense<4>", "k_diag", "k_diag_wide", "k_exchange",
            "k_dense_big", "k_dense_dmma<5>" if dtype == C128 else "k_dense5"}
    assert want <= set(worst), set(worst)


def test_row_kernel_fallback_n28(ctx, holder):
    """A 7-qubit CSR sparse op and a 9-control, 4-target op take the out-of-place row kernel (k_gather)."""
    worst = run_zoo(ctx, holder, 28, C128, fr.fullsize_zoo(28, 1028, in_place=False), 2028)
    report("n=28 f64 row kernel", worst)
    assert set(worst) == {"k_gather"}


# ---------------------------------------------------------------------------------------------------------------
# fused passes against closed forms
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jit", ["sync", "off"])
@pytest.mark.parametrize("n,dtype", SIZES, ids=SIZE_IDS)
def test_fused_qft_of_basis_state(ctx, holder, monkeypatch, n, dtype, jit):
    """Magnitudes and phases of the fused QFT of |x> against 2^(-n/2) exp(2 pi i x y / 2^n)."""
    monkeypatch.setenv("QIPB200_JIT", jit)
    (st,) = holder.take(n, dtype, 1)
    x = (1 << n) - 1 if jit == "sync" else 0xB6DB6DB7 & ((1 << n) - 1)
    st.set_basis(x)
    j0 = ctx.jit_stats()
    st.apply_schedule(circuits.qft(n))
    j1 = ctx.jit_stats()
    passes, on_generated = j1["tile_passes"] - j0["tile_passes"], j1["jit_passes"] - j0["jit_passes"]
    assert passes > 0
    # sync: every pass on a generated kernel (TMA tile moves); off: every pass on the interpreter
    assert on_generated == (passes if jit == "sync" else 0), (jit, passes, on_generated, j1["note"])
    w = 12
    rng = np.random.default_rng(n)
    bases = [0, (1 << n) - (1 << w), (1 << (n - 1)) - (1 << w), 1 << (n - 1)]
    bases += [(e // (1 << w)) << w for e in extra_windows(n)] + [int(v) << w for v in rng.integers(0, 1 << (n - w), 3)]
    bound = fr.qft_bound(n, dtype)
    worst = 0.0
    for b in bases:
        got = st.download(offset=b, length=1 << w).astype(fr.LD)
        want = fr.qft_basis_amp(n, x, np.arange(b, b + (1 << w), dtype=np.uint64))
        err = np.abs(got - want)
        i = int(np.argmax(err))
        assert err[i] <= bound, "offset %d index %d got %r want %r |diff| %.3e > %.3e" % (
            b, b + i, complex(got[i]), complex(want[i]), float(err[i]), bound)
        worst = max(worst, float(err[i]) / bound)
    report("n=%d %s fused QFT jit=%s" % (n, np.dtype(dtype).name, jit), {"tile pass": worst})


def check_analytic_windows(st, a, bases, w, src_of=None, scale=None, label="", extra=0.0):
    """Windows equal a(src_of(i)) (times `scale`) within the preparation bound (+ `extra` relative); returns the
    worst ratio."""
    eps = a.prep_rel_error() + extra
    worst = 0.0
    for b in bases:
        idx = np.arange(b, b + (1 << w), dtype=np.uint64)
        src = src_of(idx) if src_of else idx
        want = a.amp(src)
        if scale is not None:
            want = want * scale(src)
        got = st.download(offset=b, length=1 << w).astype(fr.LD)
        err = np.abs(got - want)
        zero = want == 0
        assert np.all(got[zero] == 0), (label, b)
        bound = eps * np.abs(want)
        ratio = np.where(zero, 0, err / np.where(zero, 1, bound))
        i = int(np.argmax(ratio))
        assert ratio[i] <= 1, "%s offset %d index %d got %r want %r |diff| %.3e > %.3e" % (
            label, b, b + i, complex(got[i]), complex(want[i]), float(err[i]), float(bound[i]))
        worst = max(worst, float(ratio[i]))
    return worst


def analytic_bases(n, w, seed):
    rng = np.random.default_rng(seed)
    bases = [0, (1 << n) - (1 << w), (1 << (n - 1)) - (1 << w), 1 << (n - 1)]
    bases += [(e // (1 << w)) << w for e in extra_windows(n)]
    return bases + [int(v) << w for v in rng.integers(0, 1 << (n - w), 3)]


@pytest.mark.parametrize("n,dtype", SIZES, ids=SIZE_IDS)
def test_fused_permutation_circuit(ctx, holder, n, dtype):
    """About 200 seeded permutation ops over all bits, fused, on the analytic state: windows equal a(pi^-1(i))."""
    a = fr.ProductPhaseState(n, dtype, 3000 + n)
    circ = fr.random_permutation_circuit(n, 200, 3100 + n)
    ops = [fr.perm_op(e) for e in circ]
    with_ref = n <= 31
    states = holder.take(n, dtype, 2 if with_ref else 1)
    st = states[0]
    w = 12
    bases = analytic_bases(n, w, n)
    for s in states:
        prepare(s, a)
    worst = {"preparation": check_analytic_windows(st, a, bases, w, label="prep")}
    before = windows_of(st, bases, w)
    l0 = ctx.kernel_launches()
    st.apply_schedule(ops)
    assert ctx.kernel_launches() - l0 < len(ops) // 4  # it fused
    worst["fused permutation"] = check_analytic_windows(
        st, a, bases, w, src_of=lambda idx: fr.perm_source(n, circ, idx), label="fused perm")
    if with_ref:
        states[1].apply_schedule(ops, fusion=False)
        assert st.max_abs_diff(states[1]) == 0.0
    else:
        st.apply_schedule(ops[::-1])  # every op is an involution
        after = windows_of(st, bases, w)
        for b in bases:
            assert np.array_equal(after[b], before[b]), b
    report("n=%d %s permutations" % (n, np.dtype(dtype).name), worst)


# ---------------------------------------------------------------------------------------------------------------
# measurement on the analytic state
# ---------------------------------------------------------------------------------------------------------------
MEASURE_SIZES = [(30, C128), (32, C64)]


def prob_tol(a, p, sums=1e-9):
    """2.5 eps_prep relative (|a|^2 of the prepared amplitudes) plus `sums` relative for the device's f64 sums of up to
    2^32 positive terms: 1e-9 covers the atomics of measure_probs / norm2 (about 2^20 additions per bin in any order);
    the fixed-order trees and scans of sample and measure add at most a few dozen roundings, 1e-12."""
    return (2.5 * a.prep_rel_error() + sums) * p + 1e-15


@pytest.mark.parametrize("n,dtype", MEASURE_SIZES, ids=["n30_f64", "n32_f32"])
def test_measurement_full_size(ctx, holder, n, dtype):
    a = fr.ProductPhaseState(n, dtype, 4000 + n)
    (st,) = holder.take(n, dtype, 1)
    prepare(st, a)
    w = 12
    bases = analytic_bases(n, w, 7 * n)
    worst = {"preparation": check_analytic_windows(st, a, bases, w, label="prep")}
    Q = lambda bits: [n - 1 - b for b in bits]  # noqa: E731
    total = float(a.marginal([0]).sum())
    assert abs(st.norm2() - total) <= prob_tol(a, total)
    # measure_probs / measure_prob: index bits >= 12 (whole sampling chunks) mixed with bits < 12 (inside a chunk)
    for bits in ([n - 1, 12, 3], [0, 11, 12], [n - 1, n - 10, 7, 0], [13, 31 if n > 31 else n - 2, 5]):
        idx = Q(bits)
        want = a.marginal(idx)
        got = st.measure_probs(idx)
        assert np.all(np.abs(got - want) <= prob_tol(a, want)), (bits, got, want)
        for m in (0, (1 << len(idx)) - 1, 5 % (1 << len(idx))):
            assert abs(st.measure_prob(m, idx) - want[m]) <= prob_tol(a, want[m]), (bits, m)
    # sample: 2^16 draws over all qubits (bit i of the outcome = index bit i) against the CDF descent; a draw is
    # compared on the qubits the descent decides with a margin above the error of the cumulative sums
    draws = np.random.default_rng(n).random(1 << 16)
    got = st.sample(list(range(n - 1, -1, -1)), draws=draws)
    tol = prob_tol(a, 1.0, 1e-12)
    full = levels = 0
    for r, g in zip(draws, got):
        idx, margins = a.descend(float(r))
        bad = np.nonzero(margins <= tol)[0]
        L = int(bad[0]) if bad.size else n
        if L:
            assert int(g) >> (n - L) == idx >> (n - L), (r, int(g), idx, L)
        full += L == n
        levels += L
    print("\n[full size] n=%d sample: %d of %d draws compared on all %d qubits, %.1f qubits per draw on average "
          "(the rest lie closer to a boundary than %.1e)" % (n, full, len(draws), n, levels / len(draws), tol))
    assert levels >= 8 * len(draws)
    # measure on a top and a low qubit
    circ = fr.random_permutation_circuit(n, 60, 4100 + n)
    ops = [fr.perm_op(e) for e in circ]
    for q, r in ((0, 0.3), (n - 1, 0.71)):
        prepare(st, a)
        m, p = st.measure([q], r)
        pw = a.marginal([q])[m]
        assert abs(p - pw) <= prob_tol(a, pw, 1e-12), (q, m, p, pw)
        idx, margins = a.descend(r)
        if margins[: q + 1].min() > tol:
            assert m == (idx >> (n - 1 - q)) & 1
        keep = lambda src: np.where(a.bit(src, q) == m, fr.LD(1) / np.sqrt(fr.LD(p)), fr.LD(0))  # noqa: E731
        worst["measure q=%d, download" % q] = check_analytic_windows(st, a, bases, w, scale=keep, label="collapse",
                                                                     extra=4 * fr.unit_roundoff(dtype))
        # the pending collapse folded into the next fused schedule == collapse, then the schedule
        results = []
        for explicit in (False, True):
            prepare(st, a)
            if explicit:
                st.collapse([q], m, p)
            else:
                assert st.measure([q], r) == (m, p)
            st.apply_schedule(ops)
            src_of = lambda idx: fr.perm_source(n, circ, idx)  # noqa: E731
            worst["measure q=%d, fused %s" % (q, "after collapse" if explicit else "pending")] = check_analytic_windows(
                st, a, bases, w, src_of=src_of, scale=keep, label="collapse+perm", extra=4 * fr.unit_roundoff(dtype))
            results.append(windows_of(st, bases, w))
        # both paths multiply each kept amplitude by the same collapse_multiplier(p) once (a 1-qubit diagonal folded
        # into the pass, or k_collapse) and then only move amplitudes: bit-identical
        for b in bases:
            assert np.array_equal(results[0][b], results[1][b]), (q, b, np.max(np.abs(
                results[0][b].astype(C128) - results[1][b].astype(C128))))
    report("n=%d %s measurement" % (n, np.dtype(dtype).name), worst)
