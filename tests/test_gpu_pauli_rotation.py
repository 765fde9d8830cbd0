"""Pauli-string rotations on the device (State.apply_pauli_rotations, qipb200_state_apply_pauli_rotations).

The device result is compared bit for bit (+-0 equal) with the numpy emulator of tests/pauli_rot_ref.py, and within
pauli_rot_ref.bound of its long-double reference (tests/test_pauli_rotation_cpu.py pins both to expm of Kronecker
products and to the oracle run of the MatrixOp decomposition).  The worst |got - want| / bound per group of checks is
printed (run with -s to see it)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import fullsize_ref as fr
import pauli_ref as pr
import pauli_rot_ref as rr
from rustqip_b200 import circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, pauli_rotation_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
WORST = {}


def note(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[apply_pauli_rotations] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-40s %.3e" % (k, WORST[k]))


def same_values(a, b):
    """Equal value for value (+-0 equal, no NaN)."""
    return np.array_equal(a, b)


def families(n, rng):
    """Term families: Ising step (tile pairs past n = 11), UCC-style strings, all-X / all-Y / all-Z, identities,
    random strings of every weight, and a run of over 300 X/Y terms (past the 256 descriptors kept in shared
    memory) mixed with a shared out-of-tile mask."""
    out = {"ising": rr.ising_step(n),
           "mix": [[("X", q) for q in range(n)], [], [("Y", q) for q in range(n)], [("Z", q) for q in range(n)], []]}
    out["mix"] += [[(l, q)] for q in range(n) for l in "XYZ"]
    for i in range(2 * n + 6):
        qs = rng.choice(n, size=1 + i % n, replace=False)
        out["mix"].append([(str(rng.choice(list("XYZ"))), int(q)) for q in qs])
    if n >= 4:
        out["ucc"] = rr.ucc_strings(n, 24, n)
    low = list(range(max(0, n - 6), n))  # the 4 low index bits and 2 above them
    long_run = []
    if n >= 14:  # index bits 4 and 5 become high tile bits, then 8 high bits the tile-pair mask of the sweep
        long_run = [[("X", n - 5), ("Y", n - 6)], [("X", q) for q in range(8)]]
    for i in range(300):
        qs = rng.choice(low, size=1 + i % len(low), replace=False)
        t = [(str(rng.choice(list("XY"))), int(q)) for q in qs]
        if n >= 14 and i % 3 == 0:
            t += [("X", q) for q in range(8)]  # more high bits than a tile holds: the sweep's tile-pair mask
        if i % 5 == 0:
            t += [("Z", int(q)) for q in range(n) if q not in dict((b, a) for a, b in t)][:3]
        long_run.append(t)
    out["long run"] = long_run + [[("Z", int(q)) for q in rng.choice(n, size=min(n, 3), replace=False)]
                                  for _ in range(40)]
    return out


def check_accuracy(group, psi0, n, terms, angles, got, dtype):
    ref = rr.rotate_ref(psi0, n, terms, angles)
    b = rr.bound(len(terms), float(np.linalg.norm(np.asarray(psi0).astype(C128))), dtype)
    err = float(np.max(np.abs(np.asarray(got).astype(np.clongdouble) - ref)))
    assert err <= b, (group, n, err, b)
    note(group, err / b)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_exact_against_emulator(ctx, dtype):
    name = np.dtype(dtype).name
    for n in range(1, 19):
        rng = np.random.default_rng(2000 + n)
        fam = families(n, rng)
        with State(n, dtype, ctx) as st:
            for k, (fname, terms) in enumerate(sorted(fam.items())):
                psi0 = circuits.random_state(n, 300 + 7 * n + k, dtype)
                angles = rng.uniform(-6.5, 6.5, size=len(terms))
                st.upload(psi0)
                st.apply_pauli_rotations(terms, angles)
                got = st.download()
                want = rr.emulate(psi0, n, terms, angles, dtype)
                assert same_values(got, want), (name, n, fname, int(np.sum(got != want)))
                if n <= 16 or fname != "long run":
                    check_accuracy("reference %s" % name, psi0, n, terms, angles, got, dtype)


@pytest.mark.parametrize("dtype", [C128, C64])
def test_grouping_determinism_and_zero_angles(ctx, dtype):
    n = 16
    rng = np.random.default_rng(5)
    fam = families(n, rng)
    terms = fam["ising"] + fam["ucc"] + fam["mix"][:20] + fam["long run"][:40]
    angles = rng.uniform(-3, 3, size=len(terms))
    psi0 = circuits.random_state(n, 6, dtype)
    with State(n, dtype, ctx) as st:
        st.upload(psi0)
        st.apply_pauli_rotations(terms, angles)
        one = st.download()
        st.upload(psi0)
        st.apply_pauli_rotations(terms, angles)
        again = st.download()
        assert np.array_equal(one.view(np.uint8), again.view(np.uint8))
        st.upload(psi0)
        for t, a in zip(terms, angles):
            st.apply_pauli_rotations([t], [a])
        each = st.download()
        assert same_values(one, each)
        st.upload(psi0)
        st.apply_pauli_rotations(terms, np.zeros(len(terms)))
        assert same_values(st.download(), psi0)
        st.apply_pauli_rotations([], [])
        assert same_values(st.download(), psi0)


def test_launch_count_matches_plan(ctx):
    n = 20
    rng = np.random.default_rng(9)
    fam = families(n, rng)
    cases = [rr.ising_step(n), rr.z_pairs(n), [[("X", q) for q in range(n)]], fam["ucc"], fam["long run"],
             rr.qaoa_layer(n)]
    with State(n, C128, ctx) as st:
        st.upload(circuits.random_state(n, 10, C128))
        for terms in cases:
            sweeps = pauli_rotation_plan(n, C128, terms)
            l0 = ctx.kernel_launches()
            st.apply_pauli_rotations(terms, rng.uniform(-1, 1, size=len(terms)))
            assert ctx.kernel_launches() - l0 == sweeps
        l0 = ctx.kernel_launches()
        st.apply_pauli_rotations([], [])
        assert ctx.kernel_launches() == l0
    # the long run is one tile-pair sweep with more descriptors than shared memory keeps
    assert pauli_rotation_plan(n, C128, fam["long run"]) == 1 and len(fam["long run"]) > 256


def test_cross_check_with_decomposition(ctx):
    """n = 20: the native rotations against apply_schedule of the CNOT-ladder decomposition.  Both lie within their
    own bound of the exact result: the native one within pauli_rot_ref.bound, the schedule within sqrt(2) gamma_{8k}
    for k ops (each 2x2 op rounds its two products and the sum, and the matrix entries)."""
    n = 20
    rng = np.random.default_rng(20)
    terms = rr.ising_step(n) + rr.ucc_strings(n, 16, 3) + [[("Y", q) for q in range(n)], []]
    angles = rng.uniform(-3, 3, size=len(terms))
    ops = rr.decompose_all(terms, angles)
    psi0 = circuits.random_state(n, 21, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi0)
        b.upload(psi0)
        a.apply_pauli_rotations(terms, angles)
        b.apply_schedule(ops)
        got, other = a.download(), b.download()
    bnd = rr.bound(len(terms), 1.0, C128) + math.sqrt(2) * rr.gamma(8 * len(ops), rr.U[C128])
    err = float(np.max(np.abs(got - other)))
    assert err <= bnd, (err, bnd)
    note("decomposition n=20 f64", err / bnd)


def test_validation_leaves_state_untouched(ctx):
    n = 12
    psi0 = circuits.random_state(n, 12, C128)
    long = rr.ising_step(n) * 20
    with State(n, C128, ctx) as st:
        st.upload(psi0)
        cases = [
            (long + [[("W", 1)]], INVALID_ARG, "not 'X', 'Y' or 'Z'"),
            (long + [[("X", n)]], BAD_INDEX, "out of range"),
            (long + [[("X", 1), ("Z", 1)]], BAD_INDEX, "repeated"),
        ]
        for terms, code, msg in cases:
            with pytest.raises(CircuitError) as e:
                st.apply_pauli_rotations(terms, np.ones(len(terms)))
            assert e.value.status == code and msg in str(e.value)
        for bad in (np.nan, np.inf, -np.inf):
            angles = np.ones(len(long))
            angles[-1] = bad
            with pytest.raises(CircuitError) as e:
                st.apply_pauli_rotations(long, angles)
            assert e.value.status == INVALID_ARG and "not finite" in str(e.value)
        with pytest.raises(ValueError):
            st.apply_pauli_rotations(long, np.ones(len(long) - 1))
        assert same_values(st.download(), psi0)
        # NULL angles through the C entry
        from rustqip_b200 import _lib
        from rustqip_b200.state import _marshal_paulis, _ptr
        qs, ls, lens = _marshal_paulis([[("X", 0)]])
        assert _lib.lib().qipb200_state_apply_pauli_rotations(st._h, _ptr(qs), ls, _ptr(lens), 1, None) == INVALID_ARG
        assert "NULL angles" in _lib.lib().qipb200_last_error(ctx.handle).decode()
        assert same_values(st.download(), psi0)


def test_refusal_keeps_pending_collapse_and_rotation_applies_it(ctx):
    n = 16
    psi0 = circuits.random_state(n, 31, C128)
    rng = np.random.default_rng(31)
    terms = families(n, rng)["mix"]
    angles = rng.uniform(-2, 2, size=len(terms))
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi0)
        b.upload(psi0)
        m, p = a.measure([0, 5], 0.41)
        assert p > 0
        with pytest.raises(CircuitError):
            a.apply_pauli_rotations(terms + [[("Q", 0)]], np.ones(len(terms) + 1))
        l0 = ctx.kernel_launches()
        a.apply_pauli_rotations(terms, angles)  # applies the collapse measure left pending first
        assert ctx.kernel_launches() - l0 == pauli_rotation_plan(n, C128, terms) + 1
        b.collapse([0, 5], m, p)
        collapsed = b.download()
        b.apply_pauli_rotations(terms, angles)
        got, want = a.download(), b.download()
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    assert same_values(got, rr.emulate(collapsed, n, terms, angles, C128))


def test_sharded_state_is_unsupported(ctx):
    with State(12, C128, ctx, rank=0, world_size=2) as st:
        with pytest.raises(CircuitError) as e:
            st.apply_pauli_rotations([[("Z", 0)]], [0.5])
        assert e.value.status == UNSUPPORTED


_ROTATE_WORKER = r"""
import numpy as np
import pauli_rot_ref as rr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 18
rng = np.random.default_rng(18)
terms = rr.ising_step(n) + rr.ucc_strings(n, 20, 5) + [[("Y", q) for q in range(n)], []]
angles = rng.uniform(-3, 3, size=len(terms))
ops = circuits.random_circuit(n, 10, 11, "H,T,CNOT") + circuits.qft(n)[:60]
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as a, State(n, np.complex128, ctx) as b:
        for st in (a, b):
            st.set_basis(3)
            st.apply_schedule(ops)
        before = b.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        psi = a.download()
        b.apply_pauli_rotations(terms, angles)
        assert np.array_equal(b.qubit_map(), before), "apply_pauli_rotations changed the layout"
        got = b.download()
want = rr.emulate(psi, n, terms, angles, np.complex128)
assert np.array_equal(got, want), int(np.sum(got != want))
print("ROTATE bit-exact ok")
"""


def test_permuted_layout_is_rotated_in_place():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "bit-exact ok" in p.stdout


# ---- full size ----------------------------------------------------------------------------------------------------

class Holder:
    """One full-size state at a time; freeing it returns its buffer to the device (at most 32 GiB alive)."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.st = None
        ctx.release_pool()

    def take(self, n, dtype):
        self.release()
        self.st = State(n, dtype, self.ctx)
        return self.st

    def release(self):
        if self.st is not None:
            self.st.free()
            self.st = None
        self.ctx.release_pool()


@pytest.fixture(scope="module")
def holder(ctx):
    h = Holder(ctx)
    yield h
    h.release()


W = 12  # window: 2^12 amplitudes


def window_offsets(n):
    top = (1 << n) - (1 << W)
    return sorted(set(min(o, top) for o in (0, 1 << 31, (1 << 32) - (1 << W), top, (1 << (n - 1)) + (5 << W))))


def check_windows(st, n, dtype, want_fn, bound, label):
    worst = 0.0
    for off in window_offsets(n):
        got = st.download(offset=off, length=1 << W)
        want = want_fn(np.arange(off, off + (1 << W), dtype=np.uint64))
        exact = np.zeros(1 << W, dtype=bool) if bound > 0 else np.ones(1 << W, dtype=bool)
        worst = max(worst, fr.check_window(got, want, np.ones(1 << W, dtype=np.longdouble), 1.0, exact, bound,
                                           label, off))
    return worst


@pytest.mark.parametrize("n,dtype", [(30, C128), (32, C64)], ids=["n30_f64", "n32_f32"])
def test_full_size_closed_forms(holder, n, dtype):
    name = "n%d %s" % (n, np.dtype(dtype).name)
    R = np.float64 if dtype == C128 else np.float32
    st = holder.take(n, dtype)
    # exp(-i theta/2 X^n)|0..0> = cos|0..0> - i sin|1..1>, exactly c and s rounded to the state's precision
    th = 1.1
    st.set_basis(0)
    st.apply_pauli_rotations([[("X", q) for q in range(n)]], [th])
    c, s = R(math.cos(th / 2)), R(math.sin(th / 2))

    def ghz(idx):
        w = np.zeros(idx.shape, dtype=np.clongdouble)
        w[idx == 0] = np.clongdouble(complex(c, 0))
        w[idx == (1 << n) - 1] = np.clongdouble(complex(0, -s))
        return w

    check_windows(st, n, dtype, ghz, 0.0, name + " X^n")
    assert abs(st.norm2() - (float(c) ** 2 + float(s) ** 2)) <= 1e-14
    # single-qubit X rotations from |0..0>: <Z_q> = cos theta_q, <Y_q> = -sin theta_q
    qs = [0, 1, n // 2, n - 5, n - 1]
    ths = [0.3, -1.2, 2.5, 0.9, -2.9]
    st.set_basis(0)
    st.apply_pauli_rotations([[("X", q)] for q in qs], ths)
    ev = st.expect_paulis([[("Z", q)] for q in qs] + [[("Y", q)] for q in qs])
    tol = pr.bound(n, 1.0) + 4 * rr.bound(len(qs), 1.0, dtype)
    for i, (q, t) in enumerate(zip(qs, ths)):
        for got, want in ((ev[i], math.cos(t)), (ev[len(qs) + i], -math.sin(t))):
            assert abs(got - want) <= tol, (name, q, got, want, tol)
            note("full %s X_q expect" % name, abs(got - want) / tol)
    # Z strings on |+..+>: the phase product closed form
    zt = [[("Z", 0)], [("Z", 0), ("Z", n - 1)], [("Z", q) for q in range(n)], [("Z", 3), ("Z", n // 2), ("Z", n - 2)],
          []]
    za = [0.7, -1.3, 0.4, 2.2, 0.5]
    st.set_basis(0)
    st.apply_schedule([gates.h(q) for q in range(n)])
    st.apply_pauli_rotations(zt, za)
    amp = np.longdouble(2.0) ** (-n / 2)

    def phases(idx):
        ph = np.zeros(idx.shape, dtype=np.longdouble)
        for t, a in zip(zt, za):
            _, z, _ = rr.masks(n, t)
            sgn = np.where(rr._parity(idx & np.uint64(z)), -1, 1).astype(np.longdouble)
            ph += -np.longdouble(a) / 2 * sgn
        return amp * (np.cos(ph) + 1j * np.sin(ph)).astype(np.clongdouble)

    # per element: the rotations are diagonal (relative sqrt(2) gamma_5T), plus the H layer's rounding (relative
    # gamma_8n: a few roundings per qubit on every amplitude)
    bnd = float(amp) * (math.sqrt(2) * rr.gamma(5 * len(zt), rr.U[dtype]) + rr.gamma(8 * n, rr.U[dtype]))
    note("full %s Z strings" % name, check_windows(st, n, dtype, phases, bnd, name + " Z strings"))
    holder.release()


def test_full_size_ucc_round_trip(holder):
    """N = 30 f64 from the H layer: the UCC-style strings natively, then their inverse through apply_schedule of the
    decomposition, give back 2^(-n/2) everywhere within the two bounds."""
    n = 30
    st = holder.take(n, C128)
    terms = rr.ucc_strings(n, 64, 64)
    rng = np.random.default_rng(64)
    angles = rng.uniform(-3, 3, size=len(terms))
    st.set_basis(0)
    st.apply_schedule([gates.h(q) for q in range(n)])
    st.apply_pauli_rotations(terms, angles)
    inv = rr.decompose_all(terms[::-1], -angles[::-1])
    st.apply_schedule(inv)
    amp = np.longdouble(2.0) ** (-n / 2)
    bnd = rr.bound(len(terms), 1.0, C128) + math.sqrt(2) * rr.gamma(8 * (len(inv) + n), rr.U[C128])
    ratio = check_windows(st, n, C128, lambda idx: np.full(idx.shape, amp, dtype=np.clongdouble), bnd, "ucc round trip")
    note("full n30 f64 ucc round trip", ratio)
    assert abs(st.norm2() - 1.0) <= 1e-9
    holder.release()
