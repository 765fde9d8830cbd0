"""Entanglement spectrum and von Neumann entropy of a bipartition on the device (State.entanglement_spectrum,
qipb200_state_entanglement_spectrum).

Every tolerance comes from tests/spectrum_ref.py: the eigenvalues within Weyl's bound of numpy's svd of the reshaped
state, the entropy within the Fannes-Audenaert bound, sum lambda and sum lambda^2 against norm2 and purity within the
sum of both calls' bounds.  On dyadic states the returned matrix must equal the exact G bit for bit.  The worst
|got - want| / bound per group is printed (run with -s to see it)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import purity_ref as pu
import spectrum_ref as sr
from rustqip_b200 import _lib, circuits, gates
from rustqip_b200.errors import CircuitError
from rustqip_b200.state import State, entanglement_spectrum_plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, BAD_INDEX, UNSUPPORTED = 1, 3, 7
WORST = {}
OBSERVED = {}


def note(group, got, bound):
    r = got / bound if bound > 0 else (0.0 if got == 0 else math.inf)
    WORST[group] = max(WORST.get(group, 0.0), r)
    assert got <= bound, (group, got, bound)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\n[entanglement_spectrum] worst |got - want| / bound per group")
    for k in sorted(WORST):
        print("  %-52s %.3e" % (k, WORST[k]))
    for k in sorted(OBSERVED):
        print("  observed: %s = %s" % (k, OBSERVED[k]))


def call(st, qs, rho=False):
    """(eigs, rho or None, T, S) of one call."""
    return st._spectrum(qs, rho)


def side_lists(n, s, rng):
    """Prefix (the high index bits), suffix (the low bits), scattered, and the complements of the prefix and of the
    scattered side (k = n - s: the call works on the smaller side, the qubits not passed)."""
    pre = list(range(s))
    suf = list(range(n - s, n))[::-1]
    sc = [int(q) for q in rng.permutation(n)[:s]]
    lists = [pre, suf, sc]
    if 2 * s < n:
        lists += [[q for q in range(n) if q not in pre], [q for q in range(n) if q not in sc]]
    return lists


def check_call(group, st, psi, n, qs, got=None):
    """Eigenvalues, entropy, trace and sum of squares of one call against the svd reference and norm2 / purity."""
    eigs, _, T, S = call(st, qs) if got is None else got
    s = min(len(qs), n - len(qs))
    lam, Tref = sr.schmidt_ref(psi, n, qs)
    assert eigs.size == 1 << s and np.all(np.diff(eigs) <= 0), "descending"
    e = sr.eig_bound(n, s, Tref, float(lam[0]))
    note(group + " eigs", float(np.max(np.abs(eigs - lam))), e)
    dT = sr.trace_bound(n, s, Tref) + 1e-15 * Tref
    note(group + " trace", abs(T - Tref), dT)
    Sref = sr.entropy(lam, Tref)
    note(group + " entropy", abs(S - Sref), sr.entropy_bound(s, Tref, e, dT, Sref))
    # sum lambda = T, and T against norm2
    nrm = st.norm2()
    note(group + " sum eigs vs out2[0]", abs(float(np.sum(eigs)) - T), (1 << s) * e + sr.gamma(1 << s) * Tref + dT)
    note(group + " out2[0] vs norm2", abs(T - nrm), dT + sr.gamma(1 << n) * Tref)
    # sum lambda^2 = purity, and the Renyi-2 entropy of the spectrum against renyi2_entropy
    P, Tp = st._purity2(qs)
    e_dev = sr.eig_bound(n, s, Tref, float(lam[0]), with_ref=False)
    bp, bt = pu.bound_cs(n, s, P, Tp)
    bsq = sr.sum_sq_bound(s, Tref, e_dev) + bp
    note(group + " sum eigs^2 vs purity", abs(float(np.sum(eigs ** 2)) - P), bsq)
    if P > 0:
        r2_spec = -math.log(float(np.sum(eigs ** 2)) / (T * T))
        r2 = st.renyi2_entropy(qs)
        b = bsq / (P - bsq) + 2 * (dT + bt) / (Tref - dT - bt) + 4 * sr.U_DOUBLE * (1 + abs(r2))
        note(group + " renyi2 spectrum vs renyi2_entropy", abs(r2_spec - r2), b)
    return eigs, T, S


@pytest.mark.parametrize("dtype", [C128, C64])
def test_against_reference(ctx, dtype):
    name = np.dtype(dtype).name
    for n in list(range(2, 17)) + [18, 20, 22, 24]:
        rng = np.random.default_rng(1700 + n)
        sides = range(0, n // 2 + 1) if n <= 16 else [12] if n == 24 else [1, 6, 10, 11]
        with State(n, dtype, ctx) as st:
            for kind in ("random", "circuit"):
                if kind == "random":
                    st.upload(circuits.random_state(n, 280 + n, dtype))
                else:
                    st.set_basis(2)
                    st.apply_schedule(circuits.random_circuit(n, 8, 0x5EED0700 + n, "H,T,CNOT"))
                psi = st.download()
                for s in sides:
                    lists = [list(range(n))] if s == 0 else side_lists(n, s, rng)
                    if n >= 18:  # large references: the prefix of the random state, the rest on the circuit's
                        lists = lists[:1] if kind == "random" else lists[2:] if n < 24 else []
                    for qs in lists:
                        r = sr.route(min(len(qs), n - len(qs)))
                        check_call("%s route %d" % (name, r), st, psi, n, qs)
        if n == 12:
            with State(n, dtype, ctx) as st:
                st.upload(circuits.random_state(n, 5, dtype))
                qs = [1, 4, 7, 10, 11]
                eigs = st.entanglement_spectrum(qs)
                lam = eigs[eigs > 0] / np.sum(eigs)
                assert st.entanglement_entropy(qs) == call(st, qs)[3]
                for alpha in (0.5, 2.0, 3.0):
                    assert abs(st.entanglement_entropy(qs, alpha) - sr.renyi(eigs, float(np.sum(eigs)), alpha)) <= 1e-12
                assert abs(st.entanglement_entropy(qs, math.inf) + math.log(lam.max())) <= 1e-12
                assert abs(st.entanglement_entropy(qs, 2.0) - st.renyi2_entropy(qs)) <= 1e-9


def dyadic_state(n, seed, e):
    """Re, Im in {-1, 0, 1} * 2^-e: every entry of G is an integer times 2^-2e."""
    rng = np.random.default_rng(seed)
    return (rng.integers(-1, 2, size=1 << n) + 1j * rng.integers(-1, 2, size=1 << n)) * 2.0 ** -e


def exact_gram(psi, n, qs, e):
    s = len(qs)
    if s < 12:
        return sr.gram_exact(psi, n, qs, e)
    import torch  # 2^12 and 2^13 square products: on the device, exact for the same reason
    M = sr.side_matrix(psi, n, qs) * 2.0 ** e
    re = torch.from_numpy(np.ascontiguousarray(M.real)).cuda()
    im = torch.from_numpy(np.ascontiguousarray(M.imag)).cuda()
    del M
    assert float(re.abs().max()) <= 1 and 2 * re.shape[1] < 2 ** 53
    Gr = (re @ re.T + im @ im.T).cpu().numpy()
    Gi = (im @ re.T - re @ im.T).cpu().numpy()
    del re, im
    torch.cuda.empty_cache()
    return (Gr + 1j * Gi) * 2.0 ** (-2 * e)


@pytest.mark.parametrize("s", list(range(1, 14)))
def test_rho_exact_on_dyadic_states(ctx, s):
    """rho is G bit for bit on dyadic states: the side's convention (prefix, suffix or scattered by s), the Hermitian
    mirror and the +0.0 diagonal; f32 too for s = 3, 11 and 13.  The eigenvalues are within twice the solver bound of
    eigvalsh of the exact G (both solvers backward stable)."""
    n = 2 * s if s >= 11 else max(2 * s + 2, 8)
    e = (n + 1) // 2
    psi = dyadic_state(n, 4100 + s, e)
    rng = np.random.default_rng(s)
    qs = side_lists(n, s, rng)[s % 3]
    G = exact_gram(psi, n, qs, e)
    dtypes = (C128, C64) if s in (3, 11, 13) else (C128,)
    for dtype in dtypes:
        with State(n, dtype, ctx) as st:
            st.upload(psi.astype(dtype))
            eigs, rho, T, S = call(st, qs, rho=True)
            assert np.array_equal(rho, G), (s, np.dtype(dtype).name)
            assert not np.any(np.signbit(np.diagonal(rho).imag)), "diagonal imaginary parts must be +0.0"
            assert np.array_equal(rho.T, np.conj(rho))
            assert T == float(np.sum(np.diagonal(G).real))
            if s <= 10:
                assert np.array_equal(rho.view(np.uint64), st.reduced_density(qs).view(np.uint64))
            del rho
    if s >= 12:
        import torch
        Gd = torch.from_numpy(G).cuda()
        ref = torch.linalg.eigvalsh(Gd).cpu().numpy()[::-1]
        del Gd
        torch.cuda.empty_cache()
    else:
        ref = np.linalg.eigvalsh(G)[::-1]
    note("dyadic eigs vs eigvalsh(exact G)", float(np.max(np.abs(eigs - ref))), 2 * sr.solver_bound(s, float(ref[0])))


def test_deterministic_and_launch_count(ctx):
    n = 22
    with State(n, C128, ctx) as st:
        st.upload(circuits.random_state(n, 43, C128))
        same_eigs = True
        for qs in ([0], [21, 3, 9], list(range(10)), list(range(11)), [q for q in range(n) if q % 2],
                   list(range(n)), list(range(3, n))):
            k = len(qs)
            a = call(st, qs, rho=k <= n - k)
            l0 = ctx.kernel_launches()
            b = call(st, qs, rho=k <= n - k)
            plan = entanglement_spectrum_plan(n, C128, qs)
            assert ctx.kernel_launches() - l0 == plan[2], (qs, plan)
            assert plan == sr.plan(n, qs)
            assert np.float64(a[2]).view(np.uint64) == np.float64(b[2]).view(np.uint64), qs
            if a[1] is not None:
                assert np.array_equal(a[1].view(np.uint64), b[1].view(np.uint64)), qs
            same_eigs &= bool(np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)))
            same_eigs &= np.float64(a[3]).view(np.uint64) == np.float64(b[3]).view(np.uint64)
        OBSERVED["eigenvalues and entropy bit-identical on repeat (n=22, routes 0..2)"] = same_eigs


def test_pending_set_basis_gives_a_pure_spectrum(ctx):
    for n, qs in ((12, [3, 5]), (22, list(range(11))), (24, list(range(5, 17))), (26, list(range(13)))):
        with State(n, C128, ctx) as st:
            st.set_basis((1 << n) - 7)
            l0 = ctx.kernel_launches()
            eigs, _, T, S = call(st, qs)
            assert ctx.kernel_launches() - l0 == entanglement_spectrum_plan(n, C128, qs)[2]
            want = np.zeros(eigs.size)
            want[0] = 1.0
            assert np.array_equal(eigs, want) and T == 1.0 and S == 0.0, (n, eigs[:3], T, S)


def test_sees_pending_collapse(ctx):
    n = 22
    psi = circuits.random_state(n, 22, C128)
    with State(n, C128, ctx) as a, State(n, C128, ctx) as b:
        a.upload(psi)
        b.upload(psi)
        m, p = a.measure([0, 5], 0.37)
        assert p > 0
        qs = list(range(11, 22))
        l0 = ctx.kernel_launches()
        got = call(a, qs)  # applies the collapse measure left pending (one more kernel)
        assert ctx.kernel_launches() - l0 == 1 + entanglement_spectrum_plan(n, C128, qs)[2]
        b.collapse([0, 5], m, p)
        collapsed = b.download()
        check_call("after measure f64", b, collapsed, n, qs, got)
        check_call("after measure f64 rdm route", b, collapsed, n, [3, 7], call(a, [3, 7]))


def test_refusals_leave_state_and_collapse(ctx):
    n = 14
    psi = circuits.random_state(n, 3, C128)
    lib = _lib.lib()
    with State(n, C128, ctx) as st, State(n, C128, ctx) as ref:
        st.upload(psi)
        ref.upload(psi)
        m, p = st.measure([2], 0.5)
        eigs, out2, rho = np.zeros(1 << 7), np.zeros(2), np.zeros(2 << 14)
        qs = np.array([0, 1, 2], dtype=np.uint64)
        q12 = np.arange(12, dtype=np.uint64)
        E, R, O = eigs.ctypes.data, rho.ctypes.data, out2.ctypes.data
        l0 = ctx.kernel_launches()
        raw = ((None, qs.ctypes.data, 3, E, 128, None, O, INVALID_ARG, None),
               (st._h, None, 1, E, 128, None, O, INVALID_ARG, "bad index list"),
               (st._h, qs.ctypes.data, 0, E, 128, None, O, INVALID_ARG, "bad index list"),
               (st._h, qs.ctypes.data, 3, None, 128, None, O, INVALID_ARG, "NULL eigs or out2"),
               (st._h, qs.ctypes.data, 3, E, 128, None, None, INVALID_ARG, "NULL eigs or out2"),
               (st._h, qs.ctypes.data, 3, E, 7, None, O, INVALID_ARG, "eigs_cap 7 is below the 8 eigenvalues"),
               (st._h, q12.ctypes.data, 12, E, 128, R, O, INVALID_ARG, "pass the complement"))
        for h, q, k, e, cap, r, o, code, msg in raw:
            assert lib.qipb200_state_entanglement_spectrum(h, q, k, e, cap, r, o) == code, (k, cap, msg)
            if msg:
                assert msg in lib.qipb200_last_error(ctx.handle).decode(), msg
        assert lib.qipb200_last_error(None).decode() == "entanglement_spectrum: NULL state"
        for bad, code, word in ((list(range(n)) + [0], INVALID_ARG, "bad index list"),
                                ([0, n], BAD_INDEX, "out of range"), ([4, 1, 4], BAD_INDEX, "repeated"),
                                ([], INVALID_ARG, "bad index list")):
            with pytest.raises(CircuitError) as e:
                st.entanglement_spectrum(bad)
            assert e.value.status == code and word in str(e.value), bad
        with pytest.raises(CircuitError) as e:
            st.entanglement_spectrum(list(range(9)), rho=True)  # k > n - k: rho would be the complement's
        assert e.value.status == INVALID_ARG and "pass the complement" in str(e.value)
        assert ctx.kernel_launches() == l0  # nothing ran, the collapse is still pending
        ref.collapse([2], m, p)
        assert np.array_equal(st.download().view(np.uint64), ref.download().view(np.uint64))
    # sharded states and a side of 14 qubits
    with State(12, C128, ctx, rank=0, world_size=2) as st:
        l0 = ctx.kernel_launches()
        with pytest.raises(CircuitError) as e:
            st.entanglement_spectrum([0])
        assert e.value.status == UNSUPPORTED and "entanglement_spectrum: sharded states are not supported" in str(e.value)
        assert ctx.kernel_launches() == l0
    with State(28, C64, ctx) as st:
        st.set_basis(0)
        l0 = ctx.kernel_launches()
        for qs14 in (list(range(14)), list(range(3, 17))):
            with pytest.raises(CircuitError) as e:
                st.entanglement_spectrum(qs14)
            assert e.value.status == UNSUPPORTED and "has 14 qubits" in str(e.value) and "4 GiB or more" in str(e.value)
        assert ctx.kernel_launches() == l0


_ROTATE_WORKER = r"""
import numpy as np
import spectrum_ref as sr
from rustqip_b200 import circuits
from rustqip_b200.state import Context, State

n = 22
lists = [[0, 5, 9], list(range(11)), list(range(11, 22)), [1, 3, 5, 7, 9, 11, 13, 15, 17, 19, 21], list(range(1, 22))]
worst = 0.0
with Context(0) as ctx:
    with State(n, np.complex128, ctx) as st:
        st.set_basis(3)
        st.apply_schedule(circuits.random_circuit(n, 10, 12, "H,T,CNOT") + circuits.qft(n)[:60])
        before = st.qubit_map().copy()
        assert not np.array_equal(before, np.arange(n)[::-1]), "the schedule left the canonical layout"
        got = [st._spectrum(qs, len(qs) <= n - len(qs)) for qs in lists]
        assert np.array_equal(st.qubit_map(), before), "the call restored the layout"
        psi = st.download()
    for qs, g in zip(lists, got):
        s = min(len(qs), n - len(qs))
        lam, T = sr.schmidt_ref(psi, n, qs)
        e = sr.eig_bound(n, s, T, float(lam[0]))
        err = float(np.max(np.abs(g[0] - lam)))
        assert err <= e, (qs, err, e)
        worst = max(worst, err / e)
        if g[1] is not None and s <= 10:
            import rdm_ref as rr
            want = rr.rdm_ref(psi, n, qs)
            b = rr.bound(n, s, rr.abs_weight(psi, n, qs)) * 2
            assert np.all(np.abs(g[1] - want) <= b), qs
print("ROTATE worst ratio %.3e" % worst)
"""


def test_permuted_layout_is_read_in_place():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    WORST["rotate f64 n=22 eigs"] = float(p.stdout.split("worst ratio")[1].split()[0])


# ---- full size -------------------------------------------------------------------------------------------------

def snapshot(st, n, dtype):
    """The state's bytes, copied to a device tensor chunk by chunk through a pinned buffer (it never fits the host
    twice)."""
    import torch
    item = np.dtype(dtype).itemsize
    chunk = 1 << 25
    host = torch.empty(chunk * item, dtype=torch.uint8, pin_memory=True)
    snap = torch.empty((1 << n) * item, dtype=torch.uint8, device="cuda")
    for off in range(0, 1 << n, chunk):
        st.download_ptr(host.data_ptr(), chunk, off)
        snap[off * item:(off + chunk) * item].copy_(host)
    return snap, host


def same_as_snapshot(st, n, dtype, snap, host):
    import torch
    item = np.dtype(dtype).itemsize
    chunk = host.numel() // item
    for off in range(0, 1 << n, chunk):
        st.download_ptr(host.data_ptr(), chunk, off)
        if not torch.equal(snap[off * item:(off + chunk) * item], host.cuda()):
            return False
    return True


def local_circuit(qubits, seed, exact):
    """Two layers of a one-qubit gate on every qubit of the register followed by a CNOT chain through it: Haar-random
    unitaries, or (exact) gates with entries in {0, +-1, +-i} that every kernel applies without rounding."""
    rng = np.random.default_rng(seed)
    ops = []
    for _ in range(2):
        for q in qubits:
            if exact:
                ops.append([gates.x, gates.s, gates.z, gates.y][int(rng.integers(4))](q))
            else:
                z = (rng.normal(size=(2, 2)) + 1j * rng.normal(size=(2, 2))) / math.sqrt(2)
                u, r = np.linalg.qr(z)
                u = u * (np.diag(r) / np.abs(np.diag(r)))
                ops.append(gates.mat([q], [complex(x) for x in u.reshape(-1)]))
        order = [int(q) for q in rng.permutation(qubits)]
        ops += [gates.cnot(a, b) for a, b in zip(order[:-1], order[1:])]
    return ops


@pytest.mark.parametrize("n,dtype", [(30, C128), (31, C64)], ids=["n30_f64", "n31_f32"])
def test_full_size_schmidt_form(ctx, n, dtype):
    """sum_i sqrt(lambda_i) |i>_A |i>_B with geometric lambda on A = qubits 0..12 (13 qubits), prepared as an upload of
    sqrt(lambda) on the 13 lowest index bits and 13 CNOTs onto A, then local circuits on A and on B.  The spectrum of
    A is lambda up to the state's own rounding: f64 uses Haar-random one-qubit gates applied one by one (per-gate
    kernels: each amplitude a two-term complex dot product, ||d psi|| <= sqrt(2) gamma_4 per gate, plus u for the
    upload), f32 exact gates (lambda is then the square of the f32 amplitudes, exactly).  The side of 13 and its
    complement of 17 give the same values, and the state downloads bit-identical after the calls."""
    import torch
    s = 13
    A = list(range(s))
    B = [q for q in range(n) if q not in A]
    d = 1 << s
    lam = sr.geometric_spectrum(d, 0.999)
    amp = np.sqrt(lam).astype(dtype)
    lam = amp.real.astype(np.float64) ** 2  # exact for f32 amplitudes; within u of (f64 amp)^2 for f64
    ctx.release_pool()
    exact = dtype == C64
    with State(n, dtype, ctx) as st:
        st.set_basis(0)
        st.upload(amp, 0)
        st.apply_schedule([gates.cnot(n - 1 - b, s - 1 - b) for b in range(s)])
        circ = local_circuit(A, 7, exact) + local_circuit(B, 8, exact)
        st.apply_schedule(circ, fusion=False)
        # a one-qubit gate rounds each output within sqrt(2) gamma_4 (|u00||x| + |u01||y|), and || |U| ||_2 <= sqrt(2)
        dpsi = 0.0 if exact else 2 * n * 2 * sr.gamma(4) + 2 * sr.U_DOUBLE
        T = float(np.sum(lam))
        snap, host = snapshot(st, n, dtype)
        lsum = float(np.sum(lam))
        want = np.sort(lam)[::-1]
        Sw = sr.entropy(lam, lsum)
        for qs in (A, B):
            l0 = ctx.kernel_launches()
            eigs, _, Tg, S = call(st, qs)
            assert ctx.kernel_launches() - l0 == 1
            e = (sr.eig_bound(n, s, T + 2 * dpsi, float(want[0]), with_ref=False) + 2 * dpsi + dpsi ** 2 +
                 sr.U_DOUBLE * want[0])
            tag = "full n=%d %s %s" % (n, np.dtype(dtype).name, "kept 13" if qs is A else "kept 17")
            note(tag + " eigs", float(np.max(np.abs(eigs - want))), e)
            dT = sr.trace_bound(n, s, T) + 2 * dpsi + dpsi ** 2 + sr.gamma(d) * T
            note(tag + " trace", abs(Tg - lsum), dT)
            note(tag + " entropy", abs(S - Sw), sr.entropy_bound(s, lsum, e, dT, Sw))
        assert same_as_snapshot(st, n, dtype, snap, host), "the call changed the state"
        del snap, host
        torch.cuda.empty_cache()
    ctx.release_pool()
