"""Exact density-matrix simulation on the device (DensityMatrix, qipb200_density_*).

density_apply is checked bit for bit against apply_schedule of the emitted schedule, and against the numpy reference
of tests/density_ref.py for small n.  Pure-state identities tie the readouts to the State calls; trajectory averages
of apply_kraus_channels and apply_channels are compared with the exact result; a damped product state at full size
(n = 15 f64, n = 16 f32: indices past 2^31 up to 2^32 - 1) is compared with its closed form; also the spectrum,
determinism, pending work, a permuted layout and the refusals."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import density_ref as dr
from rustqip_b200 import _lib, channels as ch, circuits, gates
from rustqip_b200.ops import make_matrix_op
from rustqip_b200.state import DensityMatrix, State, density_schedule
from test_density_cpu import random_items

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C128, C64 = np.complex128, np.complex64
INVALID_ARG, SIZE_MISMATCH, UNSUPPORTED = 1, 2, 7
TOL = {C128: 1e-12, C64: 2e-5}


def bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dtype", [C128, C64])
def test_bit_identical_to_apply_schedule(ctx, dtype, monkeypatch):
    """Both calls run the same kernels: from 2^22 amplitudes a fused pass runs on the interpreter kernel while its
    generated kernel compiles in the background (QIPB200_JIT=async, the default), and the two kernels may round
    differently, so the generated kernels are compiled before each pass there (sync)."""
    for n in range(1, 14):
        monkeypatch.setenv("QIPB200_JIT", "sync" if 2 * n >= 22 else "off")
        rng = np.random.default_rng(1000 + n)
        items = random_items(n, rng, 10 if n > 6 else 16)
        ops = density_schedule(n, dtype, items)
        i0 = int(rng.integers(1 << n))
        for fusion in (True, False):
            with DensityMatrix(n, dtype, ctx) as rho, State(2 * n, dtype, ctx) as st:
                rho.set_basis(i0)
                rho.apply(items, fusion=fusion)
                st.set_basis(i0 + (i0 << n))
                st.apply_schedule(ops, fusion=fusion)
                got = rho.download()
                assert bits_equal(got.reshape(-1), st.download()), (n, fusion)
            if n <= 6 and fusion:
                want = dr.evolve(n, items, dr.basis(n, i0))
                assert np.max(np.abs(got.astype(C128) - want)) <= TOL[dtype] * 10, n


def test_pure_state_identities(ctx):
    n = 10
    psi_h = circuits.random_state(n, 3, C128)
    phi_h = circuits.random_state(n, 4, C128) * 0.7
    ops = circuits.random_circuit(n, 6, 0x5EED0010)
    terms = [[("Z", 0)], [("X", 3), ("Y", 7)], [("Y", 1), ("Z", 2), ("X", 9)], [], [("X", 5)]]
    with DensityMatrix(n, C128, ctx) as rho, DensityMatrix(n, C128, ctx) as rho2, State(n, C128, ctx) as psi, \
            State(n, C128, ctx) as phi:
        psi.upload(psi_h)
        phi.upload(phi_h)
        rho.set_pure(psi)
        assert np.allclose(rho.download(), np.outer(psi_h, psi_h.conj()), atol=1e-15)
        assert abs(rho.fidelity(psi) - psi.norm2() ** 2) <= 1e-12
        assert abs(rho.fidelity(phi) - abs(phi.overlap(psi)) ** 2) <= 1e-12
        assert np.allclose(rho.measure_probs([2, 7, 4]), psi.measure_probs([2, 7, 4]), atol=1e-14)
        assert np.allclose(rho.expect_paulis(terms), psi.expect_paulis(terms), atol=1e-13)
        assert np.allclose(rho.reduced_density([6, 1, 8]), psi.reduced_density([6, 1, 8]), atol=1e-14)
        assert abs(rho.trace() - psi.norm2()) <= 1e-13
        rho.apply(ops)
        psi.apply_schedule(ops)
        rho2.set_pure(psi)
        assert np.max(np.abs(rho.download() - rho2.download())) <= 1e-12


def test_trajectory_averages(ctx):
    """2000 trajectories of apply_kraus_channels (a mixed layer) and of apply_channels, averaged as |psi><psi|: every
    entry within 5 sigma of the exact result."""
    n, N = 4, 2000
    rng = np.random.default_rng(44)
    psi0 = circuits.random_state(n, 44, C128)
    krs = [dr.random_kraus(2, 3, rng), ch.KrausChannel(ch.amplitude_damping(0.4)), ch.KrausChannel(ch.depolarizing(0.3))]
    kgroups = [[0, 2], [1], [3]]
    chans1 = [ch.amplitude_damping(0.3), ch.phase_damping(0.5), ch.depolarizing(0.2), ch.reset()]
    for layer, run in (
            ([(c, g) for c, g in zip(krs, kgroups)], lambda st: st.apply_kraus_channels(krs, kgroups, rng=rng)),
            ([(c, [q]) for q, c in enumerate(chans1)], lambda st: st.apply_channels(chans1, list(range(n)), rng=rng))):
        samples = np.zeros((N, 1 << n, 1 << n), dtype=C128)
        with State(n, C128, ctx) as st:
            for t in range(N):
                st.upload(psi0)
                run(st)
                v = st.download()
                samples[t] = np.outer(v, v.conj())
        with DensityMatrix(n, C128, ctx) as rho, State(n, C128, ctx) as p:
            p.upload(psi0)
            rho.set_pure(p)
            rho.apply(layer)
            exact = rho.download()
        mean = samples.mean(axis=0)
        sig = np.sqrt(samples.real.var(axis=0) / N) + 1j * np.sqrt(samples.imag.var(axis=0) / N)
        assert np.all(np.abs(mean.real - exact.real) <= 5 * sig.real + 1e-12)
        assert np.all(np.abs(mean.imag - exact.imag) <= 5 * sig.imag + 1e-12)


def _one_qubit(gamma, lam):
    """|+><+| after amplitude damping gamma, then dephasing lam."""
    r = np.array([[0.5 + gamma / 2, np.sqrt(1 - gamma) / 2], [np.sqrt(1 - gamma) / 2, (1 - gamma) / 2]])
    r[0, 1] *= np.sqrt(1 - lam)
    r[1, 0] *= np.sqrt(1 - lam)
    return r


def _entries(n, qs, idx):
    """rho[r, c] of the product state at vector indices idx (r = idx >> n, c = idx & (2^n - 1))."""
    r, c = idx >> np.uint64(n), idx & np.uint64((1 << n) - 1)
    out = np.ones(idx.shape[0])
    for q in range(n):
        sh = np.uint64(n - 1 - q)
        out = out * qs[q][((r >> sh) & np.uint64(1)).astype(np.int64), ((c >> sh) & np.uint64(1)).astype(np.int64)]
    return out


@pytest.mark.parametrize("n,dtype", [(15, C128), (16, C64)])
def test_full_size_damped_product_state(ctx, n, dtype):
    gam = [0.05 + 0.01 * q for q in range(n)]
    lam = [0.1 + 0.02 * (q % 5) for q in range(n)]
    qs = [_one_qubit(g, l) for g, l in zip(gam, lam)]
    items = [gates.h(q) for q in range(n)] + [(ch.amplitude_damping(gam[q]), [q]) for q in range(n)] + \
            [(ch.phase_damping(lam[q]), [q]) for q in range(n)]
    tol = 1e-12 if dtype == C128 else 2e-6
    with DensityMatrix(n, dtype, ctx) as rho, State(n, dtype, ctx) as plus:
        rho.set_basis(0)
        rho.apply(items)
        total = 1 << (2 * n)
        for off in [o for o in (0, 12345, (1 << 31) - 700, 1 << 31, total // 2 + 777, total - 1024) if o + 1024 <= total]:
            got = rho.state.download(offset=off, length=1024).astype(C128)
            want = _entries(n, qs, np.arange(off, off + 1024, dtype=np.uint64))
            assert np.max(np.abs(got - want)) <= tol * 4, off
        x = rho.expect_paulis([[("X", q)] for q in range(n)])
        assert np.max(np.abs(x - [2 * r[0, 1] for r in qs])) <= tol * 10
        zz = rho.expect_paulis([[("Z", q), ("Z", q + 1)] for q in range(n - 1)])
        z = [r[0, 0] - r[1, 1] for r in qs]
        assert np.max(np.abs(zz - [z[q] * z[q + 1] for q in range(n - 1)])) <= tol * 10
        for q in (0, 7, n - 1):
            assert np.max(np.abs(rho.measure_probs([q]) - np.diag(qs[q]))) <= tol * 10
        pair = rho.measure_probs([3, 1])
        assert np.max(np.abs(pair - np.kron(np.diag(qs[1]), np.diag(qs[3])))) <= tol * 10
        plus.set_basis(0)
        plus.apply_schedule([gates.h(q) for q in range(n)])
        fid = np.prod([(1 + 2 * r[0, 1]) / 2 for r in qs])
        assert abs(rho.fidelity(plus) - fid) <= tol * 10 * fid
        pur = np.prod([np.sum(r * r) for r in qs])
        assert abs(rho.purity() - pur) <= tol * 10 * pur * n
        kept = [2, 9, 0, 14, 5, 11, 7, 1, 13, 4]
        want = np.array([[1.0]])
        for q in kept:
            want = np.kron(qs[q], want)
        assert np.max(np.abs(rho.reduced_density(kept) - want)) <= tol * 10


def test_spectrum(ctx):
    for n in (1, 3, 6, 8):
        rng = np.random.default_rng(80 + n)
        with DensityMatrix(n, C128, ctx) as rho:
            rho.set_basis(1 % (1 << n))
            rho.apply(random_items(n, rng, 12))
            want = np.sort(np.linalg.eigvalsh(rho.download()))[::-1]
            assert np.max(np.abs(rho.spectrum() - want)) <= 1e-12, n
    n = 13
    gam = [0.1 + 0.05 * (q % 7) for q in range(n)]
    qs = [_one_qubit(g, 0.3) for g in gam]
    items = [gates.h(q) for q in range(n)] + [(ch.amplitude_damping(g), [q]) for q, g in enumerate(gam)] + \
            [(ch.phase_damping(0.3), [q]) for q in range(n)]
    with DensityMatrix(n, C128, ctx) as rho:
        rho.set_basis(0)
        rho.apply(items)
        ev1 = [np.linalg.eigvalsh(r) for r in qs]
        want = np.array([1.0])
        for e in ev1:
            want = np.outer(want, e).reshape(-1)
        assert np.max(np.abs(rho.spectrum() - np.sort(want)[::-1])) <= 1e-12
        h = sum(-np.sum(e[e > 0] * np.log(e[e > 0])) for e in ev1)
        assert abs(rho.entropy() - h) <= 1e-9


def test_determinism_and_pending_basis(ctx):
    n = 9
    rng = np.random.default_rng(9)
    items = random_items(n, rng, 20)
    with DensityMatrix(n, C128, ctx) as rho, State(n, C128, ctx) as psi:
        psi.upload(circuits.random_state(n, 9, C128))
        rho.set_basis(37)
        # the pending basis state; bit i of m is qubit n - 1 - i, index bit i
        assert rho.measure_probs(list(range(n))[::-1])[37] == 1.0 and rho.trace() == 1.0
        rho.set_basis(37)
        rho.apply(items)
        names = ("measure_probs", "trace", "expect_paulis", "reduced_density", "fidelity")
        reads = []
        for _ in range(3):
            reads.append((rho.measure_probs([4, 0, 8]), rho.trace(),
                          rho.expect_paulis([[("X", 1), ("Z", 3)], [("Y", 2)]]), rho.reduced_density([5, 2]),
                          rho.fidelity(psi)))
        for r in reads[1:]:
            for name, a, b in zip(names, reads[0], r):
                assert bits_equal(np.atleast_1d(a), np.atleast_1d(b)), name
        # the spectrum's input matrix is the same bits every time; cuSOLVER's eigen-solve is not promised to be
        # bit-identical on repeat (as for State.entanglement_spectrum), so its values are compared within rounding
        e0, e1 = rho.spectrum(), rho.spectrum()
        assert np.max(np.abs(e0 - e1)) <= 1e-13


_ROTATE_WORKER = r"""
import numpy as np
from test_density_cpu import random_items
from rustqip_b200 import circuits
from rustqip_b200.state import Context, DensityMatrix, State

n = 9
rng = np.random.default_rng(19)
items = circuits.noisy_random_circuit(n, 4, 0x5EED0019, gamma=0.05, lam=0.05) + random_items(n, rng, 10)
terms = [[("X", 1), ("Z", 3)], [("Y", 2), ("Y", 8)], [("Z", 0)], [("X", 4), ("X", 6), ("Z", 7)]]
with Context(0) as ctx:
    with DensityMatrix(n, np.complex128, ctx) as rho, State(n, np.complex128, ctx) as psi:
        psi.upload(circuits.random_state(n, 19, np.complex128))
        rho.set_basis(5)
        rho.apply(items)
        qmap = rho.state.qubit_map().copy()
        assert not np.array_equal(qmap, np.arange(2 * n)[::-1]), "the schedule left the canonical layout"
        def reads():
            return (rho.measure_probs([4, 0, 8]), rho.measure_probs([]), rho.expect_paulis(terms),
                    rho.reduced_density([5, 2, 7]), rho.spectrum(), rho.fidelity(psi))
        permuted = reads()
        rho.download()  # restores the canonical layout
        assert np.array_equal(rho.state.qubit_map(), np.arange(2 * n)[::-1])
        ident = reads()
        for a, b in zip(permuted[:5], ident[:5]):
            assert np.array_equal(np.asarray(a), np.asarray(b)), (a, b)
        assert abs(permuted[5] - ident[5]) <= 1e-13
print("permuted layout ok")
"""


def test_permuted_layout():
    env = dict(os.environ, QIPB200_ROTATE="1", PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", _ROTATE_WORKER], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(p.stdout[-2000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "permuted layout ok" in p.stdout


def test_refusals_leave_state_unchanged(ctx):
    L = _lib.lib()
    out = np.zeros(1 << 12)
    with State(5, C128, ctx) as odd:  # an odd qubit count
        v = circuits.random_state(5, 1, C128)
        odd.upload(v)
        assert L.qipb200_density_measure_probs(odd._h, None, 0, out.ctypes.data) == INVALID_ARG
        assert L.qipb200_density_reduced(odd._h, np.array([0], dtype=np.uint64).ctypes.data, 1,
                                         out.ctypes.data) == INVALID_ARG
        assert bits_equal(odd.download(), v)
    n = 4
    with DensityMatrix(n, C128, ctx) as rho, State(n + 1, C128, ctx) as big, State(n, C64, ctx) as f32:
        rho.set_basis(3)
        rho.apply([gates.h(0), (ch.depolarizing(0.2), [0])])
        before = rho.download().copy()
        for bad in (big, f32):
            assert L.qipb200_density_from_state(rho.state._h, bad._h) == SIZE_MISMATCH
            assert L.qipb200_density_fidelity(rho.state._h, bad._h, out.ctypes.data) == SIZE_MISMATCH
        assert bits_equal(rho.download(), before)
    with State(8, C128, ctx, rank=0, world_size=2) as sh:
        assert L.qipb200_density_measure_probs(sh._h, None, 0, out.ctypes.data) == UNSUPPORTED
        assert L.qipb200_density_apply(sh._h, None, 0, 0, None, None, None, None, None, 0) == UNSUPPORTED
    with DensityMatrix(11, C64, ctx) as rho:
        rho.set_basis(0)
        rho.apply([gates.h(3)])
        before = rho.download().copy()
        k = np.arange(11, dtype=np.uint64)
        buf = np.zeros(2 << 22)
        assert L.qipb200_density_reduced(rho.state._h, k.ctypes.data, 11, buf.ctypes.data) == UNSUPPORTED
        assert bits_equal(rho.download(), before)
    with DensityMatrix(14, C64, ctx) as rho:
        rho.set_basis(0)
        eigs = np.zeros(1 << 14)
        assert L.qipb200_density_spectrum(rho.state._h, eigs.ctypes.data) == UNSUPPORTED
        assert rho.trace() == 1.0
