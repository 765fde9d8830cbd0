"""Deterministic synthetic workloads of BASELINE.json (SURVEY.md section 8d).

All generators are pure host code; they emit lists of ``MatrixOp`` that are fed
unchanged to the GPU library and (in tests / the CPU baseline) to the oracle.
"""
from __future__ import annotations

import math
from typing import Callable, List, Sequence

import numpy as np

from . import gates
from .ops import MatrixOp

MASK64 = (1 << 64) - 1


class SplitMix64:
    def __init__(self, seed: int):
        self.state = seed & MASK64

    def next(self) -> int:
        self.state = (self.state + 0x9E3779B97F4A7C15) & MASK64
        z = self.state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)

    def uniform(self) -> float:
        return (self.next() >> 11) * (1.0 / (1 << 53))


def random_layers(seed: int, n: int, depth: int, oneq: Sequence[Callable[[int], MatrixOp]],
                  twoq: Sequence[Callable[[int, int], MatrixOp]]) -> List[MatrixOp]:
    """Generator G(seed,N,D,ONEQ,TWOQ) of SURVEY.md section 8d."""
    rng = SplitMix64(seed)
    ops: List[MatrixOp] = []
    for _ in range(depth):
        p = list(range(n))
        for i in range(n - 1, 0, -1):  # Fisher-Yates with rng.next() % (i+1)
            j = rng.next() % (i + 1)
            p[i], p[j] = p[j], p[i]
        i = 0
        while i < n:
            if n - i >= 2 and rng.next() % 3 == 0:
                g = twoq[rng.next() % len(twoq)]
                ops.append(g(p[i], p[i + 1]))
                i += 2
            else:
                g = oneq[rng.next() % len(oneq)]
                ops.append(g(p[i]))
                i += 1
    return ops


def h_layer(n: int) -> List[MatrixOp]:
    return [gates.h(q) for q in range(n)]


def random_circuit(n: int, depth: int, seed: int, gate_set: str = "H,T,CNOT") -> List[MatrixOp]:
    """Layer 0 = H on every qubit, then `depth` generated layers (configs 2 and 5)."""
    if gate_set == "H,T,CNOT":
        oneq, twoq = [gates.h, gates.t], [gates.cnot]
    elif gate_set == "H,CZ,CNOT":
        oneq, twoq = [gates.h], [gates.cz, gates.cnot]
    else:
        raise ValueError(gate_set)
    return h_layer(n) + random_layers(seed, n, depth, oneq, twoq)


def noisy_random_circuit(n: int, depth: int, seed: int, gamma: float = 1e-3, lam: float = 1e-3,
                         cnot_depolarizing: float = 0.0) -> list:
    """Items of DensityMatrix.apply: H on every qubit, then `depth` random {H, T, CNOT} layers (layer l generated as
    random_layers(seed + l, n, 1, ...)), each followed by amplitude damping (gamma) and dephasing (lam) on every qubit;
    with cnot_depolarizing > 0, two-qubit depolarizing noise follows each CNOT."""
    from . import channels as ch
    damp, deph = ch.amplitude_damping(gamma), ch.phase_damping(lam)
    items: list = h_layer(n)
    for layer in range(depth):
        for op in random_layers(seed + layer, n, 1, [gates.h, gates.t], [gates.cnot]):
            items.append(op)
            if cnot_depolarizing > 0 and op.kind == "control":
                items.append((ch.two_qubit_depolarizing(cnot_depolarizing), op.indices()))
        items += [(damp, [q]) for q in range(n)] + [(deph, [q]) for q in range(n)]
    return items


def config2(n: int = 28, depth: int = 40) -> List[MatrixOp]:
    return random_circuit(n, depth, 0x5EED0002, "H,T,CNOT")


def config5(n: int = 33, depth: int = 30) -> List[MatrixOp]:
    return random_circuit(n, depth, 0x5EED0005, "H,CZ,CNOT")


def qft(n: int) -> List[MatrixOp]:
    """Textbook QFT at the MatrixOp level (config 3; SURVEY.md quirk Q3)."""
    ops: List[MatrixOp] = []
    for i in range(n):
        ops.append(gates.h(i))
        for j in range(i + 1, n):
            ops.append(gates.cphase(j, i, math.pi / (1 << (j - i))))
    for i in range(n // 2):
        ops.append(gates.swap([i], [n - 1 - i]))
    return ops


def random_state(n: int, seed: int, dtype=np.complex128) -> np.ndarray:
    """Seeded random normalised state.  (Vectorised PCG64 normals rather than the
    scalar SplitMix64+Box-Muller of the survey: 2^30 draws in Python are not an option;
    the same array goes to the oracle and to the GPU.)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    real = np.float32 if np.dtype(dtype) == np.complex64 else np.float64
    out = np.empty(1 << n, dtype=dtype)
    chunk = 1 << 22
    acc = 0.0
    for lo in range(0, 1 << n, chunk):
        hi = min(lo + chunk, 1 << n)
        re = rng.standard_normal(hi - lo, dtype=real)
        im = rng.standard_normal(hi - lo, dtype=real)
        out[lo:hi] = re + 1j * im
        acc += float(np.vdot(re, re) + np.vdot(im, im))
    out *= real(1.0 / math.sqrt(acc))
    return out


def haar_unitary(k: int, rng: SplitMix64) -> np.ndarray:
    """Haar-random 2^k x 2^k unitary: complex Ginibre -> modified Gram-Schmidt (f64)."""
    d = 1 << k

    def normal():
        u1 = max(rng.uniform(), 1e-300)
        u2 = rng.uniform()
        r = math.sqrt(-2.0 * math.log(u1))
        return r * math.cos(2 * math.pi * u2), r * math.sin(2 * math.pi * u2)

    a = np.empty((d, d), dtype=np.complex128)
    for r in range(d):
        for c in range(d):
            re, im = normal()
            a[r, c] = complex(re, im)
    q = np.zeros_like(a)
    for c in range(d):
        v = a[:, c].copy()
        for p in range(c):
            v -= np.vdot(q[:, p], v) * q[:, p]
        q[:, c] = v / np.linalg.norm(v)
    return q


def config4(n: int = 26, blocks: int = 200, k: int = 4, seed: int = 0x5EED0004) -> List[MatrixOp]:
    """H layer, then `blocks` dense k-qubit Haar blocks on the first k of a seeded shuffle."""
    rng = SplitMix64(seed)
    ops = h_layer(n)
    for _ in range(blocks):
        p = list(range(n))
        for i in range(n - 1, 0, -1):
            j = rng.next() % (i + 1)
            p[i], p[j] = p[j], p[i]
        u = haar_unitary(k, rng)
        ops.append(gates.mat(p[:k], u.reshape(-1)))
    return ops


def sharded_parity_circuit(n: int, g: int, seed: int = 5) -> List[MatrixOp]:
    """Every op kind on the rank-held qubits 0..g-1 of a 2^g-way sharded n-qubit state (g may be 0), then
    random layers and a QFT prefix that touch them repeatedly: the circuit of the multi-GPU parity checks
    (tests/dist_worker.py) and of bench.py's `parity_ok` leg, small enough for the CPU oracle."""
    from .ops import make_matrix_op, make_swap_op
    rng = np.random.default_rng(seed)
    u2 = np.linalg.qr(rng.standard_normal((4, 4)) + 1j * rng.standard_normal((4, 4)))[0]
    hi = max(g - 1, 0)
    ops = [gates.h(0), gates.cnot(0, n - 1), gates.cnot(n - 1, 0), gates.t(0), gates.cz(0, 3),
           gates.cphase(2, 0, 0.3), gates.h(hi), gates.x(0), gates.toffoli(0, 1, 2), gates.toffoli(3, 4, 0),
           make_swap_op([0], [n - 2]), gates.rz(0, 0.4), make_matrix_op([0, 5], u2.reshape(-1)),
           make_matrix_op([4, hi], u2.reshape(-1)), make_swap_op([0], [hi]) if hi > 0 else gates.h(1)]
    # a dense 5-qubit block and a 6-qubit diagonal that include rank-held qubits (in-place wide kernels after migration)
    u5 = np.linalg.qr(rng.standard_normal((32, 32)) + 1j * rng.standard_normal((32, 32)))[0]
    ops += [make_matrix_op([0, 5, 2, 7, n - 1], u5.reshape(-1)),
            make_matrix_op([hi, 1, 6, 3, 8, n - 2] if hi != 1 else [0, 1, 6, 3, 8, n - 2],
                           np.diag(np.exp(1j * rng.standard_normal(64))).reshape(-1))]
    ops += random_circuit(n, 6, 1234 + n, "H,T,CNOT") + random_circuit(n, 4, 99 + n, "H,CZ,CNOT")
    ops += qft(n)[: 3 * n]
    return ops
