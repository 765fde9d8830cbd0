"""Single-qubit noise channels for quantum-trajectory simulation (State.apply_channels).

A ``Channel`` holds Kraus operators K_i that are each diagonal or anti-diagonal, K|b> = d(b)|b ^ flip>, and complete
(sum_i K_i^dagger K_i = I to 1e-12).  That covers amplitude and phase damping, Pauli channels, reset, the Z measurement
and their compositions, and lets a layer of such channels be drawn jointly with one sample of the state
(include/qipb200.h: qipb200_state_apply_channels)."""
from __future__ import annotations

from typing import Sequence

import numpy as np

MAX_KRAUS = 16
COMPLETE_TOL = 1e-12

_I = np.eye(2, dtype=np.complex128)
_X = np.array([[0, 1], [1, 0]], dtype=np.complex128)
_Y = np.array([[0, -1j], [1j, 0]], dtype=np.complex128)
_Z = np.array([[1, 0], [0, -1]], dtype=np.complex128)


def _weights(k):
    """|d(0)|^2, |d(1)|^2 of a monomial operator, in double as the library computes them (re^2 + im^2)."""
    flip = k[0, 0] == 0 and k[1, 1] == 0
    d = (k[1, 0], k[0, 1]) if flip else (k[0, 0], k[1, 1])
    return [float(np.float64(v.real) * np.float64(v.real) + np.float64(v.imag) * np.float64(v.imag)) for v in d]


class Channel:
    """A single-qubit channel given by its Kraus operators (a sequence of 2 x 2 complex matrices, rows as outputs,
    |0> first).  Raises ValueError unless every operator is finite, nonzero, diagonal or anti-diagonal, there are 1
    to 16 of them, and sum_i |d_i(b)|^2 is 1 within 1e-12 for b = 0 and 1: the checks the library makes."""

    def __init__(self, kraus):
        ks = np.array([np.asarray(k, dtype=np.complex128) for k in kraus], dtype=np.complex128).reshape(-1, 2, 2)
        if not 1 <= ks.shape[0] <= MAX_KRAUS:
            raise ValueError("Channel: 1 to 16 Kraus operators, got %d" % ks.shape[0])
        total = [0.0, 0.0]
        for i, k in enumerate(ks):
            if not np.all(np.isfinite(k.view(np.float64))):
                raise ValueError("Channel: operator %d has a non-finite entry" % i)
            if not np.any(k != 0):
                raise ValueError("Channel: operator %d is the zero matrix" % i)
            if not ((k[0, 1] == 0 and k[1, 0] == 0) or (k[0, 0] == 0 and k[1, 1] == 0)):
                raise ValueError("Channel: operator %d is neither diagonal nor anti-diagonal" % i)
            e = _weights(k)
            total = [total[0] + e[0], total[1] + e[1]]
        for b in (0, 1):
            if not abs(total[b] - 1.0) <= COMPLETE_TOL:
                raise ValueError("Channel: the operators are not complete (sum of |d_i(%d)|^2 - 1 = %.3g)"
                                 % (b, total[b] - 1.0))
        self.kraus = ks

    def __len__(self):
        return self.kraus.shape[0]

    def __repr__(self):
        return "Channel(%d Kraus operators)" % len(self)

    @property
    def state_dependent(self) -> bool:
        """Some operator has |d(0)|^2 != |d(1)|^2: the choice depends on the qubit's value (damping, reset)."""
        return any(e[0] != e[1] for e in map(_weights, self.kraus))

    def compose(self, other: "Channel") -> "Channel":
        """This channel, then ``other``: the Kraus operators B_j A_i (j major), zero products left out.  Products of
        diagonal or anti-diagonal matrices are again one or the other, so e.g. T1/T2 relaxation is
        ``amplitude_damping(g).compose(phase_damping(l))``."""
        ks = [b @ a for b in other.kraus for a in self.kraus]
        return Channel([k for k in ks if np.any(k != 0)])

    def superop(self, rho: np.ndarray) -> np.ndarray:
        """sum_i K_i rho K_i^dagger on a 2 x 2 density matrix (for checks)."""
        return sum(k @ rho @ k.conj().T for k in self.kraus)


def _keep(ks):
    return Channel([k for k in ks if np.any(k != 0)])


def amplitude_damping(gamma: float) -> Channel:
    """Energy relaxation |1> -> |0> with probability gamma: K0 = diag(1, sqrt(1 - gamma)), K1 = sqrt(gamma) |0><1|."""
    g = float(gamma)
    return _keep([np.diag([1.0, np.sqrt(1.0 - g)]), np.sqrt(g) * np.array([[0, 1], [0, 0]])])


def generalized_amplitude_damping(gamma: float, p: float) -> Channel:
    """Relaxation towards a thermal state with ground-state population p."""
    g, p = float(gamma), float(p)
    a, b = np.sqrt(p), np.sqrt(1.0 - p)
    return _keep([a * np.diag([1.0, np.sqrt(1.0 - g)]), a * np.sqrt(g) * np.array([[0, 1], [0, 0]]),
                  b * np.diag([np.sqrt(1.0 - g), 1.0]), b * np.sqrt(g) * np.array([[0, 0], [1, 0]])])


def phase_damping(lam: float) -> Channel:
    """Loss of phase without loss of energy: K0 = diag(1, sqrt(1 - lam)), K1 = diag(0, sqrt(lam))."""
    lam = float(lam)
    return _keep([np.diag([1.0, np.sqrt(1.0 - lam)]), np.diag([0.0, np.sqrt(lam)])])


def pauli_channel(px: float, py: float, pz: float) -> Channel:
    """X, Y, Z with probabilities px, py, pz, else nothing."""
    px, py, pz = float(px), float(py), float(pz)
    return _keep([np.sqrt(1.0 - px - py - pz) * _I, np.sqrt(px) * _X, np.sqrt(py) * _Y, np.sqrt(pz) * _Z])


def depolarizing(p: float) -> Channel:
    """rho -> (1 - p) rho + p/3 (X rho X + Y rho Y + Z rho Z): each Pauli error with probability p/3."""
    p = float(p)
    return pauli_channel(p / 3, p / 3, p / 3)


def reset() -> Channel:
    """Reset to |0>: K0 = |0><0|, K1 = |0><1|."""
    return Channel([np.diag([1.0, 0.0]), np.array([[0, 1], [0, 0]])])


def marshal(channels: Sequence[Channel]):
    """(n_kraus u32, kraus f64) arrays of the C ABI."""
    n_kraus = np.ascontiguousarray([len(c) for c in channels], dtype=np.uint32)
    kraus = np.ascontiguousarray(np.concatenate([c.kraus.reshape(-1) for c in channels]) if channels else
                                 np.zeros(0, dtype=np.complex128)).view(np.float64)
    return n_kraus, np.ascontiguousarray(kraus)
