"""Noise channels on one to four qubits for quantum-trajectory simulation (State.apply_channels,
State.apply_multiqubit_channels, State.apply_kraus_channels).

A ``Channel`` on k qubits holds Kraus operators K_i of the form K|b> = d(b)|b ^ f>, one XOR mask f per operator (every
column has at most one nonzero entry, on the same shifted diagonal; for k = 1 that is diagonal or anti-diagonal), and
is complete (sum_i K_i^dagger K_i = I to 1e-12).  That covers amplitude and phase damping, every Pauli channel (the two-
qubit depolarizing channel included), reset, the Z measurement, and their compositions and tensor products, and lets a
layer of such channels be drawn jointly with one sample of the state (include/qipb200.h:
qipb200_state_apply_channels, qipb200_state_apply_multiqubit_channels).  A ``KrausChannel`` holds any complete set of
Kraus operators (State.apply_kraus_channels: one read sweep plus about one read-write sweep per four qubits of
state-dependent channels); monomial layers are cheaper as ``Channel``.  Matrices use the qip_op MAT convention: rows as
outputs, the channel's first qubit the most significant bit of the index."""
from __future__ import annotations

import itertools
from typing import Mapping, Sequence

import numpy as np

MAX_KRAUS = 16          # operators of a single-qubit channel (qipb200_state_apply_channels)
MAX_KRAUS_MULTI = 256   # operators of a channel on 2 to 4 qubits
MAX_QUBITS = 4
COMPLETE_TOL = 1e-12

_I = np.eye(2, dtype=np.complex128)
_X = np.array([[0, 1], [1, 0]], dtype=np.complex128)
_Y = np.array([[0, -1j], [1j, 0]], dtype=np.complex128)
_Z = np.array([[1, 0], [0, -1]], dtype=np.complex128)
_PAULI = {"I": _I, "X": _X, "Y": _Y, "Z": _Z}


def _form(k):
    """(f, d) with K|b> = d[b] |b ^ f>, or None when K is not of that form (or is zero)."""
    D = k.shape[0]
    f = None
    for c in range(D):
        for r in np.flatnonzero(k[:, c] != 0):
            if f is None:
                f = int(r) ^ c
            elif int(r) ^ c != f:
                return None
    if f is None:
        return None
    return f, [k[b ^ f, b] for b in range(D)]


def _weights(k):
    """|d(b)|^2 for every b of a monomial operator, in double as the library computes them (re^2 + im^2)."""
    return [float(np.float64(v.real) * np.float64(v.real) + np.float64(v.imag) * np.float64(v.imag))
            for v in _form(k)[1]]


class Channel:
    """A channel on k = 1..4 qubits given by its Kraus operators (a sequence of 2^k x 2^k complex matrices, rows as
    outputs, the first qubit the most significant index bit).  Raises ValueError unless every operator is finite,
    nonzero and of the form K|b> = d(b)|b ^ f>, there are 1 to 16 of them (one qubit) or 1 to 256 (two to four), and
    sum_i |d_i(b)|^2 is 1 within 1e-12 for every b: the checks the library makes."""

    def __init__(self, kraus):
        mats = [np.asarray(k, dtype=np.complex128) for k in kraus]
        D = mats[0].shape[-1] if mats else 2
        if D not in (2, 4, 8, 16):
            raise ValueError("Channel: operators must be 2^k x 2^k for k = 1..4, got %r" % (mats[0].shape,))
        ks = np.array(mats, dtype=np.complex128).reshape(-1, D, D)
        nq = D.bit_length() - 1
        top = MAX_KRAUS if nq == 1 else MAX_KRAUS_MULTI
        if not 1 <= ks.shape[0] <= top:
            raise ValueError("Channel: 1 to %d Kraus operators, got %d" % (top, ks.shape[0]))
        total = [0.0] * D
        for i, k in enumerate(ks):
            if not np.all(np.isfinite(k.view(np.float64))):
                raise ValueError("Channel: operator %d has a non-finite entry" % i)
            if not np.any(k != 0):
                raise ValueError("Channel: operator %d is the zero matrix" % i)
            if _form(k) is None:
                raise ValueError("Channel: operator %d is %s" % (i, "neither diagonal nor anti-diagonal" if nq == 1
                                                                  else "not of the form d(b)|b ^ f>"))
            total = [t + e for t, e in zip(total, _weights(k))]
        for b in range(D):
            if not abs(total[b] - 1.0) <= COMPLETE_TOL:
                raise ValueError("Channel: the operators are not complete (sum of |d_i(%d)|^2 - 1 = %.3g)"
                                 % (b, total[b] - 1.0))
        self.kraus = ks

    def __len__(self):
        return self.kraus.shape[0]

    def __repr__(self):
        return "Channel(%d qubits, %d Kraus operators)" % (self.n_qubits, len(self)) if self.n_qubits > 1 else \
            "Channel(%d Kraus operators)" % len(self)

    @property
    def n_qubits(self) -> int:
        return self.kraus.shape[1].bit_length() - 1

    @property
    def state_dependent(self) -> bool:
        """Some operator's |d(b)|^2 depends on b: the choice depends on the qubits' values (damping, reset)."""
        return any(len(set(e)) > 1 for e in map(_weights, self.kraus))

    def compose(self, other: "Channel") -> "Channel":
        """This channel, then ``other`` on the same qubits: the Kraus operators B_j A_i (j major), zero products left
        out.  Products of operators of this form are again of this form, so e.g. T1/T2 relaxation is
        ``amplitude_damping(g).compose(phase_damping(l))``."""
        if other.n_qubits != self.n_qubits:
            raise ValueError("compose: channels on %d and %d qubits" % (self.n_qubits, other.n_qubits))
        ks = [b @ a for b in other.kraus for a in self.kraus]
        return Channel([k for k in ks if np.any(k != 0)])

    def tensor(self, other: "Channel") -> "Channel":
        """This channel on the first qubits and ``other`` on the ones after them: the Kraus operators A_i (x) B_j
        (i major), on at most four qubits in all."""
        if self.n_qubits + other.n_qubits > MAX_QUBITS:
            raise ValueError("tensor: %d + %d qubits, at most 4" % (self.n_qubits, other.n_qubits))
        return Channel([np.kron(a, b) for a in self.kraus for b in other.kraus])

    def superop(self, rho: np.ndarray) -> np.ndarray:
        """sum_i K_i rho K_i^dagger on a 2^k x 2^k density matrix (for checks)."""
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


def pauli_string_channel(probs: Mapping[str, float]) -> Channel:
    """A Pauli channel on k qubits: each Pauli string (e.g. ``"XZ"``: X on the first qubit, Z on the second) with its
    probability, the identity with the rest.  Strings are non-identity, distinct and all of one length k = 1..4."""
    probs = {str(s).upper(): float(p) for s, p in probs.items()}
    ks = {len(s) for s in probs}
    if len(ks) != 1 or not 1 <= next(iter(ks)) <= MAX_QUBITS:
        raise ValueError("pauli_string_channel: strings of one length 1..4, got %r" % sorted(probs))
    k = next(iter(ks))
    for s in probs:
        if set(s) - set("IXYZ") or s == "I" * k:
            raise ValueError("pauli_string_channel: %r is not a non-identity Pauli string" % s)
    def op(s):
        m = np.ones((1, 1), dtype=np.complex128)
        for c in s:
            m = np.kron(m, _PAULI[c])
        return m
    rest = 1.0 - sum(probs.values())
    return _keep([np.sqrt(rest) * op("I" * k)] + [np.sqrt(p) * op(s) for s, p in probs.items()])


def two_qubit_depolarizing(p: float) -> Channel:
    """rho -> (1 - p) rho + p/15 sum_{P != II} P rho P: each of the 15 two-qubit Pauli errors with probability p/15."""
    p = float(p)
    return pauli_string_channel({a + b: p / 15 for a, b in itertools.product("IXYZ", repeat=2) if a + b != "II"})


def _gram(k):
    """K^dagger K in double, each entry summed over the rows in ascending order (the library's order)."""
    D = k.shape[0]
    m = np.zeros((D, D), dtype=np.complex128)
    for r in range(D):
        for c in range(D):
            re = im = 0.0
            for a in range(D):
                x, y = k[a, r], k[a, c]
                re += float(x.real) * float(y.real) + float(x.imag) * float(y.imag)
                im += float(x.real) * float(y.imag) - float(x.imag) * float(y.real)
            m[r, c] = complex(re, im)
    return m


def _trace_weight(m):
    """Tr(M) / 2^k, the trace summed in ascending order."""
    t = 0.0
    for r in range(m.shape[0]):
        t += float(m[r, r].real)
    return t / m.shape[0]


class KrausChannel:
    """A channel on k = 1..4 qubits given by ANY complete set of Kraus operators (State.apply_kraus_channels): a
    sequence of 2^k x 2^k complex matrices in the qip_op MAT convention, or a ``Channel``.  Raises ValueError unless
    there are 1 to 256 operators, each finite and nonzero, and every entry of sum_i K_i^dagger K_i - I has real and
    imaginary parts within 1e-12: the checks the library makes.  A single unitary is a valid channel, so a noisy gate
    is ``KrausChannel([U]).compose(noise)``."""

    def __init__(self, kraus):
        if isinstance(kraus, (Channel, KrausChannel)):
            kraus = kraus.kraus
        mats = [np.asarray(k, dtype=np.complex128) for k in kraus]
        D = mats[0].shape[-1] if mats else 2
        if D not in (2, 4, 8, 16) or any(m.shape != (D, D) for m in mats):
            raise ValueError("KrausChannel: operators must be 2^k x 2^k for k = 1..4, got %r"
                             % (mats[0].shape if mats else (),))
        ks = np.array(mats, dtype=np.complex128).reshape(-1, D, D)
        if not 1 <= ks.shape[0] <= MAX_KRAUS_MULTI:
            raise ValueError("KrausChannel: 1 to %d Kraus operators, got %d" % (MAX_KRAUS_MULTI, ks.shape[0]))
        total = np.zeros((D, D), dtype=np.complex128)
        grams = []
        for i, k in enumerate(ks):
            if not np.all(np.isfinite(k.view(np.float64))):
                raise ValueError("KrausChannel: operator %d has a non-finite entry" % i)
            if not np.any(k != 0):
                raise ValueError("KrausChannel: operator %d is the zero matrix" % i)
            g = _gram(k)
            grams.append(g)
            total = total + g
        dev = total - np.eye(D)
        for r in range(D):
            for c in range(D):
                x = dev[r, c]
                if not (abs(x.real) <= COMPLETE_TOL and abs(x.imag) <= COMPLETE_TOL):
                    raise ValueError("KrausChannel: the operators are not complete (entry (%d, %d) of sum K^dagger K"
                                     " - I is %.3g%+.3gi)" % (r, c, x.real, x.imag))
        self.kraus = ks
        self._grams = grams

    def __len__(self):
        return self.kraus.shape[0]

    def __repr__(self):
        return "KrausChannel(%d qubits, %d Kraus operators)" % (self.n_qubits, len(self))

    @property
    def n_qubits(self) -> int:
        return self.kraus.shape[1].bit_length() - 1

    @property
    def weights(self):
        """w_i = Tr(K_i^dagger K_i) / 2^k in double, as the library computes them."""
        return [_trace_weight(g) for g in self._grams]

    @property
    def state_independent(self) -> bool:
        """Every K_i^dagger K_i is within 1e-12 (per part) of w_i I: the choice does not depend on the state (mixed-
        unitary channels such as Pauli and depolarizing channels, or {sqrt(p_i) P_i U})."""
        D = self.kraus.shape[1]
        for g in self._grams:
            d = g - _trace_weight(g) * np.eye(D)
            if not (np.all(np.abs(d.real) <= COMPLETE_TOL) and np.all(np.abs(d.imag) <= COMPLETE_TOL)):
                return False
        return True

    def compose(self, other) -> "KrausChannel":
        """This channel, then ``other`` (a KrausChannel or Channel) on the same qubits: the Kraus operators B_j A_i
        (j major), zero products left out."""
        other = other if isinstance(other, KrausChannel) else KrausChannel(other)
        if other.n_qubits != self.n_qubits:
            raise ValueError("compose: channels on %d and %d qubits" % (self.n_qubits, other.n_qubits))
        ks = [b @ a for b in other.kraus for a in self.kraus]
        return KrausChannel([k for k in ks if np.any(k != 0)])

    def tensor(self, other) -> "KrausChannel":
        """This channel on the first qubits and ``other`` on the ones after them: A_i (x) B_j (i major), at most four
        qubits in all."""
        other = other if isinstance(other, KrausChannel) else KrausChannel(other)
        if self.n_qubits + other.n_qubits > MAX_QUBITS:
            raise ValueError("tensor: %d + %d qubits, at most 4" % (self.n_qubits, other.n_qubits))
        return KrausChannel([np.kron(a, b) for a in self.kraus for b in other.kraus])

    def superop(self, rho: np.ndarray) -> np.ndarray:
        """sum_i K_i rho K_i^dagger on a 2^k x 2^k density matrix (for checks)."""
        return sum(k @ rho @ k.conj().T for k in self.kraus)


def marshal(channels: Sequence[Channel]):
    """(arity u32, n_kraus u32, kraus f64) arrays of the C ABI."""
    arity = np.ascontiguousarray([c.n_qubits for c in channels], dtype=np.uint32)
    n_kraus = np.ascontiguousarray([len(c) for c in channels], dtype=np.uint32)
    kraus = np.ascontiguousarray(np.concatenate([c.kraus.reshape(-1) for c in channels]) if channels else
                                 np.zeros(0, dtype=np.complex128)).view(np.float64)
    return arity, n_kraus, np.ascontiguousarray(kraus)
