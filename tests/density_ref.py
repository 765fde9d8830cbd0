"""numpy reference of exact noisy evolution on an n-qubit density matrix (DensityMatrix.apply, qipb200_density_*).

rho[r, c] with r, c in the qip_op index convention (qubit q at bit n - 1 - q); vec(rho) = rho.reshape(-1) is the
layout of the 2n-qubit state the library uses.  Gates are embedded through the oracle's make_op_matrix and every Kraus
operator likewise, so the reference shares nothing with the library's doubling."""
import numpy as np

from oracle import qip_oracle as qo
from rustqip_b200 import channels as ch
from rustqip_b200.ops import MatrixOp, make_matrix_op


def embed(n, qubits, K):
    """K (2^k x 2^k, the MAT convention over qubits) as a 2^n x 2^n matrix."""
    return qo.make_op_matrix(n, make_matrix_op(list(qubits), np.asarray(K, dtype=np.complex128).reshape(-1)))


def evolve(n, items, rho):
    """rho after the items of DensityMatrix.apply (MatrixOps and (channel, qubits) pairs), in complex128."""
    rho = np.array(rho, dtype=np.complex128)
    for it in items:
        if isinstance(it, MatrixOp):
            U = qo.make_op_matrix(n, it)
            rho = U @ rho @ U.conj().T
        else:
            chan, qs = it
            kc = chan if isinstance(chan, ch.KrausChannel) else ch.KrausChannel(chan)
            out = np.zeros_like(rho)
            for K in kc.kraus:
                F = embed(n, qs, K)
                out += F @ rho @ F.conj().T
            rho = out
    return rho


def basis(n, i):
    rho = np.zeros((1 << n, 1 << n), dtype=np.complex128)
    rho[i, i] = 1.0
    return rho


def superop_bits(chan, dtype):
    """sum_i kron(K_i, conj K_i) in double, terms added in ascending i starting from the first, each part rounded
    once to dtype: the superoperator the library emits, computed with separate float64 products (no FMA)."""
    kc = chan if isinstance(chan, ch.KrausChannel) else ch.KrausChannel(chan)
    acc = None
    for K in kc.kraus:
        a, b = K.real[:, None, :, None], K.imag[:, None, :, None]   # K[r1, c1]
        x, y = K.real[None, :, None, :], K.imag[None, :, None, :]   # K[r2, c2]
        re = (a * x) + (b * y)
        im = (b * x) - (a * y)
        D = K.shape[0]
        term = (re.reshape(D * D, D * D), im.reshape(D * D, D * D))
        acc = term if acc is None else (acc[0] + term[0], acc[1] + term[1])
    rd = np.float32 if dtype == np.complex64 else np.float64
    out = np.empty(acc[0].shape, dtype=dtype)
    out.real = acc[0].astype(rd)
    out.imag = acc[1].astype(rd)
    return out


def random_kraus(k, m, rng):
    """A random complete set of m Kraus operators on k qubits (a Stinespring isometry cut into blocks)."""
    D = 1 << k
    a = rng.standard_normal((m * D, D)) + 1j * rng.standard_normal((m * D, D))
    q, _ = np.linalg.qr(a)
    return ch.KrausChannel([q[i * D:(i + 1) * D, :] for i in range(m)])


def pauli_matrix(n, term):
    """The 2^n x 2^n matrix of a term [(letter, qubit), ...]."""
    P = np.eye(1 << n, dtype=np.complex128)
    mats = {"X": np.array([[0, 1], [1, 0]]), "Y": np.array([[0, -1j], [1j, 0]]), "Z": np.array([[1, 0], [0, -1]])}
    for letter, q in term:
        P = embed(n, [q], mats[letter]) @ P
    return P


def reduced(n, rho, qubits):
    """Tr_B rho with bit i of the indices the value of qubits[i] (the convention of State.reduced_density)."""
    k = len(qubits)
    out = np.zeros((1 << k, 1 << k), dtype=np.complex128)
    rest = [q for q in range(n) if q not in qubits]
    for a in range(1 << k):
        for a2 in range(1 << k):
            for b in range(1 << len(rest)):
                r = c = 0
                for i, q in enumerate(qubits):
                    r |= ((a >> i) & 1) << (n - 1 - q)
                    c |= ((a2 >> i) & 1) << (n - 1 - q)
                for j, q in enumerate(rest):
                    r |= ((b >> j) & 1) << (n - 1 - q)
                    c |= ((b >> j) & 1) << (n - 1 - q)
                out[a, a2] += rho[r, c]
    return out
