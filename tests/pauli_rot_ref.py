"""References for Pauli-string rotations (State.apply_pauli_rotations, qipb200_state_apply_pauli_rotations).

A term is a sequence of (letter, qubit) pairs as in tests/pauli_ref.py: qubit q is index bit n-1-q, x is the mask of the
X/Y letters, z of the Z/Y letters, and P = i^nY X^x Z^z, so (P psi)_j = i^nY (-1)^popc((j^x) & z) psi_{j^x}.  The call
applies exp(-i theta_T-1/2 P_T-1) ... exp(-i theta_0/2 P_0), term 0 first.

  - emulate: the device arithmetic in numpy float64 / float32, bit for bit.  Per term c = cos(theta/2) and
    s = sin(theta/2) from Python's math module (the C library the host side calls), rounded once to the state's
    precision; then psi'_j = RN(RN(c psi_j) + RN(s w_j)) per component with w_j = -i (P psi)_j, exact.
  - rotate_ref: the same rotations in long double, and bound(): the device's distance from it.  Per term the device
    rounds c and s (host cos/sin within one ulp: 2u, then the cast to f32: u), the two products and the sum; each
    component of the error is at most 4u (|c| |psi_j| + |s| |psi_j^x|) to first order, so the error vector of one term
    is at most 4u sqrt(2) |psi| in 2-norm, and later terms are unitary: the errors add.  Over T terms the max-abs error
    is at most sqrt(2) gamma_{5T} |psi|, plus gamma_{8T} in long double for the reference itself.
  - decomposition: one rotation as existing MatrixOps (basis change, CNOT ladder, rz, and back)."""
import math

import numpy as np

from rustqip_b200 import gates

U = {np.complex128: 2.0 ** -53, np.complex64: 2.0 ** -24}
U_LONGDOUBLE = float(np.finfo(np.longdouble).eps) / 2


def masks(n, term):
    x = z = ny = 0
    for letter, q in term:
        b = 1 << (n - 1 - int(q))
        if letter in ("X", "Y"):
            x |= b
        if letter in ("Z", "Y"):
            z |= b
        ny += letter == "Y"
    return x, z, ny


def _parity(v):
    return (np.bitwise_count(v) & 1).astype(bool)


def _times_i_power(ph, pr, pi):
    """i^ph (pr + i pi) as a component swap and negations."""
    return ((pr, pi), (-pi, pr), (-pr, -pi), (pi, -pr))[ph & 3]


def emulate(psi, n, terms, angles, dtype):
    """The device result, bit for bit (up to the sign of zero), as an array of dtype."""
    R = np.float64 if np.dtype(dtype) == np.complex128 else np.float32
    psi = np.asarray(psi).astype(dtype)
    re, im = psi.real.astype(R), psi.imag.astype(R)
    j = np.arange(1 << n, dtype=np.uint64)
    for term, th in zip(terms, angles):
        x, z, ny = masks(n, term)
        c, s = R(math.cos(float(th) / 2)), R(math.sin(float(th) / 2))
        p = j ^ np.uint64(x)
        neg = _parity(p & np.uint64(z))
        wr, wi = _times_i_power(ny + 3, re[p], im[p])  # w = -i * i^nY * sign * psi_{j^x}
        wr, wi = np.where(neg, -wr, wr), np.where(neg, -wi, wi)
        re, im = c * re + s * wr, c * im + s * wi
        assert re.dtype == R and im.dtype == R
    out = np.empty(1 << n, dtype=dtype)
    out.real, out.imag = re, im
    return out


def rotate_ref(psi, n, terms, angles):
    """The rotations in long double (clongdouble array)."""
    a = np.asarray(psi).astype(np.clongdouble)
    j = np.arange(1 << n, dtype=np.uint64)
    for term, th in zip(terms, angles):
        x, z, ny = masks(n, term)
        h = np.longdouble(float(th)) / 2
        c, s = np.cos(h), np.sin(h)
        p = j ^ np.uint64(x)
        pa = np.where(_parity(p & np.uint64(z)), -a[p], a[p])
        w = pa * np.clongdouble((-1j) * (1j ** (ny & 3)))
        a = c * a + s * w
    return a


def gamma(k, u):
    return k * u / (1.0 - k * u)


def bound(n_terms, norm, dtype):
    """Max-abs distance of the device result from rotate_ref, for a start state of 2-norm `norm`."""
    t = max(1, n_terms)
    return (math.sqrt(2) * gamma(5 * t, U[dtype]) + gamma(8 * t, U_LONGDOUBLE)) * norm


def sdg(q):
    return gates.mat([q], [1, 0, 0, -1j])


def decomposition(term, theta):
    """exp(-i theta/2 P) as MatrixOps: H (X) or S^dagger then H (Y) on every X/Y qubit, a CNOT ladder onto the last
    qubit of the term, rz(theta) there, the ladder back and the basis change undone.  The identity is the global phase
    e^{-i theta/2} on qubit 0."""
    if not term:
        ph = complex(math.cos(theta / 2), -math.sin(theta / 2))
        return [gates.mat([0], [ph, 0, 0, ph])]
    qs = [int(q) for _, q in term]
    into, back = [], []
    for letter, q in term:
        if letter == "X":
            into.append(gates.h(q))
            back.append(gates.h(q))
        elif letter == "Y":
            into += [sdg(q), gates.h(q)]
            back += [gates.h(q), gates.s(q)]
    ladder = [gates.cnot(qs[i], qs[i + 1]) for i in range(len(qs) - 1)]
    return into + ladder + [gates.rz(qs[-1], theta)] + ladder[::-1] + back


def decompose_all(terms, angles):
    ops = []
    for t, th in zip(terms, angles):
        ops += decomposition(t, float(th))
    return ops


# ---- the documented sweep policy (rustqip_b200/csrc/pauli_rot.h), independently of the library -------------------

def plan_policy(n, terms):
    L = min(4, n)
    m = min(7, n - L)
    low = (1 << L) - 1
    sweeps = 0
    hi = x_out = 0

    def join(x):
        nonlocal hi, x_out
        r = x & ~(low | hi)
        if r == 0 or r == x_out:
            return True
        if not (r & x_out) and bin(hi).count("1") + bin(r).count("1") <= m:
            hi |= r
            return True
        if x_out == 0:
            x_out = r
            return True
        return False

    for t in terms:
        x, _, _ = masks(n, t)
        if sweeps == 0 or not join(x):
            sweeps += 1
            hi = x_out = 0
            assert join(x)
    return sweeps


# ---- term families -------------------------------------------------------------------------------------------------

def ising_step(n):
    """One transverse-field Ising Trotter step: n Z_iZ_i+1 (periodic; Z_0 alone for n = 1), then n X_i."""
    zz = [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)] if n > 1 else [[("Z", 0)]]
    return zz + [[("X", i)] for i in range(n)]


def z_pairs(n):
    """The n + n(n-1)/2 diagonal terms Z_i and Z_iZ_j."""
    return [[("Z", i)] for i in range(n)] + [[("Z", i), ("Z", j)] for i in range(n) for j in range(i + 1, n)]


def ucc_strings(n, count, seed):
    """Jordan-Wigner double-excitation strings: X/Y on four qubits p < q < r < s (an odd number of Y), Z on the qubits
    strictly between p and q and between r and s."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        p, q, r, s = sorted(int(v) for v in rng.choice(n, size=4, replace=False))
        letters = [str(v) for v in rng.choice(list("XY"), size=4)]
        if letters.count("Y") % 2 == 0:
            letters[0] = "Y" if letters[0] == "X" else "X"
        term = [(letters[0], p)] + [("Z", k) for k in range(p + 1, q)] + [(letters[1], q), (letters[2], r)]
        term += [("Z", k) for k in range(r + 1, s)] + [(letters[3], s)]
        out.append(term)
    return out


def qaoa_layer(n):
    """A 3-regular QAOA layer on n (even) qubits: the ring and the diameters as Z_iZ_j cost terms, then X_i mixers."""
    edges = [(i, (i + 1) % n) for i in range(n)] + [(i, i + n // 2) for i in range(n // 2)]
    return [[("Z", a), ("Z", b)] for a, b in edges] + [[("X", i)] for i in range(n)]
