"""Extended-precision reference and rounding bound for transition elements <bra|P|ket> (State.transition_paulis).

With x, z and nY as in tests/pauli_ref.py (P = i^nY X^x Z^z),

    <bra|P|ket> = sum_j conj(bra_j) (P ket)_j = i^nY * sum_j (-1)^popc(j & z) * conj(bra_{j^x}) * ket_j.

transition_ref evaluates this in long double; tests/test_transition_cpu.py pins it against np.vdot with explicit
Kronecker products, and against expect_ref for bra == ket.

Rounding bound of the device kernel (k_expect in two-state mode, rustqip_b200/csrc/expect.cu), for each of Re and Im
separately, in units of S = sum_j |bra_{j^x}| |ket_j|: the summation tree is the one-state kernel's, with complex
products c_j = conj(bra_{j^x}) ket_j for every group (two double products and one add per component), both sides of a
tile pair summed explicitly for every term (two adds per visit, the count pauli_ref already allows), signs and the
+-1 of i^nY exact.  So the depth D and the bound are pauli_ref.kernel_depth / pauli_ref.bound with this S."""
import numpy as np

import pauli_ref as pr


def transition_ref(bra, ket, n, term):
    """<bra|P|ket> for one term, summed in long double (np.clongdouble)."""
    x, z, ny = pr.masks(n, term)
    b = np.asarray(bra).astype(np.clongdouble)
    k = np.asarray(ket).astype(np.clongdouble)
    j = np.arange(1 << n, dtype=np.uint64)
    c = np.conj(b[j ^ np.uint64(x)]) * k
    c = np.where(pr._parity(j & np.uint64(z)), -c, c)
    w = c.sum()
    return w * (np.clongdouble(1), np.clongdouble(1j), np.clongdouble(-1), np.clongdouble(-1j))[ny & 3]


def abs_weight(bra, ket, n, term):
    """S = sum_j |bra_{j^x}| |ket_j| (in double; it scales the bound only)."""
    x, _, _ = pr.masks(n, term)
    b = np.abs(np.asarray(bra).astype(np.complex128))
    k = np.abs(np.asarray(ket).astype(np.complex128))
    j = np.arange(1 << n, dtype=np.uint64)
    return float(np.sum(b[j ^ np.uint64(x)] * k))


def bound(n, S):
    """Bound on |Re got - Re want| and on |Im got - Im want| for a value of weight S."""
    return pr.bound(n, S)


def errors(got, want):
    """(|d Re|, |d Im|) of a complex128 device value against a long-double reference."""
    return (float(abs(np.longdouble(got.real) - want.real)), float(abs(np.longdouble(got.imag) - want.imag)))
