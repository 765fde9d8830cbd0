"""Extended-precision reference and rounding bound for Pauli-string expectation values (State.expect_paulis).

A term is a sequence of (letter, qubit) pairs; qubit q is index bit n-1-q.  With x the mask of the X/Y letters, z the
mask of the Z/Y letters and nY the number of Y letters, P = i^nY X^x Z^z and

    <psi|P|psi> = Re( i^nY * sum_j (-1)^popc(j & z) * conj(a_{j^x}) * a_j ).

expect_ref evaluates this in long double; tests/test_expect_cpu.py pins it against explicit Kronecker products.

Rounding bound of the device kernel (rustqip_b200/csrc/expect.cu), in units of S = sum_j |a_j| |a_{j^x}|:
  - each product conj(a_{j^x}) a_j (or |a_j|^2) is two double products and one add: error <= gamma_2 |a_j||a_{j^x}|;
    f32 amplitudes are exact in double;
  - inside a tile of 2^11 amplitudes a term is either a Walsh-Hadamard output (11 add levels) or a per-thread sum of
    8 products (8 adds) followed, after the tile loop, by a warp sum (5 levels) and a sum over 8 warps (8 adds);
  - signs, the conjugate of the partner tile and the coefficients 1 or 2 are exact;
  - each thread adds its tile values sequentially over the visits of its CTA: at most ceil(V / G) visits of
    V = 2^(n-11) tiles over G = 264 CTAs, twice for Z-only terms on the tile-pair path (both tiles of a pair);
  - the per-CTA partials are summed sequentially over the G CTAs.
So the depth is D = 2 + 21 + 2 ceil(V / G) + G, and |got - want| <= (gamma_D + gamma_ref) S, where gamma_ref covers the
long-double reference: its product (2 roundings) and numpy's pairwise summation of 2^n terms (sequential blocks of up
to 16 inside 128-element leaves, then a binary tree: depth at most n + 12)."""
import math

import numpy as np

U_DOUBLE = 2.0 ** -53
U_LONGDOUBLE = float(np.finfo(np.longdouble).eps) / 2
KERNEL_TILE_BITS = 11
KERNEL_GRID = 264


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


def expect_ref(psi, n, term):
    """<psi|P|psi> for one term, summed in long double (returned as a Python float of the long-double value)."""
    x, z, ny = masks(n, term)
    a = np.asarray(psi).astype(np.clongdouble)
    j = np.arange(1 << n, dtype=np.uint64)
    c = np.conj(a[j ^ np.uint64(x)]) * a
    c = np.where(_parity(j & np.uint64(z)), -c, c)
    w = c.sum()
    ph = ny & 3
    v = (w.real, -w.imag, -w.real, w.imag)[ph]
    return np.longdouble(v)


def abs_weight(psi, n, term):
    """S = sum_j |a_j| |a_{j^x}| (in double; it scales the bound only)."""
    x, _, _ = masks(n, term)
    a = np.abs(np.asarray(psi).astype(np.complex128))
    j = np.arange(1 << n, dtype=np.uint64)
    return float(np.sum(a * a[j ^ np.uint64(x)]))


def gamma(k, u):
    return k * u / (1.0 - k * u)


def kernel_depth(n):
    visits = 1 << max(0, n - KERNEL_TILE_BITS)
    return 2 + 21 + 2 * math.ceil(visits / KERNEL_GRID) + KERNEL_GRID


def bound(n, S):
    return (gamma(kernel_depth(n), U_DOUBLE) + gamma(n + 14, U_LONGDOUBLE)) * S
