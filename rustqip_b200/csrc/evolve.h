// evolve.h -- the host side of qipb200_state_evolve_pauli_sum: the Chebyshev expansion of exp(-iHt) for a real Pauli
// sum H = sum_h c_h P_h (the device recurrence is run_pauli_evolution, gradient.cu).
//
// The identity terms sum to a (in list order, from +0.0) and the others give the half-width b = sum |c_h| (in list
// order, in double, from +0.0), which bounds |H - a| since |P| = 1.  With H~ = (H - a) / b and x = RN(b t),
//   exp(-iHt) = sum_k C_k T_k(H~),   C_k = (2 - delta_k0) (-i)^k J_k(x) e^{-i RN(a t)}.
// J_0..J_M(|x|) come from Miller's backward recurrence J_(k-1) = (2k / |x|) J_k - J_(k+1) in long double (64-bit
// mantissa), started at J_(M+1) = 0 past the index M where (|x|/2)^M / M! (an upper bound of J_M) falls below
// min(tol, 1e-16) e^-60, and normalised by J_0 + 2 sum_k J_2k = 1; J_k(-x) = (-1)^k J_k(x).  Over the at most ~1.3e5
// steps the recurrence takes here its rounding stays near 1e-17 absolute, so each C_k, rounded once to double and
// multiplied by the phase (cos, -sin of RN(a t) from the C library), is within ~1e-16 absolute of the exact value for
// the same x and a t (checked against scipy.special.jv to 1e-14 for |x| up to 5000 in tests/test_evolve_cpu.py).
// The degree K is the smallest k >= 2 with tau_k = 2 sum_(j > k) |J_j(x)| <= tol; then
// |psi_K - exp(-iHt) psi| <= tau_K |psi| in exact arithmetic, since |T_k(H~)| <= 1.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "expect.h"

namespace qipb200 {

const uint32_t kEvolveMaxDegree = 65536;  // a longer series: split t over several calls

struct EvolutionPlan {
  enum Kind { kNoop, kPhase, kSeries } kind = kNoop;  // t == 0 or no terms; identity-only H (b == 0); the series
  std::vector<PauliTerm> terms;  // the non-identity terms, in list order
  std::vector<double> coeffs;    // and their coefficients
  double a = 0.0, b = 0.0;
  uint32_t degree = 0;           // K (0 unless kSeries)
  double tail = 0.0;             // tau_K (0 unless kSeries)
  std::vector<double> C;         // C_0..C_K (re, im); kNoop: C_0 = 1, kPhase: C_0 = e^{-i RN(a t)}
};

// The plan of exp(-i time H) for terms and coeffs (validated by the caller; tol in (0, 1)).  QIPB200_OK, or
// QIPB200_ERR_UNSUPPORTED with *err when K would exceed kEvolveMaxDegree or 2 / b overflows.
int plan_evolution(const std::vector<PauliTerm> &terms, const double *coeffs, double time, double tol,
                   EvolutionPlan *p, std::string *err);

}  // namespace qipb200
