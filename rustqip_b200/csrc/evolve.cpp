// evolve.cpp -- the Chebyshev plan of qipb200_state_evolve_pauli_sum (see evolve.h).
#include "evolve.h"

#include <cmath>
#include <string>

#include "../../include/qipb200.h"

namespace qipb200 {

namespace {

// J_0(x) .. J_M(x) by Miller's backward recurrence in long double (evolve.h); M grows until the upper bound
// (|x|/2)^M / M! of J_M is below e^floor_log.
std::vector<long double> bessel_j(double xd, long double floor_log) {
  const long double x = fabsl((long double)xd);
  if (x == 0.0L) return std::vector<long double>(1, 1.0L);
  uint32_t M = (uint32_t)ceill(x) + 20;
  auto log_bound = [&](uint32_t k) {  // log of (x/2)^k / k! by Stirling
    return k * logl(x / (2.0L * k)) + k - 0.5L * logl(2.0L * 3.14159265358979323846L * k);
  };
  while (log_bound(M) > floor_log) M += 8;
  std::vector<long double> J(M + 2, 0.0L);
  J[M] = 1.0L;
  for (uint32_t k = M; k >= 1; --k) {
    J[k - 1] = (2.0L * k / x) * J[k] - J[k + 1];
    if (fabsl(J[k - 1]) > 1e1000L)  // stay far inside the long double range (a tiny x grows fast)
      for (uint32_t i = k - 1; i <= M; ++i) J[i] *= 1e-1000L;
  }
  long double norm = 0.0L;
  for (uint32_t k = M - (M & 1); k >= 2; k -= 2) norm += 2.0L * J[k];
  norm += J[0];
  for (uint32_t k = 0; k <= M; ++k) J[k] = ((xd < 0 && (k & 1)) ? -J[k] : J[k]) / norm;
  J.pop_back();
  return J;
}

}  // namespace

int plan_evolution(const std::vector<PauliTerm> &terms, const double *coeffs, double time, double tol,
                   EvolutionPlan *p, std::string *err) {
  *p = EvolutionPlan();
  p->C = {1.0, 0.0};
  if (time == 0.0 || terms.empty()) return QIPB200_OK;
  for (size_t h = 0; h < terms.size(); ++h) {
    if (terms[h].x == 0 && terms[h].z == 0) {
      p->a += coeffs[h];
    } else {
      p->terms.push_back(terms[h]);
      p->coeffs.push_back(coeffs[h]);
      p->b += std::fabs(coeffs[h]);
    }
  }
  const double at = p->a * time;
  const double cp = std::cos(at), sp = -std::sin(at);  // e^{-i a t}
  if (p->b == 0.0) {
    p->kind = EvolutionPlan::kPhase;
    p->C = {cp, sp};
    return QIPB200_OK;
  }
  const double x = p->b * time;
  if (!std::isfinite(2.0 / p->b)) {
    *err = "evolve_pauli_sum: the half-width sum |c_h| = " + std::to_string(p->b) + " is too small to scale by";
    return QIPB200_ERR_UNSUPPORTED;
  }
  const std::string split = "; split the time over several calls";
  if (!(std::fabs(x) <= 2.0 * kEvolveMaxDegree)) {  // the degree grows like |x|
    *err = "evolve_pauli_sum: |t| sum |c_h| = " + std::to_string(std::fabs(x)) + " needs a degree above " +
           std::to_string(kEvolveMaxDegree) + split;
    return QIPB200_ERR_UNSUPPORTED;
  }
  const std::vector<long double> J = bessel_j(x, std::log(std::fmin(tol, 1e-16)) - 60.0);
  // tau_k = 2 sum_(j > k) |J_j|, smallest first
  std::vector<long double> tau(J.size() + 1, 0.0L);
  for (size_t k = J.size(); k-- > 0;) tau[k] = tau[k + 1] + (k + 1 < J.size() ? 2.0L * fabsl(J[k + 1]) : 0.0L);
  uint32_t K = 2;
  while (K + 1 < J.size() && tau[K] > tol) ++K;
  if (K > kEvolveMaxDegree) {
    *err = "evolve_pauli_sum: degree " + std::to_string(K) + " above " + std::to_string(kEvolveMaxDegree) +
           " for |t| sum |c_h| = " + std::to_string(std::fabs(x)) + split;
    return QIPB200_ERR_UNSUPPORTED;
  }
  p->kind = EvolutionPlan::kSeries;
  p->degree = K;
  p->tail = (double)tau[K];
  p->C.assign(2 * (K + 1), 0.0);
  for (uint32_t k = 0; k <= K; ++k) {
    const double r = (double)((k ? 2.0L : 1.0L) * (k < J.size() ? J[k] : 0.0L));
    // (-i)^k r as (re, im), then times e^{-i a t}: one of re, im is zero, so each component is one rounded product
    const double re = (k & 1) ? 0.0 : ((k & 2) ? -r : r), im = (k & 1) ? ((k & 2) ? r : -r) : 0.0;
    p->C[2 * k] = re * cp - im * sp;
    p->C[2 * k + 1] = re * sp + im * cp;
  }
  return QIPB200_OK;
}

}  // namespace qipb200
