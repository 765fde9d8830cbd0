// lanczos.h -- the lowest eigenvalue of a real Pauli sum by plain Lanczos on the device
// (qipb200_state_lanczos_pauli_sum, see lanczos.cu) and the host-side tridiagonal solve (qipb200_lanczos_ritz).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/qip_op.h"
#include "expect.h"

namespace qipb200 {

const uint32_t kLanczosMaxSteps = 4096;

// The lowest eigenvalue *theta of the m x m symmetric tridiagonal T (diagonal alpha[0..m), off-diagonal beta[1..m)),
// by Sturm-sequence bisection to the last bit; its unit eigenvector y[0..m) (may be NULL) by inverse iteration with a
// partially pivoted LU of T - theta, the sign fixed by y[0] >= 0; and *estimate = beta[m] |y[m-1]|.  m >= 1 and every
// value finite (checked by the caller).  O(m) per bisection step; no LAPACK.
void lanczos_ritz(const double *alpha, const double *beta, uint32_t m, double *theta, double *y, double *estimate);

// Kernel counts of a call on these terms (masks on physical index bits): {sum sweeps per step s, kernels per first-pass
// step (s + 1), kernels per second-pass step (s + 1), kernels outside the steps in vector mode (s + 4)}; when every
// term is the identity (b == 0 for any coefficients) {0, 0, 0, 2}.
void lanczos_plan_counts(uint32_t n, const std::vector<PauliTerm> &terms, uint32_t out4[4]);

struct LanczosResult {
  uint32_t steps = 0, converged = 0;
  double energy = 0.0, residual = 0.0, xnorm = 0.0;
  std::vector<double> alpha, beta;  // alpha_0..alpha_(m-1); beta_0 = |psi| .. beta_m
  bool zero_norm = false;           // |psi| is 0 or not finite: nothing was written
};

// The call's device work on an unsharded 2^n state (terms on physical index bits, a and b as in lanczos.cu), vector
// mode when `vector`.  Synchronises once per first-pass step.  The counts of lanczos_plan_counts.
cudaError_t run_lanczos(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                        const std::vector<PauliTerm> &terms, const double *coeffs, double a, double b,
                        uint32_t max_steps, double tol, bool vector, cudaStream_t s, uint64_t *launches,
                        LanczosResult *r);

}  // namespace qipb200
