// gradient.h -- H|psi> for a real Pauli sum H (qipb200_state_apply_pauli_sum) and the adjoint-method energy gradient of
// a Pauli-rotation circuit (qipb200_state_pauli_energy_gradient), see gradient.cu.
//
// Sum planner (the policy qipb200_pauli_sum_plan reports).  The terms of a sum commute, so they are grouped by X/Y
// mask, groups in order of first appearance and terms in list order inside a group.  A sweep's tile is the
// L = min(4, n) lowest index bits plus a set H of at most m = min(6, n - L) high bits, and the sweep may carry one
// out-of-tile X/Y mask X_out.  Sweeps are opened one at a time; each takes, in group order, every group not yet taken
// that joins by the rule of pauli_rot.h (r = x & ~(low bits | H): r == 0 or r == X_out joins; else if r & X_out == 0
// and |H| + popc(r) <= m, H |= r and it joins; else if X_out == 0, X_out = r and it joins).  Afterwards H is filled as
// in pauli_rot.h.  So a diagonal-only sum is one sweep, and the transverse-field Ising H at n = 30 takes 4.
//
// Adjoint planner (the backward sweeps qipb200_pauli_gradient_plan reports).  The rotation planner of pauli_rot.h with
// m = min(6, n - L) runs over the reversed term list, and a sweep is cut after every 256 terms.  With no terms it is one
// sweep that computes the energy only.
//
// Segment planner (the segment sweeps qipb200_pauli_geometric_tensor_plan reports).  For fork i the same walk runs over
// terms i + 1 .. T - 1 in forward order, cut after every 256 terms; the last fork has no segment.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/qip_op.h"
#include "expect.h"

namespace qipb200 {

// CTAs of a sum or adjoint sweep (fewer when it has fewer visits): two per SM of a 132-SM H100.  A fixed grid, so the
// same inputs give the same bits on any device.
const int kGradGrid = 264;

// Read-write sweeps run_pauli_sum makes for these terms (masks on physical index bits) on an unsharded 2^n state.
uint32_t pauli_sum_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms);

// Backward sweeps run_pauli_gradient makes for this ansatz on an unsharded 2^n state.
uint32_t pauli_adjoint_sweep_count(uint32_t n, const std::vector<PauliTerm> &ansatz);

// dst <- sum_h coeffs[h] P_h src (dst != src, both 2^n amplitudes of precision prec, masks on physical index bits).
// One kernel per sweep; no terms: dst is zeroed with a memset and no kernel runs.  Stream-ordered, no synchronisation.
cudaError_t run_pauli_sum(qip_prec prec, void *dst, const void *src, uint32_t n, const std::vector<PauliTerm> &terms,
                          const double *coeffs, cudaStream_t s, uint64_t *launches);

// The Chebyshev series of qipb200_state_evolve_pauli_sum (evolve.h): steps k = 1..K of the recurrence over the
// non-identity `terms` (masks on physical index bits) and their coefficients, with H~ = (H - a) / half_width, each step
// one kernel per sweep of the sum plan; state <- sum_k C_k T_k(H~) state for C = C_0..C_K (re, im), K >= 2.  work_a
// and work_b are scratch of the state's size and precision (their contents afterwards are unspecified).  Launches K x
// sweeps kernels, stream-ordered.
cudaError_t run_pauli_evolution(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                                const std::vector<PauliTerm> &terms, const double *coeffs, double half_width,
                                const std::vector<double> &C, cudaStream_t s, uint64_t *launches);

// One Lanczos sum (lanczos.cu): dst <- sum_h RN(coeffs[h] scale) P_h src, the accumulator of the first sweep started at
// RN(start from) (from NULL: at +0.0), one kernel per sweep of the sum plan.  When dot is not NULL the last sweep writes
// dot[c] = CTA c's sum of Re(conj(src_j) dst_j) over the stored dst, for c < *dot_grid (a fixed function of the plan).
// terms must not be empty.  Stream-ordered, no synchronisation.
cudaError_t run_lanczos_sum(qip_prec prec, void *dst, const void *src, const void *from, double start, uint32_t n,
                            const std::vector<PauliTerm> &terms, const double *coeffs, double scale, double *dot,
                            uint32_t *dot_grid, cudaStream_t s, uint64_t *launches);

// The adjoint gradient: state <- U state (run_pauli_rotations), work <- H state (run_pauli_sum), then the backward
// sweeps, each one adjoint kernel and one reduction kernel.  Launches forward + sum + 2 backward sweeps.  Writes
// *energy and grad[0..T); synchronises the stream.  grid: CTAs per forward sweep.
cudaError_t run_pauli_gradient(qip_prec prec, void *state, void *work, uint32_t n, const std::vector<PauliTerm> &ansatz,
                               const double *angles, const std::vector<PauliTerm> &ham, const double *coeffs, int grid,
                               cudaStream_t s, uint64_t *launches, double *energy, double *grad);

// Segment sweeps run_pauli_qgt makes for this ansatz on an unsharded 2^n state (the sum over forks i of the walk over
// terms i + 1 .. T - 1).
uint32_t pauli_qgt_sweep_count(uint32_t n, const std::vector<PauliTerm> &ansatz);

// The quantum geometric tensor of the ansatz (qipb200_state_pauli_geometric_tensor): for each term i one fork
// (state <- R_i state, work_a <- state, work_b <- P_i state) and the segment sweeps over terms i + 1 .. T - 1 on
// (work_a, work_b), each one walk kernel and one reduction kernel, then one reduction of the forks' rows.  Launches
// T + 2 S + 1 kernels (none for T = 0).  Writes qgt[0 .. 2 T^2) (G row-major, (re, im) pairs) and, when expect is not
// NULL, expect[0 .. T); synchronises the stream.
cudaError_t run_pauli_qgt(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                          const std::vector<PauliTerm> &ansatz, const double *angles, cudaStream_t s,
                          uint64_t *launches, double *qgt, double *expect);

}  // namespace qipb200
