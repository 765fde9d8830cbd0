// pauli_rot.h -- Pauli-string rotations exp(-i theta/2 P) on the device (qipb200_state_apply_pauli_rotations, see
// pauli_rot.cu).
//
// Sweep planner (the policy qipb200_pauli_rotation_plan reports).  A sweep's tile is the L = min(4, n) lowest index
// bits plus a set H of at most m = min(7, n - L) high bits; the sweep may also carry one out-of-tile X/Y mask X_out,
// shared by all its terms that reach outside the tile.  Terms are taken in order, with masks on physical index bits;
// with r = x & ~(low bits | H):
//   - r == 0 or r == X_out: the term joins;
//   - else if r & X_out == 0 and |H| + popc(r) <= m: H |= r and the term joins;
//   - else if X_out == 0: X_out = r and the term joins;
//   - else the term opens the next sweep.
// Afterwards each sweep fills H up to m bits, first with X_out bits (fewer tile pairs), then with the lowest free bits.
// So a list of only diagonal terms is one sweep, any single term is one sweep, a run whose X/Y bits lie in the low bits
// and at most m others is one sweep, and the number of sweeps is at most max(1, number of non-diagonal terms).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/qip_op.h"
#include "expect.h"

namespace qipb200 {

// Read-write sweeps run_pauli_rotations makes for these terms (masks on physical index bits) on an unsharded 2^n state.
uint32_t pauli_rotation_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms);

// psi <- exp(-i angles[T-1]/2 P_{T-1}) ... exp(-i angles[0]/2 P_0) psi in place, for terms on physical index bits of an
// unsharded 2^n state.  cos and sin of angles[t]/2 are taken in double on the host and rounded once to the state's
// precision; each amplitude pair is then updated as psi'_j = RN(RN(c psi_j) + RN(s w_j)) per component, with
// w_j = -i (P psi)_j exact.  One kernel per sweep, stream-ordered: the host tables are copied before it returns and the
// stream is not synchronised.  grid: CTAs per sweep.
cudaError_t run_pauli_rotations(qip_prec prec, void *psi, uint32_t n, const std::vector<PauliTerm> &terms,
                                const double *angles, int grid, cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
