// purity.h -- purity Tr rho_A^2 of a bipartition on the device (qipb200_state_purity, see purity.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/qip_op.h"

namespace qipb200 {

// Smallest side the Gram kernel serves; smaller sides go through run_reduced_density (which stops at kRdmMaxKept).
const uint32_t kPurityGramMinSide = 11;

// Route of qipb200_state_purity for a side of s qubits: 0 (s = 0, norm2), 1 (s <= 10, reduced_density), 2 (Gram).
uint32_t purity_route(uint32_t s);
// Blocks (I, J) of G = M M^dagger the Gram kernel visits for a side of s >= 7 qubits: 128 x 64 entries each, every
// block that touches the upper triangle, nR (nR + 1) with nR = 2^(s - 7).
uint64_t purity_gram_blocks(uint32_t s);
// Kernel launches of qipb200_state_purity for a side of s qubits (nothing pending): 1, rdm_launch_count(s), or 2.
uint64_t purity_launch_count(uint32_t s);

// out2 = {sum_{a,b} |G_ab|^2, sum_a G_aa} for G = M M^dagger, M[a][r] = psi[pdep(a, side) | pdep(r, ~side)], on an
// unsharded 2^n state; side has s >= kPurityGramMinSide bits and s <= n - s.  Synchronises the stream.
cudaError_t run_purity_gram(qip_prec prec, const void *psi, uint32_t n, uint64_t side_mask, double *out2,
                            cudaStream_t s, uint64_t *launches);

// G = M M^dagger of the side qubits at physical bits pos[0..sb) (11 <= sb <= 13, sb <= n - sb) of an unsharded 2^n
// state into the device array G (4^sb double2, row-major): bit i of a row or column index is the value of physical bit
// pos[i].  The lower triangle is the exact conjugate of the upper one and the diagonal's imaginary part is +0.0.  One
// kernel (the store epilogue of the purity Gram kernel).  Synchronises the stream.
cudaError_t run_gram_store(qip_prec prec, const void *psi, uint32_t n, const uint32_t *pos, uint32_t sb, double2 *G,
                           cudaStream_t s, uint64_t *launches);

// *out = sum_j |psi_j|^2 of an unsharded 2^n state in a fixed order (one kernel; the s = 0 route).  Synchronises.
cudaError_t run_purity_norm2(qip_prec prec, const void *psi, uint32_t n, double *out, cudaStream_t s,
                             uint64_t *launches);

}  // namespace qipb200
