// rdm.h -- reduced density matrices on the device (qipb200_state_reduced_density, see rdm.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/qip_op.h"

namespace qipb200 {

// Largest number of kept qubits (the output is 4^k complex doubles: 16 MiB at k = 10).
const uint32_t kRdmMaxKept = 10;

// Kernel launches run_reduced_density makes for k kept qubits: nB (nB + 1) with nB = 2^max(0, k - 6) (one sweep
// kernel and one reduction per block pair I <= J), so 2 for k <= 6.
uint64_t rdm_launch_count(uint32_t k);

// out[a * 2^k + b] (interleaved re/im) = sum_r psi(r, a) conj(psi(r, b)) of an unsharded 2^n state, where bit i of a
// and b is the value of physical index bit pos[i].  The lower triangle is written as the conjugate of the upper one and
// the diagonal's imaginary part is 0.0.  Synchronises the stream.
cudaError_t run_reduced_density(qip_prec prec, const void *psi, uint32_t n, const uint32_t *pos, uint32_t k,
                                double *out, cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
