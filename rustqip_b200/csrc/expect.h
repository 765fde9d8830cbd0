// expect.h -- Pauli-string expectation values on the device (qipb200_state_expect_paulis, see expect.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/qip_op.h"

namespace qipb200 {

// P = i^n_y X^x Z^z over index-bit masks x (X/Y letters) and z (Z/Y letters).
struct PauliTerm {
  uint64_t x = 0, z = 0;
  uint32_t n_y = 0;
};

// The one validation both C entries run: letters X/Y/Z only (else QIPB200_ERR_INVALID_ARG), qubits < n and distinct
// inside a term (else QIPB200_ERR_BAD_INDEX), non-NULL arrays when n_terms > 0.  Qubit q becomes index bit n-1-q.
int parse_pauli_terms(uint32_t n, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms,
                      std::vector<PauliTerm> *out, std::string *err);

// Terms of one X/Y mask: indices into the term list, in list order.
struct PauliGroup {
  uint64_t x = 0;
  std::vector<uint32_t> terms;
};

// The terms grouped by X/Y mask, groups in order of first appearance (the sweep planners of expect.cu and gradient.cu).
std::vector<PauliGroup> group_by_x(const std::vector<PauliTerm> &terms);

// Read sweeps run_expect makes for these terms (masks on physical index bits) on an unsharded 2^n state.
uint32_t expect_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms);

// out[t] = <psi|P_t|psi> (real part) for terms on physical index bits of an unsharded 2^n state.  Launches one kernel
// per sweep and one reduction kernel per batch of at most kExpectBatchTerms terms; synchronises the stream.
cudaError_t run_expect(qip_prec prec, const void *psi, uint32_t n, const std::vector<PauliTerm> &terms, double *out,
                       cudaStream_t s, uint64_t *launches);

// out2 = {read sweeps, kernels} run_transition makes for these terms on an unsharded 2^n state.
void transition_plan_counts(uint32_t n, const std::vector<PauliTerm> &terms, uint32_t *out2);

// out[2t], out[2t + 1] = Re, Im <bra|P_t|ket> for terms on physical index bits of two unsharded 2^n states of the same
// layout (bra == ket allowed).  The sweeps of run_expect over two rows per term (Re and Im), each sweep reading both
// states once; one kernel per sweep and one reduction kernel per batch; synchronises the stream.
cudaError_t run_transition(qip_prec prec, const void *bra, const void *ket, uint32_t n,
                           const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
