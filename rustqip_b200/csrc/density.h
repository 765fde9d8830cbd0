// density.h -- exact noisy simulation on density matrices (qipb200_density_*): the doubling of a circuit with Kraus
// channels into one schedule on vec(rho), and the readout kernels of density.cu.  See density.cu for the layout.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <deque>
#include <string>
#include <vector>

#include "../../include/qipb200.h"
#include "expect.h"

namespace qipb200 {

// Largest rho of qipb200_density_spectrum: 2^13 x 2^13 complex doubles is 1 GiB (kSpectrumMaxSide).
const uint32_t kDensitySpectrumMax = 13;

// The doubled schedule of a noisy circuit on an n-qubit rho, as qip_op records on 2n qubits.  Gate records are the
// caller's (they point into the caller's arrays); the conjugated copies and the superoperators own their arrays here.
struct DensitySchedule {
  std::vector<qip_op> ops;
  std::deque<qip_op> nested;
  std::deque<std::vector<uint64_t>> u64s;
  std::deque<std::vector<unsigned char>> blobs;
};

// Validate and double a circuit (the rules of include/qipb200.h, qipb200_density_apply) into *out.  Returns QIPB200_OK,
// or the status with the message (prefixed by who) in *err.
int build_density_schedule(const std::string &who, qip_prec prec, uint32_t n, const qip_op *ops, size_t n_ops,
                           size_t n_channels, const uint64_t *channel_pos, const uint32_t *arity,
                           const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, DensitySchedule *out,
                           std::string *err);

// rho = |psi><psi| (rho 2n qubits in the canonical layout, psi n qubits).  One write sweep; 1 kernel.
cudaError_t run_density_from_state(qip_prec prec, void *rho, const void *psi, uint32_t n, cudaStream_t s,
                                   uint64_t *launches);

// Sums of rho's entries over index sets (the diagonal readouts and partial traces).  Key bit j (j < nb + ke) sets the
// physical index bits key_masks[j]; entry e < 2^ke is out[e] = sum over b < 2^nb of rho[phys(b | e << nb)], in double.
// With kc > 0, e = a | a' << (ke - kc) and only the entries with a <= a' are computed (the others are left as they
// are).  out is a HOST array of 2 * 2^ke doubles (interleaved re/im).  Fixed order, no atomics.  1 kernel; synchronises.
cudaError_t run_density_sums(qip_prec prec, const void *rho, const std::vector<uint64_t> &key_masks, uint32_t nb,
                             uint32_t ke, uint32_t kc, double *out, cudaStream_t s, uint64_t *launches);

// out[t] = Re Tr(rho P_t) for terms on rho's n-qubit index bits; pol is the state's logical -> physical bit map (2n
// entries).  2 kernels per batch of terms; synchronises.
cudaError_t run_density_expect(qip_prec prec, const void *rho, uint32_t n, const std::vector<uint32_t> &pol,
                               const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches);

// out2 = {Re, Im} <psi|rho|psi> (psi in the canonical layout).  One read sweep of rho; 2 kernels; synchronises.
cudaError_t run_density_fidelity(qip_prec prec, const void *rho, const void *psi, uint32_t n,
                                 const std::vector<uint32_t> &pol, double *out2, cudaStream_t s, uint64_t *launches);

// G[r * 2^n + c] = rho_rc widened to double (device array of 4^n double2).  One read sweep; 1 kernel.
cudaError_t run_density_widen(qip_prec prec, const void *rho, uint32_t n, const std::vector<uint32_t> &pol, double2 *G,
                              cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
