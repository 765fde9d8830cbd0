// kraus.h -- one quantum-trajectory step of general Kraus channels on up to four qubits
// (qipb200_state_apply_kraus_channels): the host-side parsing, grouping and choice, and the grouped apply sweep of
// kraus.cu.  See kraus.cu for the argument and the arithmetic.
#pragma once

#include <cuda_runtime.h>

#include <complex>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/qipb200.h"

namespace qipb200 {

const uint32_t kKrausMaxArity = 4;    // qubits per channel
const uint32_t kKrausMaxOps = 256;    // operators per channel
const uint32_t kKrausGroupBits = 4;   // qubits of a group of state-dependent channels
const double kKrausTol = 1e-12;       // completeness and state independence, per matrix entry

// A validated layer.  Channel c acts on qubits[qfirst[c] .. qfirst[c + 1]) (its first qubit the most significant bit
// of the matrix index) and has the operators first[c] .. first[c + 1]; operator o's matrix is mat[o] (2^k x 2^k,
// row-major, interleaved re/im: the caller's array) and gram[o] = K^dagger K in double, summed over the row in
// ascending order.
struct KrausSet {
  std::vector<uint64_t> qubits;
  std::vector<uint32_t> qfirst;
  std::vector<uint32_t> first;
  std::vector<const double *> mat;
  std::vector<std::vector<std::complex<double>>> gram;
  std::vector<double> w;       // Tr(K^dagger K) / 2^k, the trace summed in ascending order
  std::vector<uint8_t> indep;  // state-independent: every K^dagger K within kKrausTol of w I
  size_t size() const { return indep.size(); }
  uint32_t arity(size_t c) const { return qfirst[c + 1] - qfirst[c]; }
};

// Validate n_channels channels of an n-qubit state (the rules of include/qipb200.h) into *out.  Returns QIPB200_OK,
// or the status with the message (prefixed by who) in *err.  A layer names no qubit twice; with sequential set, the
// channels run one after the other (qipb200_density_apply), so only a qubit repeated inside one channel is refused.
int parse_kraus_channels(const std::string &who, uint32_t n, size_t n_channels, const uint32_t *arity,
                         const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, KrausSet *out,
                         std::string *err, bool sequential = false);

// The groups of the state-dependent channels: runs of consecutive ones, in channel order, with at most
// kKrausGroupBits qubits each (a group closes when the next channel would exceed them).
std::vector<std::vector<size_t>> kraus_groups(const KrausSet &ks);

// out4 = {groups r, read sweeps (1 if r > 0), read-write sweeps (r), kernels of the groups (2r + 1 if r > 0)}.
void plan_kraus_channels(const KrausSet &ks, uint32_t out4[4]);

// The smallest i with u S < sum_{i' <= i} e_i' (S = sum_i e_i in order), else the last i with e_i > 0 (0 when none).
uint32_t kraus_choose(const double *e, uint32_t m, double u);

// Draw the channels of group g (channel indices in order) from rho, the group's 2^m x 2^m reduced density matrix
// (interleaved re/im) in the matrix convention over the group's qubits in order (the first the most significant).
// Writes chosen[c] and cond[c] for the group's channels and returns false when Tr rho (S) is not positive.
bool kraus_draw_group(const KrausSet &ks, const std::vector<size_t> &g, const double *rho, const double *draws,
                      uint32_t *chosen, double *cond);

// K is a positive real multiple of the identity.
bool kraus_is_scaled_identity(const double *K, uint32_t k);

// One channel of a group sweep: its physical bits in the matrix convention (pos[0] the most significant) and its
// scaled operator, already rounded to the state's precision (4^k complex<prec>, row-major).
struct KrausApplyOp {
  uint32_t k;
  uint32_t pos[kKrausMaxArity];
  std::vector<unsigned char> mat;
};

// Scratch bytes run_kraus_sweep needs.
size_t kraus_scratch_bytes();

// One read-write sweep in place: the operators of ops, in order, each a 2^k matvec on its physical bits.  When nb > 0
// it also accumulates rho[a][b] = sum_r psi'(r, a) conj(psi'(r, b)) of the stored amplitudes, bit i of a and b the
// value of physical bit bpos[i], into rho (2^nb x 2^nb, interleaved re/im; the lower triangle the conjugate of the
// upper one, the diagonal's imaginary part 0.0, as run_reduced_density writes it) and synchronises the stream.
// Launches 1 kernel, or 2 with nb > 0.
cudaError_t run_kraus_sweep(qip_prec prec, void *psi, uint32_t n, const std::vector<KrausApplyOp> &ops,
                            const uint32_t *bpos, uint32_t nb, double *rho, void *d_scratch, cudaStream_t s,
                            uint64_t *launches);

}  // namespace qipb200
