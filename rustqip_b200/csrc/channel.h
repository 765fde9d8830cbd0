// channel.h -- one quantum-trajectory step of single-qubit noise channels whose Kraus operators are diagonal or
// anti-diagonal (qipb200_state_apply_channels): the host-side parsing, choice and tables, and the two sweep kernels of
// channel.cu.  See channel.cu for the sampling argument and the arithmetic.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/qipb200.h"

namespace qipb200 {

const uint32_t kChanMaxKraus = 16;   // operators per channel
const uint32_t kChanMaxTables = 5;   // bytes of a physical index of at most 40 bits
const int kChanThreads = 256;        // both kernels
const int kChanWeightGrid = 264;     // weight: fixed grid, so the sum order does not depend on the device
const int kChanPer = 8;              // weight: amplitudes per thread and chunk
const double kChanCompleteTol = 1e-12;

// One Kraus operator K: K|b> = d[b] |b ^ flip>.
struct ChannelOp {
  double d[2][2];  // d[b] = (re, im): the nonzero entry of column b (0 when the column is zero)
  double e[2];     // |d[b]|^2 = re^2 + im^2 in double
  bool flip;       // anti-diagonal
};

struct ChannelSet {
  std::vector<uint64_t> qubits;
  std::vector<uint32_t> first;  // channel c's operators are ops[first[c] .. first[c + 1])
  std::vector<ChannelOp> ops;
  std::vector<uint8_t> dep;     // state-dependent: some operator has e[0] != e[1]
  uint32_t n_dep = 0;
};

// Validate n_channels channels of an n-qubit state (the rules of include/qipb200.h) into *out.  Returns
// QIPB200_OK, or the status with the message (prefixed by who) in *err.
int parse_channels(const std::string &who, uint32_t n, size_t n_channels, const uint64_t *qubits,
                   const uint32_t *n_kraus, const double *kraus, ChannelSet *out, std::string *err);

// The operator of channel c chosen with the uniform u for channel-qubit value b (an index into c's operators).
uint32_t channel_choose(const ChannelSet &cs, size_t c, uint32_t b, double u);

// K is a positive real multiple of the identity.
bool channel_op_is_scaled_identity(const ChannelOp &k);

// out4 = {state-dependent channels, read sweeps at most, read-write sweeps at most, kernels at most} on an unsharded
// n-qubit state with nothing pending.
void plan_channels(const ChannelSet &cs, uint32_t out4[4]);

// The per-byte tables of a product of chosen operators on distinct physical bits: table t covers index byte
// byte[t] (bytes without a channel bit are skipped), built on the host in double, bits in ascending order.
struct ChannelTables {
  uint32_t n_tab = 0;
  uint32_t byte[kChanMaxTables];
  std::vector<double2> d;  // n_tab x 256: product of d over the byte's channel bits (complex, no FMA)
  std::vector<double> e;   // n_tab x 256: product of |d|^2 over the byte's channel bits
  uint64_t flip = 0;       // F: the XOR mask of the anti-diagonal operators
};
void build_channel_tables(const uint32_t *pos, const ChannelOp *const *ops, size_t k, ChannelTables *t);

// Read sweep: *S = sum_j |psi_j|^2 prod |d(bits of j)|^2 and *N = sum_j |psi_j|^2, deterministic.  d_partials holds
// 2 kChanWeightGrid doubles.  Synchronises s.
cudaError_t run_channel_weight(qip_prec prec, const void *psi, uint32_t n, const ChannelTables &t, void *d_scratch,
                               cudaStream_t s, uint64_t *launches, double *S, double *N);
// Bytes of device scratch run_channel_weight and run_channel_apply need.
size_t channel_scratch_bytes();

// Read-write sweep in place: psi'_{j ^ F} = W(j) psi_j with W(j) = RN(prod_t d_t[byte(j)] * inv).
cudaError_t run_channel_apply(qip_prec prec, void *psi, uint32_t n, const ChannelTables &t, double inv,
                              void *d_scratch, int sm_count, cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
