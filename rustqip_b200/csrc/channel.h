// channel.h -- one quantum-trajectory step of noise channels on up to four qubits whose Kraus operators have the form
// K|b> = d(b)|b ^ f> (qipb200_state_apply_channels, qipb200_state_apply_multiqubit_channels): the host-side parsing,
// choice and tables, and the two sweep kernels of channel.cu.  See channel.cu for the sampling argument and the arithmetic.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/qipb200.h"

namespace qipb200 {

const uint32_t kChanMaxKraus = 16;          // operators per channel of qipb200_state_apply_channels
const uint32_t kChanMaxKrausMulti = 256;    // operators per channel of qipb200_state_apply_multiqubit_channels
const uint32_t kChanMaxArity = 4;           // qubits per channel
const uint32_t kChanMaxTables = 5;          // bytes of a physical index of at most 40 bits
const uint32_t kChanMaxGather = 20;         // gathered tables: each channel has at least 2 of the at most 40 bits
const uint32_t kChanMaxGatherEntries = 160; // their entries: 2^k for k bits, at most 4 per bit
const int kChanThreads = 256;               // both kernels
const int kChanWeightGrid = 264;            // weight: fixed grid, so the sum order does not depend on the device
const int kChanPer = 8;                     // weight: amplitudes per thread and chunk
const double kChanCompleteTol = 1e-12;

// One Kraus operator K on k qubits: K|b> = d[b] |b ^ f>, b and f in the matrix convention (the channel's first qubit
// is the most significant bit of b).
struct ChannelOp {
  uint32_t k;          // qubits
  uint32_t f;          // the XOR mask (k = 1: anti-diagonal)
  double d[16][2];     // d[b] = (re, im): the nonzero entry of column b (0 when the column is zero)
  double e[16];        // |d[b]|^2 = re^2 + im^2 in double
};

struct ChannelSet {
  std::vector<uint64_t> qubits;  // flat: channel c's qubits are qubits[qfirst[c] .. qfirst[c + 1])
  std::vector<uint32_t> qfirst;
  std::vector<uint32_t> first;   // channel c's operators are ops[first[c] .. first[c + 1])
  std::vector<ChannelOp> ops;
  std::vector<uint8_t> dep;      // state-dependent: some operator has e[b] != e[0]
  uint32_t n_dep = 0;
  size_t size() const { return dep.size(); }
};

// Validate n_channels channels of an n-qubit state (the rules of include/qipb200.h) into *out.  arity == NULL is the
// single-qubit form of qipb200_state_apply_channels (its limit of max_kraus operators and its messages).  Returns
// QIPB200_OK, or the status with the message (prefixed by who) in *err.
int parse_channels(const std::string &who, uint32_t n, size_t n_channels, const uint32_t *arity,
                   const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, uint32_t max_kraus,
                   ChannelSet *out, std::string *err);

// The operator of channel c chosen with the uniform u for channel value b (an index into c's operators).
uint32_t channel_choose(const ChannelSet &cs, size_t c, uint32_t b, double u);

// K is a positive real multiple of the identity.
bool channel_op_is_scaled_identity(const ChannelOp &k);

// out4 = {state-dependent channels, read sweeps at most, read-write sweeps at most, kernels at most} on an unsharded
// n-qubit state with nothing pending.
void plan_channels(const ChannelSet &cs, uint32_t out4[4]);

// The tables of a product of chosen operators on distinct physical bits, built on the host in double (complex
// products without FMA).  An operator whose bits all lie in one index byte folds into that byte's 256-entry table
// (factors in the order of their lowest bit); table t covers byte byte[t], ascending, bytes without an operator
// skipped.  Every other operator gets a gathered table of its 2^k values d[b], b gathered from its physical bits in
// the matrix convention, in operator order.  W(j) multiplies the byte tables, then the gathered ones.
struct ChannelTables {
  uint32_t n_tab = 0;
  uint32_t byte[kChanMaxTables];
  uint32_t n_gat = 0;
  uint32_t gat[kChanMaxGather];  // the physical bit of the operator's qubit i in bits 6i..6i+5, k - 1 in bits 24..25
  std::vector<double2> d;        // n_tab x 256 byte entries, then 2^k per gathered table: products of d
  std::vector<double> e;         // the same layout: products of |d|^2
  uint64_t flip = 0;             // F: the XOR of the operators' masks on their physical bits
};
// ops[i] acts on the physical bits pos[o_i .. o_i + ops[i]->k), o_i the sum of the earlier operators' k.
void build_channel_tables(const uint32_t *pos, const ChannelOp *const *ops, size_t m, ChannelTables *t);

// Read sweep: *S = sum_j |psi_j|^2 prod |d(b_c(j))|^2 and *N = sum_j |psi_j|^2, deterministic.  d_partials holds
// 2 kChanWeightGrid doubles.  Synchronises s.
cudaError_t run_channel_weight(qip_prec prec, const void *psi, uint32_t n, const ChannelTables &t, void *d_scratch,
                               cudaStream_t s, uint64_t *launches, double *S, double *N);
// Bytes of device scratch run_channel_weight and run_channel_apply need.
size_t channel_scratch_bytes();

// Read-write sweep in place: psi'_{j ^ F} = W(j) psi_j with W(j) = RN(prod_t T_t[index_t(j)] * inv).
cudaError_t run_channel_apply(qip_prec prec, void *psi, uint32_t n, const ChannelTables &t, double inv,
                              void *d_scratch, int sm_count, cudaStream_t s, uint64_t *launches);

}  // namespace qipb200
