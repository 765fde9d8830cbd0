// kernels.cuh -- launch interface of the sm_90a gate kernels (see kernels.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "opcompile.h"

namespace qipb200 {

static const int kMaxIns = 12;      // max bit positions removed from the work-item counter
static const int kMaxRegK = 4;      // largest dense block handled in registers
static const int kMaxDiagParamK = 4; // largest diagonal table passed by kernel parameter

// Launch helpers.  `psi` is the device buffer of the (local) state with 2^n_local
// amplitudes, interleaved (re,im) of R.  All return cudaError_t of the launch and
// add the number of kernels launched to *launches.
cudaError_t launch_dense(qip_prec prec, void *psi, uint32_t n_local, const FlatOp &f, cudaStream_t s,
                         uint64_t *launches);
cudaError_t launch_diag(qip_prec prec, void *psi, uint32_t n_local, uint64_t ctrl_mask,
                        const std::vector<uint32_t> &bits, const std::vector<cplx> &d, cudaStream_t s,
                        uint64_t *launches);
// Dense blocks on 5..10 target bits, in place (k = 5: groups in registers, matrix in shared memory; k >= 6: staged
// through shared memory, matrix through L1/L2), and diagonals on 5..10 bits (table in shared memory).
cudaError_t launch_dense_wide(qip_prec prec, void *psi, uint32_t n_local, const FlatOp &f, cudaStream_t s,
                              uint64_t *launches);
// The kernel launch_dense_wide runs for `f`: DENSE_WIDE_DMMA (k_dense_dmma), DENSE_WIDE_5 (k_dense5) or
// DENSE_WIDE_BIG (k_dense_big).
enum DenseWideKind { DENSE_WIDE_DMMA, DENSE_WIDE_5, DENSE_WIDE_BIG };
DenseWideKind dense_wide_kind(qip_prec prec, uint32_t n_local, const FlatOp &f);
cudaError_t launch_diag_wide(qip_prec prec, void *psi, uint32_t n_local, uint64_t ctrl_mask,
                             const std::vector<uint32_t> &bits, const std::vector<cplx> &d, cudaStream_t s,
                             uint64_t *launches);
cudaError_t launch_flip(qip_prec prec, void *psi, uint32_t n_local, uint64_t ctrl_mask, uint32_t tbit,
                        cudaStream_t s, uint64_t *launches);
cudaError_t launch_bitswap(qip_prec prec, void *psi, uint32_t n_local, uint64_t ctrl_mask, uint32_t p,
                           uint32_t q, cudaStream_t s, uint64_t *launches);

// Universal out-of-place row kernel with the reference's exact semantics
// (apply_op_row_indices, qip-iterators/src/matrix_ops.rs:62-94), offsets and
// accumulate mode included.  Device copies of the matrix / CSR are made with
// stream-ordered allocations.
cudaError_t launch_gather(qip_prec prec, const FlatOp &f, uint32_t n_qubits, const void *in,
                          uint64_t in_len, uint64_t in_off, void *out, uint64_t out_len,
                          uint64_t out_off, bool accumulate, cudaStream_t s, uint64_t *launches);
// apply_ops with several ops as the reference computes it (multi-op row iterator, accumulating; 2..8 ops).
cudaError_t launch_multi_gather(qip_prec prec, const std::vector<FlatOp> &fs, const void *in, uint64_t in_len, uint64_t in_off,
                                void *out, uint64_t out_len, uint64_t out_off, cudaStream_t s, uint64_t *launches);

// sum |a|^2 into *d_out (a device double, zeroed by the launcher).
cudaError_t launch_norm2(qip_prec prec, const void *psi, uint64_t len, double *d_out, cudaStream_t s,
                         uint64_t *launches);
// max over amplitudes of max(|re_a-re_b|, |im_a-im_b|) into *d_out (a device double).
cudaError_t launch_max_abs_diff(qip_prec prec, const void *a, const void *b, uint64_t len, double *d_out, cudaStream_t s,
                                uint64_t *launches);
cudaError_t launch_set_basis(qip_prec prec, void *psi, uint64_t len, uint64_t index, bool owns_index,
                             cudaStream_t s, uint64_t *launches);
// The same state written with memsets only (no kernel): psi[index] = 1 + 0i, every other amplitude 0.
cudaError_t write_basis_state(qip_prec prec, void *psi, uint64_t len, uint64_t index, cudaStream_t s);

// Measurement (qip/src/state_ops/measurement_ops.rs).
// hist[m] += sum of |a|^2 over amplitudes whose bits at bitpos[i] spell m (bit i of m <-> bitpos[i]).
cudaError_t launch_measure_probs(qip_prec prec, const void *psi, uint64_t len, uint64_t index_base,
                                 const uint32_t *bitpos, uint32_t n_bits, double *d_hist, cudaStream_t s,
                                 uint64_t *launches);
// per-chunk sums of |a|^2 (chunk = 2^chunk_log2 amplitudes) for inverse-CDF sampling.
cudaError_t launch_chunk_sums(qip_prec prec, const void *psi, uint64_t len, uint32_t chunk_log2,
                              double *d_sums, cudaStream_t s, uint64_t *launches);
// Sampling (qipb200_state_sample): n_draws independent soft_measure draws (measurement_ops.rs:153-176) on an
// unsharded state in canonical layout, which is not modified.  One read sweep of per-chunk sums (chunks of
// 2^sample_chunk_log2(n_local) amplitudes), a chunk-level CDF, then a second read of only the chunks some draw landed
// in.  d_out[k] gets bits bitpos[i] of draw k's index at bit i.  The number of kernels does not depend on n_draws.
struct SampleBits {
  uint32_t n_bits;
  uint32_t bitpos[64];
};
uint32_t sample_chunk_log2(uint32_t n_local);
// bytes of the device scratch launch_sample needs (one allocation, 16-byte aligned)
size_t sample_scratch_bytes(uint32_t n_local, uint64_t n_draws);
cudaError_t launch_sample(qip_prec prec, const void *psi, uint32_t n_local, const double *d_draws, uint64_t n_draws,
                          const SampleBits &bits, void *d_scratch, uint64_t *d_out, int sm_count, cudaStream_t s,
                          uint64_t *launches);
const uint32_t kSampleLaunches = 10;  // the kernels one launch_sample launches, whatever n_draws
// measure (qipb200_state_measure): the outcome m of one draw and its probability p, as one device record.
// d_draw != nullptr: m is launch_sample's result for that draw; else m must already be in d_rec (a forced outcome)
// and one read sweep computes the chunk sums.  p is summed in a fixed order from the chunk sums of the chunks whose
// high bits match m, re-reading those chunks only when some measured bit lies below sample_chunk_log2.  The number
// of kernels depends on nothing but d_draw.
struct MeasureRecord {
  uint64_t m;
  double p;
};
size_t measure_scratch_bytes(uint32_t n_local);
cudaError_t launch_measure(qip_prec prec, const void *psi, uint32_t n_local, const double *d_draw,
                           const SampleBits &bits, void *d_scratch, MeasureRecord *d_rec, int sm_count, cudaStream_t s,
                           uint64_t *launches);
// measure_state: zero where (index & row_mask) != measured_mask, else scale by p_mult.
cudaError_t launch_collapse(qip_prec prec, void *psi, uint64_t len, uint64_t index_base,
                            uint64_t row_mask, uint64_t measured_mask, double p_mult, cudaStream_t s,
                            uint64_t *launches);

}  // namespace qipb200
