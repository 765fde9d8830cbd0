// opcompile.h -- host-side validation and normalisation of a qip_op tree.
//
// Pure C++ (no CUDA): turns the borrowed C descriptor into a self-contained
// FlatOp (controls flattened, qubit numbers turned into index-bit positions,
// sparse rows densified when small) and classifies it so the launcher can pick
// an in-place kernel.  Semantics follow the reference's row iterators
// (qip-iterators/src/iterators/ops.rs:100-156, qubit_iterators.rs:8-219) and
// constructors (qip/src/state_ops/matrix_ops.rs:12-122).
#pragma once

#include <complex>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/qipb200.h"

namespace qipb200 {

typedef std::complex<double> cplx;

// Largest k for which a sparse op is expanded to a dense 2^k x 2^k matrix.
static const uint32_t kMaxDensifyK = 6;
// Largest dense k accepted at all (device matrix is 4^k complex).
static const uint32_t kMaxDenseK = 10;

enum OpClass {
  CLASS_IDENTITY = 0,  // nothing to do
  CLASS_DIAGONAL,      // diag over diag_bits, controls in ctrl_mask
  CLASS_FLIP,          // X on one bit (exact pair exchange), controls in ctrl_mask
  CLASS_BITSWAP,       // exchange of index-bit pairs (Swap), controls in ctrl_mask
  CLASS_DENSE,         // general dense block on tgt_sorted bits, controls in ctrl_mask
  CLASS_GENERAL        // anything else: out-of-place row-gather kernel
};

struct FlatOp {
  // ---- as given (reference order) ----
  int base_kind = QIP_OP_MATRIX;     // kind of the innermost non-control op
  uint32_t n = 0;                    // qubits of the state the op was compiled for
  uint32_t k = 0;                    // len(outer indices) = nc + kop
  uint32_t nc = 0;                   // total control count (nested controls summed)
  uint32_t kop = 0;                  // index count of the innermost op
  std::vector<uint32_t> idx_bits;    // index-bit position n-1-q of every outer index, reference order
  std::vector<cplx> dense;           // MATRIX (or densified SPARSE): 4^kop, row-major, reference order
  std::vector<uint64_t> sp_rowptr, sp_col;
  std::vector<cplx> sp_val;          // SPARSE kept as CSR when kop > kMaxDensifyK
  bool has_dense = false;

  // ---- normalised (for the in-place kernels) ----
  OpClass cls = CLASS_GENERAL;
  uint64_t ctrl_mask = 0;            // OR of control bit positions (incl. promoted diagonal bits)
  std::vector<uint32_t> tgt_sorted;  // target bit positions, ascending
  std::vector<cplx> m_sorted;        // dense block re-indexed so sub-index bit i <-> tgt_sorted[i]
  std::vector<uint32_t> diag_bits;   // CLASS_DIAGONAL: remaining target bits, ascending (may be empty)
  std::vector<cplx> diag;            // CLASS_DIAGONAL: 2^len(diag_bits) entries, bit i <-> diag_bits[i]
  std::vector<std::pair<uint32_t, uint32_t>> swaps;  // CLASS_BITSWAP: bit pairs to exchange
};

// Validate + flatten.  Returns QIPB200_OK or an error status with `err` set.
// `phys_of_logical` (n_qubits entries, or NULL for identity) maps logical index bit
// n-1-q to the physical bit it currently occupies (multi-GPU qubit migration).
int compile_op(const qip_op *op, qip_prec prec, uint32_t n_qubits, FlatOp *out, std::string *err,
               const uint32_t *phys_of_logical = nullptr);

// Restrict a compiled op (physical bits, non-diagonal targets all below n_local) to rank `rank` of a state sharded by
// the index bits >= n_local: controls held by the rank index either vanish or switch the op off; diagonal bits held by
// the rank index select a slice of the diagonal.  *skip = true when the op is the identity on that rank.
void restrict_flat_op(const FlatOp &f_in, uint32_t n_local, int rank, FlatOp *out, bool *skip);

// Validation only (what the reference's make_*_op constructors check + index range/distinctness).
int validate_op(const qip_op *op, qip_prec prec, uint32_t n_qubits, std::string *err);

}  // namespace qipb200

// The collapse of measure_state (measurement_ops.rs:220-269) as ordinary gates: one one-qubit diagonal QIP_OP_MATRIX
// per measured qubit, diag(1, 0) where bit i of `measured` is 0 and diag(0, 1) where it is 1, the first op carrying
// p_mult in place of its 1.  Their product zeroes the contradicting amplitudes and scales the others by p_mult, so a
// fused schedule can apply a collapse inside its first tile pass.  ops[i] borrows qubits[i] and 4 complex<prec> of
// `dense` (4 * n_qubits entries, written here); both must outlive the ops.  extern "C": the CPU planner tests call
// this construction itself.
extern "C" void qipb200_collapse_ops(qip_prec prec, const uint64_t *qubits, uint32_t n_qubits, uint64_t measured,
                                     double p_mult, qip_op *ops, void *dense);
