// opcompile.cpp -- see opcompile.h.  Host-only; no CUDA, no amplitudes.
#include "opcompile.h"

#include <algorithm>
#include <cstdio>
#include <cstring>

namespace qipb200 {

namespace {

std::string fmt(const char *f, unsigned long long a = 0, unsigned long long b = 0) {
  char buf[256];
  snprintf(buf, sizeof(buf), f, a, b);
  return std::string(buf);
}

int fail(std::string *err, int status, const std::string &msg) {
  if (err) *err = msg;
  return status;
}

cplx load_c(const void *p, qip_prec prec, uint64_t i) {
  if (prec == QIP_F32) {
    const float *f = static_cast<const float *>(p);
    return cplx(f[2 * i], f[2 * i + 1]);
  }
  const double *d = static_cast<const double *>(p);
  return cplx(d[2 * i], d[2 * i + 1]);
}

bool is_zero(const cplx &c) { return c.real() == 0.0 && c.imag() == 0.0; }
bool is_one(const cplx &c) { return c.real() == 1.0 && c.imag() == 0.0; }

}  // namespace

// Checks of the reference constructors (qip/src/state_ops/matrix_ops.rs):
//   make_matrix_op :12-27, make_sparse_matrix_op :32-59, make_swap_op :84-100,
//   make_control_op :103-108; plus index range/distinctness (an out-of-range index
//   panics in the reference's get_bit/slice indexing, a repeated one silently
//   aliases bits -- both are rejected here).
int validate_op(const qip_op *op, qip_prec prec, uint32_t n_qubits, std::string *err) {
  if (prec != QIP_F32 && prec != QIP_F64)
    return fail(err, QIPB200_ERR_INVALID_ARG, "precision must be QIP_F32 or QIP_F64");
  if (!op) return fail(err, QIPB200_ERR_INVALID_ARG, "op is NULL");
  if (n_qubits == 0 || n_qubits > 48)
    return fail(err, QIPB200_ERR_INVALID_ARG, fmt("n_qubits=%llu out of range [1,48]", n_qubits));
  if (op->kind < QIP_OP_MATRIX || op->kind > QIP_OP_CONTROL)
    return fail(err, QIPB200_ERR_INVALID_ARG, fmt("unknown op kind %llu", (unsigned)op->kind));
  if (op->n_indices == 0 || !op->indices) {
    if (op->kind == QIP_OP_SWAP)
      return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Need at least 1 swap index for a and b");
    return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Must supply at least one op index");
  }
  const uint32_t k = op->n_indices;
  if (k > n_qubits)
    return fail(err, QIPB200_ERR_BAD_INDEX, fmt("op has %llu indices but the state has %llu qubits", k, n_qubits));
  uint64_t seen = 0;
  for (uint32_t j = 0; j < k; ++j) {
    const uint64_t q = op->indices[j];
    if (q >= n_qubits)
      return fail(err, QIPB200_ERR_BAD_INDEX, fmt("qubit index %llu out of range for n=%llu", q, n_qubits));
    if (seen & (1ull << q))
      return fail(err, QIPB200_ERR_BAD_INDEX, fmt("qubit index %llu appears more than once", q));
    seen |= 1ull << q;
  }
  // walk the control chain
  const qip_op *cur = op;
  uint32_t kop = k;
  int depth = 0;
  while (cur->kind == QIP_OP_CONTROL) {
    if (cur->n_control == 0)
      return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Must supply at least one control index");
    if (!cur->inner) return fail(err, QIPB200_ERR_INVALID_ARG, "Control op without inner op");
    if (cur->n_control >= cur->n_indices)
      return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Control op leaves no indices for the inner op");
    if (cur->inner->n_indices != cur->n_indices - cur->n_control)
      return fail(err, QIPB200_ERR_SIZE_MISMATCH,
                  fmt("Control op: inner op has %llu indices, expected %llu", cur->inner->n_indices,
                      cur->n_indices - cur->n_control));
    if (++depth > 32) return fail(err, QIPB200_ERR_INVALID_ARG, "Control ops nested too deeply");
    kop = cur->n_indices - cur->n_control;
    cur = cur->inner;
    if (cur->kind < QIP_OP_MATRIX || cur->kind > QIP_OP_CONTROL)
      return fail(err, QIPB200_ERR_INVALID_ARG, fmt("unknown inner op kind %llu", (unsigned)cur->kind));
  }
  if (kop == 0) return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Must supply at least one op index");
  switch (cur->kind) {
    case QIP_OP_MATRIX: {
      if (!cur->dense) return fail(err, QIPB200_ERR_INVALID_ARG, "Matrix op without data");
      if (kop > kMaxDenseK)
        return fail(err, QIPB200_ERR_UNSUPPORTED,
                    fmt("dense op on %llu qubits exceeds the supported maximum of %llu", kop, kMaxDenseK));
      if (cur->n_entries != (1ull << (2 * kop)))
        return fail(err, QIPB200_ERR_SIZE_MISMATCH,
                    fmt("Matrix data has %llu entries versus expected 2^2*%llu", cur->n_entries, kop));
      break;
    }
    case QIP_OP_SPARSE: {
      // the row count is checked BEFORE sp_rowptr is touched: a record with n_rows = 0 (e.g. from a parsed,
      // untrusted schedule) owns a one-element rowptr
      if (!cur->sp_rowptr) return fail(err, QIPB200_ERR_INVALID_ARG, "Sparse op without data");
      if (kop > 20) return fail(err, QIPB200_ERR_UNSUPPORTED, "sparse op on more than 20 qubits");
      if (cur->n_entries != (1ull << kop))
        return fail(err, QIPB200_ERR_SIZE_MISMATCH,
                    fmt("Sparse matrix has %llu rows versus expected 2^%llu", cur->n_entries, kop));
      if (!cur->sp_col && cur->sp_rowptr[0] != cur->sp_rowptr[1])
        return fail(err, QIPB200_ERR_INVALID_ARG, "Sparse op without data");
      for (uint64_t r = 0; r < (1ull << kop); ++r) {
        if (cur->sp_rowptr[r + 1] <= cur->sp_rowptr[r])
          return fail(err, QIPB200_ERR_SIZE_MISMATCH,
                      fmt("All rows of sparse matrix must have data (%llu is empty)", r));
        for (uint64_t e = cur->sp_rowptr[r]; e < cur->sp_rowptr[r + 1]; ++e)
          if (cur->sp_col[e] >= (1ull << kop))
            return fail(err, QIPB200_ERR_BAD_INDEX, fmt("sparse column %llu out of range in row %llu", cur->sp_col[e], r));
      }
      if (!cur->sp_val) return fail(err, QIPB200_ERR_INVALID_ARG, "Sparse op without values");
      break;
    }
    case QIP_OP_SWAP: {
      if (kop < 2) return fail(err, QIPB200_ERR_SIZE_MISMATCH, "Need at least 1 swap index for a and b");
      if (kop & 1)
        return fail(err, QIPB200_ERR_SIZE_MISMATCH,
                    fmt("Swap must be performed on two sets of indices of equal length, found %llu vs %llu",
                        (kop + 1) / 2, kop / 2));
      break;
    }
    default:
      return fail(err, QIPB200_ERR_INVALID_ARG, "malformed op tree");
  }
  return QIPB200_OK;
}

// Re-index a dense block from the reference's sub-index order (indices[0] = MSB,
// matrix_ops.rs:12-30) to "sorted" order where sub-index bit i <-> i-th smallest
// target bit position.  The data is permuted on the host instead of the state.
static void sort_block(const std::vector<uint32_t> &tgt_ref_bits, const std::vector<cplx> &m_ref,
                       std::vector<uint32_t> *tgt_sorted, std::vector<cplx> *m_sorted) {
  const uint32_t k = (uint32_t)tgt_ref_bits.size();
  std::vector<uint32_t> order(k);
  for (uint32_t i = 0; i < k; ++i) order[i] = i;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return tgt_ref_bits[a] < tgt_ref_bits[b]; });
  tgt_sorted->resize(k);
  for (uint32_t i = 0; i < k; ++i) (*tgt_sorted)[i] = tgt_ref_bits[order[i]];
  const uint64_t side = 1ull << k;
  std::vector<uint64_t> to_ref(side);
  for (uint64_t u = 0; u < side; ++u) {
    uint64_t r = 0;
    for (uint32_t i = 0; i < k; ++i)
      if ((u >> i) & 1) r |= 1ull << (k - 1 - order[i]);  // reference position j=order[i] <-> sub bit k-1-j
    to_ref[u] = r;
  }
  m_sorted->resize(side * side);
  for (uint64_t u = 0; u < side; ++u)
    for (uint64_t v = 0; v < side; ++v) (*m_sorted)[u * side + v] = m_ref[to_ref[u] * side + to_ref[v]];
}

int compile_op(const qip_op *op, qip_prec prec, uint32_t n_qubits, FlatOp *out, std::string *err,
               const uint32_t *phys_of_logical) {
  int st = validate_op(op, prec, n_qubits, err);
  if (st != QIPB200_OK) return st;
  FlatOp &f = *out;
  f = FlatOp();
  f.n = n_qubits;
  f.k = op->n_indices;
  f.idx_bits.resize(f.k);
  for (uint32_t j = 0; j < f.k; ++j) {
    const uint32_t logical = n_qubits - 1 - (uint32_t)op->indices[j];  // matrix_ops.rs:18
    f.idx_bits[j] = phys_of_logical ? phys_of_logical[logical] : logical;
  }
  const qip_op *cur = op;
  f.kop = f.k;
  while (cur->kind == QIP_OP_CONTROL) {  // ops.rs:111-115,147-153: nested controls add up
    f.nc += cur->n_control;
    f.kop = cur->n_indices - cur->n_control;
    cur = cur->inner;
  }
  if (f.nc + f.kop != f.k)
    return fail(err, QIPB200_ERR_SIZE_MISMATCH, "nested Control ops: control counts do not add up to the index count");
  f.base_kind = cur->kind;
  const uint64_t side = 1ull << f.kop;
  if (cur->kind == QIP_OP_MATRIX) {
    f.dense.resize(side * side);
    for (uint64_t i = 0; i < side * side; ++i) f.dense[i] = load_c(cur->dense, prec, i);
    f.has_dense = true;
  } else if (cur->kind == QIP_OP_SPARSE) {
    const uint64_t nnz = cur->sp_rowptr[side];
    if (f.kop <= kMaxDensifyK) {
      // Densify: duplicate columns of a row are summed in stored order.
      f.dense.assign(side * side, cplx(0, 0));
      for (uint64_t r = 0; r < side; ++r)
        for (uint64_t e = cur->sp_rowptr[r]; e < cur->sp_rowptr[r + 1]; ++e)
          f.dense[r * side + cur->sp_col[e]] += load_c(cur->sp_val, prec, e);
      f.has_dense = true;
    } else {
      f.sp_rowptr.assign(cur->sp_rowptr, cur->sp_rowptr + side + 1);
      f.sp_col.assign(cur->sp_col, cur->sp_col + nnz);
      f.sp_val.resize(nnz);
      for (uint64_t e = 0; e < nnz; ++e) f.sp_val[e] = load_c(cur->sp_val, prec, e);
    }
  }

  // ---- classification -------------------------------------------------------
  for (uint32_t j = 0; j < f.nc; ++j) f.ctrl_mask |= 1ull << f.idx_bits[j];
  std::vector<uint32_t> tgt_ref(f.idx_bits.begin() + f.nc, f.idx_bits.end());

  if (f.base_kind == QIP_OP_SWAP) {
    // Swap(m, a ++ b): sub-index [a|b] <- column [b|a] (qubit_iterators.rs:208-218):
    // m independent exchanges of index bits a_j <-> b_j.
    const uint32_t m = f.kop / 2;
    for (uint32_t j = 0; j < m; ++j) {
      uint32_t p = tgt_ref[j], q = tgt_ref[m + j];
      f.swaps.push_back(std::make_pair(std::min(p, q), std::max(p, q)));
    }
    f.cls = CLASS_BITSWAP;
    return QIPB200_OK;
  }
  if (!f.has_dense) {
    f.cls = CLASS_GENERAL;
    return QIPB200_OK;
  }
  sort_block(tgt_ref, f.dense, &f.tgt_sorted, &f.m_sorted);

  bool diagonal = true, identity = true;
  for (uint64_t u = 0; u < side && diagonal; ++u)
    for (uint64_t v = 0; v < side; ++v) {
      const cplx &c = f.m_sorted[u * side + v];
      if (u != v && !is_zero(c)) {
        diagonal = false;
        identity = false;
        break;
      }
      if (u == v && !is_one(c)) identity = false;
    }
  if (identity) {
    f.cls = CLASS_IDENTITY;
    return QIPB200_OK;
  }
  if (diagonal) {
    // Promote every bit whose "0" half of the diagonal is exactly 1 to a control:
    // diag(1, w) on t == phase w where bit t is set (the reference multiplies by
    // exactly 1 there: same values).  T, S, Z, CZ, controlled phases all reduce to
    // a scalar on a bit mask.
    std::vector<uint32_t> bits = f.tgt_sorted;
    std::vector<cplx> d(side);
    for (uint64_t u = 0; u < side; ++u) d[u] = f.m_sorted[u * side + u];
    bool changed = true;
    while (changed && !bits.empty()) {
      changed = false;
      for (size_t i = 0; i < bits.size(); ++i) {
        bool ones = true;
        for (uint64_t u = 0; u < d.size(); ++u)
          if (!((u >> i) & 1) && !is_one(d[u])) {
            ones = false;
            break;
          }
        if (!ones) continue;
        std::vector<cplx> nd;
        for (uint64_t u = 0; u < d.size(); ++u)
          if ((u >> i) & 1) nd.push_back(d[u]);  // keeps relative bit order of the others
        f.ctrl_mask |= 1ull << bits[i];
        bits.erase(bits.begin() + i);
        d.swap(nd);
        changed = true;
        break;
      }
    }
    f.diag_bits = bits;
    f.diag = d;
    f.cls = CLASS_DIAGONAL;
    return QIPB200_OK;
  }
  if (f.kop == 1 && is_zero(f.m_sorted[0]) && is_zero(f.m_sorted[3]) && is_one(f.m_sorted[1]) &&
      is_one(f.m_sorted[2])) {
    f.cls = CLASS_FLIP;  // X (CNOT / Toffoli with controls): exact index permutation
    return QIPB200_OK;
  }
  f.cls = CLASS_DENSE;
  return QIPB200_OK;
}

void restrict_flat_op(const FlatOp &f_in, uint32_t n_local, int rank, FlatOp *out, bool *skip) {
  const uint32_t nl = n_local;
  const uint64_t lo_mask = (nl >= 64) ? ~0ull : ((1ull << nl) - 1ull);
  const uint64_t rank_val = (uint64_t)rank << nl;
  *skip = false;
  *out = f_in;
  if (f_in.cls == CLASS_IDENTITY) {
    *skip = true;
    return;
  }
  const uint64_t hc = f_in.ctrl_mask & ~lo_mask;
  if ((rank_val & hc) != hc) {  // a control held by the rank index is 0 here
    *skip = true;
    return;
  }
  out->ctrl_mask = f_in.ctrl_mask & lo_mask;
  if (f_in.cls == CLASS_DIAGONAL) {
    std::vector<cplx> d = f_in.diag;
    std::vector<uint32_t> all = f_in.diag_bits;
    for (int i = (int)all.size() - 1; i >= 0; --i) {  // highest first keeps indices valid
      if (all[i] < nl) continue;
      const int v = (int)((rank_val >> all[i]) & 1ull);
      std::vector<cplx> nd;
      for (uint64_t u = 0; u < d.size(); ++u)
        if ((int)((u >> i) & 1) == v) nd.push_back(d[u]);
      d.swap(nd);
      all.erase(all.begin() + i);
    }
    bool all_one = true;
    for (size_t u = 0; u < d.size(); ++u)
      if (!(d[u].real() == 1.0 && d[u].imag() == 0.0)) all_one = false;
    if (all_one) {
      *skip = true;
      return;
    }
    out->diag_bits = all;
    out->diag = d;
  }
}

}  // namespace qipb200

extern "C" void qipb200_collapse_ops(qip_prec prec, const uint64_t *qubits, uint32_t n_qubits, uint64_t measured,
                                     double p_mult, qip_op *ops, void *dense) {
  for (uint32_t i = 0; i < n_qubits; ++i) {
    const uint64_t bit = (measured >> i) & 1ull;
    const double keep = i == 0 ? p_mult : 1.0;
    const double re[4] = {bit ? 0.0 : keep, 0.0, 0.0, bit ? keep : 0.0};  // row-major 2x2
    for (int j = 0; j < 4; ++j) {
      if (prec == QIP_F32) {
        float *d = static_cast<float *>(dense) + 8 * i + 2 * j;
        d[0] = (float)re[j];
        d[1] = 0.0f;
      } else {
        double *d = static_cast<double *>(dense) + 8 * i + 2 * j;
        d[0] = re[j];
        d[1] = 0.0;
      }
    }
    qip_op &op = ops[i];
    memset(&op, 0, sizeof(op));
    op.kind = QIP_OP_MATRIX;
    op.n_indices = 1;
    op.n_entries = 4;
    op.indices = qubits + i;
    op.dense = prec == QIP_F32 ? (const void *)(static_cast<float *>(dense) + 8 * i)
                               : (const void *)(static_cast<double *>(dense) + 8 * i);
  }
}
