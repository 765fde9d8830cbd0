// qipb200.hpp -- header-only C++ host mirror of the reference's operator interface for the
// gate-application path, on top of the C ABI (include/qipb200.h).
//
// The reference is Rust; this image has no Rust toolchain, so the host side above the C ABI
// is C++ (the reference is compiled code).  Names, argument order and error behaviour follow
// the reference so that call sites read the same:
//
//   qip::MatrixOp<P>                       <- enum MatrixOp<P>            (qip-iterators/src/iterators/ops.rs:11-91)
//   qip::make_matrix_op / make_swap_op /   <- qip::state_ops::matrix_ops  (qip/src/state_ops/matrix_ops.rs:12-122)
//        make_control_op / make_sparse_matrix_op
//   qip::apply_op / apply_op_overwrite /   <- qip_iterators::matrix_ops   (qip-iterators/src/matrix_ops.rs:98-219)
//        apply_ops                            (host slices in, host slices out; executed on the H100)
//   qip::B200State<P>                      <- the two Vec<Complex<P>> of LocalBuilder::calculate_state_with_init
//                                             (qip/src/builder.rs:406-407,423-514): amplitudes stay in HBM between gates
//   qip::CircuitError                      <- qip::errors::CircuitError   (qip/src/errors.rs:6-22)
//
// P is float or double (trait Precision, qip/src/types.rs:6-13).
#pragma once

#include <algorithm>
#include <complex>
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "qipb200.h"

namespace qip {

struct CircuitError : std::runtime_error {
  int status;
  explicit CircuitError(const std::string &msg, int status_ = 0) : std::runtime_error(msg), status(status_) {}
};

template <typename P>
struct Prec;
template <>
struct Prec<float> {
  static constexpr qip_prec value = QIP_F32;
};
template <>
struct Prec<double> {
  static constexpr qip_prec value = QIP_F64;
};

// enum MatrixOp<P> { Matrix(indices, data), SparseMatrix(indices, rows), Swap(n, indices), Control(nc, indices, Box<op>) }
template <typename P>
class MatrixOp {
 public:
  typedef std::complex<P> C;
  enum Kind { Matrix = QIP_OP_MATRIX, SparseMatrix = QIP_OP_SPARSE, Swap = QIP_OP_SWAP, Control = QIP_OP_CONTROL };

  static MatrixOp new_matrix(std::vector<uint64_t> indices, std::vector<C> data) {  // ops.rs:49-55
    MatrixOp op(Matrix);
    op.indices_ = std::move(indices);
    op.data_ = std::move(data);
    return op;
  }
  static MatrixOp new_sparse(std::vector<uint64_t> indices, const std::vector<std::vector<std::pair<uint64_t, C>>> &rows) {
    MatrixOp op(SparseMatrix);  // ops.rs:58-64
    op.indices_ = std::move(indices);
    op.rowptr_.push_back(0);
    for (const auto &row : rows) {
      for (const auto &e : row) {
        op.cols_.push_back(e.first);
        op.vals_.push_back(e.second);
      }
      op.rowptr_.push_back(op.cols_.size());
    }
    return op;
  }
  static MatrixOp new_swap(std::vector<uint64_t> a, const std::vector<uint64_t> &b) {  // ops.rs:67-78
    MatrixOp op(Swap);
    op.swap_n_ = a.size();
    a.insert(a.end(), b.begin(), b.end());
    op.indices_ = std::move(a);
    return op;
  }
  static MatrixOp new_control(std::vector<uint64_t> c, const std::vector<uint64_t> &r, MatrixOp inner) {  // ops.rs:81-91
    MatrixOp op(Control);
    op.n_control_ = (uint32_t)c.size();
    c.insert(c.end(), r.begin(), r.end());
    op.indices_ = std::move(c);
    op.inner_ = std::make_shared<MatrixOp>(std::move(inner));
    return op;
  }

  size_t num_indices() const { return kind_ == Swap ? 2 * swap_n_ : indices_.size(); }  // ops.rs:24-36
  const std::vector<uint64_t> &indices() const { return indices_; }                     // ops.rs:39-46
  Kind kind() const { return kind_; }
  uint32_t n_control() const { return n_control_; }
  const MatrixOp *inner() const { return inner_.get(); }

  // Borrowed C view; valid while *this lives and is not modified.
  const qip_op *c_op() const {
    c_.kind = kind_;
    c_.n_indices = (uint32_t)indices_.size();
    c_.n_control = n_control_;
    c_.reserved = 0;
    c_.n_entries = kind_ == Matrix ? data_.size() : (kind_ == SparseMatrix ? rowptr_.size() - 1 : 0);
    c_.indices = indices_.data();
    c_.dense = data_.empty() ? nullptr : data_.data();
    c_.sp_rowptr = rowptr_.empty() ? nullptr : rowptr_.data();
    c_.sp_col = cols_.empty() ? nullptr : cols_.data();
    c_.sp_val = vals_.empty() ? nullptr : vals_.data();
    c_.inner = inner_ ? inner_->c_op() : nullptr;
    return &c_;
  }

 private:
  explicit MatrixOp(Kind k) : kind_(k) {}
  Kind kind_;
  std::vector<uint64_t> indices_;
  std::vector<C> data_;
  std::vector<uint64_t> rowptr_, cols_;
  std::vector<C> vals_;
  size_t swap_n_ = 0;
  uint32_t n_control_ = 0;
  std::shared_ptr<MatrixOp> inner_;
  mutable qip_op c_{};
};

// ---- qip/src/state_ops/matrix_ops.rs:12-122 (validating constructors) ------------------------
template <typename P>
MatrixOp<P> make_matrix_op(std::vector<uint64_t> indices, std::vector<std::complex<P>> dat) {
  const size_t n = indices.size();
  if (n == 0) throw CircuitError("Must supply at least one op index");
  if (dat.size() != (size_t(1) << (2 * n)))
    throw CircuitError("Matrix data has " + std::to_string(dat.size()) + " entries versus expected 2^2*" + std::to_string(n));
  return MatrixOp<P>::new_matrix(std::move(indices), std::move(dat));
}
template <typename P>
MatrixOp<P> make_swap_op(std::vector<uint64_t> a, std::vector<uint64_t> b) {
  if (a.empty() || b.empty()) throw CircuitError("Need at least 1 swap index for a and b");
  if (a.size() != b.size())
    throw CircuitError("Swap must be performed on two sets of indices of equal length, found " +
                       std::to_string(a.size()) + " vs " + std::to_string(b.size()));
  return MatrixOp<P>::new_swap(std::move(a), b);
}
template <typename P>
MatrixOp<P> make_control_op(std::vector<uint64_t> c, MatrixOp<P> op) {
  if (c.empty()) throw CircuitError("Must supply at least one control index");
  if (op.kind() == MatrixOp<P>::Control) {  // nested controls are flattened (:112-115)
    std::vector<uint64_t> rest(op.indices().begin() + op.n_control(), op.indices().end());
    c.insert(c.end(), op.indices().begin(), op.indices().begin() + op.n_control());
    return MatrixOp<P>::new_control(std::move(c), rest, *op.inner());
  }
  std::vector<uint64_t> r = op.indices();
  return MatrixOp<P>::new_control(std::move(c), r, std::move(op));
}

// ---- context -----------------------------------------------------------------------------------
class Context {
 public:
  explicit Context(int device = 0) {
    int st = qipb200_init(&ctx_, device);
    if (st != QIPB200_OK) throw CircuitError(qipb200_last_error(nullptr), st);  // no CPU fallback
  }
  // ONE context over several devices of this process (a power-of-two count): states created on it are sharded
  // over the devices inside the library -- what a single-process host like LocalBuilder needs to use a whole box
  explicit Context(const std::vector<int> &devices) {
    int st = qipb200_init_multi(&ctx_, (int)devices.size(), devices.data());
    if (st != QIPB200_OK) throw CircuitError(qipb200_last_error(nullptr), st);
  }
  ~Context() { qipb200_shutdown(ctx_); }
  Context(const Context &) = delete;
  Context &operator=(const Context &) = delete;
  qipb200_ctx *get() const { return ctx_; }
  void check(int st) const {
    if (st != QIPB200_OK) throw CircuitError(qipb200_last_error(ctx_), st);
  }

 private:
  qipb200_ctx *ctx_ = nullptr;
};

// ---- qip_iterators::matrix_ops drop-ins (host slices) -------------------------------------------
template <typename P>
void apply_op(Context &ctx, size_t n, const MatrixOp<P> &op, const std::vector<std::complex<P>> &input,
              std::vector<std::complex<P>> &output, size_t input_offset, size_t output_offset) {  // matrix_ops.rs:98-123
  ctx.check(qipb200_apply_op(ctx.get(), Prec<P>::value, (uint32_t)n, op.c_op(), input.data(), input.size(),
                             output.data(), output.size(), input_offset, output_offset));
}
template <typename P>
void apply_op_overwrite(Context &ctx, size_t n, const MatrixOp<P> &op, const std::vector<std::complex<P>> &input,
                        std::vector<std::complex<P>> &output, size_t input_offset, size_t output_offset) {  // :127-152
  ctx.check(qipb200_apply_op_overwrite(ctx.get(), Prec<P>::value, (uint32_t)n, op.c_op(), input.data(), input.size(),
                                       output.data(), output.size(), input_offset, output_offset));
}

// ---- classical functions on the device (FunctionOpIterator, qip-iterators/src/iterators/qubit_iterators.rs:221-271) --
// U|x>|y> = e^{i theta(x)} |x>|y ^ f(x)> for a table of 2^n_in entries, checked and uploaded once; bit i of x is qubit
// in_qubits[i], bit i of f(x) goes to out_qubits[i] (B200State::apply_function).  f may be empty when n_out == 0,
// theta empty for a pure permutation.
//
// B200Function::from_code: the same op for f and theta given as CUDA source (qipb200_function_new_code), compiled with
// NVRTC and evaluated on the device, so n_in may cover the whole state.  A compile error throws with the NVRTC log.
class B200Function {
 public:
  B200Function(Context &ctx, uint32_t n_in, uint32_t n_out, const std::vector<uint64_t> &f,
               const std::vector<double> &theta = {})
      : ctx_(ctx), n_in_(n_in), n_out_(n_out) {
    const size_t size = n_in < 64 ? size_t(1) << n_in : 0;
    if ((!f.empty() && f.size() != size) || (!theta.empty() && theta.size() != size))
      throw CircuitError("B200Function: f and theta need 2^n_in = " + std::to_string(size) + " entries each");
    ctx.check(qipb200_function_new(ctx.get(), n_in, n_out, f.empty() ? nullptr : f.data(),
                                   theta.empty() ? nullptr : theta.data(), &fn_));
  }
  // source defines qip_f (n_out > 0) and, with theta, qip_theta(x, p) over n_params parameters (0 until set_params)
  static B200Function from_code(Context &ctx, uint32_t n_in, uint32_t n_out, const std::string &source,
                                bool theta = false, uint32_t n_params = 0) {
    return B200Function(ctx, n_in, n_out, source, theta, n_params);
  }
  ~B200Function() { qipb200_function_free(fn_); }
  B200Function(const B200Function &) = delete;
  B200Function &operator=(const B200Function &) = delete;
  uint32_t n_in() const { return n_in_; }
  uint32_t n_out() const { return n_out_; }
  const qipb200_function *get() const { return fn_; }
  // code functions: the parameters theta is evaluated with (checked finite for every x; refused: the old ones stay)
  void set_params(const std::vector<double> &params) {
    ctx_.check(qipb200_function_set_params(fn_, params.empty() ? nullptr : params.data(), (uint32_t)params.size()));
  }
  // f(x) and (cos theta(x), sin theta(x)) (interleaved) for x in [x0, x0 + count), evaluated on the device
  void tabulate(uint64_t x0, uint64_t count, std::vector<uint64_t> *f, std::vector<double> *cs) const {
    if (f) f->assign(count, 0);
    if (cs) cs->assign(2 * count, 0.0);
    ctx_.check(qipb200_function_tabulate(fn_, x0, count, f ? f->data() : nullptr, cs ? cs->data() : nullptr));
  }

 private:
  B200Function(Context &ctx, uint32_t n_in, uint32_t n_out, const std::string &source, bool theta, uint32_t n_params)
      : ctx_(ctx), n_in_(n_in), n_out_(n_out) {
    // the NVRTC log of a compile error is in the last error, which check() throws
    ctx.check(qipb200_function_new_code(ctx.get(), n_in, n_out, source.c_str(), theta ? QIPB200_FN_CODE_THETA : 0u,
                                        n_params, nullptr, 0, &fn_));
  }
  Context &ctx_;
  uint32_t n_in_, n_out_;
  qipb200_function *fn_ = nullptr;
};

// ---- device-resident state: the body of LocalBuilder::calculate_state_with_init -------------------
template <typename P>
class B200State {
 public:
  B200State(Context &ctx, size_t n) : ctx_(ctx), n_(n) { ctx_.check(qipb200_state_new(ctx.get(), Prec<P>::value, (uint32_t)n, &st_)); }
  ~B200State() { qipb200_state_free(st_); }
  B200State(const B200State &) = delete;
  B200State &operator=(const B200State &) = delete;

  void set_basis(uint64_t index) { ctx_.check(qipb200_state_set_basis(st_, index)); }  // builder.rs:421
  void apply(const MatrixOp<P> &op) { ctx_.check(qipb200_state_apply_op(st_, op.c_op())); }  // builder.rs:499,514
  void apply_all(const std::vector<MatrixOp<P>> &ops, bool fusion = true) {              // builder.rs:423-514
    std::vector<qip_op> c(ops.size());
    for (size_t i = 0; i < ops.size(); ++i) c[i] = *ops[i].c_op();
    ctx_.check(qipb200_state_apply_schedule(st_, c.data(), c.size(), fusion ? QIPB200_SCHED_DEFAULT : QIPB200_SCHED_NO_FUSION));
  }
  std::vector<std::complex<P>> into_state() {  // builder.rs:518
    std::vector<std::complex<P>> out(size_t(1) << n_);
    ctx_.check(qipb200_state_download(st_, out.data(), 0, out.size()));
    return out;
  }
  double prob_magnitude() {  // measurement_ops.rs:11-13
    double v = 0;
    ctx_.check(qipb200_state_norm2(st_, &v));
    return v;
  }
  uint64_t soft_measure(const std::vector<uint64_t> &indices, double r) {  // measurement_ops.rs:153-176, draw supplied
    uint64_t m = 0;
    ctx_.check(qipb200_state_soft_measure(st_, indices.data(), (uint32_t)indices.size(), r, &m));
    return m;
  }
  // draws.size() soft_measure draws on the uncollapsed state (shots without rerunning the circuit)
  std::vector<uint64_t> sample(const std::vector<uint64_t> &indices, const std::vector<double> &draws) {
    std::vector<uint64_t> m(draws.size());
    ctx_.check(qipb200_state_sample(st_, indices.data(), (uint32_t)indices.size(), draws.data(), draws.size(), m.data()));
    return m;
  }
  // measure (measurement_ops.rs:190-214): draw with r in [0,1), take the probability, collapse; returns (m, p)
  std::pair<uint64_t, double> measure(const std::vector<uint64_t> &indices, double r) {
    uint64_t m = 0;
    double p = 0.0;
    ctx_.check(qipb200_state_measure(st_, indices.data(), (uint32_t)indices.size(), r, 0u, &m, &p));
    return {m, p};
  }
  // ... with a forced outcome, and its probability when known (MeasuredCondition { measured, prob })
  std::pair<uint64_t, double> measure(const std::vector<uint64_t> &indices, uint64_t measured, std::optional<double> prob) {
    uint64_t m = measured;
    double p = prob ? *prob : 0.0;
    const uint32_t flags = QIPB200_MEASURE_FORCED | (prob ? (uint32_t)QIPB200_MEASURE_FORCED_PROB : 0u);
    ctx_.check(qipb200_state_measure(st_, indices.data(), (uint32_t)indices.size(), 0.0, flags, &m, &p));
    return {m, p};
  }
  void collapse(const std::vector<uint64_t> &indices, uint64_t measured, double prob) {  // measure_state, :220-269
    ctx_.check(qipb200_state_collapse(st_, indices.data(), (uint32_t)indices.size(), measured, prob));
  }
  std::vector<double> measure_probs(const std::vector<uint64_t> &indices) {  // measurement_ops.rs:115-127
    std::vector<double> out(size_t(1) << indices.size());
    ctx_.check(qipb200_state_measure_probs(st_, indices.data(), (uint32_t)indices.size(), out.data()));
    return out;
  }
  // <psi|P_t|psi> for Pauli strings, each a list of (letter, qubit) pairs, e.g. {{'Z', 0}, {'Z', 1}} (absent in the
  // reference); weighted sums are the caller's dot product
  std::vector<double> expect_paulis(const std::vector<std::vector<std::pair<char, uint64_t>>> &terms) {
    std::vector<uint64_t> qubits;
    std::vector<char> letters;
    std::vector<uint32_t> lens;
    for (const auto &t : terms) {
      lens.push_back((uint32_t)t.size());
      for (const auto &lq : t) {
        letters.push_back(lq.first);
        qubits.push_back(lq.second);
      }
    }
    std::vector<double> out(terms.size());
    // a list of identities has no letters: pass non-NULL (unread) arrays, the C entry refuses NULL ones
    const uint64_t no_qubit = 0;
    const char no_letter = 'Z';
    ctx_.check(qipb200_state_expect_paulis(st_, qubits.empty() ? &no_qubit : qubits.data(),
                                           letters.empty() ? &no_letter : letters.data(), lens.data(), terms.size(),
                                           out.data()));
    return out;
  }
  // <this|P_t|ket> for Pauli strings encoded as in expect_paulis; ket is a state of the same context, precision and
  // size (it may be this one), and the empty term gives the overlap (absent in the reference)
  std::vector<std::complex<double>> transition_paulis(B200State &ket,
                                                      const std::vector<std::vector<std::pair<char, uint64_t>>> &terms) {
    Flat f(terms);
    std::vector<std::complex<double>> out(terms.size());
    ctx_.check(qipb200_state_transition_paulis(st_, ket.st_, f.q(), f.l(), f.lens.data(), terms.size(),
                                               reinterpret_cast<double *>(out.data())));
    return out;
  }
  // <this|ket>
  std::complex<double> overlap(B200State &ket) {
    return transition_paulis(ket, std::vector<std::vector<std::pair<char, uint64_t>>>(1))[0];
  }
  // psi <- exp(-i angles[T-1]/2 P_{T-1}) ... exp(-i angles[0]/2 P_0) psi for Pauli strings encoded as in
  // expect_paulis, term 0 first (absent in the reference)
  void apply_pauli_rotations(const std::vector<std::vector<std::pair<char, uint64_t>>> &terms,
                             const std::vector<double> &angles) {
    if (angles.size() != terms.size())
      throw CircuitError("apply_pauli_rotations: " + std::to_string(terms.size()) + " terms but " +
                         std::to_string(angles.size()) + " angles");
    std::vector<uint64_t> qubits;
    std::vector<char> letters;
    std::vector<uint32_t> lens;
    for (const auto &t : terms) {
      lens.push_back((uint32_t)t.size());
      for (const auto &lq : t) {
        letters.push_back(lq.first);
        qubits.push_back(lq.second);
      }
    }
    // a list of identities has no letters: pass non-NULL (unread) arrays, the C entry refuses NULL ones
    const uint64_t no_qubit = 0;
    const char no_letter = 'Z';
    ctx_.check(qipb200_state_apply_pauli_rotations(st_, qubits.empty() ? &no_qubit : qubits.data(),
                                                   letters.empty() ? &no_letter : letters.data(), lens.data(),
                                                   terms.size(), angles.data()));
  }
  // One quantum-trajectory step of single-qubit channels on distinct qubits: n_kraus[c] operators of 8 doubles each
  // for channel c (row-major, re/im interleaved), 1 + qubits.size() draws in [0, 1); returns (chosen, prob).
  std::pair<std::vector<uint32_t>, double> apply_channels(const std::vector<uint64_t> &qubits,
                                                          const std::vector<uint32_t> &n_kraus,
                                                          const std::vector<double> &kraus,
                                                          const std::vector<double> &draws) {
    if (n_kraus.size() != qubits.size() || draws.size() != qubits.size() + 1)
      throw CircuitError("apply_channels: " + std::to_string(qubits.size()) + " qubits need as many n_kraus and " +
                         std::to_string(qubits.size() + 1) + " draws");
    std::vector<uint32_t> chosen(qubits.size());
    double p = 0.0;
    ctx_.check(qipb200_state_apply_channels(st_, qubits.size(), qubits.data(), n_kraus.data(), kraus.data(),
                                            draws.data(), chosen.data(), &p));
    return {chosen, p};
  }
  // The same for channels on 1..4 qubits each: channel c acts on the arity[c] qubits that follow channel c-1's in
  // `qubits` and has n_kraus[c] operators of 2 * 4^arity[c] doubles each; returns (chosen, prob).
  std::pair<std::vector<uint32_t>, double> apply_multiqubit_channels(const std::vector<uint32_t> &arity,
                                                                     const std::vector<uint64_t> &qubits,
                                                                     const std::vector<uint32_t> &n_kraus,
                                                                     const std::vector<double> &kraus,
                                                                     const std::vector<double> &draws) {
    if (n_kraus.size() != arity.size() || draws.size() != arity.size() + 1)
      throw CircuitError("apply_multiqubit_channels: " + std::to_string(arity.size()) +
                         " channels need as many n_kraus and " + std::to_string(arity.size() + 1) + " draws");
    std::vector<uint32_t> chosen(arity.size());
    double p = 0.0;
    ctx_.check(qipb200_state_apply_multiqubit_channels(st_, arity.size(), arity.data(), qubits.data(), n_kraus.data(),
                                                       kraus.data(), draws.data(), chosen.data(), &p));
    return {chosen, p};
  }
  // The same for any complete Kraus sets on 1..4 qubits each, one draw per channel; returns (chosen, cond, prob).
  std::tuple<std::vector<uint32_t>, std::vector<double>, double> apply_kraus_channels(
      const std::vector<uint32_t> &arity, const std::vector<uint64_t> &qubits, const std::vector<uint32_t> &n_kraus,
      const std::vector<double> &kraus, const std::vector<double> &draws) {
    if (n_kraus.size() != arity.size() || draws.size() != arity.size())
      throw CircuitError("apply_kraus_channels: " + std::to_string(arity.size()) +
                         " channels need as many n_kraus and draws");
    std::vector<uint32_t> chosen(arity.size());
    std::vector<double> cond(arity.size());
    double p = 0.0;
    ctx_.check(qipb200_state_apply_kraus_channels(st_, arity.size(), arity.data(), qubits.data(), n_kraus.data(),
                                                  kraus.data(), draws.data(), chosen.data(), cond.data(), &p));
    return std::make_tuple(chosen, cond, p);
  }
  // ---- this state as the vec of an n-qubit density matrix (2n qubits; rho_rc at index r 2^n + c) ----
  // gates and channels interleaved in one fused schedule: channel c runs after ops[0 .. channel_pos[c]), channels
  // encoded as for apply_kraus_channels (a qubit may appear in several)
  void density_apply(const std::vector<qip_op> &ops, const std::vector<uint64_t> &channel_pos,
                     const std::vector<uint32_t> &arity, const std::vector<uint64_t> &qubits,
                     const std::vector<uint32_t> &n_kraus, const std::vector<double> &kraus, bool fusion = true) {
    if (channel_pos.size() != arity.size() || n_kraus.size() != arity.size())
      throw CircuitError("density_apply: " + std::to_string(arity.size()) +
                         " channels need as many positions and n_kraus");
    ctx_.check(qipb200_density_apply(st_, ops.data(), ops.size(), arity.size(), channel_pos.data(), arity.data(),
                                     qubits.data(), n_kraus.data(), kraus.data(),
                                     fusion ? QIPB200_SCHED_DEFAULT : QIPB200_SCHED_NO_FUSION));
  }
  // rho = |psi><psi| for a state psi of n qubits
  void density_from_state(const B200State &psi) { ctx_.check(qipb200_density_from_state(st_, psi.st_)); }
  // out[m] = sum of rho_rr over the r whose bits on indices equal m (bit i of m is indices[i])
  std::vector<double> density_measure_probs(const std::vector<uint64_t> &indices) {
    std::vector<double> out(1ull << indices.size());
    ctx_.check(qipb200_density_measure_probs(st_, indices.empty() ? nullptr : indices.data(),
                                             (uint32_t)indices.size(), out.data()));
    return out;
  }
  // Re Tr(rho P_t), terms as for expect_paulis
  std::vector<double> density_expect_paulis(const std::vector<std::vector<std::pair<char, uint64_t>>> &terms) {
    Flat f(terms);
    std::vector<double> out(terms.size());
    ctx_.check(qipb200_density_expect_paulis(st_, f.q(), f.l(), f.lens.data(), terms.size(), out.data()));
    return out;
  }
  // rho_A of 1..10 kept qubits: row-major 2^k x 2^k complex values
  std::vector<std::complex<double>> density_reduced(const std::vector<uint64_t> &qubits) {
    std::vector<std::complex<double>> out(1ull << (2 * std::min<size_t>(qubits.size(), 10)));
    ctx_.check(qipb200_density_reduced(st_, qubits.data(), (uint32_t)qubits.size(), (double *)out.data()));
    return out;
  }
  // <psi|rho|psi>
  std::complex<double> density_fidelity(const B200State &psi) {
    double out2[2] = {0.0, 0.0};
    ctx_.check(qipb200_density_fidelity(st_, psi.st_, out2));
    return {out2[0], out2[1]};
  }
  // the 2^n eigenvalues of rho, descending (n <= 13)
  std::vector<double> density_spectrum(uint32_t n) {
    std::vector<double> eigs(1ull << std::min<uint32_t>(n, 13));
    ctx_.check(qipb200_density_spectrum(st_, eigs.data()));
    return eigs;
  }
  // psi <- U psi for U|x>|y> = e^{i theta(x)} |x>|y ^ f(x)>: x on in_qubits, y on out_qubits (absent from the
  // reference's MatrixOp)
  void apply_function(const B200Function &fn, const std::vector<uint64_t> &in_qubits,
                      const std::vector<uint64_t> &out_qubits = {}) {
    if (in_qubits.size() != fn.n_in() || out_qubits.size() != fn.n_out())
      throw CircuitError("apply_function: the function takes " + std::to_string(fn.n_in()) + " input and " +
                         std::to_string(fn.n_out()) + " output qubits");
    ctx_.check(qipb200_state_apply_function(st_, fn.get(), in_qubits.empty() ? nullptr : in_qubits.data(),
                                            out_qubits.empty() ? nullptr : out_qubits.data()));
  }
  // <psi|D|psi> = sum_j |psi_j|^2 theta(x(j)) for D = diag theta of a code function with theta, x on in_qubits
  double expect_function(const B200Function &fn, const std::vector<uint64_t> &in_qubits) {
    if (in_qubits.size() != fn.n_in())
      throw CircuitError("expect_function: the function takes " + std::to_string(fn.n_in()) + " input qubits");
    double out = 0.0;
    ctx_.check(qipb200_state_expect_function(st_, fn.get(), in_qubits.data(), &out));
    return out;
  }
  // this state <- H src for H = sum_h coeffs[h] P_h, Pauli strings encoded as in expect_paulis; src is another state
  // of the same context, precision and size, and this state takes its layout (absent in the reference)
  void apply_pauli_sum(const B200State &src, const std::vector<std::vector<std::pair<char, uint64_t>>> &terms,
                       const std::vector<double> &coeffs) {
    if (coeffs.size() != terms.size())
      throw CircuitError("apply_pauli_sum: " + std::to_string(terms.size()) + " terms but " +
                         std::to_string(coeffs.size()) + " coefficients");
    Flat f(terms);
    ctx_.check(qipb200_state_apply_pauli_sum(st_, src.st_, f.q(), f.l(), f.lens.data(), terms.size(), coeffs.data()));
  }
  // energy and gradient of <psi0|U^dagger H U|psi0> by the adjoint method: this state holds psi0 (and ends there up
  // to rounding), U applies exp(-i angles[t]/2 P_t) for the ansatz strings, term 0 first, H = sum_h coeffs[h] Q_h;
  // work is scratch of the same size and precision.  A parameter shared by several strings has the sum of their
  // entries as its derivative (absent in the reference)
  std::pair<double, std::vector<double>> energy_gradient(
      B200State &work, const std::vector<std::vector<std::pair<char, uint64_t>>> &ansatz,
      const std::vector<double> &angles, const std::vector<std::vector<std::pair<char, uint64_t>>> &hamiltonian,
      const std::vector<double> &coeffs) {
    if (angles.size() != ansatz.size() || coeffs.size() != hamiltonian.size())
      throw CircuitError("energy_gradient: " + std::to_string(ansatz.size()) + " terms, " +
                         std::to_string(angles.size()) + " angles, " + std::to_string(hamiltonian.size()) +
                         " Hamiltonian terms, " + std::to_string(coeffs.size()) + " coefficients");
    Flat a(ansatz), h(hamiltonian);
    std::pair<double, std::vector<double>> out(0.0, std::vector<double>(ansatz.size()));
    ctx_.check(qipb200_state_pauli_energy_gradient(st_, work.st_, a.q(), a.l(), a.lens.data(), ansatz.size(),
                                                   angles.data(), h.q(), h.l(), h.lens.data(), hamiltonian.size(),
                                                   coeffs.data(), &out.first, out.second.data()));
    return out;
  }
  // the quantum geometric tensor of the ansatz (strings encoded as in expect_paulis, term 0 first): returns (G row-major
  // T x T, e) with G_ij = <d_i psi|d_j psi> - <d_i psi|psi><psi|d_j psi> and e_t = <psi_t|P_t|psi_t>; this state ends
  // at U psi0, work_a and work_b are scratch of the same context, precision and size (absent in the reference)
  std::pair<std::vector<std::complex<double>>, std::vector<double>> geometric_tensor(
      B200State &work_a, B200State &work_b, const std::vector<std::vector<std::pair<char, uint64_t>>> &ansatz,
      const std::vector<double> &angles) {
    if (angles.size() != ansatz.size())
      throw CircuitError("geometric_tensor: " + std::to_string(ansatz.size()) + " terms but " +
                         std::to_string(angles.size()) + " angles");
    Flat a(ansatz);
    std::pair<std::vector<std::complex<double>>, std::vector<double>> out(
        std::vector<std::complex<double>>(ansatz.size() * ansatz.size()), std::vector<double>(ansatz.size()));
    ctx_.check(qipb200_state_pauli_geometric_tensor(st_, work_a.st_, work_b.st_, a.q(), a.l(), a.lens.data(),
                                                    ansatz.size(), angles.data(),
                                                    reinterpret_cast<double *>(out.first.data()), out.second.data()));
    return out;
  }
  // this state <- exp(-i time H) this state for H = sum_h coeffs[h] P_h, by a Chebyshev series cut at the smallest
  // degree K >= 2 whose tail bound is <= tol; work_a and work_b are scratch of the same context, precision and size.
  // Returns (K, tail bound) (absent in the reference)
  std::pair<uint32_t, double> evolve_pauli_sum(B200State &work_a, B200State &work_b,
                                               const std::vector<std::vector<std::pair<char, uint64_t>>> &terms,
                                               const std::vector<double> &coeffs, double time, double tol) {
    if (coeffs.size() != terms.size())
      throw CircuitError("evolve_pauli_sum: " + std::to_string(terms.size()) + " terms but " +
                         std::to_string(coeffs.size()) + " coefficients");
    Flat f(terms);
    std::pair<uint32_t, double> out(0, 0.0);
    ctx_.check(qipb200_state_evolve_pauli_sum(st_, work_a.st_, work_b.st_, f.q(), f.l(), f.lens.data(), terms.size(),
                                              coeffs.data(), time, tol, &out.first, &out.second));
    return out;
  }
  // the lowest eigenvalue of H = sum_h coeffs[h] P_h reachable from this state, by plain Lanczos until the Ritz
  // estimate is <= tol sum |c_h| (non-identity terms) or max_steps; with vector, this state ends as the normalised
  // Ritz vector.  work_a and work_b are scratch of the same context, precision and size (absent in the reference)
  struct LanczosResult {
    double energy = 0.0, residual = 0.0, ritz_norm = 0.0;
    uint32_t steps = 0;
    bool converged = false;
    std::vector<double> alpha, beta;  // alpha_0..alpha_(steps-1); beta_0 = |psi| .. beta_steps
  };
  LanczosResult lanczos_pauli_sum(B200State &work_a, B200State &work_b,
                                  const std::vector<std::vector<std::pair<char, uint64_t>>> &terms,
                                  const std::vector<double> &coeffs, uint32_t max_steps, double tol,
                                  bool vector = true) {
    if (coeffs.size() != terms.size())
      throw CircuitError("lanczos_pauli_sum: " + std::to_string(terms.size()) + " terms but " +
                         std::to_string(coeffs.size()) + " coefficients");
    Flat f(terms);
    LanczosResult r;
    const size_t cap = max_steps ? max_steps : 1;
    r.alpha.assign(cap, 0.0);
    r.beta.assign(cap + 1, 0.0);
    double out3[3] = {0.0, 0.0, 0.0};
    uint32_t conv = 0;
    ctx_.check(qipb200_state_lanczos_pauli_sum(st_, work_a.st_, work_b.st_, f.q(), f.l(), f.lens.data(), terms.size(),
                                               coeffs.data(), max_steps, tol, vector ? QIPB200_LANCZOS_VECTOR : 0u,
                                               &r.steps, &conv, r.alpha.data(), r.beta.data(), out3));
    r.alpha.resize(r.steps);
    r.beta.resize(r.steps + 1);
    r.energy = out3[0];
    r.residual = out3[1];
    r.ritz_norm = out3[2];
    r.converged = conv != 0;
    return r;
  }
  // reduced density matrix of up to 10 qubits, row-major 2^k x 2^k; bit i of the row and column index is the value of
  // qubits[i], as in measure_probs (absent in the reference)
  std::vector<std::complex<double>> reduced_density(const std::vector<uint64_t> &qubits) {
    const size_t dim = qubits.size() <= 10 ? (size_t)1 << qubits.size() : 1;
    std::vector<std::complex<double>> out(dim * dim);
    ctx_.check(qipb200_state_reduced_density(st_, qubits.data(), (uint32_t)qubits.size(),
                                             reinterpret_cast<double *>(out.data())));
    return out;
  }
  // {Tr rho_A^2, Tr rho_A} of the qubits `qubits` on the state as it is; purity = first / second^2 (absent in the
  // reference)
  std::pair<double, double> purity(const std::vector<uint64_t> &qubits) {
    double out2[2] = {0.0, 0.0};
    ctx_.check(qipb200_state_purity(st_, qubits.data(), (uint32_t)qubits.size(), out2));
    return std::make_pair(out2[0], out2[1]);
  }
  // eigenvalues (descending, not renormalised) of the reduced density matrix across the cut of `qubits`, for a smaller
  // side of s <= 13 qubits; *entropy (if given) gets the von Neumann entropy in nats of the normalised spectrum
  // (absent in the reference)
  std::vector<double> entanglement_spectrum(const std::vector<uint64_t> &qubits, double *entropy = nullptr) {
    const size_t k = qubits.size(), s = std::min(k, n_ >= k ? n_ - k : 0);
    std::vector<double> eigs((size_t)1 << std::min<size_t>(s, 13));
    double out2[2] = {0.0, 0.0};
    ctx_.check(qipb200_state_entanglement_spectrum(st_, qubits.data(), (uint32_t)k, eigs.data(), eigs.size(), nullptr,
                                                   out2));
    if (entropy) *entropy = out2[1];
    return eigs;
  }
  // a schedule parsed from the QIPS wire format (owned by the library): builder.rs:423-514 on foreign circuits
  void apply_parsed(const qip_op *ops, size_t n_ops, bool fusion = true) {
    ctx_.check(qipb200_state_apply_schedule(st_, ops, n_ops, fusion ? QIPB200_SCHED_DEFAULT : QIPB200_SCHED_NO_FUSION));
  }
  qipb200_state *get() const { return st_; }

 private:
  // Pauli strings as the flat arrays of the C ABI; a list of identities has no letters, so q() and l() point at
  // non-NULL (unread) values then, since the C entries refuse NULL arrays
  struct Flat {
    std::vector<uint64_t> qubits;
    std::vector<char> letters;
    std::vector<uint32_t> lens;
    uint64_t no_qubit = 0;
    char no_letter = 'Z';
    explicit Flat(const std::vector<std::vector<std::pair<char, uint64_t>>> &terms) {
      for (const auto &t : terms) {
        lens.push_back((uint32_t)t.size());
        for (const auto &lq : t) {
          letters.push_back(lq.first);
          qubits.push_back(lq.second);
        }
      }
    }
    const uint64_t *q() const { return qubits.empty() ? &no_qubit : qubits.data(); }
    const char *l() const { return letters.empty() ? &no_letter : letters.data(); }
  };
  Context &ctx_;
  size_t n_;
  qipb200_state *st_ = nullptr;
};

// ---- QIPS schedule wire format (SURVEY section 8f, N3): RAII over qipb200_schedule_parse ------------
class ParsedSchedule {
 public:
  ParsedSchedule(const void *bytes, size_t len) {
    char err[256];
    if (qipb200_schedule_parse(bytes, len, &s_, err, sizeof(err)) != QIPB200_OK) throw CircuitError(err);
    ops_ = qipb200_schedule_ops(s_, &n_ops_, &n_qubits_, &prec_);
  }
  ~ParsedSchedule() { qipb200_schedule_free(s_); }
  ParsedSchedule(const ParsedSchedule &) = delete;
  ParsedSchedule &operator=(const ParsedSchedule &) = delete;
  const qip_op *ops() const { return ops_; }
  size_t size() const { return n_ops_; }
  uint32_t n_qubits() const { return n_qubits_; }
  qip_prec prec() const { return prec_; }

 private:
  qipb200_schedule *s_ = nullptr;
  const qip_op *ops_ = nullptr;
  size_t n_ops_ = 0;
  uint32_t n_qubits_ = 0;
  qip_prec prec_ = QIP_F64;
};

}  // namespace qip
