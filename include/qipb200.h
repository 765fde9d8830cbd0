/*
 * qipb200.h -- C ABI of libqipb200: H100-native (sm_90a) state-vector gate
 * application behind RustQIP's operator API.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point names
 * the reference interface it replaces (paths relative to the RustQIP tree).
 * A Rust `extern "C"` block / bindgen run over this header is all a
 * maintainer needs (INTEGRATION.md shows the shim).
 *
 * Conventions
 *   - amplitudes: interleaved (re,im) of float (QIP_F32) or double (QIP_F64),
 *     i.e. the memory layout of `&[Complex<P>]`; lengths/offsets are counted
 *     in amplitudes, not bytes.
 *   - qubit q <-> index bit n-1-q; see include/qip_op.h for the op descriptor.
 *   - every function returns a qipb200_status (0 == OK) and never aborts the
 *     process; the message of the last failure is available through
 *     qipb200_last_error().  (The reference's constructors return
 *     CircuitResult<T>, qip/src/errors.rs:6-22; apply_op* itself panics on
 *     misuse -- here both surface as status codes.)
 *   - there is NO CPU fallback: without a CUDA device qipb200_init() fails
 *     with QIPB200_ERR_CUDA and nothing else can be called.
 *   - a ctx / state handle is not thread-safe (it is the `&mut` of the
 *     reference); distinct handles may be driven from distinct host threads.
 */
#ifndef QIPB200_H
#define QIPB200_H

#include "qip_op.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum qipb200_status {
  QIPB200_OK = 0,
  QIPB200_ERR_INVALID_ARG = 1,   /* null pointer, bad enum, malformed op tree            */
  QIPB200_ERR_SIZE_MISMATCH = 2, /* len(dense) != 4^k, swap halves differ, empty indices */
  QIPB200_ERR_BAD_INDEX = 3,     /* qubit index >= n, or repeated                        */
  QIPB200_ERR_CUDA = 4,          /* CUDA runtime/driver error (message has the details)  */
  QIPB200_ERR_COMM = 5,          /* multi-GPU exchange set-up or peer access failure     */
  QIPB200_ERR_OOM = 6,           /* device allocation failed                             */
  QIPB200_ERR_UNSUPPORTED = 7    /* valid request this build cannot serve (e.g. k too large) */
} qipb200_status;

typedef struct qipb200_ctx qipb200_ctx;     /* one CUDA device + stream + scratch         */
typedef struct qipb200_state qipb200_state; /* device-resident 2^n amplitudes (or a shard) */

/* Schedule flags for qipb200_state_apply_schedule / qipb200_calculate_state. */
enum {
  QIPB200_SCHED_DEFAULT = 0u,   /* fusion allowed: sequential PRODUCT of the ops        */
  QIPB200_SCHED_NO_FUSION = 1u  /* one kernel sweep per op, exactly as the reference's
                                   per-entry loop (qip/src/builder.rs:423-514)          */
};

/* ---- library / context ------------------------------------------------------- */

/* ABI version of this header (major*1000 + minor). */
int qipb200_abi_version(void);

/* Create a context bound to CUDA device `device_id` (one process per GPU).
 * Replaces nothing in the reference (it has no device); owns the stream the
 * gate kernels run on.  Fails with QIPB200_ERR_CUDA when no usable sm_90
 * device exists -- there is no CPU path. */
int qipb200_init(qipb200_ctx **ctx, int device_id);
/* One context over SEVERAL devices of this process (n_devices a power of two; device_ids == NULL means 0..n-1):
 * the drop-in for a single-process host such as LocalBuilder::calculate_state_with_init
 * (qip/src/builder.rs:400-519), which has no notion of ranks.  States created on it with qipb200_state_new are
 * sharded over the devices by their top log2(n_devices) index bits; every state call is served by one host thread
 * per device inside the library, the devices map each other with CUDA peer access (NVLink / NVSwitch) and run
 * the same exchange kernels as the one-process-per-GPU path.  upload/download address the whole 2^n vector. */
int qipb200_init_multi(qipb200_ctx **ctx, int n_devices, const int *device_ids);
void qipb200_shutdown(qipb200_ctx *ctx);

/* Message of the last failing call on `ctx` (or, with ctx == NULL, of the last
 * failing call on this thread that had no ctx yet).  Never NULL. */
const char *qipb200_last_error(const qipb200_ctx *ctx);

/* The CUDA stream (a `cudaStream_t`) every kernel of `ctx` is launched on, so that a
 * caller can bracket work with its own CUDA events. */
int qipb200_stream_handle(const qipb200_ctx *ctx, void **stream);

/* Number of this library's kernels launched through `ctx` so far. */
uint64_t qipb200_kernel_launches(const qipb200_ctx *ctx);
/* out4 = { all kernels, fused tile passes, NVLink exchange kernels, reference ops folded into tile passes }. */
int qipb200_launch_stats(const qipb200_ctx *ctx, uint64_t *out4);

/* Per-gate kernels launched through `ctx` so far (qipb200_state_apply_op and unfused schedules), by kernel:
 * out[QIPB200_KC_*] for the first min(n, QIPB200_KC_COUNT) entries.  Lets a caller see which kernel an op took,
 * e.g. that it ran in place rather than on the out-of-place row kernel. */
enum {
  QIPB200_KC_DENSE = 0,      /* k_dense, k <= 4 in registers */
  QIPB200_KC_DIAG = 1,       /* k_diag */
  QIPB200_KC_DIAG_WIDE = 2,  /* k_diag_wide */
  QIPB200_KC_EXCHANGE = 3,   /* k_exchange (X / CNOT / Toffoli-X / Swap pairs) */
  QIPB200_KC_DENSE5 = 4,     /* k_dense5 */
  QIPB200_KC_DENSE_DMMA = 5, /* k_dense_dmma (f64, k = 5, 6) */
  QIPB200_KC_DENSE_BIG = 6,  /* k_dense_big */
  QIPB200_KC_GATHER = 7,     /* k_gather, the out-of-place row kernel */
  QIPB200_KC_COUNT = 8
};
int qipb200_kernel_counts(const qipb200_ctx *ctx, uint64_t *out, size_t n);

/* Free the one state buffer the context keeps after a state is freed (for the next state of the same size), so
 * that the device memory of freed states is returned at once.  The next state allocates afresh. */
int qipb200_release_pool(qipb200_ctx *ctx);

/* Generated kernels (absent in the reference): fused tile passes of big states are compiled by NVRTC into
 * kernels specialised to the pass (rustqip_b200/csrc/jit_codegen.cpp); a pass whose kernel is still being compiled
 * in the background runs the generic kernel meanwhile.  With wait != 0 this call blocks until the background
 * compilations have finished.  out4 = { tile passes run by generated kernels, all tile passes (this context),
 * programs compiled so far (process, valid with wait), their total compile time in ms (valid with wait) };
 * `note` (may be NULL) receives the reason the generated path was last declined, if any.
 * Environment: QIPB200_JIT = off | async (default from 22 local qubits) | sync (compile before launching). */
int qipb200_jit_stats(qipb200_ctx *ctx, int wait, double *out4, char *note, size_t note_len);
/* Host-only (no GPU, ctx-free): plan the schedule for an n-qubit single-device state, generate and NVRTC-compile
 * the kernel of every fused pass into the process-wide cache (a later qipb200_state_apply_schedule of the same
 * schedule then starts on generated kernels at once).  out5 = { passes, passes covered by the generator, compiled
 * without error, wall ms, sum of per-program compile ms }; `log` (may be NULL) receives the last compiler message. */
int qipb200_jit_precompile(qip_prec prec, uint32_t n_qubits, const qip_op *ops, size_t n_ops, double *out5, char *log,
                           size_t log_len);

/* Optional device timing by category (absent in the reference): while enabled, every fused tile pass and every
 * NVLink exchange (kernel + its two flag barriers) is bracketed by a CUDA-event pair on the context's stream.
 * profile_read synchronises the stream and returns
 *   out4 = { tile-pass ms, tile passes, exchange ms, exchanges }  since the previous read, then resets. */
int qipb200_profile_enable(qipb200_ctx *ctx, int on);
int qipb200_profile_read(qipb200_ctx *ctx, double *out4);

/* Validate an op exactly as the reference's constructors do
 * (qip/src/state_ops/matrix_ops.rs:12-122: non-empty indices, len(dense)==4^k,
 * sparse row count 2^k and no empty row, equal swap halves, >=1 control) plus
 * index range / distinctness for an n-qubit state.  Needs no GPU (ctx may be NULL). */
int qipb200_validate_op(const qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, const qip_op *op);

/* ---- stateless drop-ins for qip_iterators::matrix_ops (HOST buffers) ---------- */

/* qip_iterators::matrix_ops::apply_op (qip-iterators/src/matrix_ops.rs:98-123):
 * output[o] += row(output_offset+o) . input, partners outside
 * [input_offset, input_offset+input_len) read as zero.  Copies both buffers to
 * the device, runs the gate kernel, copies `output` back. */
int qipb200_apply_op(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, const qip_op *op,
                     const void *input, uint64_t input_len, void *output, uint64_t output_len,
                     uint64_t input_offset, uint64_t output_offset);

/* qip_iterators::matrix_ops::apply_op_overwrite (matrix_ops.rs:127-152):
 * same with `=` instead of `+=`; `output` is write-only. */
int qipb200_apply_op_overwrite(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, const qip_op *op,
                               const void *input, uint64_t input_len, void *output,
                               uint64_t output_len, uint64_t input_offset, uint64_t output_offset);

/* qip_iterators::matrix_ops::apply_ops (matrix_ops.rs:158-219).
 *   n_ops == 0 : copy of the overlapping index range (matrix_ops.rs:170-183);
 *   n_ops == 1 : apply_op;
 *   n_ops  > 1 : output += the reference's multi-op row sum (matrix_ops.rs:184-217 with
 *                sum_for_ops_cols, iterators/iterator_mapper.rs:8-31, and MultiOpIterator,
 *                qubit_multi_iterator.rs:38-78), restated AS IT IS: op i reads its row from
 *                the low bits left of the sub-row while columns are composed first-op-high
 *                (SURVEY.md section 8 quirk Q5), so for ops that are not all alike the
 *                result is not their tensor product -- exactly what the reference returns.
 *                Offsets and ragged windows as in apply_op.  2..8 ops, at most 40 indices
 *                in total (else QIPB200_ERR_UNSUPPORTED).  To apply gates one after the
 *                other use a state + qipb200_state_apply_schedule. */
int qipb200_apply_ops(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, const qip_op *ops,
                      size_t n_ops, const void *input, uint64_t input_len, void *output,
                      uint64_t output_len, uint64_t input_offset, uint64_t output_offset);

/* ---- device-resident state: the body of LocalBuilder::calculate_state_with_init
 *      (qip/src/builder.rs:400-519) ------------------------------------------------ */

/* `let mut state = vec![Complex::zero(); 1 << n]` (builder.rs:406); all zero. */
int qipb200_state_new(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, qipb200_state **state);
void qipb200_state_free(qipb200_state *state);

/* `state[initial_index] = Complex::one()` after clearing (builder.rs:421). */
int qipb200_state_set_basis(qipb200_state *state, uint64_t index);

/* Copy `len` amplitudes host<->device starting at amplitude `offset`
 * (the reference returns/accepts the Vec itself, builder.rs:518). */
int qipb200_state_upload(qipb200_state *state, const void *host, uint64_t offset, uint64_t len);
int qipb200_state_download(qipb200_state *state, void *host, uint64_t offset, uint64_t len);

/* One pipeline entry: `apply_op_overwrite(n,&uop,&state,&mut arena,0,0)` followed by
 * the buffer swap (builder.rs:499,514); logically state <- U state.  Stream-ordered. */
int qipb200_state_apply_op(qipb200_state *state, const qip_op *op);

/* The whole fold over the pipeline (builder.rs:423-514) for unitary entries:
 * state <- ops[n_ops-1] ... ops[0] state.  With QIPB200_SCHED_NO_FUSION every op
 * is one sweep; otherwise runs of ops are fused into shared-memory tile passes. */
int qipb200_state_apply_schedule(qipb200_state *state, const qip_op *ops, size_t n_ops,
                                 uint32_t flags);

/* sum |a|^2 over the WHOLE state: prob_magnitude, measurement_ops.rs:11-13.  On a sharded state the call is
 * COLLECTIVE (every rank calls it; the per-rank sums are added through the peers' reduction slots over NVLink)
 * and every rank receives the same total. */
int qipb200_state_norm2(qipb200_state *state, double *out);

/* max over the (local) amplitudes of max(|re_a - re_b|, |im_a - im_b|), computed on the device: the
 * comparison behind the fused-vs-unfused parity checks at sizes no host oracle reaches (two 16 GiB
 * states at N=30).  Both states must live on the same context and have the same shape and layout.
 * Replaces nothing in the reference (its tests compare Vecs on the host). */
int qipb200_state_max_abs_diff(qipb200_state *a, qipb200_state *b, double *out);

/* Block until everything queued on the state's stream has finished. */
int qipb200_state_sync(qipb200_state *state);

/* One call == LocalBuilder::calculate_state_with_init for a unitary pipeline:
 * allocate, set |init_index>, run the schedule, copy the 2^n amplitudes to
 * `host_out` (HOST memory, 2^n complex<prec>).  This is the end-to-end entry
 * bench.py's `e2e` times. */
int qipb200_calculate_state(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, uint64_t init_index,
                            const qip_op *ops, size_t n_ops, uint32_t flags, void *host_out);

/* ---- measurement on the device (qip/src/state_ops/measurement_ops.rs) ----------
 * On a sharded state all four calls are COLLECTIVE: every rank calls with the same arguments and every rank
 * receives the result for the whole 2^n vector (histograms / scalars are summed across the ranks in rank order
 * through peer-mapped reduction slots, so the values are bit-identical on all ranks and can be fed to
 * qipb200_state_collapse as they are).  measure_probs is limited to 16 measured qubits there. */

/* measure_probs (measurement_ops.rs:115-127): out[m] for m in 0..2^n_indices,
 * bit i of m <-> indices[i].  `out` is HOST memory of 2^n_indices doubles. */
int qipb200_state_measure_probs(qipb200_state *state, const uint64_t *indices, uint32_t n_indices,
                                double *out);
/* measure_prob (measurement_ops.rs:44-58). */
int qipb200_state_measure_prob(qipb200_state *state, uint64_t measured, const uint64_t *indices,
                               uint32_t n_indices, double *out);
/* soft_measure (measurement_ops.rs:153-176) with the uniform draw r in [0,1)
 * supplied by the caller (the reference calls rand::random). */
int qipb200_state_soft_measure(qipb200_state *state, const uint64_t *indices, uint32_t n_indices,
                               double r, uint64_t *measured);
/* K = n_draws independent soft_measure draws (measurement_ops.rs:153-176) on one state, which is NOT collapsed:
 * measured[k] is what qipb200_state_soft_measure(state, indices, n_indices, draws[k], ..) returns, up to
 * summation order (a draw within rounding distance of a cumulative boundary may land on the neighbouring index).
 * bit i of measured[k] <-> indices[i].  draws / measured are HOST arrays of n_draws entries; the draws are not
 * range-checked (a draw at or above the state's total, or NaN, gives index 0, as in the reference).
 * Reads the state at most twice whatever K (per-chunk sums, then only the chunks some draw landed in); the
 * number of kernels does not depend on K; the same state and draws give bit-identical results.  Synchronises.
 * n_draws == 0 is a no-op.  Sharded states: QIPB200_ERR_UNSUPPORTED. */
int qipb200_state_sample(qipb200_state *state, const uint64_t *indices, uint32_t n_indices,
                         const double *draws, uint64_t n_draws, uint64_t *measured);
/* measure_state (measurement_ops.rs:220-269): zero the amplitudes that
 * contradict `measured`, scale the rest by 1/sqrt(measured_prob); in place. */
int qipb200_state_collapse(qipb200_state *state, const uint64_t *indices, uint32_t n_indices,
                           uint64_t measured, double measured_prob);

enum {
  QIPB200_MEASURE_FORCED = 1u,      /* *measured is an input: MeasuredCondition { measured, prob: None } */
  QIPB200_MEASURE_FORCED_PROB = 2u  /* with FORCED: *prob is an input too (prob: Some(p)); no read sweep */
};
/* measure (measurement_ops.rs:190-214): draw the outcome as soft_measure does with the uniform r in [0,1)
 * (ignored when FORCED), take its probability as measure_prob does (unless FORCED_PROB), collapse as
 * measure_state does, and return both.  bit i of *measured <-> indices[i].  Synchronises.
 *   *measured is what qipb200_state_soft_measure(state, indices, n_indices, r, ..) returns, up to summation order
 *   (as for qipb200_state_sample); *prob is qipb200_state_measure_prob(state, *measured, ..) up to summation order;
 *   the state afterwards is qipb200_state_collapse(state, indices, n_indices, *measured, *prob).  *prob == 0 leaves
 *   the state untouched.  The same state and arguments give bit-identical results.
 * Unsharded states: one read sweep plus the chunk the draw landed in when every measured qubit q satisfies
 * q <= n-13 (at most two sweeps otherwise), a fixed number of kernels, and no collapse sweep: the collapse is kept
 * pending on the state and runs as diagonal gates inside the first tile pass of the next fused apply_schedule (any
 * other call that touches the amplitudes applies it first; set_basis and load drop it).
 * Sharded and multi-device states: soft_measure, measure_prob and collapse in turn (collective). */
int qipb200_state_measure(qipb200_state *state, const uint64_t *indices, uint32_t n_indices, double r,
                          uint32_t flags, uint64_t *measured, double *prob);

/* <psi|P_t|psi> for n_terms Pauli strings on the state AS IT IS (not renormalised, like measure_probs); absent in the
 * reference.  Term t is the term_len[t] pairs (qubits[k], paulis[k]) that follow term t-1 in the flat arrays.  The
 * letters are 'X', 'Y' and 'Z' (else QIPB200_ERR_INVALID_ARG), a qubit >= n or repeated inside one term gives
 * QIPB200_ERR_BAD_INDEX, NULL arrays with n_terms > 0 give QIPB200_ERR_INVALID_ARG, n_terms == 0 is a no-op, and an
 * empty term is the identity (= norm2).  out[t] (HOST, n_terms doubles) is real: P_t is Hermitian, and the imaginary
 * part is rounding and is not returned.  Deterministic (same state and terms -> bit-identical out), accumulated in
 * double for both precisions, synchronises.  A read sweep carries up to 16384 terms: terms with equal X/Y masks share
 * one sweep (a mask with more than 16384 terms takes one per 16384), Z-only terms fill the room of the other sweeps and
 * take one sweep per 16384 of what is left, and distinct masks share a sweep when their bits fit one tile
 * (qipb200_expect_plan reports the count); one kernel per sweep plus one reduction kernel per batch of sweeps of at
 * most 16384 terms, so the device scratch stays below 35 MB for any number of terms.  A pending collapse is applied first; a permuted
 * layout is read as it is.  Sharded and multi-device states: QIPB200_ERR_UNSUPPORTED. */
int qipb200_state_expect_paulis(qipb200_state *state, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, double *out);
/* Host-only (no GPU, ctx-free), like qipb200_plan_exchanges: the number of read sweeps the call above makes for these
 * terms on an unsharded n-qubit state in canonical layout (0 for n_terms == 0).  Validates as the call above does. */
int qipb200_expect_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *sweeps);

/* <bra|P_t|ket> for n_terms Pauli strings, on the two states AS THEY ARE (not renormalised); absent in the reference.
 * Terms are encoded and validated as for qipb200_state_expect_paulis (same codes and messages).  With P = i^nY X^x Z^z,
 *   <bra|P|ket> = sum_j conj(bra_j) (P ket)_j = i^nY sum_j (-1)^popc(j & z) conj(bra_{j ^ x}) ket_j.
 * out (HOST, 2 * n_terms doubles) receives (Re, Im) of term t at out[2t], out[2t + 1]; the empty term gives the overlap
 * <bra|ket>, and <bra|P|ket> is conj(<ket|P|bra>).  bra == ket is allowed (then out[2t] is expect_paulis' value up to
 * rounding).  Accumulated in double for both precisions (f32 amplitudes are widened before they are multiplied) over a
 * fixed grid with fixed-order per-CTA partials and one reduction kernel per batch, no floating-point atomics: the same
 * states and terms give bit-identical out; synchronises.  The summation order and its rounding bound are documented in
 * rustqip_b200/csrc/expect.cu.  Sweeps are planned as for expect_paulis with two rows (Re and Im) per term, so a read
 * sweep of both states carries up to 8192 terms; one kernel per sweep plus one reduction kernel per batch of at most
 * 16384 rows (qipb200_transition_plan reports both counts).
 * Errors, all before any device work (a refused call leaves both states and a pending collapse as they were): NULL bra
 * or ket, and NULL out with n_terms > 0, give QIPB200_ERR_INVALID_ARG; a term error the code and message of
 * expect_paulis; states of different contexts, precisions or sizes QIPB200_ERR_SIZE_MISMATCH; sharded or multi-device
 * states QIPB200_ERR_UNSUPPORTED.  n_terms == 0 is a no-op.  A collapse pending on either state is applied first (one
 * kernel each).  Layouts: two states with the same qubit map (canonical, or permuted alike by QIPB200_ROTATE) are read
 * where they are and keep their layout; otherwise each permuted state is first restored to the canonical layout, with
 * the kernels of that restore (swap-only tile passes under QIPB200_ROTATE, one bit-swap kernel per transposition
 * otherwise), and its amplitudes stay logically the same, as before a download. */
int qipb200_state_transition_paulis(qipb200_state *bra, qipb200_state *ket, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, double *out);
/* Host-only (no GPU, ctx-free): out2 = {read sweeps, kernels} of the call above on unsharded n-qubit states in
 * canonical layout with nothing pending ({0, 0} for n_terms == 0).  Validates as the call above does; NULL out2, a bad
 * precision or n_qubits not in 1..40 give QIPB200_ERR_INVALID_ARG. */
int qipb200_transition_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *out2);

/* Reduced density matrix of the k = n_qubits_kept qubits `qubits` on the state AS IT IS (not renormalised, like
 * measure_probs); absent in the reference.  out (HOST, 2 * 4^k doubles, interleaved re/im) receives
 *   rho[a * 2^k + b] = sum_r psi(r, a) conj(psi(r, b))      (partial trace over every other qubit)
 * where bit i of a and b is the value of qubit qubits[i] (the convention of measure_probs: diag(rho) equals
 * measure_probs(qubits) up to rounding, and the trace is norm2).  The lower triangle is the conjugate of the upper one
 * and the diagonal's imaginary part is exactly 0.0.  Double for f32 and f64 states (f32 amplitudes are widened before
 * they are multiplied), deterministic (same state and qubits -> bit-identical out), synchronises.  NULL qubits, k == 0
 * or k > n give QIPB200_ERR_INVALID_ARG, a qubit >= n or repeated QIPB200_ERR_BAD_INDEX, NULL out
 * QIPB200_ERR_INVALID_ARG, k > 10 QIPB200_ERR_UNSUPPORTED.  One read sweep for k <= 6 (2 kernels); for k = 7..10,
 * nB = 2^(k-6) sweeps in nB (nB + 1) kernels.  A pending collapse is applied first; a permuted layout is read as it is.
 * Sharded and multi-device states: QIPB200_ERR_UNSUPPORTED. */
int qipb200_state_reduced_density(qipb200_state *state, const uint64_t *qubits, uint32_t n_qubits_kept, double *out);

/* out2[0] = Tr rho_A^2 = sum_{a,b} |rho_ab|^2, out2[1] = Tr rho_A = sum_j |psi_j|^2, for rho_A the reduced density
 * matrix of the k qubits `qubits` (as qipb200_state_reduced_density defines it), on the state AS IT IS (not
 * renormalised): purity = out2[0] / out2[1]^2 and the Renyi-2 entropy is -ln of it; absent in the reference.  With
 * s = min(k, n - k), the smaller side, the route depends on s only: s = 0 (k = n) is one norm2 sweep (out2 = {norm2^2,
 * norm2}); 1 <= s <= 10 is qipb200_state_reduced_density of the side's qubits, with ||rho||_F^2 summed on the host in a
 * fixed order; s >= 11 is a Gram product G = M M^dagger on the FP64 tensor pipe over the side (M: the state reshaped
 * to 2^s x 2^(n-s)), two kernels, documented with its summation order and error bound in rustqip_b200/csrc/purity.cu.
 * Double for f32 and f64 states (f32 amplitudes are widened before they are multiplied), deterministic (same state and
 * qubits -> bit-identical out2), no floating-point atomics, synchronises.  Errors, all before any device work: NULL
 * state, NULL qubits, NULL out2, k == 0 or k > n give QIPB200_ERR_INVALID_ARG, a qubit >= n or repeated
 * QIPB200_ERR_BAD_INDEX, sharded and multi-device states QIPB200_ERR_UNSUPPORTED.  A pending collapse is applied first;
 * a permuted layout is read as it is. */
int qipb200_state_purity(qipb200_state *state, const uint64_t *qubits, uint32_t k, double *out2);
/* Host-only (no GPU, ctx-free): out4 = {route (0 norm2, 1 reduced_density, 2 Gram), s, kernels, Gram blocks} of the
 * call above on an unsharded n-qubit state with nothing pending.  Kernels: 1, 2^m (2^m + 1) with m = max(0, s - 6), or
 * 2; Gram blocks (128 x 64 entries of G, those touching its upper triangle): 2^(s-7) (2^(s-7) + 1) on route 2, else 0.
 * Validates the qubits as the call above does; NULL out4, a bad precision or n_qubits not in 1..40 give
 * QIPB200_ERR_INVALID_ARG. */
int qipb200_purity_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, uint32_t k, uint32_t *out4);

/* Entanglement spectrum and von Neumann entropy of the cut between the k qubits `qubits` and the rest, on the state
 * AS IT IS (not renormalised); absent in the reference.  The side is taken as by qipb200_state_purity: the qubits
 * passed when k <= n - k, else their complement; s is its size and G its 2^s x 2^s matrix sum_r psi(r, a)
 * conj(psi(r, b)) in the convention of qipb200_state_reduced_density (bit i of a row index is the value of side qubit
 * i).  The nonzero spectra of both sides agree, so the eigenvalues do not depend on which side is passed.
 *   eigs (HOST, eigs_cap >= 2^s doubles): the 2^s eigenvalues of G in descending order (the solver's values sorted
 *     on the host: cuSOLVER's own order is ascending only up to rounding among nearly equal ones), not renormalised (the
 *     squared Schmidt coefficients times the norm); values that come out slightly negative through rounding are
 *     returned as computed.
 *   out2[0] = T = sum_a G_aa in index order; out2[1] = -sum p_i ln p_i (nats) over the eigenvalues > 0 in ascending
 *     order, p_i = lambda_i / T; 0 if T == 0.
 *   rho (HOST, may be NULL; 2 * 4^s doubles, interleaved re/im, row-major): G.  The lower triangle is the exact
 *     conjugate of the upper one and the diagonal's imaginary part is +0.0.  For s <= 10 these are the bits
 *     qipb200_state_reduced_density returns; for s = 11..13 it extends that call.  Needs k <= n - k (rho is the
 *     matrix of the qubits passed); otherwise QIPB200_ERR_INVALID_ARG asks for the complement.
 * Routes by s alone, as qipb200_state_purity: s = 0 one norm2 sweep (eigs = {norm2}); 1 <= s <= 10
 * qipb200_state_reduced_density of the side; 11 <= s <= 13 the purity Gram kernel with a store epilogue (one kernel,
 * G on the device: 16 * 4^s bytes, 1 GiB at s = 13; order and error bound in rustqip_b200/csrc/purity.cu).  On routes
 * 1 and 2 G is solved on the device by cuSOLVER (cusolverDnZheevd, eigenvalues only), loaded at run time with dlopen
 * (libcusolver.so.11, then /usr/local/cuda/lib64); the library does not link it.  cuSOLVER's own kernels are not
 * counted by qipb200_kernel_launches, which counts this library's kernels only.  Determinism: rho and out2[0] are
 * bit-identical on repeated calls (fixed-order sums, no atomics); the eigenvalues are whatever cuSOLVER returns, and
 * were bit-identical on repeated calls on an H100 (CUDA 12.9, cuSOLVER 11.7), which cuSOLVER does not promise.
 * Synchronises; the state is read only.  A pending collapse is applied first (after the device buffers are
 * allocated); a pending set_basis state is written first; a permuted layout is read as it is.
 * Errors, all before any device work (a refused call leaves the state and anything pending on it as they were): NULL
 * state, qubits, eigs or out2, k == 0 or k > n, eigs_cap < 2^s, and rho with k > n - k give QIPB200_ERR_INVALID_ARG;
 * a qubit >= n or repeated QIPB200_ERR_BAD_INDEX; s >= 14, sharded and multi-device states, and a cuSOLVER that
 * cannot be loaded (the message gives the loader's reason) QIPB200_ERR_UNSUPPORTED; G or the solver's workspace not
 * allocatable QIPB200_ERR_OOM. */
int qipb200_state_entanglement_spectrum(qipb200_state *state, const uint64_t *qubits, uint32_t k,
                                        double *eigs, size_t eigs_cap, double *rho, double *out2);
/* Host-only (no GPU, ctx-free): out5 = {route (0 norm2, 1 reduced_density, 2 Gram store), s, kernels this library
 * launches (1, 2^m (2^m + 1) with m = max(0, s - 6), or 1), bytes of the device matrix (16 * 4^s; 0 on route 0),
 * 1 if cuSOLVER loads in this process else 0} of the call above on an unsharded n-qubit state with nothing pending.
 * Validates as qipb200_purity_plan does; s >= 14 gives QIPB200_ERR_UNSUPPORTED as the call does. */
int qipb200_entanglement_spectrum_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, uint32_t k,
                                       uint32_t *out5);

/* psi <- exp(-i angles[T-1]/2 P_{T-1}) ... exp(-i angles[0]/2 P_0) psi: Pauli-string rotations, term 0 first; absent in
 * the reference.  Terms are encoded and validated as for qipb200_state_expect_paulis (same codes and messages), with
 * P = i^nY X^x Z^z, so a single 'Z' term is rz(q, angle) and a single 'X' term is Rx(angle); an empty term is the
 * global phase e^{-i angle/2}.  NULL angles with n_terms > 0, or a non-finite angle, give QIPB200_ERR_INVALID_ARG.
 * Every term and angle is checked before any device work: a refused call leaves the amplitudes (and a pending
 * collapse) as they were.  n_terms == 0 is a no-op.  Arithmetic (fixed, so that it can be emulated bit for bit): per
 * term c = cos(angle/2) and s = sin(angle/2) are computed in double on the host and rounded once to the state's
 * precision; each pair (j, j ^ x) is updated from its old values as
 *   psi'_j = (RN(RN(c re psi_j) + RN(s re w_j)), RN(RN(c im psi_j) + RN(s im w_j))),   w_j = -i (P psi)_j (exact)
 * in the state's precision, without FMA, so the result depends neither on how terms share sweeps nor on the layout.
 * Stream-ordered like apply_schedule (does not synchronise; the host arrays are copied before it returns).  One kernel
 * per read-write sweep of the state; a sweep carries a run of consecutive terms whose X/Y letters fit one tile (plus
 * one shared out-of-tile mask); qipb200_pauli_rotation_plan reports the count.  A pending collapse is applied first
 * (one more kernel); a permuted layout is rotated in place and stays as it is.  Sharded and multi-device states:
 * QIPB200_ERR_UNSUPPORTED. */
int qipb200_state_apply_pauli_rotations(qipb200_state *state, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *angles);
/* Host-only (no GPU, ctx-free): the number of read-write sweeps the call above makes for these terms on an unsharded
 * n-qubit state in canonical layout (0 for n_terms == 0).  Validates the terms as the call above does. */
int qipb200_pauli_rotation_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *sweeps);

/* One quantum-trajectory step of n_channels single-qubit channels on distinct qubits (absent in the reference): each
 * channel applies one of its Kraus operators, drawn with its Born probability, and the state is renormalised.
 * Averaging the states of many trajectories gives the channels' density matrix.  Channel c acts on qubits[c] and has
 * n_kraus[c] (1..16) operators that follow those of channel c-1 in `kraus`: 2 x 2 complex matrices of 8 doubles each,
 * row-major, interleaved re/im, rows as outputs, |0> first (the orientation of a qip_op MAT).  Every operator must be
 * diagonal (K01 = K10 = 0) or anti-diagonal (K00 = K11 = 0), so that K|b> = d(b)|b ^ flip>: amplitude and generalised
 * amplitude damping, phase damping, bit and phase flips, depolarizing and any Pauli channel, reset, the Z measurement
 * and their compositions.  A channel is complete when |sum_i |d_i(b)|^2 - 1| <= 1e-12 for b = 0 and 1 (sum K^dagger K
 * = I), and state-dependent when some operator has |d_i(0)|^2 != |d_i(1)|^2 (damping and reset, not Pauli channels).
 * draws (HOST, 1 + n_channels uniforms in [0, 1)) and chosen (HOST, n_channels) are arrays of the caller:
 *   1. x: when some channel is state-dependent, qipb200_state_sample(state, the state-dependent qubits in channel
 *      order, draws[0]) by the same kernels, so bit-identical (bit k of x <-> the k-th such channel); it assumes a
 *      unit-norm state and restores a permuted layout first.  Otherwise no sweep runs and draws[0] is unused.
 *   2. chosen[c] = the smallest i with draws[1 + c] S_b < sum_{i' <= i} e_{i'}, with e_i = re^2 + im^2 of d_i(b) in
 *      double, S_b = sum_i e_i in Kraus order, b = x_c (0 for a state-independent channel); when rounding leaves no
 *      such i, the last i with e_i > 0.  The tuple is then drawn with exactly its probability <psi|(x)_c E_i|psi>.
 *   3. Chosen operators that are positive real multiples of the identity are dropped (they scale psi and p alike):
 *      when every chosen operator is one, no further kernel runs and the state is unchanged bit for bit.
 *   4. q: when a remaining operator has |d(0)|^2 != |d(1)|^2, one read sweep computes S = sum_j |psi_j|^2 prod
 *      |d(bits of j)|^2 and N = sum_j |psi_j|^2 in a fixed order (per-CTA partials added on the host) and q = S / N;
 *      otherwise q is the product of the remaining operators' uniform weights, on the host.
 *   5. *prob = q x (the dropped operators' weights): the probability of the tuple for the normalised state.
 *   6. Unless q == 0 (a zero state, left untouched), one read-write sweep in place on physical bits (a permuted layout
 *      keeps its qubit map): psi'_{j ^ F} = W(j) psi_j, F the XOR mask of the anti-diagonal choices, with
 *      W(j) = RN_prec(((T_0[byte_0(j)] T_1[byte_1(j)]) ...) (1/sqrt q)): T_k are 256-entry complex tables of the
 *      products of d over the channel bits in physical index byte k (bytes without one skipped), built on the host in
 *      double in ascending bit order, all complex products in double without FMA; then, for (a, b) = psi_j,
 *      (RN(RN(Wr a) - RN(Wi b)), RN(RN(Wr b) + RN(Wi a))) in the state's precision without FMA.
 * Errors, all before any device work (a refused call leaves the state and a pending collapse as they were): NULL
 * state or prob, NULL arrays with n_channels > 0, n_kraus not in 1..16, a non-finite entry, the zero matrix, an
 * operator neither diagonal nor anti-diagonal, an incomplete channel (the message names the channel and the
 * operator), and a draw outside [0, 1) give QIPB200_ERR_INVALID_ARG; a qubit >= n or repeated across channels
 * QIPB200_ERR_BAD_INDEX; sharded and multi-device states QIPB200_ERR_UNSUPPORTED.  n_channels == 0 is a no-op
 * (*prob = 1).  A pending collapse is applied first and a pending set_basis state written first.  Synchronises (it
 * returns chosen and prob).  At most three read sweeps (the sample's two, the second only of the chunk its draw
 * landed in, and the weight) and one read-write sweep; qipb200_channels_plan gives the counts. */
int qipb200_state_apply_channels(qipb200_state *state, size_t n_channels, const uint64_t *qubits,
                                 const uint32_t *n_kraus, const double *kraus, const double *draws,
                                 uint32_t *chosen, double *prob);
/* Host-only (no GPU, ctx-free): validates as the call does.  out4 = {state-dependent channels, read sweeps at most,
 * read-write sweeps at most, kernels at most} on an unsharded n-qubit state with nothing pending.  NULL out4, a bad
 * precision or n_qubits not in 1..40 give QIPB200_ERR_INVALID_ARG. */
int qipb200_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels, const uint64_t *qubits,
                          const uint32_t *n_kraus, const double *kraus, uint32_t *out4);

/* qipb200_state_apply_channels for channels on k = 1..4 qubits each (absent in the reference): two-qubit depolarizing
 * and any multi-qubit Pauli channel, correlated dephasing, tensor products of the single-qubit channels above, a
 * multi-qubit reset or Z measurement.  Channel c acts on the arity[c] qubits that follow those of channel c-1 in
 * `qubits` (no qubit twice in the layer) and has n_kraus[c] (1..256) operators that follow those of channel c-1 in
 * `kraus`: 2^k x 2^k complex matrices of 2 4^k doubles each, row-major, interleaved re/im, rows as outputs, in the
 * qip_op MAT sub-index convention: the channel's first qubit is the most significant bit of the row and column index
 * (for k = 1 exactly the input of qipb200_state_apply_channels).  Every operator must have the form K|b> = d(b)|b ^ f>:
 * every column at most one nonzero entry, at row b ^ f for one f shared by all nonzero columns (whole zero columns are
 * allowed: the reset |00><b| is one operator per b), and not the zero matrix.  Complete: |sum_i |d_i(b)|^2 - 1| <= 1e-12
 * for every b in 0..2^k-1; state-dependent: some operator's |d_i(b)|^2 depends on b.  draws, chosen and prob, and the
 * six steps, are those of qipb200_state_apply_channels with these changes:
 *   1. x samples the qubits of the state-dependent channels in channel order and, within a channel, in its qubit order:
 *      bit i of x is the i-th qubit so listed (the measure_probs convention).  The channel value b_c is the channel's
 *      bits of x in the matrix convention, so the two run in opposite directions: for a channel whose qubits sit at
 *      bits s .. s+k-1 of x, b_c = sum_i ((x >> (s + i)) & 1) << (k - 1 - i).
 *   3. A dropped operator has f = 0 and the same positive real d(b) for every b.
 *   4. w(j) = prod_c |d_c(b_c(j))|^2 over the remaining operators, b_c(j) the channel's bits of physical index j.
 *   6. F is the XOR of the chosen masks on their physical bits, and W(j) = RN_prec(((T_0[i_0(j)] T_1[i_1(j)]) ...)
 *      (1/sqrt q)) with two kinds of table: an operator whose physical bits all lie in one index byte folds into that
 *      byte's 256-entry table (its factors multiplied in the order of their lowest physical bit, so a layer of
 *      single-qubit channels gives the tables of qipb200_state_apply_channels), bytes ascending; every other operator
 *      has a table of its 2^k values d(b), indexed by its physical bits gathered in the matrix convention, in channel
 *      order after the byte tables.
 * A layer of single-qubit channels gives the same chosen, prob and state, bit for bit, as qipb200_state_apply_channels.
 * Errors, all before any device work (a refused call leaves the state and a pending collapse as they were): NULL state
 * or prob, NULL arrays with n_channels > 0, an arity not in 1..4, n_kraus not in 1..256, a non-finite entry, the zero
 * matrix, an operator not of the form above (the message names the channel and the operator), an incomplete channel
 * (it names the channel and b) and a draw outside [0, 1) give QIPB200_ERR_INVALID_ARG; a qubit >= n or repeated
 * anywhere in the layer QIPB200_ERR_BAD_INDEX; sharded and multi-device states QIPB200_ERR_UNSUPPORTED.  Sweeps as for
 * qipb200_state_apply_channels; qipb200_multiqubit_channels_plan gives the counts. */
int qipb200_state_apply_multiqubit_channels(qipb200_state *state, size_t n_channels, const uint32_t *arity,
                                            const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus,
                                            const double *draws, uint32_t *chosen, double *prob);
/* Host-only (no GPU, ctx-free): validates as the call does; out4 as for qipb200_channels_plan. */
int qipb200_multiqubit_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels, const uint32_t *arity,
                                     const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus,
                                     uint32_t *out4);

/* One quantum-trajectory step of channels on k = 1..4 qubits each with ANY complete set of Kraus operators (absent in
 * the reference): Kraus sets fitted by process tomography, noisy gates given as one channel ({(A_i (x) A_j) CNOT},
 * {sqrt(p_i) P_i U}), relaxation with a coherent part, damping along any axis.  Channels are encoded as for
 * qipb200_state_apply_multiqubit_channels (arity 1..4, 1..256 operators, 2^k x 2^k matrices in the qip_op MAT
 * convention, no qubit twice in the layer), but any finite nonzero operator is accepted.  Complete: every entry of
 * sum_i K_i^dagger K_i - I (computed in double, operators in order, K^dagger K summed over rows in ascending order) has
 * real and imaginary parts within 1e-12.  draws (HOST, n_channels uniforms in [0, 1), one per channel; there is no
 * sample draw), chosen (HOST, n_channels) and cond (HOST, n_channels, may be NULL) are arrays of the caller; chosen[c]
 * is the operator chosen for channel c, cond[c] the conditional probability of that choice given the earlier ones as
 * computed here, and *prob the product of the cond values in channel order.  Monomial layers (every operator
 * K|b> = d(b)|b ^ f>) are cheaper through qipb200_state_apply_multiqubit_channels (its draws differ: 1 + n).
 *   1. State-independent channels: every K_i^dagger K_i within 1e-12 (per part) of w_i I, w_i = Tr(K_i^dagger K_i) /
 *      2^k (mixed-unitary channels: Pauli and depolarizing channels, {sqrt(p_i) P_i U}).  Drawn without reading the
 *      state: chosen[c] = the rule of step 3 on the w_i, cond[c] = w_i; the operator K / sqrt(w_i) is unitary.
 *   2. Groups: the other channels, cut in channel order into runs of consecutive ones with at most 4 qubits in all (a
 *      group closes when the next channel would exceed 4).
 *   3. Drawing group g on the host in double: rho_g is the reduced density matrix of the group's qubits, indexed in
 *      the matrix convention over the group's qubits in channel order.  Channel by channel, numerator_i =
 *      Re Tr[(M_{i_1} (x) .. (x) M_{i_{j-1}} (x) M_i (x) I) rho_g], M = K^dagger K of the choices already made in the
 *      group and the identity on its later channels, each numerator clamped at 0; S = sum_i numerator_i in order; the
 *      choice is the smallest i with draw S < sum_{i' <= i} numerator_i', else the last i with numerator_i > 0; cond =
 *      numerator_i / S.
 *   4. Sweeps: one read sweep (qipb200_state_reduced_density's kernels) gives rho_1; then one read-write sweep per
 *      group applies its chosen operators, each as K / sqrt(cond[c]), and accumulates rho_{g+1} from the amplitudes
 *      as stored (fixed grid and order, no atomics: deterministic).  After the groups, the state-independent channels'
 *      operators K / sqrt(w_i) run through qipb200_state_apply_schedule as MAT ops in channel order (the planner fuses
 *      them); a chosen operator that is a positive real multiple of the identity is dropped.  They commute with the
 *      groups: the qubits are disjoint.
 *   5. Arithmetic of a group's apply: each scaled operator K' = K * (1 / sqrt(cond)) is computed in double on the host
 *      and each part rounded once to the state's precision; per channel, in channel order, every fibre x of its
 *      physical bits (x_b at column b in the matrix convention) becomes y_r = ((t_r0 + t_r1) + t_r2) + ...,
 *      t_rb = (RN(RN(K'_re x_re) - RN(K'_im x_im)), RN(RN(K'_re x_im) + RN(K'_im x_re))), in the state's precision
 *      without FMA, columns ascending.  So the state can be reproduced bit for bit from chosen and cond.
 *   6. When some group finds S = 0 (a zero state, or one that became zero), the call stops there: chosen and cond are
 *      0 for every channel, *prob = 0, and a zero input state is left untouched.
 * Errors, all before any device work (a refused call leaves the state and anything pending as they were): NULL state
 * or prob, NULL arrays with n_channels > 0, an arity not in 1..4, n_kraus not in 1..256, a non-finite entry, the zero
 * matrix, an incomplete channel (the message names the channel and the matrix entry) and a draw outside [0, 1) give
 * QIPB200_ERR_INVALID_ARG; a qubit >= n or repeated anywhere in the layer QIPB200_ERR_BAD_INDEX; sharded and
 * multi-device states QIPB200_ERR_UNSUPPORTED.  n_channels == 0 is a no-op (*prob = 1).  A pending collapse is
 * applied first and a pending set_basis state written first; a permuted layout is worked on in physical bits.
 * Synchronises.  qipb200_kraus_channels_plan gives the counts. */
int qipb200_state_apply_kraus_channels(qipb200_state *state, size_t n_channels, const uint32_t *arity,
                                       const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus,
                                       const double *draws, uint32_t *chosen, double *cond, double *prob);
/* Host-only (no GPU, ctx-free): validates as the call does.  out4 = {groups r, read sweeps (1 if r > 0), read-write
 * sweeps of the groups (r), kernels of the groups (2r + 1 if r > 0)} on an unsharded n-qubit state with nothing
 * pending; the passes of the state-independent channels' schedule are not counted.  NULL out4, a bad precision or
 * n_qubits not in 1..40 give QIPB200_ERR_INVALID_ARG. */
int qipb200_kraus_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels, const uint32_t *arity,
                                const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, uint32_t *out4);

/* ---- Exact noisy simulation on density matrices (absent in the reference) ------------------------------------------
 * The exact mixed state of a noisy circuit, where the trajectory calls above give one pure sample: purity, entropy
 * and fidelity are not averages of trajectory quantities, and effects of 1e-3 noise are below the statistical error
 * of thousands of trajectories.
 * Representation: a density matrix rho of n >= 1 qubits is a qipb200_state of 2n qubits (no new handle).  Row qubit q
 * is state qubit q and column qubit q is state qubit n + q, so in the qip_op convention rho_rc is the amplitude at
 * index r * 2^n + c: rows are contiguous and the downloaded vector, read as a row-major 2^n x 2^n matrix, is rho.
 * |i><i| is qipb200_state_set_basis(rho, i * 2^n + i) (it stays pending: the first fused pass is load-free), and
 * Tr rho^2 = sum |rho_rc|^2 is qipb200_state_norm2 of the vector for Hermitian rho.  The qipb200_state_* entries keep
 * their meaning on the raw vector.  The qipb200_density_* entries take the 2n-qubit state: an odd qubit count gives
 * QIPB200_ERR_INVALID_ARG, sharded and multi-device states QIPB200_ERR_UNSUPPORTED; all checks run before any device
 * work, so a refused call leaves rho (and anything pending on it) as it was.  A pending set_basis or collapse is
 * applied first, and a permuted layout (QIPB200_ROTATE) is read where it is.  The readouts synchronise; those computed
 * by this library's kernels are deterministic (fixed grids and orders, no atomics); the spectrum's eigen-solve is
 * cuSOLVER's, whose bits are not promised to repeat. */

/* Gates and channels, interleaved, in one fused schedule on vec(rho).  Channel c runs after ops[0 .. channel_pos[c]);
 * channels at one position run in channel order; channel_pos is non-decreasing and at most n_ops.  Channels are
 * encoded and checked as for qipb200_state_apply_kraus_channels (arity 1..4, 1..256 operators, complete to 1e-12),
 * except that a qubit may appear in several channels: they run one after the other.  Ops are checked by
 * qipb200_validate_op on n qubits.  The doubled schedule: each op, then its conjugate on the column qubits (every
 * index + n, MAT and sparse values conjugated, Swap and Control structure unchanged); each channel one MAT op on
 * [q_1..q_k, q_1 + n..q_k + n] with S = sum_i kron(K_i, conj K_i), formed in double, terms added in ascending i, each
 * part rounded once to the state's precision.  It runs through qipb200_state_apply_schedule with flags, so the result
 * is bit-identical to that call on the schedule qipb200_density_schedule writes when both run the same kernels (with
 * the default QIPB200_JIT=async a pass may run on the interpreter kernel while its generated kernel compiles, and the
 * two may round differently).  Errors: QIPB200_ERR_INVALID_ARG for
 * NULL arrays, a bad channel_pos and the channel refusals of apply_kraus_channels; a qubit >= n gives
 * QIPB200_ERR_BAD_INDEX (channels) or validate_op's status (ops). */
int qipb200_density_apply(qipb200_state *rho, const qip_op *ops, size_t n_ops, size_t n_channels,
                          const uint64_t *channel_pos, const uint32_t *arity, const uint64_t *qubits,
                          const uint32_t *n_kraus, const double *kraus, uint32_t flags);
/* Host-only (no GPU, ctx-free): checks as qipb200_density_apply does for an n-qubit rho (n in 1..20, a known
 * precision) and writes the doubled schedule in the QIPS v1 format (n_qubits = 2n) to buf.  *len is set to the size;
 * when buf is NULL or cap is smaller the call returns QIPB200_ERR_SIZE_MISMATCH.  A Rust or C caller exports a noisy
 * circuit with it. */
int qipb200_density_schedule(qip_prec prec, uint32_t n, const qip_op *ops, size_t n_ops, size_t n_channels,
                             const uint64_t *channel_pos, const uint32_t *arity, const uint64_t *qubits,
                             const uint32_t *n_kraus, const double *kraus, void *buf, size_t cap, size_t *len);
/* rho = |psi><psi| (not normalised): psi has n qubits, rho's context and precision, and is unsharded (else
 * QIPB200_ERR_SIZE_MISMATCH / QIPB200_ERR_UNSUPPORTED).  rho's pending work is dropped and its layout becomes the
 * canonical one; a permuted psi is restored first.  One write sweep of rho. */
int qipb200_density_from_state(qipb200_state *rho, qipb200_state *psi);
/* out[m] = sum of Re rho_rr over the r whose bits on indices equal m; bit i of m is indices[i] (the convention of
 * qipb200_state_measure_probs); n_indices = 0 gives out[0] = Tr rho.  Reads only the 2^n diagonal entries.  A qubit
 * >= n or repeated gives QIPB200_ERR_BAD_INDEX. */
int qipb200_density_measure_probs(qipb200_state *rho, const uint64_t *indices, uint32_t n_indices, double *out);
/* out[t] = Re Tr(rho P_t) for Pauli strings encoded and checked as for qipb200_state_expect_paulis on n qubits.  Each
 * term gathers 2^n entries of rho; up to 4096 terms per launch. */
int qipb200_density_expect_paulis(qipb200_state *rho, const uint64_t *qubits, const char *paulis,
                                  const uint32_t *term_len, size_t n_terms, double *out);
/* rho_A = Tr_B rho for k = 1..min(n, 10) kept qubits: out is row-major 2^k x 2^k, interleaved re/im, bit i of the
 * indices the value of qubits[i] (the layout of qipb200_state_reduced_density).  Exactly Hermitian: the entries a <= a'
 * are summed and mirrored, the diagonal's imaginary part is 0.0.  k > 10 gives QIPB200_ERR_UNSUPPORTED. */
int qipb200_density_reduced(qipb200_state *rho, const uint64_t *qubits, uint32_t k, double *out);
/* out2 = {Re, Im} <psi|rho|psi>, psi as for qipb200_density_from_state.  One read sweep of rho, accumulated in double;
 * the fidelity of a normalised rho with a unit vector psi is out2[0]. */
int qipb200_density_fidelity(qipb200_state *rho, qipb200_state *psi, double *out2);
/* The 2^n eigenvalues of rho in descending order into eigs (HOST, 2^n doubles), for n <= 13 (else
 * QIPB200_ERR_UNSUPPORTED): rho is widened to double on the device and solved by cuSOLVER (as
 * qipb200_state_entanglement_spectrum); when cuSOLVER cannot be loaded the call returns QIPB200_ERR_UNSUPPORTED. */
int qipb200_density_spectrum(qipb200_state *rho, double *eigs);

/* Classical functions applied to a register: U |x>|y> = e^{i theta(x)} |x>|y XOR f(x)> for a function given as a table
 * (the row rule of the reference's FunctionOpIterator, qip-iterators/src/iterators/qubit_iterators.rs:221-271, which
 * no MatrixOp reaches): Grover and Shor oracles, modular arithmetic, cost-table phases.
 * Bit convention (that of measure_probs): bit i of x is the value of qubit in_qubits[i], and bit i of f(x) is XORed
 * into qubit out_qubits[i].  In the reference's numbering of the op's rows (indices = in ++ out, indices[0] the most
 * significant bit), row (x, y) therefore reads column (x, y ^ flip_bits(n_out, f(flip_bits(n_in, x)))).
 *
 * A function is a handle bound to the context it was made on, kept on its device, and applies to states of either
 * precision.  function_new validates and uploads the table once (an oracle is applied many times): f[x] for
 * x < 2^n_in (n_out-bit values, kept as u32; may be NULL when n_out == 0) and, when theta is not NULL, the pair
 * (cos theta[x], sin theta[x]) computed in double on the host.  Errors: NULL ctx or out, n_in == 0, f NULL with
 * n_out > 0, n_out == 0 with theta NULL (nothing to apply), f[x] >= 2^n_out or a non-finite theta[x] (the message
 * names the first such x) give QIPB200_ERR_INVALID_ARG; n_in > 26 (the tables would exceed 1.25 GiB), n_out > 32 and
 * multi-device contexts QIPB200_ERR_UNSUPPORTED; a failed device allocation QIPB200_ERR_OOM.  Synchronises.
 * function_free is stream-ordered (cudaFreeAsync on the context's stream), so it may follow an apply at once; free
 * every function before its context is shut down. */
typedef struct qipb200_function qipb200_function;
int qipb200_function_new(qipb200_ctx *ctx, uint32_t n_in, uint32_t n_out, const uint64_t *f, const double *theta, qipb200_function **out);
void qipb200_function_free(qipb200_function *fn);
/* psi <- U psi with x on the fn's n_in qubits in_qubits and y on its n_out qubits out_qubits (may be NULL when
 * n_out == 0).  Arithmetic (fixed, so that it can be emulated bit for bit): without theta the op moves amplitudes and
 * is exact (-0 is preserved); with theta, c = RN(cos theta(x)) and s = RN(sin theta(x)) in the state's precision and,
 * for the partner amplitude (a, b) = psi_{j ^ d},
 *   psi'_j = (RN(RN(c a) - RN(s b)), RN(RN(c b) + RN(s a)))
 * without FMA, so the result depends neither on the path nor on the layout.  Errors, all before any device work (a
 * refused call leaves the state and a pending collapse as they were): NULL state or fn, or NULL qubit arrays where
 * their count is > 0, QIPB200_ERR_INVALID_ARG; a qubit >= n, or one repeated within or across the two registers,
 * QIPB200_ERR_BAD_INDEX; sharded and multi-device states QIPB200_ERR_UNSUPPORTED; fn made on another context
 * QIPB200_ERR_INVALID_ARG.  A pending collapse is applied first (one more kernel); a permuted layout is worked on where
 * it is and keeps its qubit map.  Stream-ordered like apply_schedule (does not synchronise); exactly one kernel, one
 * read-write sweep of the state: a staged tile path when the low 4 index bits and the out register's index bits fit
 * one tile of T_max = 11 (f64) or 12 (f32) bits, a pair path otherwise (rustqip_b200/csrc/function.h). */
int qipb200_state_apply_function(qipb200_state *state, const qipb200_function *fn, const uint64_t *in_qubits, const uint64_t *out_qubits);
/* Host-only (no GPU, ctx-free): out2 = {path: 0 staged tile / 1 pair, tile bits of the staged path (0 for pair)} of the
 * call above on an unsharded n-qubit state in canonical layout.  NULL out2, a bad precision or n_qubits not in 1..40
 * give QIPB200_ERR_INVALID_ARG; n_in and n_out are checked as function_new checks them, the qubits as the call does. */
int qipb200_function_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *in_qubits, uint32_t n_in, const uint64_t *out_qubits, uint32_t n_out, uint32_t *out2);

/* Functions given as CUDA source (absent in the reference): the same op U |x>|y> = e^{i theta(x)} |x>|y XOR f(x)> with f
 * and theta evaluated on the device, so no table is built or uploaded and n_in may span the whole state.  `source` is
 * CUDA C++ that defines
 *   __device__ uint64_t qip_f(uint64_t x)                   when n_out > 0, and
 *   __device__ double qip_theta(uint64_t x, const double *p) with QIPB200_FN_CODE_THETA,
 * where p holds the handle's n_params parameters (set by function_set_params, all 0 at creation); the bit convention
 * is that of function_new.  The source is compiled with NVRTC for sm_90a together with the kernels of the table path
 * (--fmad=false, the options of the generated pass kernels), through the same process cache and QIPB200_JIT_CACHE_DIR
 * on-disk cache.  Before the handle is returned, one kernel evaluates f over every x < 2^n_in and one evaluates theta
 * with the zero parameters: f(x) >= 2^n_out or a non-finite theta(x) refuses the handle, naming the first such x.
 * Errors: NULL ctx or out, NULL or empty source, n_in == 0, unknown flags, n_out == 0 without THETA (nothing to apply),
 * n_params > 16, an NVRTC compile error (the NVRTC log goes to `log`, when log_len > 0, and to last_error) and the
 * refusals above give QIPB200_ERR_INVALID_ARG; n_out > 32, n_in + n_out > 34, multi-device contexts, and a process
 * without NVRTC or the driver API (the reason in `log`) QIPB200_ERR_UNSUPPORTED.  Synchronises.
 * A code handle applies with qipb200_state_apply_function exactly as a table does (same checks, path plan, one kernel
 * and one read-write sweep), with c = RN(cos theta(x)) and s = RN(sin theta(x)) from sincos evaluated in double on the
 * device.  function_free of a code handle waits for the context's stream before it unloads the program. */
enum { QIPB200_FN_CODE_THETA = 1u /* the source defines qip_theta */ };
int qipb200_function_new_code(qipb200_ctx *ctx, uint32_t n_in, uint32_t n_out, const char *source, uint32_t flags, uint32_t n_params, char *log, size_t log_len, qipb200_function **out);
/* Set the n_params parameters theta is evaluated with (n_params must equal the handle's).  With THETA, one kernel first
 * evaluates theta(x, params) for every x < 2^n_in; a non-finite value gives QIPB200_ERR_INVALID_ARG naming the first
 * such x and keeps the previous parameters.  NULL fn, or NULL params with n_params > 0, QIPB200_ERR_INVALID_ARG; a
 * table handle QIPB200_ERR_UNSUPPORTED.  Synchronises.  Applies queued before keep the parameters they were queued
 * with. */
int qipb200_function_set_params(qipb200_function *fn, const double *params, uint32_t n_params);
/* Host-only (no GPU, ctx-free): build and compile the program of function_new_code, as qipb200_jit_precompile does for
 * passes, so that code can be checked without a GPU.  Same argument checks and codes as function_new_code; the NVRTC
 * log (errors, or warnings) goes to `log`. */
int qipb200_function_code_compile(uint32_t n_in, uint32_t n_out, const char *source, uint32_t flags, uint32_t n_params, char *log, size_t log_len);
/* f(x) into f_out[i] and (cos theta(x), sin theta(x)) in double into cs_out[2i], cs_out[2i + 1], for x = x0 + i,
 * i < count, evaluated ON THE DEVICE by the functions the apply kernels use (the table lookups, or the compiled code
 * with the current parameters): the apply rounds these (c, s) once to the state's precision.  Either output may be
 * NULL; without a phase cs_out gets (1, 0) and without an out register f_out gets 0.  x0 + count > 2^n_in or NULL fn
 * give QIPB200_ERR_INVALID_ARG.  Synchronises. */
int qipb200_function_tabulate(const qipb200_function *fn, uint64_t x0, uint64_t count, uint64_t *f_out, double *cs_out);
/* *out = sum_j |psi_j|^2 theta(x(j), p) = <psi|D|psi> for D = diag theta, x(j) the value of in_qubits in index j: the
 * diagonal expectation value of a code handle with THETA (e.g. the QAOA energy <C> of any cost C), on the state AS IT
 * IS (not renormalised, like expect_paulis).  One kernel, one read sweep.  Accumulated in double for both precisions
 * (f32 amplitudes are widened before use) over a fixed grid with per-CTA partials summed on the host in a fixed order,
 * no floating-point atomics: the same state and parameters give bit-identical out.  The order and the first-order
 * rounding bound are documented in rustqip_b200/csrc/function.cu.  Synchronises.  Errors, all before any device work (a
 * refused call leaves the state and a pending collapse as they were): NULL state, fn or out QIPB200_ERR_INVALID_ARG; a
 * table handle or a code handle without THETA QIPB200_ERR_UNSUPPORTED (a table keeps cos theta and sin theta, not
 * theta); in_qubits checked as apply_function checks them; sharded and multi-device states QIPB200_ERR_UNSUPPORTED; fn
 * made on another context QIPB200_ERR_INVALID_ARG.  A pending collapse is applied first (one more kernel); a permuted
 * layout is read where it is. */
int qipb200_state_expect_function(qipb200_state *state, const qipb200_function *fn, const uint64_t *in_qubits, double *out);

/* dst <- sum_h coeffs[h] P_h src, out of place: H|psi> for a Hamiltonian given as a real Pauli sum (absent in the
 * reference).  Terms are encoded and validated as for qipb200_state_expect_paulis (same codes and messages); an empty
 * term is coeffs[h] times the identity.  NULL coeffs with n_terms > 0, a non-finite coefficient or dst == src give
 * QIPB200_ERR_INVALID_ARG; states of different contexts, precisions or sizes QIPB200_ERR_SIZE_MISMATCH; sharded and
 * multi-device states QIPB200_ERR_UNSUPPORTED.  Every check runs before any device work: a refused call leaves both
 * states (and a pending collapse) as they were.  n_terms == 0 sets dst to zero.  A collapse pending on src is applied
 * first, one pending on dst is dropped (dst is overwritten), and dst takes src's layout.  Arithmetic: per amplitude the
 * terms of one X/Y mask sum their signed coefficients in double, the products with the partner amplitude (widened to
 * double) are added in a fixed order, and each read-write sweep stores the sum rounded to the state's precision; the
 * order and the forward error bound are documented in rustqip_b200/csrc/gradient.cu.  The terms are grouped into
 * sweeps on physical index bits, so a permuted layout may round differently; the same inputs in the same layout give
 * the same bits.
 * Stream-ordered (does not synchronise).  One kernel per sweep; qipb200_pauli_sum_plan reports the count. */
int qipb200_state_apply_pauli_sum(qipb200_state *dst, const qipb200_state *src, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *coeffs);
/* Host-only (no GPU, ctx-free): the number of sweeps qipb200_state_apply_pauli_sum makes for these terms on an
 * unsharded n-qubit state in canonical layout (0 for n_terms == 0).  Validates the terms as the call does. */
int qipb200_pauli_sum_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *sweeps);

/* Energy and gradient of a Pauli-rotation circuit by the adjoint method (absent in the reference).  With
 * U = R_{T-1} ... R_0, R_t = exp(-i angles[t]/2 P_t) (the convention of qipb200_state_apply_pauli_rotations) and
 * H = sum_h coeffs[h] Q_h, on entry `state` holds psi0 and the call
 *   1. state <- U state, exactly qipb200_state_apply_pauli_rotations;
 *   2. work <- H state, exactly qipb200_state_apply_pauli_sum;
 *   3. for t = T-1 down to 0: grad[t] = Im <work|P_t|state>, then state <- R_t^dagger state, work <- R_t^dagger work;
 *      *energy = Re <work|state> before the first undo.
 * In exact arithmetic grad[t] = dE/dangles[t] for E = <psi0|U^dagger H U|psi0>.  A parameter shared by several terms
 * (one QAOA angle on many strings) has the sum of their entries as its derivative.  The undo uses the rotation update
 * with the same host-rounded c and the negated s, so `state` ends bit-identical to that arithmetic run forward and then
 * backward: psi0 only up to rounding (re-prepare it when it is needed exactly); `work` ends holding U^dagger H U psi0.
 * Inner products are accumulated in double in a fixed order: the same inputs give the same bits.  Validation as above
 * for both term lists; NULL or non-finite angles or coeffs (when their list is not empty), NULL energy, NULL grad with
 * n_terms > 0 or state == work give QIPB200_ERR_INVALID_ARG, mismatched states QIPB200_ERR_SIZE_MISMATCH, sharded
 * states QIPB200_ERR_UNSUPPORTED, all before any device work.  Pending collapses and layout: `work` plays dst and
 * `state` src of qipb200_state_apply_pauli_sum.  Synchronises.  Launches f + s + 2 b kernels for the three counts
 * {f, s, b} of qipb200_pauli_gradient_plan (plus one for a pending collapse on `state`). */
int qipb200_state_pauli_energy_gradient(qipb200_state *state, qipb200_state *work, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *angles, const uint64_t *ham_qubits, const char *ham_paulis, const uint32_t *ham_term_len, size_t n_ham, const double *coeffs, double *energy, double *grad);
/* Host-only (no GPU, ctx-free): out3 = {forward, sum, backward} sweeps of the call above on an unsharded n-qubit state
 * in canonical layout.  Validates both term lists as the call does. */
int qipb200_pauli_gradient_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const uint64_t *ham_qubits, const char *ham_paulis, const uint32_t *ham_term_len, size_t n_ham, uint32_t *out3);

/* The quantum geometric tensor of a Pauli-rotation circuit (absent in the reference).  With U = R_{T-1} ... R_0,
 * R_t = exp(-i angles[t]/2 P_t) (the convention of qipb200_state_apply_pauli_rotations), psi0 the state on entry,
 * psi_t = R_t ... R_0 psi0, psi = U psi0 and d_t psi = R_{T-1} ... R_{t+1} (-i/2) P_t psi_t:
 *   qgt[2 (i T + j) + {0, 1}] = Re, Im of G_ij = <d_i psi|d_j psi> - <d_i psi|psi><psi|d_j psi>,
 *   expect[t] = e_t = <psi_t|P_t|psi_t> (also <P_t> just before R_t; expect may be NULL).
 * Re G is the Fubini-Study metric (the matrix of a quantum-natural-gradient step and of McLachlan's imaginary-time
 * equation), 4 Re G the quantum Fisher information, Im G the antisymmetric part of variational real-time evolution.
 * In exact arithmetic that is the tensor for a unit-norm psi0; the call computes
 *   G_tt = (|psi_t|^2 - e_t^2) / 4,   G_ij = (M_ij - e_i e_j) / 4 for i < j,   G_ji = conj(G_ij) (Im G_tt = +0.0),
 * with M_ij = <mu|P_j|phi>, phi = psi_i and mu = P_i psi_i both carried forward through R_{i+1} .. R_{j-1}.  For
 * i = 0 .. T-1 in order: a fork (state <- R_i state with the arithmetic of apply_pauli_rotations, work_a <- state,
 * work_b <- P_i state exactly, |psi_i|^2 and e_i summed in double), then the segment: the sweeps of terms i+1 .. T-1,
 * each term j adding Re and Im of <work_b|P_j|work_a> and then rotating both work states by R_j with the same
 * host-rounded c and s.  The order is fixed, so the same inputs give the same bits; the forward error bound is
 * documented in rustqip_b200/csrc/gradient.cu.  At exit `state` holds U psi0 bit-identical to
 * qipb200_state_apply_pauli_rotations, `work_a` the same bits and `work_b` P_{T-1} U psi0 exactly.  An empty string
 * is a global phase: its row and column of G are zero up to rounding.  A parameter shared by several strings gets
 * A^T G A for its term-to-parameter matrix A (on the host).
 * Terms are validated as for qipb200_state_expect_paulis (same codes and messages).  A state passed twice, NULL or
 * non-finite angles or NULL qgt (n_terms > 0) give QIPB200_ERR_INVALID_ARG; states of different contexts, precisions
 * or sizes QIPB200_ERR_SIZE_MISMATCH; sharded or multi-device states, and n_terms > 2048 (the result alone is 2 T^2
 * doubles), QIPB200_ERR_UNSUPPORTED; all before any device work (a refused call leaves the three states and a pending
 * collapse as they were).  A collapse pending on state is applied first; ones pending on the work states are dropped,
 * and they take the state's layout (a permuted layout is worked on in physical bits and keeps its qubit map).
 * n_terms == 0 launches no kernel beyond a pending collapse on state and leaves the work states as they are.
 * Synchronises once, at the end.  Launches the kernel count of qipb200_pauli_geometric_tensor_plan (plus one for a
 * pending collapse). */
int qipb200_state_pauli_geometric_tensor(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *angles, double *qgt, double *expect);
/* Host-only (no GPU, ctx-free): out3 = {forks (= T), segment sweeps (the sum over i of the sweeps of terms
 * i+1 .. T-1), kernels the call launches (T + 2 sweeps + 1, or 0 for T == 0)} on an unsharded n-qubit state in
 * canonical layout.  Validates the terms as the call does (n_terms > 2048: QIPB200_ERR_UNSUPPORTED). */
int qipb200_pauli_geometric_tensor_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *out3);

/* state <- exp(-i time H) state for a real Pauli sum H = sum_h coeffs[h] P_h, by a Chebyshev expansion (absent in the
 * reference).  Terms are encoded and validated as for qipb200_state_apply_pauli_sum (same codes and messages).  The
 * identity terms sum to a; the others give the half-width b = sum |coeffs[h]| >= |H - a|; with H~ = (H - a) / b,
 *   exp(-iHt) = e^{-iat} sum_k (2 - delta_k0) (-i)^k J_k(bt) T_k(H~),
 * cut at the smallest degree K >= 2 whose tail bound tau_K = 2 sum_(j > K) |J_j(bt)| is <= tol, so in exact arithmetic
 * |result - exp(-iHt) state| <= tau_K |state|.  *degree = K and *tail = tau_K.  The recurrence T_(k+1) = 2 H~ T_k -
 * T_(k-1) runs in work_a and work_b (scratch: their contents afterwards are unspecified) with one read-write sweep of
 * the sum plan per kernel, and state accumulates the series; the arithmetic is fixed and its forward error bound is
 * documented in rustqip_b200/csrc/gradient.cu, the coefficients in rustqip_b200/csrc/evolve.h.  time == 0 or
 * n_terms == 0: a no-op (K = 0, no kernel).  b == 0 (identity terms only): the global phase e^{-iat}, exactly
 * qipb200_state_apply_pauli_rotations of one empty term by the angle 2 RN(a time) (K = 0, one kernel).
 * Errors, all before any device work (a refused call leaves the three states and a pending collapse as they were):
 * a state passed twice, NULL or non-finite coeffs (n_terms > 0), a non-finite time, tol not in (0, 1) or NULL
 * degree / tail give QIPB200_ERR_INVALID_ARG; states of different contexts, precisions or sizes
 * QIPB200_ERR_SIZE_MISMATCH; sharded or multi-device states, and K > 65536 (split the time over several calls),
 * QIPB200_ERR_UNSUPPORTED.  A collapse pending on state is applied first; ones pending on the work states are dropped,
 * and they take the state's layout.  Stream-ordered (the host arrays are copied before it returns); launches
 * K x sweeps kernels (qipb200_pauli_evolution_plan), plus one for a pending collapse. */
int qipb200_state_evolve_pauli_sum(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *coeffs, double time, double tol, uint32_t *degree, double *tail);
/* Host-only (no GPU, ctx-free): the plan of the call above on an unsharded n-qubit state in canonical layout.
 * out3 = {degree K, sweeps per step, kernels}, *tail = tau_K, and when coeffs_out is not NULL and coeffs_cap (in
 * doubles) is at least 2 (K + 1), coeffs_out = C_0..C_K as (re, im) pairs, the series coefficients including
 * e^{-iat} (C_0 = 1 for a no-op, e^{-iat} alone for identity-only H).  Validates as the call does. */
int qipb200_pauli_evolution_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *coeffs, double time, double tol, uint32_t *out3, double *tail, double *coeffs_out, size_t coeffs_cap);

/* The lowest eigenvalue of a real Pauli sum H = sum_h coeffs[h] P_h reachable from the start state, by plain Lanczos
 * (no reorthogonalisation) on the device (absent in the reference).  Terms are encoded and validated as for
 * qipb200_state_apply_pauli_sum (same codes and messages).  The identity terms sum to a; the others give the scale
 * b = sum |coeffs[h]|.  From v_0 = state / |state| step j forms alpha_j = <v_j|H v_j> and beta_(j+1) =
 * |H v_j - alpha_j v_j - beta_j v_(j-1)|; after m steps the host takes the lowest eigenvalue theta of the tridiagonal
 * T_m and its unit eigenvector y (qipb200_lanczos_ritz) and stops at the first m with the estimate
 * rho_m = beta_m |y_(m-1)| <= tol b (*converged = 1; a breakdown, beta_m = 0, counts), else at max_steps
 * (*converged = 0, the best estimate returned).  Only the part of H's spectrum the state has weight on is reachable: a
 * start state in a symmetry sector (fixed S_z, parity, ...) gives that sector's ground state.  *steps = m;
 * alpha[0..m) and beta[0..m] (beta[0] = |state|) are written when not NULL (room for max_steps and max_steps + 1).
 * flags 0 (energy only): the state is read and not written; out3 = {theta, rho_m, 0}.  QIPB200_LANCZOS_VECTOR: a
 * second pass reruns the recurrence with the same scalars (so the same bits) and accumulates x = sum_j y_j v_j into
 * the state, which ends as x / |x|; out3 = {E, |H x - E x|, |x| before normalisation}, E = <x|H x>, both computed on
 * the device after the pass (|x| far from 1 shows loss of orthogonality).  In exact arithmetic some eigenvalue of H
 * lies within out3[1] of out3[0] in both modes.  The arithmetic, its order and the rounding bounds of alpha and beta
 * are documented in rustqip_b200/csrc/lanczos.cu; the same inputs give the same bits.  work_a and work_b are scratch
 * (their contents afterwards are unspecified).  b == 0 (no terms, or identity terms only): every vector is an
 * eigenvector: out3 = {a, 0, 1 or 0}, *steps = 0, *converged = 1, and vector mode normalises the state.
 * Errors: a state passed twice, NULL or non-finite coeffs (n_terms > 0), max_steps 0 or above 4096, tol not in
 * (0, 1), unknown flags or NULL steps / converged / out3 give QIPB200_ERR_INVALID_ARG; states of different contexts,
 * precisions or sizes QIPB200_ERR_SIZE_MISMATCH; sharded or multi-device states QIPB200_ERR_UNSUPPORTED; all before
 * any device work (a refused call leaves the three states and a pending collapse as they were).  A start state of zero
 * (or non-finite) norm gives QIPB200_ERR_INVALID_ARG after the first read sweep, the state unchanged.  A collapse
 * pending on state is applied first; ones pending on the work states are dropped, and they take the state's layout.
 * Synchronises once per first-pass step.  With {s, k1, k2, k0} = qipb200_pauli_lanczos_plan it launches 1 + m k1
 * kernels (energy only) or m k1 + (m - 1) k2 + k0 (vector mode), plus one for a pending collapse; b == 0 launches 1
 * (2 in vector mode). */
enum { QIPB200_LANCZOS_VECTOR = 1u };
int qipb200_state_lanczos_pauli_sum(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, const double *coeffs, uint32_t max_steps, double tol, uint32_t flags, uint32_t *steps, uint32_t *converged, double *alpha, double *beta, double *out3);
/* Host-only (no GPU, ctx-free): out4 = {sum sweeps per step, kernels per first-pass step, kernels per second-pass step,
 * kernels outside the steps in vector mode} of the call above on an unsharded n-qubit state in canonical layout
 * ({0, 0, 0, 2} when every term is the identity).  Validates the terms as the call does. */
int qipb200_pauli_lanczos_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms, uint32_t *out4);
/* Host-only (no GPU, ctx-free): the tridiagonal solve the call runs after each step, on alpha[0..m) and beta[0..m]
 * laid out as above: the lowest eigenvalue *theta of T_m (diagonal alpha, off-diagonal beta[1..m)), its unit
 * eigenvector y (m doubles, sign fixed by y[0] >= 0; may be NULL) and *estimate = beta[m] |y[m-1]|.  NULL alpha, beta,
 * theta or estimate, m == 0 or a non-finite value give QIPB200_ERR_INVALID_ARG. */
int qipb200_lanczos_ritz(const double *alpha, const double *beta, uint32_t m, double *theta, double *y, double *estimate);

/* ---- multi-GPU: the 2^n state sharded by its top log2(world) index bits,
 *      one process per GPU (absent in the reference; its only hook is the
 *      input_offset/output_offset slice model, matrix_ops.rs:74-89) -------------- */

#define QIPB200_IPC_HANDLE_BYTES 64

/* Create rank `rank`'s shard (2^(n - log2 world) amplitudes) of an n-qubit state.
 * world_size must be a power of two. */
int qipb200_state_new_sharded(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, int rank,
                              int world_size, qipb200_state **state);
/* Export this shard's CUDA-IPC handles (amplitude buffer + flag page), each
 * QIPB200_IPC_HANDLE_BYTES long, for the caller to all-gather. */
int qipb200_state_ipc_export(qipb200_state *state, void *amp_handle, void *flag_handle);
/* Import all peers' handles (world_size * QIPB200_IPC_HANDLE_BYTES each, rank order):
 * maps every peer shard over NVLink so exchange kernels can load/store it directly. */
int qipb200_state_ipc_import(qipb200_state *state, const void *amp_handles, const void *flag_handles);
/* Current logical-qubit -> physical-index-bit map of a sharded state (n entries):
 * the exchange pass migrates "hot" qubits to local bits instead of moving them back. */
int qipb200_state_qubit_map(qipb200_state *state, uint32_t *bit_of_qubit);
/* Bytes this rank has pulled/pushed over NVLink so far. */
int qipb200_state_exchange_bytes(qipb200_state *state, uint64_t *bytes);

/* Host-side plan only (no GPU, ctx may be NULL): for each op, report whether a
 * world_size-way sharded n-qubit state needs an exchange to apply it
 * (needs_exchange[i] = number of rank bits the op acts on non-diagonally). */
int qipb200_plan_exchanges(qip_prec prec, uint32_t n_qubits, int world_size, const qip_op *ops,
                           size_t n_ops, uint32_t *needs_exchange);

/* ---- N3: gate-schedule wire format "QIPS" -----------------------------------------
 * The reference's only export is OpenQASM 2.0 (qip/src/qasm.rs:112-184), which drops MAT
 * entries; QIPS carries exactly the `qip_op` records this ABI consumes (byte layout:
 * rustqip_b200/wire.py, rustqip_b200/csrc/wire.cpp).  Host-only: no GPU, no context.
 *
 * parse: builds an owned schedule from `len` bytes; on a malformed buffer returns
 * QIPB200_ERR_INVALID_ARG with a message in errbuf (may be NULL).  The returned records stay valid
 * until qipb200_schedule_free and can be passed to qipb200_state_apply_schedule /
 * qipb200_calculate_state as they are.
 * serialise: returns the number of bytes the schedule needs and writes them when cap suffices
 * (call with buf=NULL to size the buffer); 0 on a malformed op tree. */
typedef struct qipb200_schedule qipb200_schedule;
int qipb200_schedule_parse(const void *buf, size_t len, qipb200_schedule **out, char *errbuf, size_t errlen);
const qip_op *qipb200_schedule_ops(const qipb200_schedule *s, size_t *n_ops, uint32_t *n_qubits, qip_prec *prec);
void qipb200_schedule_free(qipb200_schedule *s);
size_t qipb200_schedule_serialise(qip_prec prec, uint32_t n_qubits, const qip_op *ops, size_t n_ops, void *buf,
                                  size_t cap);

/* State files "QIPA" (checkpoint / resume; the reference keeps its state in two Vecs for the duration of one call,
 * qip/src/builder.rs:406-407, and has no equivalent): one file per shard -- 40-byte header {magic "QIPA", version 1,
 * prec, n_qubits, rank, world, first_index, n_amplitudes} followed by the shard's amplitudes in canonical index
 * order, streamed through a 64 MiB bounce buffer.  load checks the header against the target state.  On a
 * multi-device state (qipb200_init_multi) the shards go to "<path>.<rank>".  Byte-compatible with
 * rustqip_b200.wire.dump_state / load_state. */
int qipb200_state_save(qipb200_state *state, const char *path);
int qipb200_state_load(qipb200_state *state, const char *path);

#ifdef __cplusplus
}
#endif
#endif /* QIPB200_H */
