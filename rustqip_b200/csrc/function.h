// function.h -- function ops |x>|y> -> e^{i theta(x)} |x>|y ^ f(x)> on the device for functions given as tables or as
// CUDA source (qipb200_state_apply_function, qipb200_state_expect_function; see function.cu).
//
// Path plan (the policy qipb200_function_plan reports), on physical index bits.  With L = min(4, n) low bits and
// T = min(T_max, n), T_max = 11 for f64 and 12 for f32 (one tile buffer is 32 KiB either way):
//   - staged tile path when L + |{out bits >= L}| <= T: the tile is the L low bits, the out bits above them, and the
//     lowest free bits from L up until it has T bits (as sweep_fill fills a Pauli-rotation tile);
//   - pair path otherwise.
// So an op without output qubits (phase only) always takes the tile path.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/qip_op.h"

namespace qipb200 {

const uint32_t kFnMaxIn = 26;   // 2^26 entries: 256 MiB of f and 1 GiB of (cos, sin)
const uint32_t kFnMaxOut = 32;  // f is kept as u32
const uint32_t kFnCodeMaxBits = 34;    // n_in + n_out of a code function: no state on one H100 is larger
const uint32_t kFnCodeMaxParams = 16;  // parameters of a code function's theta

struct FnPlan {
  uint32_t path = 0;       // 0: staged tile, 1: pair
  uint32_t tile_bits = 0;  // T of the tile path, 0 for the pair path
  uint64_t hi = 0;         // tile path: the tile bits above the L low bits
};

// The plan above for out-register bits out_pos[0..n_out) of an unsharded 2^n state.
FnPlan plan_function(qip_prec prec, uint32_t n, const uint32_t *out_pos, uint32_t n_out);

// psi <- U psi in place, U|x>|y> = e^{i theta(x)} |x>|y ^ f(x)>, where bit i of x is index bit in_pos[i] and bit i of
// f(x) goes to index bit out_pos[i] (physical bits of an unsharded 2^n state).  f: the device table of f (NULL when
// n_out == 0); cs: (cos, sin) of theta per x, in double (NULL: no phase).  Exactly one kernel, stream-ordered.
cudaError_t run_function(qip_prec prec, void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                         const uint32_t *out_pos, uint32_t n_out, const uint32_t *f, const double2 *cs, int sm_count,
                         cudaStream_t s, uint64_t *launches);

// ---- code functions: the user's qip_f / qip_theta compiled with NVRTC into the kernels of the table path ----

struct FnCode;  // a code function's program, loaded on its context's device

// Compile (or find in the process or on-disk cache) the program of a code function without loading it: QIPB200_OK,
// QIPB200_ERR_INVALID_ARG with the NVRTC log in *msg, or QIPB200_ERR_UNSUPPORTED without NVRTC (*msg: why).
int function_code_compile(uint32_t n_out, const char *source, bool theta, std::string *msg);
// The same, then load it on the current device: also QIPB200_ERR_UNSUPPORTED without the driver entry points and
// QIPB200_ERR_CUDA when the module does not load (*msg: why).
int function_code_load(uint32_t n_out, const char *source, bool theta, FnCode **out, std::string *msg);
// Unload (no kernel of c may still be queued).
void function_code_free(FnCode *c);

// *first = the first x < 2^n_in with f(x) >= 2^n_out (range) or a non-finite theta(x, params) (!range), or
// UINT64_MAX when there is none.  One kernel; d_word is one u64 of device scratch.  Synchronises on s.
cudaError_t function_code_first_bad(const FnCode *c, bool range, uint32_t n_in, uint32_t n_out, const double *params,
                                    uint64_t *d_word, int sm_count, cudaStream_t s, uint64_t *first, std::string *err);

// run_function for a code function with kFnCodeMaxParams params: the same plan, kernels and arithmetic, with f and
// (cos, sin) of theta evaluated on the device.  Exactly one kernel, stream-ordered.
cudaError_t run_function_code(qip_prec prec, void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                              const uint32_t *out_pos, uint32_t n_out, const FnCode *c, const double *params,
                              int sm_count, cudaStream_t s, uint64_t *launches, std::string *err);

const int kFnExpPartials = 264;  // the fixed expect grid (function_dev.cuh: kFnExpGrid)

// *out = sum_j |psi_j|^2 theta(x(j), params) in double, in the fixed order of function.cu.  One kernel;
// d_partials holds kFnExpPartials doubles of device scratch.  Synchronises on s.
cudaError_t expect_function_code(qip_prec prec, const void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                                 const FnCode *c, const double *params, double *d_partials, cudaStream_t s,
                                 uint64_t *launches, double *out, std::string *err);

// f(x) (f_out) and (cos theta(x), sin theta(x)) (cs_out, interleaved) for x in [x0, x0 + count), by the device
// functions the apply kernels use: those of c (with params) when c is not NULL, else the tables f / cs.  Either output
// may be NULL; cs_out needs a phase (c->theta or cs).  Synchronises on s.
cudaError_t tabulate_function(const FnCode *c, const double *params, const uint32_t *f, const double2 *cs,
                              uint64_t x0, uint64_t count, uint64_t *f_out, double *cs_out, int sm_count,
                              cudaStream_t s, std::string *err);

}  // namespace qipb200
