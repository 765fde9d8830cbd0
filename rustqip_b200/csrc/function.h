// function.h -- table-defined function ops |x>|y> -> e^{i theta(x)} |x>|y ^ f(x)> on the device
// (qipb200_state_apply_function, see function.cu).
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

#include "../../include/qip_op.h"

namespace qipb200 {

const uint32_t kFnMaxIn = 26;   // 2^26 entries: 256 MiB of f and 1 GiB of (cos, sin)
const uint32_t kFnMaxOut = 32;  // f is kept as u32

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

}  // namespace qipb200
