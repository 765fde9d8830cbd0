// pauli_rot_dev.cuh -- what pauli_rot.cu (qipb200_state_apply_pauli_rotations) and gradient.cu (the adjoint
// gradient and qipb200_state_apply_pauli_sum) share: the term descriptors of a rotation sweep, the sweep planner
// parameterised by the number of high tile bits, the descriptor builder and the device arithmetic of one rotation.  The
// tile geometry is sweep.cuh's.  See pauli_rot.cu for the arithmetic and pauli_rot.h for the planner policy.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/qip_op.h"
#include "expect.h"
#include "sweep.cuh"

namespace qipb200 {

const uint32_t kRotMaxM = 7;  // the most chosen high tile bits any sweep geometry uses
static_assert(kRotMaxM <= kSweepMaxHi, "the high tile bits fit SweepTiles::hi_pos");

enum : uint32_t {
  kRotPhase = 3u,     // w = i^phase (+-1) psi_partner
  kRotPair = 4u,      // the term's partner is in the other tile of the pair
  kRotBarrier = 8u,   // ownership differs from the previous term's: __syncthreads first
  kRotDiag = 16u,     // x == 0
};

struct RotTermDev {
  uint64_t z_out;  // Z/Y bits outside the tile
  uint32_t x_in;   // tile-local X/Y mask
  uint32_t z_in;   // tile-local Z/Y mask
  double c, s;     // cos and sin of theta/2, rounded to the state's precision (s negated for the inverse rotation)
  uint32_t flags;
  uint32_t aux;    // kRotDiag: length of the diagonal run this term starts; one-tile terms: lowest bit of x_in
};

struct RotArgs {
  SweepTiles geo;
  uint32_t n_terms;
};

struct RotSweep {
  uint64_t hi = 0;     // chosen high tile bits
  uint64_t x_out = 0;  // out-of-tile X/Y mask shared by the sweep
  uint32_t first = 0, end = 0;
};

// ---- host ----------------------------------------------------------------------------------------------------------

// The join rule of pauli_rot.h for a sweep with at most m chosen high tile bits (low: the mask of the L low bits):
// true when a term or group of X/Y mask x fits S, after growing S.hi or setting S.x_out as the rule says; false leaves S
// as it was.
bool rot_sweep_join(RotSweep *S, uint64_t x, uint64_t low, uint32_t m);

// The policy of pauli_rot.h with at most m (<= kRotMaxM) chosen high tile bits: consecutive terms per sweep.
void plan_rot_sweeps(uint32_t n, uint32_t m, const std::vector<PauliTerm> &terms, std::vector<RotSweep> *out);

// Geometry and term descriptors of every sweep: args[k] for sw[k], ht[t] for terms[t].  c and s come from the host's
// cos and sin of angles[t]/2, rounded once to the state's precision; negate_s stores -s (the inverse rotation).
// Returns false when a term breaks the planner's invariant (a different out-of-tile mask).
bool build_rot_tables(qip_prec prec, uint32_t n, const std::vector<PauliTerm> &terms, const double *angles,
                      bool negate_s, const std::vector<RotSweep> &sw, std::vector<RotArgs> *args,
                      std::vector<RotTermDev> *ht);

// ---- device --------------------------------------------------------------------------------------------------------

namespace {

__device__ __forceinline__ float flip_sign(float v, uint32_t bit) {
  return __int_as_float(__float_as_int(v) ^ (int)(bit << 31));
}
__device__ __forceinline__ double flip_sign(double v, uint32_t bit) {
  return __hiloint2double(__double2hiint(v) ^ (int)(bit << 31), __double2loint(v));
}

// c a + s w with w = i^ph (+-1) p, for s that already carries the sign (-1)^(ph >> 1) (+-1) and swap = ph & 1:
// w = (-p.y, p.x) or (p.x, p.y) up to that sign.  RN(s (-v)) = -RN(s v), so these are the bits of the definition.
template <typename R, typename V>
__device__ __forceinline__ V rot1(V a, V p, R c, R s, bool swap) {
  V o;
  if (swap) {
    o.x = add_rn(mul_rn(c, a.x), -mul_rn(s, p.y));
    o.y = add_rn(mul_rn(c, a.y), mul_rn(s, p.x));
  } else {
    o.x = add_rn(mul_rn(c, a.x), mul_rn(s, p.x));
    o.y = add_rn(mul_rn(c, a.y), mul_rn(s, p.y));
  }
  return o;
}

}  // namespace

}  // namespace qipb200
