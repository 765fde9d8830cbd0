// sweep.cuh -- the tile geometry of the kernels that sweep the state tile by tile (expect.cu, rdm.cu, pauli_rot.cu,
// gradient.cu, lanczos.cu, function.cu) and the generic device helpers they share.
//
// A tile is the L = min(kSweepL, n) lowest index bits (runs of 16 contiguous amplitudes) plus chosen high bits hi_pos,
// in increasing order; tile element e sits at offset tile_offset(e).  The other index bits form the visit index, spread
// over out_pos, except the pair bit (the lowest bit of x_out: a sweep with x_out != 0 visits the tile pair
// (B, B ^ x_out) from the side whose pair bit is clear) and the bits a caller skips (rdm.cu's block bits).  Visit v has
// base visit_base(v).
#pragma once

#include <cuda_runtime.h>

#include <cassert>
#include <cstdint>
#include <cstring>

namespace qipb200 {

const uint32_t kSweepL = 4;      // low index bits of a tile (runs of 16 amplitudes)
const uint32_t kSweepMaxHi = 8;  // the most chosen high tile bits any sweep uses (f32 function tiles: 12 - 4)

struct SweepTiles {
  uint64_t x_out;     // 0, or the out-of-tile X/Y mask shared by the sweep
  uint64_t n_visits;  // tiles (x_out == 0) or tile pairs
  uint32_t L, tb;     // low bits, tile bits
  uint32_t n_out;     // bits of the visit index, spread over out_pos
  uint8_t hi_pos[kSweepMaxHi];
  uint8_t out_pos[64];
};

// ---- host ----------------------------------------------------------------------------------------------------------

// The geometry of a sweep with tile bits low(L) | hi (at most kSweepMaxHi high bits) and out-of-tile mask x_out; the
// bits of skip are neither tile nor visit bits.
inline SweepTiles sweep_tiles(uint32_t n, uint32_t L, uint64_t hi, uint64_t x_out, uint64_t skip = 0) {
  assert(__builtin_popcountll(hi) <= (int)kSweepMaxHi);  // hi_pos has room for kSweepMaxHi bits
  SweepTiles g;
  memset(&g, 0, sizeof(g));
  g.x_out = x_out;
  g.L = g.tb = L;
  for (uint32_t b = 0; b < n; ++b)
    if ((hi >> b) & 1) g.hi_pos[g.tb++ - L] = (uint8_t)b;
  const uint64_t tile = ((1ull << L) - 1) | hi, pair_bit = x_out & (~x_out + 1);
  for (uint32_t b = 0; b < n; ++b)
    if (!(((tile | pair_bit | skip) >> b) & 1)) g.out_pos[g.n_out++] = (uint8_t)b;
  g.n_visits = 1ull << g.n_out;
  return g;
}

// Index bits of mask on the tile (the L low bits, then hi_pos in order) packed into a tile-local index.
inline uint32_t tile_local(const SweepTiles &g, uint64_t mask) {
  uint32_t r = (uint32_t)(mask & ((1ull << g.L) - 1));
  for (uint32_t i = 0; i < g.tb - g.L; ++i) r |= (uint32_t)((mask >> g.hi_pos[i]) & 1ull) << (g.L + i);
  return r;
}

// Fill the free high tile bits of a planned sweep up to m: first x_out bits (fewer tile pairs), then the lowest free
// bits from L up (longer contiguous runs).
inline void sweep_fill(uint64_t *hi, uint64_t *x_out, uint32_t n, uint32_t L, uint32_t m) {
  for (uint32_t b = 0; b < n && (uint32_t)__builtin_popcountll(*hi) < m; ++b)
    if ((*x_out >> b) & 1) {
      *hi |= 1ull << b;
      *x_out &= ~(1ull << b);
    }
  for (uint32_t b = L; b < n && (uint32_t)__builtin_popcountll(*hi) < m; ++b) *hi |= 1ull << b;
}

// ---- device --------------------------------------------------------------------------------------------------------

namespace {

template <typename R>
struct SweepV;
template <>
struct SweepV<float> {
  typedef float2 type;
};
template <>
struct SweepV<double> {
  typedef double2 type;
};

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

__device__ __forceinline__ bool parity(uint64_t v) { return __popcll(v) & 1; }

// Offset of tile element e from the visit's base.
__device__ __forceinline__ uint64_t tile_offset(const SweepTiles &g, uint32_t e) {
  uint64_t o = e & ((1u << g.L) - 1);
  for (uint32_t i = 0; i < g.tb - g.L; ++i) o |= (uint64_t)((e >> (g.L + i)) & 1u) << g.hi_pos[i];
  return o;
}

// Base index of visit v: the bits of v spread over out_pos.
__device__ __forceinline__ uint64_t visit_base(const SweepTiles &g, uint64_t v) {
  uint64_t b = 0;
  for (uint32_t i = 0; i < g.n_out; ++i) b |= ((v >> i) & 1ull) << g.out_pos[i];
  return b;
}

template <int B>
__device__ __forceinline__ void cp_async(void *sdst, const void *gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(sdst);
  if (B == 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

}  // namespace

}  // namespace qipb200
