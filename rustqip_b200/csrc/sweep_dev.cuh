// sweep_dev.cuh -- the tile geometry record of sweep.cuh and the generic device helpers of the sweep kernels.  It
// compiles with nvcc and with NVRTC alone: function.cu embeds its text in the programs of code functions (function.h).
#pragma once

#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>

#include <cstdint>
#else
typedef unsigned char uint8_t;
typedef unsigned int uint32_t;
typedef unsigned long long uint64_t;
#endif

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
