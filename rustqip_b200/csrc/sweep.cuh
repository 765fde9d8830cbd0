// sweep.cuh -- the tile geometry of the kernels that sweep the state tile by tile (expect.cu, rdm.cu, pauli_rot.cu,
// gradient.cu, lanczos.cu, function.cu): its host builders here, the record and the generic device helpers the
// kernels share in sweep_dev.cuh.
//
// A tile is the L = min(kSweepL, n) lowest index bits (runs of 16 contiguous amplitudes) plus chosen high bits hi_pos,
// in increasing order; tile element e sits at offset tile_offset(e).  The other index bits form the visit index, spread
// over out_pos, except the pair bit (the lowest bit of x_out: a sweep with x_out != 0 visits the tile pair
// (B, B ^ x_out) from the side whose pair bit is clear) and the bits a caller skips (rdm.cu's block bits).  Visit v has
// base visit_base(v).
#pragma once

#include <cassert>
#include <cstring>

#include "sweep_dev.cuh"

namespace qipb200 {

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

}  // namespace qipb200
