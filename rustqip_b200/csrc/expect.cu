// expect.cu -- <psi|P|psi> for many Pauli strings P per read sweep of the state (qipb200_state_expect_paulis).
//
// Write P = i^nY X^x Z^z (x: index-bit mask of the X/Y letters, z: of the Z/Y letters).  Then
//   <P> = i^nY * sum_j (-1)^popc(j & z) * c_j,   c_j = conj(a_{j^x}) a_j,
// so terms with the same x share the products c_j and differ only in the sign pattern.
//
// Sweep = tile geometry + x_out.  A tile (sweep.cuh) is the kSweepL lowest index bits plus up to kExpM chosen high bits
// (2^11 amplitudes, read as runs of 16 contiguous amplitudes).  Each mask splits as x = x_in ^ x_out with x_in on tile
// bits; the masks of one sweep share x_out.  With x_out == 0 a CTA holds one tile; otherwise it holds the pair of tiles
// (B, B ^ x_out), visited once from the side whose lowest x_out bit is clear: the partner's half of the sum is
// (-1)^popc(x & z) * conj(sum over B), so every amplitude is still read exactly once per sweep.
//
// Per mask group the CTA forms c over its tile in registers, then either
//   - "direct": each of at most kExpMaxDirect terms of the sweep is a signed sum per thread, kept in a register
//     accumulator across the tiles the CTA walks (groups of few terms, e.g. the single X_i of an Ising field), or
//   - "WHT": an in-place Walsh-Hadamard transform of c over the 11 tile bits (3 stages in registers, 5 through warp
//     shuffles, 3 through shared memory); every term is then one shared-memory read at its tile-local z pattern,
//     added by the thread that owns the term into a shared-memory accumulator.
// z bits outside the tile give a CTA-uniform sign, popc(tile_base & z_out).  Only the real part of i^nY * sum is
// kept (P is Hermitian): each term accumulates one real component with a coefficient in {0, +-1, +-2}.
//
// Determinism: a fixed grid of kExpGrid CTAs with a static tile assignment, per-thread accumulation in tile order,
// shuffle/shared-memory block sums in a fixed order, per-CTA partials [CTA][term] summed by one reduction kernel in
// CTA order.  No floating-point atomics.
//
// Terms per sweep: up to kExpBatchTerms.  The first kExpSmemTerms accumulators of a sweep live in shared memory, the
// rest in the CTA's own column of the partials (each owned by one thread, so still no atomics).  A mask group of more
// than kExpBatchTerms terms takes one sweep per kExpBatchTerms of them; Z-only terms fill the room the other sweeps
// leave before opening sweeps of their own.
//
// Scratch: at most kExpBatchTerms rows per batch, 8 B per row and CTA (34.6 MB for kExpGrid = 264) plus the term
// tables; a longer term list runs in several batches, each with its own reduction kernel.  Shared memory: at most
// 111.4 KiB per CTA (f64 tile pair), so two CTAs fit on an SM.
//
// Two-state mode (k_expect<R, true>, qipb200_state_transition_paulis): <bra|P|ket> = i^nY sum_j (-1)^popc(j & z) c_j
// with c_j = conj(bra_{j^x}) ket_j.  The conjugate-symmetry shortcut needs bra == ket, so a tile pair (B, B') sums both
// sides explicitly for every group: side B from conj(bra_B') ket_B, side B' from conj(bra_B) ket_B', the diagonal group
// from conj(bra_B) ket_B and conj(bra_B') ket_B'; every amplitude of each state is still read once per sweep.  c_j is
// complex for the diagonal group too, so every term keeps both components: it is two rows, Re(i^nY w) and Im(i^nY w),
// i.e. a +-1 times one component of w (nY = 0..3: (re, im), (-im, re), (-re, -im), (im, -re)).  The planner and the
// batches count rows, so a sweep carries up to kExpBatchTerms / 2 terms.  Staged tiles: ket_B and bra_B (the one-state
// pair footprint, 111.4 KiB at f64), on a tile pair also ket_B' and bra_B' (175.4 KiB at f64: one CTA per SM; 111.4 KiB
// at f32).
// Rounding, each component, in units of S = sum_j |bra_{j^x}| |ket_j| (tests/transition_ref.py):
//   - c_j: two double products and one add per component (f32 amplitudes are exact in double): gamma_2;
//   - per tile: a Walsh-Hadamard output (11 add levels), or a per-thread sum of 8 (8 adds), a warp sum (5) and a sum
//     over 8 warps (8 adds) after the tile loop: at most 21;
//   - signs and the +-1 of i^nY are exact;
//   - each thread adds its tile values sequentially over the visits of its CTA, both sides of a pair for every term:
//     at most 2 ceil(V / G) adds for V = 2^(n-11) tiles over G = 264 CTAs;
//   - the per-CTA partials are summed sequentially over the G CTAs.
// Depth D = 2 + 21 + 2 ceil(V / G) + G, the one-state depth, and |got - want| <= gamma_D S per component.
#include "expect.h"

#include <algorithm>
#include <cstdio>
#include <map>

#include "../../include/qipb200.h"
#include "sweep.cuh"

namespace qipb200 {

namespace {

const uint32_t kExpM = 7;               // chosen high bits of a tile
const uint32_t kExpTileLog2 = kSweepL + kExpM;
const uint32_t kExpTile = 1u << kExpTileLog2;
const int kExpThreads = 256;
const int kExpPer = kExpTile / kExpThreads;  // tile amplitudes per thread (8: three in-register WHT stages)
const uint32_t kExpMaxDirect = 16;      // register accumulators per thread
const uint32_t kExpDirectGroupTerms = 4;  // groups of at most this many terms are evaluated directly
const uint32_t kExpBatchTerms = 16384;  // terms per reduction batch, and so per sweep
const uint32_t kExpSmemTerms = 1024;    // accumulators in shared memory; a sweep's later terms accumulate in global
const uint32_t kExpSmemGroups = 256;    // group descriptors staged in shared memory; later ones are read from global
const int kExpGrid = 264;               // CTAs per sweep: two per SM of a 132-SM H100
static_assert(kExpPer == 8, "the WHT below assumes 8 amplitudes per thread");
static_assert(kExpM <= kSweepMaxHi, "the high tile bits fit SweepTiles::hi_pos");

struct ExpGroupDev {
  uint32_t x_in;          // tile-local X/Y mask
  uint32_t diag;          // x == 0: c_j = |a_j|^2
  uint32_t first, end;    // the group's terms (sweep-local)
  uint32_t dfirst, dend;  // its direct slots (empty: WHT)
};

struct ExpTermDev {
  uint64_t z_out;  // Z/Y bits outside the tile
  uint32_t z_in;   // tile-local Z/Y pattern
  uint32_t comp;   // 0: real part, 1: imaginary part of the sum
  double coef;     // sign of i^nY on that component, times (1 +- eta) on the tile-pair path
};

struct ExpArgs {
  SweepTiles geo;
  uint32_t n_terms, n_direct;
  uint32_t row_off;   // partial row of the sweep's first term in the batch
  uint32_t rows;      // rows of the batch (length of a CTA's column of partials)
  uint32_t n_groups;
  uint16_t direct_term[kExpMaxDirect];
  ExpTermDev direct[kExpMaxDirect];  // the direct slots' terms (staged in shared memory by every CTA)
};

__device__ __forceinline__ double parity_sign(uint64_t v) { return parity(v) ? -1.0 : 1.0; }

template <int NC>
__device__ __forceinline__ void butterflies8(double (&c)[kExpPer][2]) {
#pragma unroll
  for (int s = 1; s < kExpPer; s <<= 1)
#pragma unroll
    for (int k = 0; k < kExpPer; ++k)
      if (!(k & s))
#pragma unroll
        for (int q = 0; q < NC; ++q) {
          const double u = c[k][q], v = c[k | s][q];
          c[k][q] = u + v;
          c[k | s][q] = u - v;
        }
}

// Walsh-Hadamard transform over the 11 tile-local bits of c (thread t holds elements t + 256 k) into cbuf[e*NC+q]:
// bits 8-10 in registers, bits 0-4 through shuffles, bits 5-7 after a transpose through cbuf.
template <int NC>
__device__ __forceinline__ void wht_tile(double (&c)[kExpPer][2], double *cbuf) {
  const int t = threadIdx.x, lane = t & 31;
  butterflies8<NC>(c);
#pragma unroll
  for (int b = 1; b < 32; b <<= 1)
#pragma unroll
    for (int k = 0; k < kExpPer; ++k)
#pragma unroll
      for (int q = 0; q < NC; ++q) {
        const double p = __shfl_xor_sync(0xffffffffu, c[k][q], b);
        c[k][q] = (lane & b) ? p - c[k][q] : c[k][q] + p;
      }
  __syncthreads();  // the previous group's readers of cbuf are done
#pragma unroll
  for (int k = 0; k < kExpPer; ++k)
#pragma unroll
    for (int q = 0; q < NC; ++q) cbuf[(t + kExpThreads * k) * NC + q] = c[k][q];
  __syncthreads();
  const int e0 = lane | ((t >> 5) << 8);
#pragma unroll
  for (int k = 0; k < kExpPer; ++k)
#pragma unroll
    for (int q = 0; q < NC; ++q) c[k][q] = cbuf[(e0 | (k << 5)) * NC + q];
  butterflies8<NC>(c);
#pragma unroll
  for (int k = 0; k < kExpPer; ++k)
#pragma unroll
    for (int q = 0; q < NC; ++q) cbuf[(e0 | (k << 5)) * NC + q] = c[k][q];
  __syncthreads();
}

// TWO (qipb200_state_transition_paulis): psi is the ket, bra the bra.  Tiles staged in shared memory: ket_B, bra_B
// (and ket_B', bra_B' on a tile pair, B' = B ^ x_out).  Every group is summed over both sides of a pair (side B from
// conj(bra_B') ket_B, side B' from conj(bra_B) ket_B'; the diagonal group from conj(bra_B) ket_B and
// conj(bra_B') ket_B'), its products are complex (the diagonal group too) and each term is two rows, Re and Im.
template <typename R, bool TWO>
__global__ void __launch_bounds__(kExpThreads, 2)
    k_expect(const R *__restrict__ psi, const __grid_constant__ ExpArgs a, const ExpGroupDev *__restrict__ groups,
             const ExpTermDev *__restrict__ terms, double *__restrict__ partials, const R *__restrict__ bra) {
  typedef typename SweepV<R>::type V;
  extern __shared__ __align__(16) unsigned char smem[];
  const bool pair = a.geo.x_out != 0;
  V *sA = reinterpret_cast<V *>(smem);
  V *sP = sA + kExpTile;
  double *cbuf = reinterpret_cast<double *>(smem + (TWO ? (pair ? 4 : 2) : (pair ? 2 : 1)) * kExpTile * sizeof(V));
  double *red = cbuf + 2 * kExpTile;                          // [warp][direct slot]
  const uint32_t n_smem_terms = min(a.n_terms, kExpSmemTerms), n_smem_groups = min(a.n_groups, kExpSmemGroups);
  double *acc_s = red + (kExpThreads / 32) * kExpMaxDirect;                  // [sweep term < kExpSmemTerms]
  ExpTermDev *sd = reinterpret_cast<ExpTermDev *>(acc_s + n_smem_terms);     // the direct slots' terms
  ExpGroupDev *sg = reinterpret_cast<ExpGroupDev *>(sd + kExpMaxDirect);   // the first groups
  // this CTA's column of the batch's partials [CTA][row]; the accumulators of terms >= kExpSmemTerms live there
  double *gcol = partials + (uint64_t)blockIdx.x * a.rows + a.row_off;
  const int t = threadIdx.x;
  if ((uint32_t)t < kExpMaxDirect) sd[t] = a.direct[t];
  for (uint32_t i = t; i < n_smem_terms; i += kExpThreads) acc_s[i] = 0.0;
  for (uint32_t i = kExpSmemTerms + t; i < a.n_terms; i += kExpThreads) gcol[i] = 0.0;
  for (uint32_t i = t; i < n_smem_groups; i += kExpThreads) sg[i] = groups[i];
  double acc[kExpMaxDirect];
#pragma unroll
  for (uint32_t d = 0; d < kExpMaxDirect; ++d) acc[d] = 0.0;
  const uint32_t tsize = 1u << a.geo.tb;
  uint64_t off[kExpPer];
#pragma unroll
  for (int k = 0; k < kExpPer; ++k) off[k] = tile_offset(a.geo, t + kExpThreads * k);
  for (uint64_t v = blockIdx.x; v < a.geo.n_visits; v += gridDim.x) {
    const uint64_t base = visit_base(a.geo, v);
    __syncthreads();  // the previous tile's readers are done
#pragma unroll
    for (int k = 0; k < kExpPer; ++k) {
      const uint32_t e = t + kExpThreads * k;
      V u, w;
      u.x = u.y = w.x = w.y = (R)0;
      if (TWO) {  // ket_B, bra_B, then ket_B', bra_B'
        V u2, w2;
        u2.x = u2.y = w2.x = w2.y = (R)0;
        if (e < tsize) {
          u = *reinterpret_cast<const V *>(psi + 2 * (base | off[k]));
          w = *reinterpret_cast<const V *>(bra + 2 * (base | off[k]));
          if (pair) {
            u2 = *reinterpret_cast<const V *>(psi + 2 * ((base ^ a.geo.x_out) | off[k]));
            w2 = *reinterpret_cast<const V *>(bra + 2 * ((base ^ a.geo.x_out) | off[k]));
          }
        }
        sA[e] = u;
        sP[e] = w;
        if (pair) {
          sA[2 * kExpTile + e] = u2;
          sA[3 * kExpTile + e] = w2;
        }
        continue;
      }
      if (e < tsize) {
        u = *reinterpret_cast<const V *>(psi + 2 * (base | off[k]));
        if (pair) w = *reinterpret_cast<const V *>(psi + 2 * ((base ^ a.geo.x_out) | off[k]));
      }
      sA[e] = u;
      if (pair) sP[e] = w;
    }
    __syncthreads();
    for (uint32_t g = 0; g < a.n_groups; ++g) {
      const ExpGroupDev G = g < kExpSmemGroups ? sg[g] : groups[g];
      // the diagonal group sums over both tiles of a pair; with two states every group does
      const int sides = TWO ? (pair ? 2 : 1) : ((G.diag && pair) ? 2 : 1);
      for (int side = 0; side < sides; ++side) {
        const uint64_t sbase = side ? base ^ a.geo.x_out : base;
        double c[kExpPer][2];
#pragma unroll
        for (int k = 0; k < kExpPer; ++k) {
          const uint32_t e = t + kExpThreads * k;
          if (TWO) {  // conj(bra_{j ^ x}) ket_j: the bra of the same side for the diagonal group, else the other one
            const V *sk = sA + (side ? 2 * kExpTile : 0);
            const V *sb = sA + (((G.diag ? side : side ^ 1) && pair) ? 3 * kExpTile : kExpTile);
            const V u = sk[e];
            const V w = sb[e ^ G.x_in];
            c[k][0] = (double)w.x * (double)u.x + (double)w.y * (double)u.y;
            c[k][1] = (double)w.x * (double)u.y - (double)w.y * (double)u.x;
          } else if (G.diag) {
            const V u = (side ? sP : sA)[e];
            c[k][0] = (double)u.x * (double)u.x + (double)u.y * (double)u.y;
            c[k][1] = 0.0;
          } else {
            const V u = sA[e];
            const V w = (pair ? sP : sA)[e ^ G.x_in];
            c[k][0] = (double)w.x * (double)u.x + (double)w.y * (double)u.y;  // conj(w) * u
            c[k][1] = (double)w.x * (double)u.y - (double)w.y * (double)u.x;
          }
        }
        if (G.dend > G.dfirst) {
#pragma unroll
          for (uint32_t d = 0; d < kExpMaxDirect; ++d) {
            if (d < G.dfirst || d >= G.dend) continue;
            const uint32_t z_in = sd[d].z_in, comp = sd[d].comp;
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < kExpPer; ++k) {
              const double cv = comp ? c[k][1] : c[k][0];
              s += (__popc((t + kExpThreads * k) & z_in) & 1) ? -cv : cv;
            }
            acc[d] += sd[d].coef * parity_sign(sbase & sd[d].z_out) * s;
          }
        } else {
          if (G.diag && !TWO)
            wht_tile<1>(c, cbuf);
          else
            wht_tile<2>(c, cbuf);
          const uint32_t nc = (G.diag && !TWO) ? 1 : 2;
          for (uint32_t i = G.first + t; i < G.end; i += kExpThreads) {
            const ExpTermDev T = terms[i];
            const double v = T.coef * parity_sign(sbase & T.z_out) * cbuf[T.z_in * nc + T.comp];
            if (i < kExpSmemTerms)
              acc_s[i] += v;
            else
              gcol[i] += v;  // owned by this thread like the shared-memory ones: coalesced, no atomics
          }
        }
      }
    }
  }
  // direct slots: warp sums, then the warps in order
  const int lane = t & 31, warp = t >> 5;
#pragma unroll
  for (uint32_t d = 0; d < kExpMaxDirect; ++d) {
    double v = acc[d];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp * kExpMaxDirect + d] = v;
  }
  __syncthreads();
  if ((uint32_t)t < a.n_direct) {
    double s = 0.0;
    for (int w = 0; w < kExpThreads / 32; ++w) s += red[w * kExpMaxDirect + t];
    acc_s[a.direct_term[t]] = s;  // the direct groups come first in a sweep: their terms are < kExpMaxDirect
  }
  __syncthreads();
  for (uint32_t i = t; i < n_smem_terms; i += kExpThreads) gcol[i] = acc_s[i];
}

__global__ void __launch_bounds__(256) k_expect_reduce(const double *__restrict__ partials, uint32_t rows, uint32_t grid,
                                                        double *__restrict__ res) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s = 0.0;
  for (uint32_t c = 0; c < grid; ++c) s += partials[(uint64_t)c * rows + r];
  res[r] = s;
}

// ---- host: grouping and greedy packing ----------------------------------------------

struct Group : PauliGroup {
  bool direct = false;
};

struct Sweep {
  uint64_t hi = 0;     // chosen high tile bits
  uint64_t x_out = 0;  // out-of-tile X/Y bits shared by every group
  uint32_t n_terms = 0;
  std::vector<Group> groups;
};

void plan_sweeps(uint32_t n, const std::vector<PauliTerm> &terms, std::vector<Sweep> *out) {
  const uint32_t L = std::min(kSweepL, n), m = std::min(kExpM, n - L);
  const uint64_t low = (1ull << L) - 1;
  // groups of equal X/Y mask in order of first appearance, cut into units of at most kExpBatchTerms terms
  std::vector<Group> units;
  std::vector<uint32_t> diag;
  for (const PauliGroup &g : group_by_x(terms))
    if (g.x == 0) {
      diag = g.terms;
    } else {
      for (size_t s = 0; s < g.terms.size(); s += kExpBatchTerms) {
        Group u;
        u.x = g.x;
        u.terms.assign(g.terms.begin() + s, g.terms.begin() + std::min(g.terms.size(), s + kExpBatchTerms));
        units.push_back(u);
      }
    }
  // greedy: a unit joins the sweep when the high bits where it differs from the sweep's x_out fit in the tile
  std::vector<bool> used(units.size(), false);
  size_t left = units.size();
  std::vector<Sweep> &sw = *out;
  sw.clear();
  while (left) {
    Sweep s;
    bool started = false;
    for (size_t i = 0; i < units.size(); ++i) {
      if (used[i] || s.n_terms + units[i].terms.size() > kExpBatchTerms) continue;
      const uint64_t hx = units[i].x & ~low;
      if (!started) {
        s.x_out = hx;
        started = true;
      } else {
        const uint64_t h2 = s.hi | ((hx ^ s.x_out) & ~s.hi);
        if ((uint32_t)__builtin_popcountll(h2) > m) continue;
        s.hi = h2;
        s.x_out &= ~h2;
      }
      used[i] = true;
      --left;
      s.n_terms += (uint32_t)units[i].terms.size();
      s.groups.push_back(units[i]);
    }
    sw.push_back(s);
  }
  // diagonal terms fill the room the sweeps leave, in sweep order; only what is left opens sweeps of its own
  for (size_t done = 0, k = 0; done < diag.size(); ++k) {
    if (k == sw.size()) sw.push_back(Sweep());
    const size_t take = std::min<size_t>(kExpBatchTerms - sw[k].n_terms, diag.size() - done);
    if (take == 0) continue;
    Group d;
    d.terms.assign(diag.begin() + done, diag.begin() + done + take);
    done += take;
    sw[k].n_terms += (uint32_t)take;
    sw[k].groups.push_back(d);
  }
  for (Sweep &s : sw) {
    sweep_fill(&s.hi, &s.x_out, n, L, m);
    uint32_t slots = 0;
    for (Group &g : s.groups)
      if (g.terms.size() <= kExpDirectGroupTerms && slots + g.terms.size() <= kExpMaxDirect) {
        g.direct = true;
        slots += (uint32_t)g.terms.size();
      }
    std::stable_partition(s.groups.begin(), s.groups.end(), [](const Group &g) { return g.direct; });
  }
}

// Shared memory of a sweep past its staged tiles: the transform buffer, the warp sums of the direct slots, the first
// accumulators, the direct slots' terms and the first groups.
constexpr size_t kExpSmemRest = 2 * kExpTile * sizeof(double) + (kExpThreads / 32) * kExpMaxDirect * sizeof(double) +
                                kExpSmemTerms * sizeof(double) + kExpMaxDirect * sizeof(ExpTermDev) +
                                kExpSmemGroups * sizeof(ExpGroupDev);
static_assert(2 * kExpTile * sizeof(double2) + kExpSmemRest <= 113 * 1024,
              "two CTAs per SM: at most 113 KiB of shared memory each (one state, or two states on one tile)");
static_assert(4 * kExpTile * sizeof(double2) + kExpSmemRest <= 227 * 1024,
              "two states on a tile pair: four tiles, one CTA per SM");

// Tiles a sweep stages: ket (and partner), times two with a bra.
uint32_t staged_tiles(bool two, bool pair) { return (two ? 2u : 1u) * (pair ? 2u : 1u); }

template <typename R, bool TWO>
cudaError_t launch_sweep(const void *psi, const void *bra, const ExpArgs &a, const ExpGroupDev *g,
                         const ExpTermDev *t, double *partials, cudaStream_t s) {
  const size_t smem = staged_tiles(TWO, a.geo.x_out != 0) * kExpTile * sizeof(typename SweepV<R>::type) +
                      2 * kExpTile * sizeof(double) + (kExpThreads / 32) * kExpMaxDirect * sizeof(double) +
                      std::min(a.n_terms, kExpSmemTerms) * sizeof(double) + kExpMaxDirect * sizeof(ExpTermDev) +
                      std::min(a.n_groups, kExpSmemGroups) * sizeof(ExpGroupDev);
  const size_t smem_max = staged_tiles(TWO, true) * kExpTile * sizeof(double2) + kExpSmemRest;
  cudaError_t e = cudaFuncSetAttribute(k_expect<R, TWO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
  if (e != cudaSuccess) return e;
  k_expect<R, TWO><<<kExpGrid, kExpThreads, smem, s>>>((const R *)psi, a, g, t, partials, (const R *)bra);
  return cudaGetLastError();
}

// End of the reduction batch that starts at sweep k: whole sweeps of at most kExpBatchTerms rows in all.
size_t batch_end(const std::vector<Sweep> &sw, size_t k) {
  size_t e = k, rows = 0;
  while (e < sw.size() && rows + sw[e].n_terms <= kExpBatchTerms) rows += sw[e++].n_terms;
  return e;
}

// The rows a call sums: one per term (one state: the real part), or two (two states: Re at row 2t, Im at 2t + 1).
std::vector<PauliTerm> term_rows(const std::vector<PauliTerm> &terms, bool two) {
  if (!two) return terms;
  std::vector<PauliTerm> rows;
  rows.reserve(2 * terms.size());
  for (const PauliTerm &p : terms) {
    rows.push_back(p);
    rows.push_back(p);
  }
  return rows;
}

cudaError_t run_sweeps(qip_prec prec, const void *psi, const void *bra, uint32_t n,
                       const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches);

}  // namespace

int parse_pauli_terms(uint32_t n, const uint64_t *qubits, const char *paulis, const uint32_t *term_len, size_t n_terms,
                      std::vector<PauliTerm> *out, std::string *err) {
  out->clear();
  if (n_terms == 0) return QIPB200_OK;
  if (!qubits || !paulis || !term_len) {
    *err = "expect: NULL qubits, paulis or term_len";
    return QIPB200_ERR_INVALID_ARG;
  }
  char msg[160];
  out->reserve(n_terms);
  size_t k = 0;
  for (size_t t = 0; t < n_terms; ++t) {
    PauliTerm p;
    uint64_t seen = 0;
    for (uint32_t j = 0; j < term_len[t]; ++j, ++k) {
      const char c = paulis[k];
      const uint64_t q = qubits[k];
      if (c != 'X' && c != 'Y' && c != 'Z') {
        snprintf(msg, sizeof(msg), "expect: term %zu: Pauli letter 0x%02x is not 'X', 'Y' or 'Z'", t, (unsigned)(unsigned char)c);
        *err = msg;
        return QIPB200_ERR_INVALID_ARG;
      }
      if (q >= n) {
        snprintf(msg, sizeof(msg), "expect: term %zu: qubit %llu out of range for %u qubits", t, (unsigned long long)q, n);
        *err = msg;
        return QIPB200_ERR_BAD_INDEX;
      }
      const uint64_t bit = 1ull << (n - 1 - q);
      if (seen & bit) {
        snprintf(msg, sizeof(msg), "expect: term %zu: qubit %llu repeated", t, (unsigned long long)q);
        *err = msg;
        return QIPB200_ERR_BAD_INDEX;
      }
      seen |= bit;
      if (c != 'Z') p.x |= bit;
      if (c != 'X') p.z |= bit;
      if (c == 'Y') ++p.n_y;
    }
    out->push_back(p);
  }
  return QIPB200_OK;
}

std::vector<PauliGroup> group_by_x(const std::vector<PauliTerm> &terms) {
  std::vector<PauliGroup> gr;
  std::map<uint64_t, size_t> where;
  for (uint32_t t = 0; t < (uint32_t)terms.size(); ++t) {
    auto it = where.find(terms[t].x);
    if (it == where.end()) {
      it = where.emplace(terms[t].x, gr.size()).first;
      gr.push_back(PauliGroup());
      gr.back().x = terms[t].x;
    }
    gr[it->second].terms.push_back(t);
  }
  return gr;
}

uint32_t expect_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms) {
  std::vector<Sweep> sw;
  plan_sweeps(n, terms, &sw);
  return (uint32_t)sw.size();
}

void transition_plan_counts(uint32_t n, const std::vector<PauliTerm> &terms, uint32_t *out2) {
  std::vector<Sweep> sw;
  plan_sweeps(n, term_rows(terms, true), &sw);
  uint32_t batches = 0;
  for (size_t k = 0; k < sw.size(); k = batch_end(sw, k)) ++batches;
  out2[0] = (uint32_t)sw.size();
  out2[1] = (uint32_t)sw.size() + batches;
}

cudaError_t run_expect(qip_prec prec, const void *psi, uint32_t n, const std::vector<PauliTerm> &terms, double *out,
                       cudaStream_t s, uint64_t *launches) {
  return run_sweeps(prec, psi, nullptr, n, terms, out, s, launches);
}

cudaError_t run_transition(qip_prec prec, const void *bra, const void *ket, uint32_t n,
                           const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches) {
  return run_sweeps(prec, ket, bra, n, terms, out, s, launches);
}

namespace {

// One state (bra == NULL): out[t] = Re <psi|P_t|psi>.  Two: out[2t], out[2t + 1] = Re, Im <bra|P_t|psi>.
cudaError_t run_sweeps(qip_prec prec, const void *psi, const void *bra, uint32_t n,
                       const std::vector<PauliTerm> &terms_in, double *out, cudaStream_t s, uint64_t *launches) {
  if (terms_in.empty()) return cudaSuccess;
  const bool two = bra != nullptr;
  const std::vector<PauliTerm> terms = term_rows(terms_in, two);
  std::vector<Sweep> sw;
  plan_sweeps(n, terms, &sw);
  const uint32_t L = std::min(kSweepL, n);
  const uint64_t low = (1ull << L) - 1;
  // host tables of every sweep, rows in sweep order; batches of whole sweeps of at most kExpBatchTerms rows
  std::vector<ExpArgs> args(sw.size());
  std::vector<ExpGroupDev> hg;
  std::vector<ExpTermDev> ht;
  std::vector<uint32_t> orig;
  std::vector<size_t> g_off(sw.size()), t_off(sw.size());
  for (size_t k = 0; k < sw.size(); ++k) {
    const Sweep &S = sw[k];
    ExpArgs &a = args[k];
    memset(&a, 0, sizeof(a));
    a.geo = sweep_tiles(n, L, S.hi, S.x_out);
    const uint64_t tile = low | S.hi;
    a.n_groups = (uint32_t)S.groups.size();
    a.n_terms = S.n_terms;
    g_off[k] = hg.size();
    t_off[k] = ht.size();
    uint32_t first = 0;
    for (const Group &G : S.groups) {
      ExpGroupDev gd;
      gd.x_in = tile_local(a.geo, G.x & tile);
      gd.diag = G.x == 0;
      gd.first = first;
      gd.end = first + (uint32_t)G.terms.size();
      gd.dfirst = gd.dend = 0;
      if (G.direct) {
        gd.dfirst = a.n_direct;
        gd.dend = a.n_direct + (uint32_t)G.terms.size();
      }
      for (uint32_t j = 0; j < G.terms.size(); ++j) {
        const PauliTerm &P = terms[G.terms[j]];
        ExpTermDev td;
        td.z_out = P.z & ~tile;
        td.z_in = tile_local(a.geo, P.z & tile);
        const uint32_t ph = P.n_y & 3;  // Re(i^ph w): +Re, -Im, -Re, +Im
        td.comp = ph & 1;
        td.coef = (ph == 0 || ph == 3) ? 1.0 : -1.0;
        if (two && (G.terms[j] & 1)) {  // Im(i^ph w): +Im, +Re, -Im, -Re
          td.comp = (ph & 1) ^ 1;
          td.coef = ph < 2 ? 1.0 : -1.0;
        }
        if (S.x_out && !gd.diag && !two) {  // + the partner tile: w + eta conj(w)
          const double eta = (__builtin_popcountll(P.x & P.z) & 1) ? -1.0 : 1.0;
          td.coef *= td.comp ? 1.0 - eta : 1.0 + eta;
        }
        if (G.direct) {
          a.direct[a.n_direct] = td;
          a.direct_term[a.n_direct++] = (uint16_t)(first + j);
        }
        ht.push_back(td);
        orig.push_back(G.terms[j]);
      }
      first = gd.end;
      hg.push_back(gd);
    }
  }
  std::vector<std::pair<size_t, size_t>> batches;  // [first sweep, end sweep)
  size_t rows_cap = 0, groups_cap = 0;
  for (size_t k = 0; k < sw.size();) {
    const size_t e = batch_end(sw, k);
    size_t rows = 0;
    for (size_t i = k; i < e; ++i) rows += sw[i].n_terms;
    batches.push_back(std::make_pair(k, e));
    rows_cap = std::max(rows_cap, rows);
    groups_cap = std::max(groups_cap, (e < sw.size() ? g_off[e] : hg.size()) - g_off[k]);
    k = e;
  }
  const size_t part_bytes = rows_cap * kExpGrid * sizeof(double);
  const size_t res_bytes = rows_cap * sizeof(double);
  const size_t term_bytes = rows_cap * sizeof(ExpTermDev);
  const size_t bytes = part_bytes + res_bytes + term_bytes + groups_cap * sizeof(ExpGroupDev);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, bytes, s);
  if (e != cudaSuccess) return e;
  double *d_part = (double *)d;
  double *d_res = (double *)(d + part_bytes);
  ExpTermDev *d_terms = (ExpTermDev *)(d + part_bytes + res_bytes);
  ExpGroupDev *d_groups = (ExpGroupDev *)(d + part_bytes + res_bytes + term_bytes);
  std::vector<double> res(ht.size());
  for (size_t b = 0; b < batches.size() && e == cudaSuccess; ++b) {
    const size_t k0 = batches[b].first, k1 = batches[b].second;
    const size_t t_end = k1 < sw.size() ? t_off[k1] : ht.size();
    const size_t g_end = k1 < sw.size() ? g_off[k1] : hg.size();
    const uint32_t rows = (uint32_t)(t_end - t_off[k0]);
    e = cudaMemcpyAsync(d_terms, ht.data() + t_off[k0], rows * sizeof(ExpTermDev), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(d_groups, hg.data() + g_off[k0], (g_end - g_off[k0]) * sizeof(ExpGroupDev),
                          cudaMemcpyHostToDevice, s);
    for (size_t k = k0; k < k1 && e == cudaSuccess; ++k) {
      ExpArgs a = args[k];
      a.row_off = (uint32_t)(t_off[k] - t_off[k0]);
      a.rows = rows;
      const ExpGroupDev *g = d_groups + (g_off[k] - g_off[k0]);
      const ExpTermDev *t = d_terms + a.row_off;
      if (two)
        e = prec == QIP_F32 ? launch_sweep<float, true>(psi, bra, a, g, t, d_part, s)
                            : launch_sweep<double, true>(psi, bra, a, g, t, d_part, s);
      else
        e = prec == QIP_F32 ? launch_sweep<float, false>(psi, nullptr, a, g, t, d_part, s)
                            : launch_sweep<double, false>(psi, nullptr, a, g, t, d_part, s);
      ++*launches;
    }
    if (e == cudaSuccess) {
      k_expect_reduce<<<(rows + 255) / 256, 256, 0, s>>>(d_part, rows, kExpGrid, d_res);
      ++*launches;
      e = cudaGetLastError();
    }
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(res.data() + t_off[k0], d_res, rows * sizeof(double), cudaMemcpyDeviceToHost, s);
  }
  const cudaError_t ef = cudaFreeAsync(d, s);
  if (e == cudaSuccess) e = ef;
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = es;
  if (e != cudaSuccess) return e;
  for (size_t r = 0; r < res.size(); ++r) out[orig[r]] = res[r];
  return cudaSuccess;
}

}  // namespace

}  // namespace qipb200
