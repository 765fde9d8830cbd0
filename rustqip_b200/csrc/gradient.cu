// gradient.cu -- dst <- H src for a real Pauli sum H = sum_h c_h P_h (qipb200_state_apply_pauli_sum), and the
// adjoint-method gradient of E = <psi0|U^dagger H U|psi0> for U = R_{T-1} ... R_0, R_t = exp(-i theta_t/2 P_t)
// (qipb200_state_pauli_energy_gradient).  Planner policies: gradient.h.
//
// Geometry.  Both kernels stage two states per CTA, so their tile (sweep.cuh) is the kSweepL = 4 lowest index bits plus
// up to kGradM = 6 chosen high bits: 2^10 amplitudes, four per thread of 256.  One tile or tile pair of each of two
// states is 64 KiB at f64 (four 16 KiB tiles), which keeps two CTAs per SM at under 113 KiB each.
//
// k_pauli_sum.  (P src)_j = i^nY (-1)^popc(k & z) src_k with k = j ^ x, so the terms of one X/Y mask x (a group) share
// src_k and differ by a real or imaginary sign: the group's coefficient at j is a + i b with
//   a = sum of +-c_h over the group's terms with nY even, b = the same over nY odd, in list order, in double,
// (the sign is Re / Im of i^nY times (-1)^popc(k & z_h); the first addition is to +0.0).  Per amplitude, in double and
// with no FMA contraction:
//   re = RN(RN(a p.x) - RN(b p.y)), im = RN(RN(a p.y) + RN(b p.x)), acc = (RN(acc.x + re), RN(acc.y + im)),
// p = src_k widened to double, groups in the sweep's order (gradient.h), sweeps in plan order.  acc starts at +0.0 in
// the first sweep, which writes dst without reading it, and at the stored dst in later ones; each sweep stores acc
// rounded to the state's precision (exact at f64).  So dst is a fixed function of the inputs and the plan (made on
// physical index bits, so it follows the layout), emulated bit for bit in tests/gradient_ref.py.  Forward error, per
// amplitude j with A_j = sum_h |c_h| |src_(j^x_h)|:
//   |dst_j - (H src)_j| <= 2 (gamma_(T+G+2)(2^-53) + gamma_S(u)) A_j     (T terms, G groups, S sweeps, u the state's
// unit roundoff: each component is a sum of at most T + G + 2 rounded double operations on terms bounded by
// |c_h| (|p.x| + |p.y|), plus one rounding to the state's precision per sweep).  A thread owns its four amplitudes of
// each tile: src is read from shared memory only, so no barrier separates groups.
//
// k_pauli_sum, evolution mode (EVO = true; qipb200_state_evolve_pauli_sum, host plan in evolve.h).  Step k of the
// Chebyshev recurrence T_1 = H~ S, T_k = 2 H~ T_(k-1) - T_(k-2) runs the s sweeps of plan_sum over the non-identity
// terms with the coefficients RN(c_h / b) (step 1) or RN(c_h (2 / b)) (later steps) in place of c_h.  T_k is in
// work_a for odd k, work_b for even k; src = T_(k-1) (S for k = 1) is the only operand read at partner indices and is
// never written in the step, so no sweep has a read-after-write hazard.  Per amplitude, in double, no FMA:
//   - the first sweep's acc starts at +0.0 (k = 1), at -S (k = 2) or at -T_(k-2) (k >= 3, read from dst, which it
//     overwrites in place), RN(start v) of the value v widened to double with start = -1, so an exact negation; later
//     sweeps start at the stored dst (start = 1);
//   - the groups add as above, and each sweep stores acc rounded to the state's precision;
//   - the last sweep of step k >= 2 then updates S at the own index from the stored (rounded) t = T_k, with
//     cmul(c, v) = (RN(RN(c.x v.x) - RN(c.y v.y)), RN(RN(c.x v.y) + RN(c.y v.x))) and RN additions:
//       k = 2: S <- RN_prec((cmul(C_0, S) + cmul(C_1, T_1)) + cmul(C_2, t))   (T_1 = src at the own index)
//       k > 2: S <- RN_prec(S + cmul(C_k, t)).
// S and T_(k-2) are read before they are written, by the thread that owns the amplitude; T_(k-2) (the accumulator
// start) is staged in the dst tiles, S is loaded straight into registers before the groups.  Emulated bit for bit in
// tests/evolve_ref.py.  Forward error in 2-norm, to first order, for |psi| = |S| on entry: with
//   delta = 2 (gamma_(T+G+4)(2^-53) + gamma_s(u))   (T non-identity terms, G groups, s sweeps; the extra operations are
// the start value and the rounding of RN(c_h / b)), step k adds a local error e_k with |e_1| <= delta |psi| and
// |e_k| <= 3 delta |psi| (|A| <= sum_h |2 c_h / b| |T| = 2 |T|, plus |T_(k-2)|).  The error of T_k is
// sum_(m <= k) U_(k-m)(H~) e_m, and |U_j(H~)| <= j + 1 (Chebyshev polynomials of the second kind), so it is at most
// 3 delta k (k + 1) / 2 |psi|: quadratic in k.  A Lanczos step (run_lanczos_sum, lanczos.cu) uses the same mode with
// update = 0, start = -RN(beta_j / beta_(j-1)) (an inexact scaling, rounded once), and in its last sweep adds
// Re(conj(src_j) dst_j) of the stored dst_j (src_j is staged at the own index) into a per-thread double, reduced per
// warp, then per CTA in warp order into dot[CTA].  With C = sum_k |C_k| (|S| <= C |psi| after any step),
//   |S_device - sum_k C_k T_k(H~) psi| <= [3 delta sum_k |C_k| k (k + 1) / 2 + sqrt(2) (2 gamma_4(2^-53) + u) K C]
//                                        x (1 + 3 delta K (K + 1) / 2) |psi|,
// the second term for the K accumulations into S.  tests/evolve_ref.py: bound().
//
// k_pauli_adjoint.  The backward pass runs over the sweeps of the reversed term list (gradient.h) with the descriptors
// of pauli_rot.cu for c and -s: R_t^dagger = exp(+i theta_t/2 P_t) is exactly the rotation update of pauli_rot.cu with
// s negated, so phi (= state) and lambda (= work) go back bit for bit as the emulator says.  Per term, on the pairs
// (or the diagonal elements) the thread owns by the rules of pauli_rot.cu, barriers included, it first adds
// Im<lambda|P_t|phi> = sum_j Re(conj(lambda_j) w_j), w_j = -i (P phi)_j, in a double register (f32 amplitudes widened,
// fma), then undoes R_t on both states.  The first backward sweep adds Re<lambda|phi> (the energy) from the staged tiles
// before any term, then waits at a CTA barrier: the first term of a sweep carries no barrier of its own (the loop
// otherwise starts right after the staging barrier), and its pairs may belong to threads of other warps.  Per term the
// 32 lanes of a warp reduce by butterfly shuffles and lane 0 adds into the warp's slot in shared memory (one slot per warp and row, visits in order); when the CTA has done its tiles it sums its 8 warp slots
// in warp order into scratch[row][CTA], and k_adjoint_reduce sums each row over the CTAs in CTA order.  The grid is a
// fixed kGradGrid CTAs (or the visit count, when smaller): the same inputs give the same bits on any device.
// A sweep holds at most kAdjMaxTerms terms so the slots fit shared memory: 64 KiB of tiles, 8 x 257 slots and the
// staged descriptors, at most 91 KiB per CTA.
//
// The quantum geometric tensor (qipb200_state_pauli_geometric_tensor, run_pauli_qgt).  For each term i in order:
//   - fork i (k_qgt_fork): state <- R_i state with the arithmetic of pauli_rot.cu (the same host-rounded c and s, the
//     same rot1 per pair), work_a <- the rotated state, work_b <- P_i of it (a permutation, signs and component swaps:
//     exact).  One thread per amplitude pair (j, j ^ x) of P_i, j with the lowest bit h of x clear, or per element when
//     x == 0, kForkUnroll pairs in flight, loaded straight from global memory: the two loads of a warp touch the same
//     32-byte sectors (h < 2 at f64) or two contiguous runs, so the fork reads the state once and writes three states.
//     It adds |psi'_j|^2 = fma(x, x, y y) and Re(conj(psi'_j) (P psi')_j) = fma(x, px, y py) per element into two
//     per-thread doubles, reduced by butterfly in the warp, then the 8 warps in order into scratch[2i + {0, 1}][CTA] on
//     a fixed grid of min(kForkGrid, 2^(n-1) / 256) CTAs; one k_qgt_reduce at the end sums every fork's rows over the
//     CTAs in order.
//   - segment i: the walk of gradient.h over terms i + 1 .. T - 1 (the descriptors built with c and +s, so the walk
//     runs forward) with k_pauli_adjoint in complex-row mode (QGT = true) on phi = work_a, lambda = work_b: per term it
//     adds Re<lambda|P_j|phi> = sum Re(conj(lambda_k) i w_k) (dot_w_re: the fma policy of dot_w with the other swap)
//     next to Im<lambda|P_j|phi> (dot_w), two rows per term, no energy row, then rotates both states by R_j.  The
//     reduction is the adjoint's: per-thread double, warp butterfly, warp slots, CTA sums in warp order, then
//     k_qgt_reduce sums each row over the CTAs in CTA order into M_ij at res[2 (i T + j)].  Shared memory: 64 KiB of
//     tiles, 8 warps x 512 rows x 8 B and 256 descriptors x 40 B, 106 KiB per CTA: still two CTAs per SM.
// The host downloads res (2 T^2 + 2 T doubles) once and forms G_tt = (|psi_t|^2 - e_t^2) / 4, G_ij = (M_ij - e_i e_j) / 4
// for i < j and G_ji = conj(G_ij).  The grids, the plan and the order of every sum are fixed: the same inputs give the
// same bits.  Forward error, to first order, for |psi0| = N and u the state's unit roundoff: a state after k rotations
// is within sqrt(2) gamma_(5k)(u) N of exact (pauli_rot.cu), and psi_t, phi and mu have had at most T rotations (P is
// exact), so each inner product M_ij, e_t and |psi_t|^2 errs by at most
//   delta = (2 sqrt(2) gamma_(5T)(u) + gamma_D(2^-53)) N^2,   D = 2^n / 256 + 300 (elements per thread and visit, the
// warp butterfly, the slots over visits, the warps and the CTAs), with f32 amplitudes widened exactly; |e_t| <= N^2, so
// |G - G_exact| <= delta (1 + 2 N^2) / 4 + gamma_3(2^-53) N^4 per entry (the host's three roundings).  tests/qgt_ref.py:
// qgt_bound().
#include "gradient.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "../../include/qipb200.h"
#include "pauli_rot.h"
#include "pauli_rot_dev.cuh"

namespace qipb200 {

namespace {

const uint32_t kGradM = 6;
static_assert(kGradM <= kSweepMaxHi, "the high tile bits fit SweepTiles::hi_pos");
const uint32_t kGradTile = 1u << (kSweepL + kGradM);
const int kGradThreads = 256;
const int kGradPer = kGradTile / kGradThreads;  // tile amplitudes per thread
const int kGradWarps = kGradThreads / 32;
const uint32_t kAdjMaxTerms = 256;       // terms of one backward sweep
const uint32_t kAdjRows = kAdjMaxTerms + 1;  // + the energy
const uint32_t kQgtRows = 2 * kAdjMaxTerms;  // complex rows: Re and Im per term
const int kForkThreads = 256;
const int kForkWarps = kForkThreads / 32;
const int kForkUnroll = 2;   // amplitude pairs per thread in flight
const int kForkGrid = 528;   // CTAs of a fork (fewer when the state has fewer items)

struct SumGroupDev {
  uint32_t x_in;   // tile-local X/Y mask
  uint32_t pair;   // the group's partner amplitudes are in the other tile of the pair
  uint32_t first, end;  // its terms
};

struct SumTermDev {
  uint64_t z_out;  // Z/Y bits outside the tile
  uint32_t z_in;   // tile-local Z/Y mask
  uint32_t odd;    // nY odd: the term adds to b, else to a
  double c;        // c_h times the sign of Re / Im of i^nY
};

// One sweep of a Chebyshev step or a Lanczos step (k_pauli_sum<R, PAIR, true>), see "k_pauli_sum, evolution mode"
// above and lanczos.cu.
struct EvoSweep {
  const void *from;  // the accumulator starts at RN(start from) at the own index; NULL: at +0.0
  void *state;       // S, updated at the own index after the store when update != 0
  double start;      // -1 (a Chebyshev step's first sweep), RN(-beta_j / beta_(j-1)) (a Lanczos step's) or 1
  uint32_t update;   // 0: none; 1: S <- c0 S + c1 src + c2 dst (step 2); 2: S <- S + c2 dst (steps >= 3)
  double2 c0, c1, c2;
  double *dot;       // not NULL: dot[CTA] = the CTA's sum of Re(conj(src_j) dst_j), dst_j as stored (Lanczos)
};

__device__ __forceinline__ double2 widen(float2 v) { return make_double2(v.x, v.y); }
__device__ __forceinline__ double2 widen(double2 v) { return v; }
__device__ __forceinline__ void narrow(double2 a, float2 *o) { *o = make_float2((float)a.x, (float)a.y); }
__device__ __forceinline__ void narrow(double2 a, double2 *o) { *o = a; }

// c v and a + v, complex, in double with every product and sum rounded (no FMA)
__device__ __forceinline__ double2 cmul_rn(double2 c, double2 v) {
  return make_double2(__dadd_rn(__dmul_rn(c.x, v.x), -__dmul_rn(c.y, v.y)),
                      __dadd_rn(__dmul_rn(c.x, v.y), __dmul_rn(c.y, v.x)));
}
__device__ __forceinline__ double2 cadd_rn(double2 a, double2 v) {
  return make_double2(__dadd_rn(a.x, v.x), __dadd_rn(a.y, v.y));
}

template <typename R, bool PAIR, bool EVO>
__global__ void __launch_bounds__(kGradThreads, 2)
    k_pauli_sum(R *__restrict__ dst, const R *__restrict__ src, const __grid_constant__ RotArgs a,
                const SumGroupDev *__restrict__ groups, const SumTermDev *__restrict__ terms, uint32_t accumulate,
                const __grid_constant__ EvoSweep ev) {
  typedef typename SweepV<R>::type V;
  extern __shared__ __align__(16) unsigned char smem[];
  // single tiles: [buffer][src, from] double-buffered; pairs: src A, src B, from A, from B
  V *tiles = reinterpret_cast<V *>(smem);
  const int t = threadIdx.x;
  const uint32_t tsize = 1u << a.geo.tb;
  // where the accumulator starts: the stored partial (dst) or, in the first sweep of a Chebyshev step, T_(k-1)
  const R *from = EVO ? (const R *)ev.from : dst;
  const bool load = EVO ? ev.from != nullptr : accumulate != 0;
  uint64_t off[kGradPer];
#pragma unroll
  for (int k = 0; k < kGradPer; ++k) off[k] = tile_offset(a.geo, t + kGradThreads * k);
  auto issue = [&](uint64_t v, V *S, V *D, V *S2, V *D2) {  // S2, D2: the pair's B tiles
    const uint64_t b = visit_base(a.geo, v);
#pragma unroll
    for (int k = 0; k < kGradPer; ++k) {
      const uint32_t e = t + kGradThreads * k;
      if (e >= tsize) continue;
      cp_async<sizeof(V)>(S + e, src + 2 * (b | off[k]));
      if (load) cp_async<sizeof(V)>(D + e, from + 2 * (b | off[k]));
      if (PAIR) {
        cp_async<sizeof(V)>(S2 + e, src + 2 * ((b ^ a.geo.x_out) | off[k]));
        if (load) cp_async<sizeof(V)>(D2 + e, from + 2 * ((b ^ a.geo.x_out) | off[k]));
      }
    }
  };
  uint64_t v = blockIdx.x;
  if (!PAIR) {
    if (v < a.geo.n_visits) issue(v, tiles, tiles + kGradTile, nullptr, nullptr);
    cp_async_commit();
  }
  int cur = 0;
  double dsum = 0.0;  // Lanczos: this thread's share of Re<src|dst>, over its amplitudes in visit order
  for (; v < a.geo.n_visits; v += gridDim.x) {
    V *sA, *sB, *dA, *dB;
    if (PAIR) {
      sA = tiles;
      sB = tiles + kGradTile;
      dA = tiles + 2 * kGradTile;
      dB = tiles + 3 * kGradTile;
      issue(v, sA, dA, sB, dB);
      cp_async_commit();
      cp_async_wait<0>();
    } else {
      sA = tiles + cur * 2 * kGradTile;
      dA = sA + kGradTile;
      sB = dB = nullptr;
      const uint64_t nv = v + gridDim.x;
      V *nS = tiles + (cur ^ 1) * 2 * kGradTile;
      if (nv < a.geo.n_visits) issue(nv, nS, nS + kGradTile, nullptr, nullptr);
      cp_async_commit();
      cp_async_wait<1>();
    }
    __syncthreads();
    const uint64_t bA = visit_base(a.geo, v), bB = bA ^ a.geo.x_out;
#pragma unroll 1
    for (int side = 0; side < (PAIR ? 2 : 1); ++side) {
      const V *own = side ? sB : sA, *other = side ? sA : sB;
      const V *D = side ? dB : dA;
      const uint64_t b = side ? bB : bA, bo = side ? bA : bB;
      double2 acc[kGradPer];
      V sv[kGradPer];  // S at the own index, loaded before the groups for the update after the store
#pragma unroll
      for (int k = 0; k < kGradPer; ++k) {
        const uint32_t e = t + kGradThreads * k;
        acc[k] = make_double2(0.0, 0.0);
        if (load && e < tsize) acc[k] = widen(D[e]);
        if (EVO) acc[k] = make_double2(__dmul_rn(ev.start, acc[k].x), __dmul_rn(ev.start, acc[k].y));
        if (EVO && ev.update && e < tsize)
          sv[k] = *reinterpret_cast<const V *>((const R *)ev.state + 2 * (b | off[k]));
      }
      for (uint32_t g = 0; g < a.n_terms; ++g) {
        const SumGroupDev G = groups[g];
        const V *S = (PAIR && G.pair) ? other : own;
        const uint64_t bk = (PAIR && G.pair) ? bo : b;  // base of the tile that holds k = j ^ x
        double ca[kGradPer], cb[kGradPer];
#pragma unroll
        for (int k = 0; k < kGradPer; ++k) ca[k] = cb[k] = 0.0;
        for (uint32_t h = G.first; h < G.end; ++h) {
          const SumTermDev T = terms[h];
          const uint32_t so = (uint32_t)parity(bk & T.z_out);
#pragma unroll
          for (int k = 0; k < kGradPer; ++k) {
            const uint32_t e = t + kGradThreads * k;
            const double cv = flip_sign(T.c, so ^ (__popc((e ^ G.x_in) & T.z_in) & 1));
            if (T.odd)
              cb[k] = __dadd_rn(cb[k], cv);
            else
              ca[k] = __dadd_rn(ca[k], cv);
          }
        }
#pragma unroll
        for (int k = 0; k < kGradPer; ++k) {
          const uint32_t e = t + kGradThreads * k;
          if (e >= tsize) continue;
          const double2 p = widen(S[e ^ G.x_in]);
          const double re = __dadd_rn(__dmul_rn(ca[k], p.x), -__dmul_rn(cb[k], p.y));
          const double im = __dadd_rn(__dmul_rn(ca[k], p.y), __dmul_rn(cb[k], p.x));
          acc[k].x = __dadd_rn(acc[k].x, re);
          acc[k].y = __dadd_rn(acc[k].y, im);
        }
      }
#pragma unroll
      for (int k = 0; k < kGradPer; ++k) {
        const uint32_t e = t + kGradThreads * k;
        if (e >= tsize) continue;
        narrow(acc[k], reinterpret_cast<V *>(dst + 2 * (b | off[k])));
        if (EVO && ev.dot) {
          V o;
          narrow(acc[k], &o);
          const double2 u = widen(own[e]), w = widen(o);
          dsum = fma(u.x, w.x, fma(u.y, w.y, dsum));
        }
        if (EVO && ev.update) {
          V o;
          narrow(acc[k], &o);
          const double2 sk = widen(sv[k]), tk = widen(o);
          const double2 r = ev.update == 1 ? cadd_rn(cadd_rn(cmul_rn(ev.c0, sk), cmul_rn(ev.c1, widen(own[e]))),
                                                     cmul_rn(ev.c2, tk))
                                           : cadd_rn(sk, cmul_rn(ev.c2, tk));
          narrow(r, reinterpret_cast<V *>((R *)ev.state + 2 * (b | off[k])));
        }
      }
    }
    __syncthreads();  // every thread has read this buffer before the next cp.async writes it
    if (!PAIR) cur ^= 1;
  }
  cp_async_wait<0>();
  if (EVO && ev.dot) {  // butterfly in the warp, then the 8 warps in order: fixed for a fixed grid
    __shared__ double wsum[kGradWarps];
#pragma unroll
    for (int o = 16; o; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
    if ((t & 31) == 0) wsum[t >> 5] = dsum;
    __syncthreads();
    if (t == 0) {
      double s = 0.0;
      for (int w = 0; w < kGradWarps; ++w) s += wsum[w];
      ev.dot[blockIdx.x] = s;
    }
  }
}

// Re(conj(l) w) for w = i^ph (+-1) p as rot1 forms it: swap: w = (-p.y, p.x), else (p.x, p.y), times (-1)^neg.
__device__ __forceinline__ double dot_w(double2 l, double2 p, bool swap, uint32_t neg) {
  const double d = swap ? fma(l.y, p.x, -l.x * p.y) : fma(l.x, p.x, l.y * p.y);
  return neg ? -d : d;
}

// Re(conj(l) i w) = Re<l|P|p> for the same w: dot_w with the other swap and one more negation when swap is set.
__device__ __forceinline__ double dot_w_re(double2 l, double2 p, bool swap, uint32_t neg) {
  return dot_w(l, p, !swap, neg ^ (uint32_t)swap);
}

template <uint32_t ROWS>
__device__ __forceinline__ void slot_add(double *red, uint32_t row, double g) {
#pragma unroll
  for (int o = 16; o; o >>= 1) g += __shfl_xor_sync(0xffffffffu, g, o);
  if ((threadIdx.x & 31) == 0) red[(threadIdx.x >> 5) * ROWS + row] += g;
}

// QGT = false: the adjoint gradient (rows: Im<lambda|P_t|phi> per term, then the energy).  QGT = true: a segment of
// the geometric tensor (rows 2r, 2r + 1: Re and Im of <lambda|P_t|phi> for the sweep's term r, no energy); the
// direction of the walk comes from the descriptors alone.
template <typename R, bool PAIR, bool QGT>
__global__ void __launch_bounds__(kGradThreads, 2)
    k_pauli_adjoint(R *__restrict__ phi, R *__restrict__ lam, const __grid_constant__ RotArgs a,
                    const RotTermDev *__restrict__ terms, uint32_t energy, double *__restrict__ scratch) {
  typedef typename SweepV<R>::type V;
  constexpr uint32_t kRows = QGT ? kQgtRows : kAdjRows;
  extern __shared__ __align__(16) unsigned char smem[];
  // single tiles: [buffer][phi, lambda] double-buffered; pairs: phi A, phi B, lambda A, lambda B
  V *tiles = reinterpret_cast<V *>(smem);
  double *red = reinterpret_cast<double *>(smem + 4 * kGradTile * sizeof(V));  // [warp][row]
  RotTermDev *sT = reinterpret_cast<RotTermDev *>(red + kGradWarps * kRows);
  const int t = threadIdx.x;
  // the energy is row n_terms
  const uint32_t rows = QGT ? 2 * a.n_terms : a.n_terms + (energy ? 1u : 0u);
  for (uint32_t i = t; i < a.n_terms; i += kGradThreads) sT[i] = terms[i];
  for (uint32_t i = t; i < kGradWarps * kRows; i += kGradThreads) red[i] = 0.0;  // ordered by the loop's barrier
  const uint32_t tsize = 1u << a.geo.tb;
  uint64_t off[kGradPer];
#pragma unroll
  for (int k = 0; k < kGradPer; ++k) off[k] = tile_offset(a.geo, t + kGradThreads * k);
  auto issue = [&](uint64_t v, V *P, V *Lm, V *P2, V *L2) {  // P2, L2: the pair's B tiles
    const uint64_t b = visit_base(a.geo, v);
#pragma unroll
    for (int k = 0; k < kGradPer; ++k) {
      const uint32_t e = t + kGradThreads * k;
      if (e >= tsize) continue;
      cp_async<sizeof(V)>(P + e, phi + 2 * (b | off[k]));
      cp_async<sizeof(V)>(Lm + e, lam + 2 * (b | off[k]));
      if (PAIR) {
        cp_async<sizeof(V)>(P2 + e, phi + 2 * ((b ^ a.geo.x_out) | off[k]));
        cp_async<sizeof(V)>(L2 + e, lam + 2 * ((b ^ a.geo.x_out) | off[k]));
      }
    }
  };
  uint64_t v = blockIdx.x;
  if (!PAIR) {
    if (v < a.geo.n_visits) issue(v, tiles, tiles + kGradTile, nullptr, nullptr);
    cp_async_commit();
  }
  int cur = 0;
  for (; v < a.geo.n_visits; v += gridDim.x) {
    V *pA, *pB, *lA, *lB;
    if (PAIR) {
      pA = tiles;
      pB = tiles + kGradTile;
      lA = tiles + 2 * kGradTile;
      lB = tiles + 3 * kGradTile;
      issue(v, pA, lA, pB, lB);
      cp_async_commit();
      cp_async_wait<0>();
    } else {
      pA = tiles + cur * 2 * kGradTile;
      lA = pA + kGradTile;
      pB = lB = nullptr;
      const uint64_t nv = v + gridDim.x;
      V *nP = tiles + (cur ^ 1) * 2 * kGradTile;
      if (nv < a.geo.n_visits) issue(nv, nP, nP + kGradTile, nullptr, nullptr);
      cp_async_commit();
      cp_async_wait<1>();
    }
    __syncthreads();
    const uint64_t bA = visit_base(a.geo, v), bB = bA ^ a.geo.x_out;
    if (!QGT && energy) {  // Re<lambda|phi> on the thread's own elements, before any term is undone
      double g = 0.0;
      for (int side = 0; side < (PAIR ? 2 : 1); ++side) {
        const V *P = side ? pB : pA, *Lm = side ? lB : lA;
#pragma unroll
        for (int k = 0; k < kGradPer; ++k) {
          const uint32_t e = t + kGradThreads * k;
          if (e < tsize) g += dot_w(widen(Lm[e]), widen(P[e]), false, 0);
        }
      }
      slot_add<kRows>(red, a.n_terms, g);
      // the first term of a sweep carries no barrier and may update elements other warps have yet to read here
      __syncthreads();
    }
    for (uint32_t i = 0; i < a.n_terms;) {
      const RotTermDev T = sT[i];
      if (T.flags & kRotBarrier) __syncthreads();
      if (T.flags & kRotDiag) {  // a run of diagonal terms on the thread's own elements, in registers, tile by tile
        const uint32_t end = i + T.aux;
#pragma unroll 1
        for (int side = 0; side < (PAIR ? 2 : 1); ++side) {
          V *P = side ? pB : pA, *Lm = side ? lB : lA;
          const uint64_t b = side ? bB : bA;
          V r[kGradPer], q[kGradPer];
#pragma unroll
          for (int k = 0; k < kGradPer; ++k) {
            const uint32_t e = t + kGradThreads * k;
            r[k].x = r[k].y = q[k].x = q[k].y = (R)0;  // elements past a small tile add 0 and are never stored
            if (e < tsize) {
              r[k] = P[e];
              q[k] = Lm[e];
            }
          }
          for (uint32_t j = i; j < end; ++j) {
            const RotTermDev D = sT[j];
            const uint32_t ph = D.flags & kRotPhase;
            const bool swap = ph & 1;
            const R c = (R)D.c, s = flip_sign((R)D.s, ph >> 1);
            // sign of element k (e = t + 256 k): parity(t & z_in) ^ parity(k & z_in >> 8) ^ parity(base & z_out)
            const uint32_t zk = D.z_in >> 8;
            const uint32_t par4 = ((zk & 1) ? 0xAu : 0u) ^ ((zk & 2) ? 0xCu : 0u);
            const uint32_t f = par4 ^ (((__popc((uint32_t)t & D.z_in) & 1) ^ (uint32_t)parity(b & D.z_out)) ? 0xFu : 0u);
            double g = 0.0, gr = 0.0;
#pragma unroll
            for (int k = 0; k < kGradPer; ++k) {
              const uint32_t nk = (f >> k) & 1;
              g += dot_w(widen(q[k]), widen(r[k]), swap, nk ^ (ph >> 1));
              if (QGT) gr += dot_w_re(widen(q[k]), widen(r[k]), swap, nk ^ (ph >> 1));
              r[k] = rot1<R, V>(r[k], r[k], c, flip_sign(s, nk), swap);
              q[k] = rot1<R, V>(q[k], q[k], c, flip_sign(s, nk), swap);
            }
            if (QGT) {
              slot_add<kRows>(red, 2 * j, gr);
              slot_add<kRows>(red, 2 * j + 1, g);
            } else {
              slot_add<kRows>(red, j, g);
            }
          }
#pragma unroll
          for (int k = 0; k < kGradPer; ++k) {
            const uint32_t e = t + kGradThreads * k;
            if (e < tsize) {
              P[e] = r[k];
              Lm[e] = q[k];
            }
          }
        }
        i = end;
        continue;
      }
      const uint32_t ph = T.flags & kRotPhase;
      const bool swap = ph & 1;
      const R c = (R)T.c, s = flip_sign((R)T.s, ph >> 1);
      double g = 0.0, gr = 0.0;
      if (PAIR && (T.flags & kRotPair)) {  // (A[e], B[e ^ x_in]) for the thread's own e
        const uint32_t nA = parity(bA & T.z_out), nB = parity(bB & T.z_out);
#pragma unroll
        for (int k = 0; k < kGradPer; ++k) {
          const uint32_t e = t + kGradThreads * k;
          if (e >= tsize) continue;
          const uint32_t f = e ^ T.x_in;
          const uint32_t sa = nB ^ (__popc(f & T.z_in) & 1), sb = nA ^ (__popc(e & T.z_in) & 1);
          const V u = pA[e], w = pB[f], lu = lA[e], lw = lB[f];
          g += dot_w(widen(lu), widen(w), swap, sa ^ (ph >> 1)) + dot_w(widen(lw), widen(u), swap, sb ^ (ph >> 1));
          if (QGT)
            gr += dot_w_re(widen(lu), widen(w), swap, sa ^ (ph >> 1)) +
                  dot_w_re(widen(lw), widen(u), swap, sb ^ (ph >> 1));
          pA[e] = rot1<R, V>(u, w, c, flip_sign(s, sa), swap);
          pB[f] = rot1<R, V>(w, u, c, flip_sign(s, sb), swap);
          lA[e] = rot1<R, V>(lu, lw, c, flip_sign(s, sa), swap);
          lB[f] = rot1<R, V>(lw, lu, c, flip_sign(s, sb), swap);
        }
      } else {  // the thread's pairs (e, e ^ x_in) with bit aux of e clear, on each tile
        const uint32_t h = T.aux;
#pragma unroll 1
        for (int side = 0; side < (PAIR ? 2 : 1); ++side) {
          V *P = side ? pB : pA, *Lm = side ? lB : lA;
          const uint32_t no = parity((side ? bB : bA) & T.z_out);
#pragma unroll
          for (int k = 0; k < kGradPer / 2; ++k) {
            const uint32_t p = t + kGradThreads * k;
            if (2 * p >= tsize) continue;
            const uint32_t e = ((p >> h) << (h + 1)) | (p & ((1u << h) - 1)), f = e ^ T.x_in;
            const uint32_t se = no ^ (__popc(f & T.z_in) & 1), sf = no ^ (__popc(e & T.z_in) & 1);
            const V u = P[e], w = P[f], lu = Lm[e], lw = Lm[f];
            g += dot_w(widen(lu), widen(w), swap, se ^ (ph >> 1)) + dot_w(widen(lw), widen(u), swap, sf ^ (ph >> 1));
            if (QGT)
              gr += dot_w_re(widen(lu), widen(w), swap, se ^ (ph >> 1)) +
                    dot_w_re(widen(lw), widen(u), swap, sf ^ (ph >> 1));
            P[e] = rot1<R, V>(u, w, c, flip_sign(s, se), swap);
            P[f] = rot1<R, V>(w, u, c, flip_sign(s, sf), swap);
            Lm[e] = rot1<R, V>(lu, lw, c, flip_sign(s, se), swap);
            Lm[f] = rot1<R, V>(lw, lu, c, flip_sign(s, sf), swap);
          }
        }
      }
      if (QGT) {
        slot_add<kRows>(red, 2 * i, gr);
        slot_add<kRows>(red, 2 * i + 1, g);
      } else {
        slot_add<kRows>(red, i, g);
      }
      ++i;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kGradPer; ++k) {
      const uint32_t e = t + kGradThreads * k;
      if (e >= tsize) continue;
      *reinterpret_cast<V *>(phi + 2 * (bA | off[k])) = pA[e];
      *reinterpret_cast<V *>(lam + 2 * (bA | off[k])) = lA[e];
      if (PAIR) {
        *reinterpret_cast<V *>(phi + 2 * (bB | off[k])) = pB[e];
        *reinterpret_cast<V *>(lam + 2 * (bB | off[k])) = lB[e];
      }
    }
    __syncthreads();  // the stores have read this buffer before the next cp.async writes it
    if (!PAIR) cur ^= 1;
  }
  cp_async_wait<0>();
  __syncthreads();
  for (uint32_t r = t; r < rows; r += kGradThreads) {
    double s = 0.0;
    for (int w = 0; w < kGradWarps; ++w) s += red[w * kRows + r];
    scratch[(uint64_t)r * gridDim.x + blockIdx.x] = s;
  }
}

// res[idx] = sum over CTAs in order of scratch[row][CTA]; row i < n_terms is reversed position first + i, that is term
// T - 1 - first - i, at res[1 + that term]; row n_terms (energy sweeps) is the energy at res[0].
__global__ void __launch_bounds__(256) k_adjoint_reduce(const double *__restrict__ scratch, uint32_t rows,
                                                         uint32_t grid, uint32_t n_terms, uint32_t T, uint32_t first,
                                                         double *__restrict__ res) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s = 0.0;
  for (uint32_t c = 0; c < grid; ++c) s += scratch[(uint64_t)r * grid + c];
  res[r == n_terms ? 0 : T - first - r] = s;
}

// res[r] = sum over CTAs in order of scratch[r][CTA], r < rows (a segment sweep's rows or every fork's two rows).
__global__ void __launch_bounds__(256) k_qgt_reduce(const double *__restrict__ scratch, uint32_t rows, uint32_t grid,
                                                     double *__restrict__ res) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s = 0.0;
  for (uint32_t c = 0; c < grid; ++c) s += scratch[(uint64_t)r * grid + c];
  res[r] = s;
}

struct ForkArgs {
  uint64_t x, z;     // the term's X/Y and Z/Y masks on physical index bits
  uint64_t n_items;  // amplitude pairs (x != 0) or amplitudes (x == 0)
  uint32_t h;        // lowest bit of x (x != 0)
  uint32_t ny;       // number of Y letters, mod 4
  double c, s;       // as the term's RotTermDev: cos and sin of theta/2 rounded to the state's precision
};

// i^ny (-1)^neg p: (P psi)_j for the partner value p = psi_(j ^ x), a component swap and negations (exact)
template <typename V>
__device__ __forceinline__ V pauli_value(V p, uint32_t ny, uint32_t neg) {
  V o = p;
  if (ny & 1) {
    o.x = -p.y;
    o.y = p.x;
  }
  if (((ny >> 1) ^ neg) & 1) {
    o.x = -o.x;
    o.y = -o.y;
  }
  return o;
}

// The fork of the geometric tensor: state <- R state, work_a <- R state, work_b <- P R state, in one read of state and
// three writes; scratch[0][CTA] and scratch[1][CTA] get the CTA's sums of |psi'_j|^2 and Re(conj(psi'_j) (P psi')_j).
// One thread per pair (j, j ^ x) with bit h of j clear, or per element when x == 0, loaded straight from global memory.
template <typename R>
__global__ void __launch_bounds__(kForkThreads, 4)
    k_qgt_fork(R *__restrict__ state, R *__restrict__ wa, R *__restrict__ wb, const __grid_constant__ ForkArgs f,
               double *__restrict__ scratch) {
  typedef typename SweepV<R>::type V;
  V *S = reinterpret_cast<V *>(state), *A = reinterpret_cast<V *>(wa), *B = reinterpret_cast<V *>(wb);
  const uint32_t ph = (f.ny + 3) & 3;  // w = -i (P psi) = i^ph (+-1) psi_partner, as the rotation descriptors say
  const bool swap = ph & 1;
  const R c = (R)f.c, s = flip_sign((R)f.s, ph >> 1);
  const uint64_t lo = (1ull << f.h) - 1, stride = (uint64_t)gridDim.x * kForkThreads;
  double nrm = 0.0, ex = 0.0;
  for (uint64_t p0 = (uint64_t)blockIdx.x * kForkThreads + threadIdx.x; p0 < f.n_items;
       p0 += kForkUnroll * stride) {
    uint64_t j[kForkUnroll];
    V u[kForkUnroll], w[kForkUnroll];
#pragma unroll
    for (int k = 0; k < kForkUnroll; ++k) {  // every load of the group before any arithmetic
      const uint64_t p = p0 + k * stride;
      if (p >= f.n_items) continue;
      j[k] = f.x ? ((p & ~lo) << 1) | (p & lo) : p;
      u[k] = S[j[k]];
      if (f.x) w[k] = S[j[k] ^ f.x];
    }
#pragma unroll
    for (int k = 0; k < kForkUnroll; ++k) {
      const uint64_t p = p0 + k * stride;
      if (p >= f.n_items) continue;
      const uint64_t jj = j[k], kk = jj ^ f.x;
      const uint32_t sj = parity(kk & f.z), sk = parity(jj & f.z);  // the signs of (P psi)_j and (P psi)_k
      if (f.x) {
        const V a = rot1<R, V>(u[k], w[k], c, flip_sign(s, sj), swap);
        const V b = rot1<R, V>(w[k], u[k], c, flip_sign(s, sk), swap);
        const V pa = pauli_value(b, f.ny, sj), pb = pauli_value(a, f.ny, sk);
        S[jj] = a;
        S[kk] = b;
        A[jj] = a;
        A[kk] = b;
        B[jj] = pa;
        B[kk] = pb;
        const double2 da = widen(a), db = widen(b), dpa = widen(pa), dpb = widen(pb);
        nrm += fma(da.x, da.x, da.y * da.y) + fma(db.x, db.x, db.y * db.y);
        ex += fma(da.x, dpa.x, da.y * dpa.y) + fma(db.x, dpb.x, db.y * dpb.y);
      } else {
        const V a = rot1<R, V>(u[k], u[k], c, flip_sign(s, sj), swap);
        const V pa = pauli_value(a, f.ny, sj);
        S[jj] = a;
        A[jj] = a;
        B[jj] = pa;
        const double2 da = widen(a), dpa = widen(pa);
        nrm += fma(da.x, da.x, da.y * da.y);
        ex += fma(da.x, dpa.x, da.y * dpa.y);
      }
    }
  }
  __shared__ double wsum[kForkWarps][2];
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
    ex += __shfl_xor_sync(0xffffffffu, ex, o);
  }
  if ((threadIdx.x & 31) == 0) {
    wsum[threadIdx.x >> 5][0] = nrm;
    wsum[threadIdx.x >> 5][1] = ex;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
    for (int w = 0; w < kForkWarps; ++w) t += wsum[w][threadIdx.x];
    scratch[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x] = t;
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------

struct SumSweep {
  RotSweep geo;
  std::vector<uint32_t> groups;  // indices into the group list, in order
};

void plan_sum(uint32_t n, const std::vector<PauliTerm> &terms, std::vector<PauliGroup> *groups_out,
              std::vector<SumSweep> *out) {
  const uint32_t L = std::min(kSweepL, n), m = std::min(kGradM, n - L);
  const uint64_t low = (1ull << L) - 1;
  std::vector<PauliGroup> &gr = *groups_out;
  gr = group_by_x(terms);
  std::vector<SumSweep> &sw = *out;
  sw.clear();
  std::vector<bool> used(gr.size(), false);
  size_t left = gr.size();
  while (left) {
    SumSweep S;
    for (size_t g = 0; g < gr.size(); ++g)
      if (!used[g] && rot_sweep_join(&S.geo, gr[g].x, low, m)) {
        used[g] = true;
        --left;
        S.groups.push_back((uint32_t)g);
      }
    sw.push_back(S);
  }
  for (SumSweep &S : sw) sweep_fill(&S.geo.hi, &S.geo.x_out, n, L, m);
}

// The walk of pauli_rot.h's planner with kGradM high tile bits over `terms`, a sweep cut after every kAdjMaxTerms
// terms (no terms: no sweeps).
void plan_walk(uint32_t n, const std::vector<PauliTerm> &terms, std::vector<RotSweep> *out) {
  std::vector<RotSweep> sw;
  plan_rot_sweeps(n, kGradM, terms, &sw);
  out->clear();
  for (const RotSweep &S : sw)
    for (uint32_t f = S.first; f < S.end; f += kAdjMaxTerms) {
      RotSweep P = S;
      P.first = f;
      P.end = std::min(S.end, f + kAdjMaxTerms);
      out->push_back(P);
    }
}

void plan_adjoint(uint32_t n, const std::vector<PauliTerm> &rev, std::vector<RotSweep> *out) {
  plan_walk(n, rev, out);
  if (out->empty()) {  // no terms: one sweep for the energy, on the tile of the lowest bits
    const uint32_t L = std::min(kSweepL, n), m = std::min(kGradM, n - L);
    RotSweep S;
    sweep_fill(&S.hi, &S.x_out, n, L, m);
    out->push_back(S);
  }
}

template <typename R, bool PAIR, bool EVO>
cudaError_t launch_sum(void *dst, const void *src, const RotArgs &a, const SumGroupDev *g, const SumTermDev *t,
                       uint32_t accumulate, const EvoSweep &ev, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  static_assert(4 * kGradTile * sizeof(double2) <= 113 * 1024, "two CTAs per SM: at most 113 KiB of shared memory each");
  const size_t smem = 4 * kGradTile * sizeof(V);
  cudaError_t e =
      cudaFuncSetAttribute(k_pauli_sum<R, PAIR, EVO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int grid = (int)std::min<uint64_t>(a.geo.n_visits, (uint64_t)kGradGrid);
  k_pauli_sum<R, PAIR, EVO><<<grid, kGradThreads, smem, s>>>((R *)dst, (const R *)src, a, g, t, accumulate, ev);
  return cudaGetLastError();
}

template <bool EVO>
cudaError_t launch_sum_any(qip_prec prec, void *dst, const void *src, const RotArgs &a, const SumGroupDev *g,
                           const SumTermDev *t, uint32_t accumulate, const EvoSweep &ev, cudaStream_t s) {
  if (prec == QIP_F32)
    return a.geo.x_out ? launch_sum<float, true, EVO>(dst, src, a, g, t, accumulate, ev, s)
                       : launch_sum<float, false, EVO>(dst, src, a, g, t, accumulate, ev, s);
  return a.geo.x_out ? launch_sum<double, true, EVO>(dst, src, a, g, t, accumulate, ev, s)
                     : launch_sum<double, false, EVO>(dst, src, a, g, t, accumulate, ev, s);
}

// The device tables of plan_sum: args[k] (n_terms = its group count) and the groups of sweep k from (*hg)[(*g_off)[k]]
// for every sweep, and the terms they index, with c = RN(scale coeffs[h]) times the sign of Re / Im of i^nY.  False
// when a group breaks the planner's invariant (a different out-of-tile mask).
bool build_sum_tables(uint32_t n, const std::vector<PauliTerm> &terms, const double *coeffs, double scale,
                      std::vector<RotArgs> *args, std::vector<SumGroupDev> *hg, std::vector<SumTermDev> *ht,
                      std::vector<size_t> *g_off) {
  std::vector<PauliGroup> gr;
  std::vector<SumSweep> sw;
  plan_sum(n, terms, &gr, &sw);
  const uint32_t L = std::min(kSweepL, n);
  const uint64_t low = (1ull << L) - 1;
  args->assign(sw.size(), RotArgs());
  g_off->assign(sw.size(), 0);
  hg->clear();
  ht->clear();
  for (size_t k = 0; k < sw.size(); ++k) {
    const SumSweep &S = sw[k];
    RotArgs &a = (*args)[k];
    memset(&a, 0, sizeof(a));
    a.geo = sweep_tiles(n, L, S.geo.hi, S.geo.x_out);
    const uint64_t tile = low | S.geo.hi;
    a.n_terms = (uint32_t)S.groups.size();  // groups, for this kernel
    (*g_off)[k] = hg->size();
    for (uint32_t gi : S.groups) {
      const PauliGroup &G = gr[gi];
      const uint64_t xo = G.x & ~tile;
      if (xo != 0 && xo != S.geo.x_out) return false;
      SumGroupDev gd;
      gd.x_in = tile_local(a.geo, G.x & tile);
      gd.pair = xo ? 1u : 0u;
      gd.first = (uint32_t)ht->size();
      for (uint32_t t : G.terms) {
        const PauliTerm &P = terms[t];
        SumTermDev td;
        td.z_out = P.z & ~tile;
        td.z_in = tile_local(a.geo, P.z & tile);
        td.odd = P.n_y & 1;
        const double c = scale * coeffs[t];
        td.c = ((P.n_y & 3) >= 2) ? -c : c;  // i^nY = 1, i, -1, -i
        ht->push_back(td);
      }
      gd.end = (uint32_t)ht->size();
      hg->push_back(gd);
    }
  }
  return true;
}

template <typename R, bool PAIR, bool QGT>
cudaError_t launch_adjoint(void *phi, void *lam, const RotArgs &a, const RotTermDev *terms, uint32_t energy,
                           double *scratch, int grid, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  static_assert(kGradThreads == 256 && kGradPer == 4, "the diagonal path's sign table assumes e = t + 256 k, k < 4");
  const size_t fixed = 4 * kGradTile * sizeof(V) + kGradWarps * (QGT ? kQgtRows : kAdjRows) * sizeof(double);
  static_assert(4 * kGradTile * sizeof(double2) + kGradWarps * kAdjRows * sizeof(double) +
                        kAdjMaxTerms * sizeof(RotTermDev) <= 113 * 1024,
                "two CTAs per SM: at most 113 KiB of shared memory each");
  static_assert(4 * kGradTile * sizeof(double2) + kGradWarps * kQgtRows * sizeof(double) +
                        kAdjMaxTerms * sizeof(RotTermDev) <= 113 * 1024,
                "complex rows: still two CTAs per SM, at most 113 KiB of shared memory each");
  const size_t smem = fixed + a.n_terms * sizeof(RotTermDev);
  cudaError_t e = cudaFuncSetAttribute(k_pauli_adjoint<R, PAIR, QGT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(fixed + kAdjMaxTerms * sizeof(RotTermDev)));
  if (e != cudaSuccess) return e;
  k_pauli_adjoint<R, PAIR, QGT><<<grid, kGradThreads, smem, s>>>((R *)phi, (R *)lam, a, terms, energy, scratch);
  return cudaGetLastError();
}

template <bool QGT>
cudaError_t launch_adjoint_any(qip_prec prec, void *phi, void *lam, const RotArgs &a, const RotTermDev *terms,
                               uint32_t energy, double *scratch, int grid, cudaStream_t s) {
  if (prec == QIP_F32)
    return a.geo.x_out ? launch_adjoint<float, true, QGT>(phi, lam, a, terms, energy, scratch, grid, s)
                       : launch_adjoint<float, false, QGT>(phi, lam, a, terms, energy, scratch, grid, s);
  return a.geo.x_out ? launch_adjoint<double, true, QGT>(phi, lam, a, terms, energy, scratch, grid, s)
                     : launch_adjoint<double, false, QGT>(phi, lam, a, terms, energy, scratch, grid, s);
}

// The segments of the geometric tensor: for fork i, the walk over terms i + 1 .. T - 1 (sw[i]).
void plan_segments(uint32_t n, const std::vector<PauliTerm> &ansatz, std::vector<std::vector<RotSweep>> *sw) {
  sw->assign(ansatz.size(), std::vector<RotSweep>());
  for (size_t i = 0; i + 1 < ansatz.size(); ++i)
    plan_walk(n, std::vector<PauliTerm>(ansatz.begin() + i + 1, ansatz.end()), &(*sw)[i]);
}

}  // namespace

uint32_t pauli_sum_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms) {
  std::vector<PauliGroup> gr;
  std::vector<SumSweep> sw;
  plan_sum(n, terms, &gr, &sw);
  return (uint32_t)sw.size();
}

uint32_t pauli_adjoint_sweep_count(uint32_t n, const std::vector<PauliTerm> &ansatz) {
  std::vector<PauliTerm> rev(ansatz.rbegin(), ansatz.rend());
  std::vector<RotSweep> sw;
  plan_adjoint(n, rev, &sw);
  return (uint32_t)sw.size();
}

cudaError_t run_pauli_sum(qip_prec prec, void *dst, const void *src, uint32_t n, const std::vector<PauliTerm> &terms,
                          const double *coeffs, cudaStream_t s, uint64_t *launches) {
  const size_t amp_bytes = (prec == QIP_F32 ? 2 * sizeof(float) : 2 * sizeof(double)) << n;
  if (terms.empty()) return cudaMemsetAsync(dst, 0, amp_bytes, s);  // the empty sum
  std::vector<RotArgs> args;
  std::vector<SumGroupDev> hg;
  std::vector<SumTermDev> ht;
  std::vector<size_t> g_off;
  if (!build_sum_tables(n, terms, coeffs, 1.0, &args, &hg, &ht, &g_off)) return cudaErrorInvalidValue;
  const size_t gbytes = hg.size() * sizeof(SumGroupDev), tbytes = ht.size() * sizeof(SumTermDev);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, tbytes + gbytes, s);
  if (e != cudaSuccess) return e;
  SumTermDev *dt = (SumTermDev *)d;
  SumGroupDev *dg = (SumGroupDev *)(d + tbytes);
  // pageable sources: the copies are staged before cudaMemcpyAsync returns
  e = cudaMemcpyAsync(dt, ht.data(), tbytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dg, hg.data(), gbytes, cudaMemcpyHostToDevice, s);
  const EvoSweep none = {};
  for (size_t k = 0; k < args.size() && e == cudaSuccess; ++k) {
    e = launch_sum_any<false>(prec, dst, src, args[k], dg + g_off[k], dt, k > 0, none, s);
    ++*launches;
  }
  const cudaError_t ef = cudaFreeAsync(d, s);
  return e != cudaSuccess ? e : ef;
}

cudaError_t run_pauli_evolution(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                                const std::vector<PauliTerm> &terms, const double *coeffs, double half_width,
                                const std::vector<double> &C, cudaStream_t s, uint64_t *launches) {
  const uint32_t K = (uint32_t)(C.size() / 2) - 1;
  if (terms.empty() || K < 2) return cudaErrorInvalidValue;
  // H~ = (H - a) / b: step 1 applies it with coefficients RN(c_h / b), later steps 2 H~ with RN(c_h (2 / b))
  std::vector<RotArgs> args, args2;
  std::vector<SumGroupDev> hg, hg2;
  std::vector<SumTermDev> h1, h2;
  std::vector<size_t> g_off, g_off2;
  if (!build_sum_tables(n, terms, coeffs, 1.0 / half_width, &args, &hg, &h1, &g_off) ||
      !build_sum_tables(n, terms, coeffs, 2.0 / half_width, &args2, &hg2, &h2, &g_off2))
    return cudaErrorInvalidValue;
  const size_t gbytes = hg.size() * sizeof(SumGroupDev), tbytes = h1.size() * sizeof(SumTermDev);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, 2 * tbytes + gbytes, s);
  if (e != cudaSuccess) return e;
  SumTermDev *dt1 = (SumTermDev *)d, *dt2 = (SumTermDev *)(d + tbytes);
  SumGroupDev *dg = (SumGroupDev *)(d + 2 * tbytes);
  e = cudaMemcpyAsync(dt1, h1.data(), tbytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dt2, h2.data(), tbytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dg, hg.data(), gbytes, cudaMemcpyHostToDevice, s);
  const uint32_t S = (uint32_t)args.size();
  EvoSweep ev = {};
  ev.state = state;
  ev.c0 = make_double2(C[0], C[1]);
  ev.c1 = make_double2(C[2], C[3]);
  // T_k lives in work_a for odd k and in work_b for even k; step k >= 3 overwrites T_(k-2) in place
  for (uint32_t k = 1; k <= K && e == cudaSuccess; ++k) {
    void *dst = (k & 1) ? work_a : work_b;
    const void *src = k == 1 ? state : (k & 1) ? work_b : work_a;
    ev.c2 = make_double2(C[2 * k], C[2 * k + 1]);
    for (uint32_t j = 0; j < S && e == cudaSuccess; ++j) {
      ev.from = j > 0 ? dst : k == 1 ? nullptr : k == 2 ? state : dst;
      ev.start = j == 0 && k >= 2 ? -1.0 : 1.0;
      ev.update = j + 1 < S ? 0u : k == 1 ? 0u : k == 2 ? 1u : 2u;
      e = launch_sum_any<true>(prec, dst, src, args[j], dg + g_off[j], k == 1 ? dt1 : dt2, 0, ev, s);
      ++*launches;
    }
  }
  const cudaError_t ef = cudaFreeAsync(d, s);
  return e != cudaSuccess ? e : ef;
}

cudaError_t run_lanczos_sum(qip_prec prec, void *dst, const void *src, const void *from, double start, uint32_t n,
                            const std::vector<PauliTerm> &terms, const double *coeffs, double scale, double *dot,
                            uint32_t *dot_grid, cudaStream_t s, uint64_t *launches) {
  std::vector<RotArgs> args;
  std::vector<SumGroupDev> hg;
  std::vector<SumTermDev> ht;
  std::vector<size_t> g_off;
  if (terms.empty() || !build_sum_tables(n, terms, coeffs, scale, &args, &hg, &ht, &g_off))
    return cudaErrorInvalidValue;
  const size_t gbytes = hg.size() * sizeof(SumGroupDev), tbytes = ht.size() * sizeof(SumTermDev);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, tbytes + gbytes, s);
  if (e != cudaSuccess) return e;
  SumTermDev *dt = (SumTermDev *)d;
  SumGroupDev *dg = (SumGroupDev *)(d + tbytes);
  e = cudaMemcpyAsync(dt, ht.data(), tbytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dg, hg.data(), gbytes, cudaMemcpyHostToDevice, s);
  EvoSweep ev = {};
  const size_t S = args.size();
  for (size_t j = 0; j < S && e == cudaSuccess; ++j) {
    ev.from = j > 0 ? dst : from;
    ev.start = j > 0 ? 1.0 : start;
    ev.dot = j + 1 == S ? dot : nullptr;
    e = launch_sum_any<true>(prec, dst, src, args[j], dg + g_off[j], dt, 0, ev, s);
    ++*launches;
  }
  *dot_grid = (uint32_t)std::min<uint64_t>(args.back().geo.n_visits, (uint64_t)kGradGrid);
  const cudaError_t ef = cudaFreeAsync(d, s);
  return e != cudaSuccess ? e : ef;
}

cudaError_t run_pauli_gradient(qip_prec prec, void *state, void *work, uint32_t n, const std::vector<PauliTerm> &ansatz,
                               const double *angles, const std::vector<PauliTerm> &ham, const double *coeffs, int grid,
                               cudaStream_t s, uint64_t *launches, double *energy, double *grad) {
  const uint32_t T = (uint32_t)ansatz.size();
  cudaError_t e = run_pauli_rotations(prec, state, n, ansatz, angles, grid, s, launches);
  if (e == cudaSuccess) e = run_pauli_sum(prec, work, state, n, ham, coeffs, s, launches);
  if (e != cudaSuccess) return e;
  std::vector<PauliTerm> rev(ansatz.rbegin(), ansatz.rend());
  std::vector<double> rev_angles(angles ? std::vector<double>(angles, angles + T) : std::vector<double>());
  std::reverse(rev_angles.begin(), rev_angles.end());
  std::vector<RotSweep> sw;
  plan_adjoint(n, rev, &sw);
  std::vector<RotArgs> args;
  std::vector<RotTermDev> ht;
  if (!build_rot_tables(prec, n, rev, rev_angles.data(), true, sw, &args, &ht)) return cudaErrorInvalidValue;
  const size_t tbytes = std::max<size_t>(1, ht.size()) * sizeof(RotTermDev);
  const size_t sbytes = (size_t)kAdjRows * kGradGrid * sizeof(double), rbytes = (T + 1) * sizeof(double);
  char *d = nullptr;
  e = cudaMallocAsync((void **)&d, tbytes + sbytes + rbytes, s);
  if (e != cudaSuccess) return e;
  RotTermDev *dt = (RotTermDev *)d;
  double *scratch = (double *)(d + tbytes);
  double *res = (double *)(d + tbytes + sbytes);
  if (!ht.empty()) e = cudaMemcpyAsync(dt, ht.data(), ht.size() * sizeof(RotTermDev), cudaMemcpyHostToDevice, s);
  for (size_t k = 0; k < sw.size() && e == cudaSuccess; ++k) {
    RotArgs &a = args[k];
    const uint32_t en = k == 0, g = (uint32_t)std::min<uint64_t>(a.geo.n_visits, (uint64_t)kGradGrid);
    const RotTermDev *td = dt + sw[k].first;
    e = launch_adjoint_any<false>(prec, state, work, a, td, en, scratch, g, s);
    ++*launches;
    if (e != cudaSuccess) break;
    const uint32_t rows = a.n_terms + en;
    k_adjoint_reduce<<<(rows + 255) / 256, 256, 0, s>>>(scratch, rows, g, a.n_terms, T, sw[k].first, res);
    e = cudaGetLastError();
    ++*launches;
  }
  std::vector<double> host(T + 1);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host.data(), res, rbytes, cudaMemcpyDeviceToHost, s);
  const cudaError_t ef = cudaFreeAsync(d, s);
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  if (ef != cudaSuccess) return ef;
  if (es != cudaSuccess) return es;
  *energy = host[0];
  for (uint32_t t = 0; t < T; ++t) grad[t] = host[1 + t];
  return cudaSuccess;
}

uint32_t pauli_qgt_sweep_count(uint32_t n, const std::vector<PauliTerm> &ansatz) {
  std::vector<std::vector<RotSweep>> sw;
  plan_segments(n, ansatz, &sw);
  uint64_t count = 0;
  for (const std::vector<RotSweep> &v : sw) count += v.size();
  return (uint32_t)count;
}

cudaError_t run_pauli_qgt(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                          const std::vector<PauliTerm> &ansatz, const double *angles, cudaStream_t s,
                          uint64_t *launches, double *qgt, double *expect) {
  const uint32_t T = (uint32_t)ansatz.size();
  if (T == 0) return cudaSuccess;
  std::vector<std::vector<RotSweep>> sw;
  plan_segments(n, ansatz, &sw);
  // every segment's descriptors (they depend on its sweeps), uploaded once: segment i's from ht[t_off[i]]
  std::vector<RotArgs> args;
  std::vector<RotTermDev> ht;
  std::vector<size_t> t_off(T), a_off(T);
  for (uint32_t i = 0; i < T; ++i) {
    t_off[i] = ht.size();
    a_off[i] = args.size();
    if (sw[i].empty()) continue;
    std::vector<PauliTerm> seg(ansatz.begin() + i + 1, ansatz.end());
    std::vector<RotArgs> a;
    std::vector<RotTermDev> h;
    if (!build_rot_tables(prec, n, seg, angles + i + 1, false, sw[i], &a, &h)) return cudaErrorInvalidValue;
    args.insert(args.end(), a.begin(), a.end());
    ht.insert(ht.end(), h.begin(), h.end());
  }
  // one fork grid per call, so that every fork's two rows reduce over the same CTAs at the end
  const uint32_t gf = (uint32_t)std::min<uint64_t>(kForkGrid, std::max<uint64_t>(1, (1ull << (n - 1)) / kForkThreads));
  const size_t tbytes = std::max<size_t>(1, ht.size()) * sizeof(RotTermDev);
  const size_t sbytes = (size_t)kQgtRows * kGradGrid * sizeof(double);
  const size_t fbytes = (size_t)2 * T * gf * sizeof(double);
  const size_t rcount = (size_t)2 * T * T + 2 * T, rbytes = rcount * sizeof(double);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, tbytes + sbytes + fbytes + rbytes, s);
  if (e != cudaSuccess) return e;
  RotTermDev *dt = (RotTermDev *)d;
  double *scratch = (double *)(d + tbytes);
  double *fscratch = (double *)(d + tbytes + sbytes);
  double *res = (double *)(d + tbytes + sbytes + fbytes);  // M (2 T^2), then (|psi_t|^2, e_t) per fork
  if (!ht.empty()) e = cudaMemcpyAsync(dt, ht.data(), ht.size() * sizeof(RotTermDev), cudaMemcpyHostToDevice, s);
  for (uint32_t i = 0; i < T && e == cudaSuccess; ++i) {
    const PauliTerm &P = ansatz[i];
    ForkArgs fa;
    fa.x = P.x;
    fa.z = P.z;
    fa.n_items = P.x ? 1ull << (n - 1) : 1ull << n;
    fa.h = P.x ? (uint32_t)__builtin_ctzll(P.x) : 0u;
    fa.ny = P.n_y & 3;
    // c and s exactly as build_rot_tables rounds them, so the fork rotates as the sweeps and pauli_rot.cu do
    double c = cos(angles[i] / 2), sn = sin(angles[i] / 2);
    if (prec == QIP_F32) {
      c = (double)(float)c;
      sn = (double)(float)sn;
    }
    fa.c = c;
    fa.s = sn;
    double *fs = fscratch + (size_t)2 * i * gf;
    if (prec == QIP_F32)
      k_qgt_fork<float><<<gf, kForkThreads, 0, s>>>((float *)state, (float *)work_a, (float *)work_b, fa, fs);
    else
      k_qgt_fork<double><<<gf, kForkThreads, 0, s>>>((double *)state, (double *)work_a, (double *)work_b, fa, fs);
    e = cudaGetLastError();
    ++*launches;
    for (size_t k = 0; k < sw[i].size() && e == cudaSuccess; ++k) {
      const RotArgs &a = args[a_off[i] + k];
      const uint32_t g = (uint32_t)std::min<uint64_t>(a.geo.n_visits, (uint64_t)kGradGrid);
      e = launch_adjoint_any<true>(prec, work_a, work_b, a, dt + t_off[i] + sw[i][k].first, 0, scratch, g, s);
      ++*launches;
      if (e != cudaSuccess) break;
      // rows 2r + {0, 1} of the sweep belong to term j = i + 1 + first + r: M_ij at res[2 (i T + j)]
      const uint32_t rows = 2 * a.n_terms;
      k_qgt_reduce<<<(rows + 255) / 256, 256, 0, s>>>(scratch, rows, g,
                                                      res + 2 * ((size_t)i * T + i + 1 + sw[i][k].first));
      e = cudaGetLastError();
      ++*launches;
    }
  }
  if (e == cudaSuccess) {
    k_qgt_reduce<<<(2 * T + 255) / 256, 256, 0, s>>>(fscratch, 2 * T, gf, res + (size_t)2 * T * T);
    e = cudaGetLastError();
    ++*launches;
  }
  std::vector<double> host(rcount);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host.data(), res, rbytes, cudaMemcpyDeviceToHost, s);
  const cudaError_t ef = cudaFreeAsync(d, s);
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  if (ef != cudaSuccess) return ef;
  if (es != cudaSuccess) return es;
  const double *M = host.data(), *F = host.data() + (size_t)2 * T * T;
  for (uint32_t i = 0; i < T; ++i) {
    const double ei = F[2 * i + 1];
    if (expect) expect[i] = ei;
    qgt[2 * ((size_t)i * T + i)] = 0.25 * (F[2 * i] - ei * ei);
    qgt[2 * ((size_t)i * T + i) + 1] = 0.0;
    for (uint32_t j = i + 1; j < T; ++j) {
      const size_t ij = (size_t)i * T + j, ji = (size_t)j * T + i;
      const double re = 0.25 * (M[2 * ij] - ei * F[2 * j + 1]), im = 0.25 * M[2 * ij + 1];
      qgt[2 * ij] = re;
      qgt[2 * ij + 1] = im;
      qgt[2 * ji] = re;
      qgt[2 * ji + 1] = -im;
    }
  }
  return cudaSuccess;
}

}  // namespace qipb200
