// purity.cu -- the purity Tr rho_A^2 of a bipartition as a Gram product on the FP64 tensor pipe (qipb200_state_purity).
//
// For the side S (s physical index bits, the smaller side of the cut) and the other bits O (n - s of them):
//
//   M[a][r] = psi[pdep(a, S) | pdep(r, O)],   G = M M^dagger (2^s x 2^s),   P = sum_{a,b} |G_ab|^2,   T = sum_a G_aa
//
// P is Tr rho^2 of either side, and T is the squared norm.  G is never stored (16 GiB at the N = 30 half cut): each CTA
// owns one block of G, accumulates it in registers over the whole inner dimension 2^(n-s) and folds it into P.
//
// Blocks: 128 rows (block row I) x 64 columns (block column J).  G is Hermitian, so only the blocks that touch the
// upper triangle run: J = 2I .. 2^(s-6) - 1, nR (nR + 1) blocks with nR = 2^(s-7).  Blocks are numbered row by row, so
// co-resident CTAs share the 128-row panel of their I and read it once from HBM between them (L2).  In a block with
// J >= 2I + 2 every entry lies above the diagonal; J = 2I and 2I + 1 straddle it.  Weights: 2 above the diagonal, 1 on
// it, 0 below; diagonal entries also add Re G_aa to T.
//
// Per CTA: 256 threads, 8 warps of 64 x 16 entries (4 x 2 tiles of mma.m16n8k8.f64), 64 accumulator doubles per thread
// (Re and Im, 128 KiB per CTA).  The inner dimension runs in chunks of 16: the two panels of a chunk (128 and 64 rows
// x 16 amplitudes) are staged with cp.async through three shared-memory buffers (147 KiB for f64), column-major with a
// pad that makes the fragment loads conflict-free.  The 16 inner indices of a chunk are the 4 lowest bits of O: when O
// holds index bits 0..3 (the side is high, a prefix cut) a row of a panel is 16 contiguous amplitudes, and when S holds
// the low bits (a suffix cut) a panel column is 64 or 128 contiguous ones; whole sectors either way.  f32 amplitudes are
// widened to double (exactly) when the fragments are read.  Per chunk and 8 inner indices:
//   Re G += Ar Br^T + Ai Bi^T,   Im G += Ai Br^T + Ar (-Bi)^T          (four DMMA per 16 x 8 tile)
//
// Determinism and order: every accumulator is one sequence of DMMA in chunk order.  Then each thread sums its 32
// entries as p = fma(w re, re, p), p = fma(w im, im, p) in tile order (w re is exact), the 256 thread sums of a CTA are
// added by a fixed binary tree (depth 8), and the CTA writes one (P, T) slot.  One reduction kernel (256 threads) has
// thread t add slots t, t + 256, ... in order, then a fixed binary tree (depth 8).  No floating-point atomics; the same
// state and side give the same bits.  Launches: the Gram kernel and the reduction, 2.  The s = 0 route (k = n) is
// k_purity_norm2: one read sweep of the state in a fixed order, and one kernel.
//
// Error bound (first order, u = 2^-53, gamma_m = m u / (1 - m u)).  A DMMA m16n8k8 result is taken to be no less
// accurate than 8 sequential fused multiply-adds into the accumulator (the f64 tensor pipe is IEEE round-to-nearest).
// Each component of G_ab then sums D = 2 * 2^(n-s) exact products in sequence, the moduli of which add to at most
// W_ab = sum_r |M_ar| |M_br| (|xr yr| + |xi yi| <= |x| |y|), so
//   |dG_ab| <= delta_ab = sqrt(2) gamma_D W_ab.
// The final sum adds non-negative terms w |G_ab|^2 along a chain of E = 64 + 8 + ceil(B / 256) + 8 roundings (B
// blocks), and |G + dG|^2 - |G|^2 <= 2 |G| delta + delta^2, so
//   |P_got - P| <= sum_{a,b} (2 |G_ab| delta_ab + delta_ab^2) (1 + gamma_E) + gamma_E P,
//   |T_got - T| <= gamma_{D+E} T.
// By Cauchy-Schwarz sum_{a,b} |G_ab| W_ab <= T^2, which gives a bound from the outputs alone.  tests/purity_ref.py
// evaluates both forms.
//
// The store epilogue (qipb200_state_entanglement_spectrum, sides of 11..13 qubits) runs the same main loop and writes
// G instead of folding it: k_purity_gram<R, true> stores every accumulator entry of its block that lies on or above
// the diagonal into a device G of 4^s double2 (1 GiB at s = 13), row-major in the side-qubit convention of
// reduced_density (bit i of a row index is the value of side qubit i).  The rows' indices in that convention, a' and
// b', are built with the physical offsets into the same shared-memory tables (sideA / sideB next to rowA / rowB).
// Entry (a, b) with a < b writes G_a'b' = (Re, Im) and G_b'a' = (Re, -Im), the exact conjugate; a diagonal entry
// writes (Re, +0.0); entries below the diagonal of a straddling block write nothing (their mirror is written by the
// block holding (b, a), which also runs).  Each entry is the accumulator of one fixed DMMA sequence, so G is
// deterministic, and every stored entry is within |dG_ab| <= sqrt(2) gamma_D W_ab of the exact one, hence
// ||dG||_F <= sqrt(2) gamma_D ||W||_F <= sqrt(2) gamma_D T (W = |M| |M|^T, ||W||_F <= || |M| ||_F^2 = T).  One kernel.
#include "purity.h"

#include <algorithm>

#include "rdm.h"
#include "sweep.cuh"

namespace qipb200 {

namespace {

const int kGramThreads = 256;
const int kGramBM = 128;  // rows of a block (block row I)
const int kGramBN = 64;   // columns of a block (block column J)
const int kGramBK = 16;   // inner indices per chunk: the 4 lowest bits of O
const int kGramStages = 3;
const int kGramGridPerSm = 2;   // CTAs per SM of the s = 0 sweep (a 132-SM H100)
const uint32_t kGramBMLog2 = 7;

struct GramArgs {
  uint64_t side;       // S: physical bits of the side
  uint64_t other;      // O: every other bit below 2^n
  uint64_t other_hi;   // O without its 4 lowest bits: the chunk index bits
  uint64_t n_chunks;   // 2^(n - s) / kGramBK
  uint32_t n_rows;     // nR = 2^(s - 7)
  uint32_t k_fast;     // 1 when index bit 0 is in O: the inner index is the fast one of a panel load
};

// Shared memory per stage: the two panels, column-major (inner index k, then row), each column padded so that the
// 8 (16-byte) or 16 (8-byte) lanes of a fragment load hit distinct banks.
// The store epilogue adds the rows' side indices (uint32) after the offset tables.
template <typename V, bool Store>
struct GramSmem {
  static constexpr int PAD = sizeof(V) == 16 ? 2 : 4;
  static constexpr int LDA = kGramBM + PAD, LDB = kGramBN + PAD;
  static constexpr int STAGE = kGramBK * (LDA + LDB);  // elements of V
  static constexpr size_t TABLE_BYTES =
      (kGramBM + kGramBN + kGramBK) * sizeof(uint64_t) + (Store ? (kGramBM + kGramBN) * sizeof(uint32_t) : 0);
  static constexpr size_t BYTES = TABLE_BYTES + (size_t)kGramStages * STAGE * sizeof(V);
};

__device__ __forceinline__ uint64_t pdep(uint64_t x, uint64_t mask) {
  uint64_t r = 0;
  for (uint64_t m = mask; m; m &= m - 1, x >>= 1)
    if (x & 1) r |= m & (~m + 1);
  return r;
}

__device__ __forceinline__ void dmma(double (&c)[4], const double (&a)[4], double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b0), "d"(b1));
}

// The row index of G in the side-qubit convention: bit r of x (the r-th lowest bit of S) moves to bit lbits[r], the
// 4-bit field r of lbits.
__device__ __forceinline__ uint32_t side_index(uint64_t x, uint64_t lbits) {
  uint32_t r = 0;
  for (; x; x >>= 1, lbits >>= 4)
    if (x & 1) r |= 1u << (lbits & 15);
  return r;
}

// Store == false: the purity epilogue, out = the CTA slots, lbits unused.  Store == true: out = G (4^s entries,
// row-major in the side-qubit convention), lbits as side_index takes it.
template <typename R, bool Store>
__global__ void __launch_bounds__(kGramThreads, 1)
    k_purity_gram(const R *__restrict__ psi, const __grid_constant__ GramArgs g, double2 *__restrict__ out,
                  uint64_t lbits) {
  typedef typename SweepV<R>::type V;
  typedef GramSmem<V, Store> SM;
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t *rowA = reinterpret_cast<uint64_t *>(smem);
  uint64_t *rowB = rowA + kGramBM;
  uint64_t *koff = rowB + kGramBN;
  uint32_t *sideA = reinterpret_cast<uint32_t *>(koff + kGramBK);  // Store only: a' of each row of the block
  uint32_t *sideB = sideA + kGramBM;                                 // and b' of each column
  V *stages = reinterpret_cast<V *>(smem + SM::TABLE_BYTES);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int gid = lane >> 2, tig = lane & 3;
  const int wm = warp >> 2, wn = warp & 3;  // the warp's 64 rows and 16 columns of the block

  // block (I, J): row I holds the 2 (nR - I) blocks J = 2I .. 2 nR - 1
  uint32_t I = 0;
  uint64_t b = blockIdx.x;
  while (b >= 2ull * (g.n_rows - I)) b -= 2ull * (g.n_rows - I++);
  const uint32_t J = 2 * I + (uint32_t)b;

  if (t < kGramBM) {
    rowA[t] = pdep(((uint64_t)I << kGramBMLog2) + t, g.side);
    if constexpr (Store) sideA[t] = side_index(((uint64_t)I << kGramBMLog2) + t, lbits);
  } else if (t < kGramBM + kGramBN) {
    rowB[t - kGramBM] = pdep(((uint64_t)J << (kGramBMLog2 - 1)) + (t - kGramBM), g.side);
    if constexpr (Store) sideB[t - kGramBM] = side_index(((uint64_t)J << (kGramBMLog2 - 1)) + (t - kGramBM), lbits);
  } else if (t < kGramBM + kGramBN + kGramBK)
    koff[t - kGramBM - kGramBN] = pdep(t - kGramBM - kGramBN, g.other);
  __syncthreads();

  // Stage chunk c (chunk bits kb) into buffer buf: 2048 + 1024 amplitudes, 12 per thread.
  auto load = [&](uint64_t kb, int buf) {
    V *sA = stages + (size_t)buf * SM::STAGE;
    V *sB = sA + kGramBK * SM::LDA;
#pragma unroll
    for (int j = 0; j < kGramBM * kGramBK / kGramThreads; ++j) {
      const int e = t + kGramThreads * j;
      const int k = g.k_fast ? e & (kGramBK - 1) : e >> kGramBMLog2;
      const int row = g.k_fast ? e >> 4 : e & (kGramBM - 1);
      cp_async<sizeof(V)>(sA + k * SM::LDA + row, psi + 2 * (rowA[row] | koff[k] | kb));
    }
#pragma unroll
    for (int j = 0; j < kGramBN * kGramBK / kGramThreads; ++j) {
      const int e = t + kGramThreads * j;
      const int k = g.k_fast ? e & (kGramBK - 1) : e >> (kGramBMLog2 - 1);
      const int row = g.k_fast ? e >> 4 : e & (kGramBN - 1);
      cp_async<sizeof(V)>(sB + k * SM::LDB + row, psi + 2 * (rowB[row] | koff[k] | kb));
    }
  };
  // the chunk bits of the next chunk: a masked increment over O without its 4 lowest bits
  const uint64_t step = g.other_hi & (~g.other_hi + 1);
  auto next = [&](uint64_t kb) { return ((kb | ~g.other_hi) + step) & g.other_hi; };

  double re[4][2][4], im[4][2][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) re[mt][nt][c] = im[mt][nt][c] = 0.0;

  uint64_t kb = 0;
#pragma unroll
  for (int st = 0; st < kGramStages - 1; ++st) {
    if ((uint64_t)st < g.n_chunks) {
      load(kb, st);
      kb = next(kb);
    }
    cp_async_commit();
  }
  int buf = 0;
  for (uint64_t c = 0; c < g.n_chunks; ++c) {
    cp_async_wait<kGramStages - 2>();
    __syncthreads();  // chunk c is in buf for every thread, and buffer (c - 1) % stages is free again
    if (c + kGramStages - 1 < g.n_chunks) {
      int lb = buf + kGramStages - 1;
      if (lb >= kGramStages) lb -= kGramStages;
      load(kb, lb);
      kb = next(kb);
    }
    cp_async_commit();
    const V *sA = stages + (size_t)buf * SM::STAGE + wm * 64;
    const V *sB = stages + (size_t)buf * SM::STAGE + kGramBK * SM::LDA + wn * 16;
#pragma unroll
    for (int kk = 0; kk < kGramBK; kk += 8) {
      // B fragments (k = tig, tig + 4; column gid) of the warp's two 8-column tiles: Br, Bi and -Bi
      double br[2][2], bi[2][2], nbi[2][2];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const V u = sB[(kk + tig + 4 * h) * SM::LDB + nt * 8 + gid];
          br[nt][h] = (double)u.x;
          bi[nt][h] = (double)u.y;
          nbi[nt][h] = -(double)u.y;
        }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        // A fragment: (gid, tig), (gid + 8, tig), (gid, tig + 4), (gid + 8, tig + 4)
        double ar[4], ai[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const V u = sA[(kk + tig + 4 * (q >> 1)) * SM::LDA + mt * 16 + gid + 8 * (q & 1)];
          ar[q] = (double)u.x;
          ai[q] = (double)u.y;
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          dmma(re[mt][nt], ar, br[nt][0], br[nt][1]);
          dmma(re[mt][nt], ai, bi[nt][0], bi[nt][1]);
          dmma(im[mt][nt], ai, br[nt][0], br[nt][1]);
          dmma(im[mt][nt], ar, nbi[nt][0], nbi[nt][1]);
        }
      }
    }
    if (++buf == kGramStages) buf = 0;
  }
  cp_async_wait<0>();

  // accumulator c of tile (mt, nt) is entry (gid + 8 (c >> 1), 2 tig + (c & 1)) of the tile
  if constexpr (Store) {
    const uint64_t K = (uint64_t)g.n_rows << kGramBMLog2;
    const int64_t a0 = ((int64_t)I << kGramBMLog2) + wm * 64 + gid, b0 = ((int64_t)J << (kGramBMLog2 - 1)) + wn * 16 + 2 * tig;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int ra = wm * 64 + mt * 16 + gid + 8 * (c >> 1), rb = wn * 16 + nt * 8 + 2 * tig + (c & 1);
          const int64_t a = a0 + mt * 16 + 8 * (c >> 1), bb = b0 + nt * 8 + (c & 1);
          const uint64_t la = sideA[ra], lb = sideB[rb];
          if (a == bb) {
            out[la * K + la] = make_double2(re[mt][nt][c], 0.0);
          } else if (a < bb) {
            out[la * K + lb] = make_double2(re[mt][nt][c], im[mt][nt][c]);
            out[lb * K + la] = make_double2(re[mt][nt][c], -im[mt][nt][c]);
          }
        }
    return;
  }
  double p = 0.0, tr = 0.0;
  const int64_t a0 = ((int64_t)I << kGramBMLog2) + wm * 64 + gid, b0 = ((int64_t)J << (kGramBMLog2 - 1)) + wn * 16 + 2 * tig;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int64_t a = a0 + mt * 16 + 8 * (c >> 1), bb = b0 + nt * 8 + (c & 1);
        const double w = a < bb ? 2.0 : a == bb ? 1.0 : 0.0;
        p = fma(w * re[mt][nt][c], re[mt][nt][c], p);
        p = fma(w * im[mt][nt][c], im[mt][nt][c], p);
        if (a == bb) tr += re[mt][nt][c];
      }
  __syncthreads();
  double2 *red = reinterpret_cast<double2 *>(smem);
  red[t] = make_double2(p, tr);
  __syncthreads();
  for (int h = kGramThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      red[t].x += red[t + h].x;
      red[t].y += red[t + h].y;
    }
    __syncthreads();
  }
  if (t == 0) out[blockIdx.x] = red[0];
}

// out2 = the sum of the slots in block order, by one CTA: thread t adds slots t, t + 256, ..., then a fixed binary tree.
__device__ void reduce_slots(const double2 *__restrict__ slots, uint64_t n_slots, double *__restrict__ out2) {
  __shared__ double2 red[kGramThreads];
  const int t = threadIdx.x;
  double2 s = make_double2(0.0, 0.0);
  for (uint64_t i = t; i < n_slots; i += kGramThreads) {
    const double2 v = __ldcg(slots + i);
    s.x += v.x;
    s.y += v.y;
  }
  red[t] = s;
  __syncthreads();
  for (int h = kGramThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      red[t].x += red[t + h].x;
      red[t].y += red[t + h].y;
    }
    __syncthreads();
  }
  if (t == 0) {
    out2[0] = red[0].x;
    out2[1] = red[0].y;
  }
}

__global__ void __launch_bounds__(kGramThreads) k_purity_reduce(const double2 *__restrict__ slots, uint64_t n_slots,
                                                                double *__restrict__ out2) {
  reduce_slots(slots, n_slots, out2);
}

// The s = 0 route: out2[0] = sum_j |psi_j|^2 in one kernel and a fixed order.  Each thread adds its amplitudes (grid
// stride) with two fma each, a CTA adds its threads by a fixed binary tree into its slot, and the CTA that finishes
// last (an integer counter) sums the slots as reduce_slots does.
template <typename R>
__global__ void __launch_bounds__(kGramThreads) k_purity_norm2(const R *__restrict__ psi, uint64_t len,
                                                               double2 *__restrict__ slots, unsigned *counter,
                                                               double *__restrict__ out2) {
  typedef typename SweepV<R>::type V;
  __shared__ double red[kGramThreads];
  __shared__ bool last;
  const int t = threadIdx.x;
  double acc = 0.0;
  for (uint64_t i = (uint64_t)blockIdx.x * kGramThreads + t; i < len; i += (uint64_t)gridDim.x * kGramThreads) {
    const V v = reinterpret_cast<const V *>(psi)[i];
    acc = fma((double)v.x, (double)v.x, acc);
    acc = fma((double)v.y, (double)v.y, acc);
  }
  red[t] = acc;
  __syncthreads();
  for (int h = kGramThreads / 2; h > 0; h >>= 1) {
    if (t < h) red[t] += red[t + h];
    __syncthreads();
  }
  if (t == 0) {
    slots[blockIdx.x] = make_double2(red[0], 0.0);
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last) {
    __threadfence();
    reduce_slots(slots, gridDim.x, out2);
  }
}

template <typename R, bool Store>
cudaError_t launch_gram(const void *psi, const GramArgs &g, uint64_t n_blocks, double2 *out, uint64_t lbits,
                        cudaStream_t s) {
  typedef GramSmem<typename SweepV<R>::type, Store> SM;
  static_assert(SM::BYTES <= 227 * 1024, "one CTA per SM: at most 227 KiB of shared memory");
  static_assert(kGramThreads * sizeof(double2) <= SM::BYTES, "the CTA reduction reuses the stage buffers");
  cudaError_t e =
      cudaFuncSetAttribute(k_purity_gram<R, Store>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM::BYTES);
  if (e != cudaSuccess) return e;
  k_purity_gram<R, Store><<<(unsigned)n_blocks, kGramThreads, SM::BYTES, s>>>((const R *)psi, g, out, lbits);
  return cudaGetLastError();
}

// The kernel's arguments for the side side_mask (s = popcount >= 7) of an unsharded 2^n state.
GramArgs gram_args(uint32_t n, uint64_t side_mask) {
  const uint32_t sb = (uint32_t)__builtin_popcountll(side_mask);
  GramArgs g;
  g.side = side_mask;
  g.other = ((n >= 64 ? 0ull : 1ull << n) - 1) & ~side_mask;
  uint64_t low = g.other;
  for (int i = 0; i < 4; ++i) low &= low - 1;  // clear the 4 lowest bits of O
  g.other_hi = low;
  g.n_chunks = 1ull << (n - sb - 4);
  g.n_rows = 1u << (sb - kGramBMLog2);
  g.k_fast = g.other & 1;
  return g;
}

}  // namespace

cudaError_t run_purity_norm2(qip_prec prec, const void *psi, uint32_t n, double *out, cudaStream_t s,
                             uint64_t *launches) {
  const unsigned grid = kGramGridPerSm * 132;
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, (grid + 1) * sizeof(double2) + sizeof(unsigned), s);
  if (e != cudaSuccess) return e;
  double2 *slots = (double2 *)d;
  double *d_out = (double *)(slots + grid);
  unsigned *counter = (unsigned *)(slots + grid + 1);
  e = cudaMemsetAsync(counter, 0, sizeof(unsigned), s);
  if (e == cudaSuccess) {
    if (prec == QIP_F32)
      k_purity_norm2<float><<<grid, kGramThreads, 0, s>>>((const float *)psi, 1ull << n, slots, counter, d_out);
    else
      k_purity_norm2<double><<<grid, kGramThreads, 0, s>>>((const double *)psi, 1ull << n, slots, counter, d_out);
    ++*launches;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, sizeof(double), cudaMemcpyDeviceToHost, s);
  const cudaError_t ef = cudaFreeAsync(d, s);
  if (e == cudaSuccess) e = ef;
  const cudaError_t es = cudaStreamSynchronize(s);
  return e == cudaSuccess ? es : e;
}

uint32_t purity_route(uint32_t s) { return s == 0 ? 0 : s < kPurityGramMinSide ? 1 : 2; }

uint64_t purity_gram_blocks(uint32_t s) {
  const uint64_t nr = 1ull << (s - kGramBMLog2);
  return nr * (nr + 1);
}

uint64_t purity_launch_count(uint32_t s) {
  switch (purity_route(s)) {
    case 0: return 1;
    case 1: return rdm_launch_count(s);
    default: return 2;
  }
}

cudaError_t run_purity_gram(qip_prec prec, const void *psi, uint32_t n, uint64_t side_mask, double *out2,
                            cudaStream_t s, uint64_t *launches) {
  const uint32_t sb = (uint32_t)__builtin_popcountll(side_mask);
  const GramArgs g = gram_args(n, side_mask);
  const uint64_t n_blocks = purity_gram_blocks(sb);
  double2 *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, (n_blocks + 1) * sizeof(double2), s);
  if (e != cudaSuccess) return e;
  double2 *d_out = d + n_blocks;
  e = prec == QIP_F32 ? launch_gram<float, false>(psi, g, n_blocks, d, 0, s)
                      : launch_gram<double, false>(psi, g, n_blocks, d, 0, s);
  ++*launches;
  if (e == cudaSuccess) {
    k_purity_reduce<<<1, kGramThreads, 0, s>>>(d, n_blocks, reinterpret_cast<double *>(d_out));
    ++*launches;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out2, d_out, 2 * sizeof(double), cudaMemcpyDeviceToHost, s);
  const cudaError_t ef = cudaFreeAsync(d, s);
  if (e == cudaSuccess) e = ef;
  const cudaError_t es = cudaStreamSynchronize(s);
  return e == cudaSuccess ? es : e;
}

cudaError_t run_gram_store(qip_prec prec, const void *psi, uint32_t n, const uint32_t *pos, uint32_t sb, double2 *G,
                           cudaStream_t s, uint64_t *launches) {
  uint64_t side_mask = 0;
  for (uint32_t i = 0; i < sb; ++i) side_mask |= 1ull << pos[i];
  // field r of lbits: the side qubit i whose physical bit pos[i] is the r-th lowest bit of the mask
  uint64_t lbits = 0;
  for (uint32_t i = 0; i < sb; ++i)
    lbits |= (uint64_t)i << (4 * __builtin_popcountll(side_mask & ((1ull << pos[i]) - 1)));
  const GramArgs g = gram_args(n, side_mask);
  const uint64_t n_blocks = purity_gram_blocks(sb);
  const cudaError_t e = prec == QIP_F32 ? launch_gram<float, true>(psi, g, n_blocks, G, lbits, s)
                                        : launch_gram<double, true>(psi, g, n_blocks, G, lbits, s);
  ++*launches;
  const cudaError_t es = cudaStreamSynchronize(s);
  return e == cudaSuccess ? es : e;
}

}  // namespace qipb200
