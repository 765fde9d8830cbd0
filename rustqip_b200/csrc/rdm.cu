// rdm.cu -- reduced density matrices of up to kRdmMaxKept qubits (qipb200_state_reduced_density).
//
//   rho[a][b] = sum_r psi(r, a) conj(psi(r, b))     (partial trace over every index bit not kept)
//
// Tile geometry of sweep.cuh: the kSweepL lowest index bits plus up to kRdmM chosen high bits, 2^11 amplitudes.  Up to
// six kept bits ("columns") are tile bits; the other tile bits and the visit index are the traced-out rows r.  A tile is
// then a block X of rows x C entries (C = 2^min(k, 6)), and a CTA accumulates X_I^T conj(X_J) over the tiles it visits.
//   - k <= 6: every kept bit is a column, I = J, one read sweep gives all of rho.
//   - 7 <= k <= 10: the other k - 6 kept bits are block bits outside the tile, rho has nB x nB blocks of 64 x 64
//     (nB = 2^(k-6)), and block (I, J) with I <= J reads the tile pair (base | I, base | J): nB sweeps of the state in
//     all.  The lower blocks are the conjugate transposes of the upper ones.
// Work per tile: each thread owns a register block of RB x RB entries (columns a = ablk + Q i, b = bblk + Q j) and a
// share of the rows; for C = 64 a thread owns one 4 x 4 block and every row (8 shared-memory loads per 16 complex
// multiply-adds), for smaller C the rows are split over S threads and their partials summed in a fixed order at the
// end.  On a diagonal block (I = J) the entries with i > j lie strictly below the diagonal and are skipped: the host
// writes the lower triangle as the conjugate of the upper one.  Amplitudes are staged with cp.async; single tiles are
// double-buffered (the next tile loads while the current one is multiplied).  f32 amplitudes are converted to double
// as they are read from shared memory, and every sum is in double.
//
// Determinism: a fixed grid of kRdmGrid CTAs with a static tile assignment, per-thread accumulation in tile and row
// order with explicit fma, the row splits summed in thread order, per-CTA partials [CTA][entry] summed by one reduction
// kernel per block pair in CTA order.  No floating-point atomics.
//
// Launches: one sweep kernel and one reduction per block pair, nB (nB + 1) in all (2 for k <= 6).  Scratch: one block
// pair's partials (kRdmGrid x 4096 x 16 B = 17.3 MB) plus the device copy of rho (16 MiB at k = 10), below 40 MB.
// Shared memory: 64 KiB per CTA at most (two f64 tiles, or the row-split partials), so two CTAs fit on an SM.
#include "rdm.h"

#include <algorithm>
#include <complex>
#include <cstring>
#include <vector>

#include "sweep.cuh"

namespace qipb200 {

namespace {

const uint32_t kRdmM = 7;          // chosen high bits of a tile
const uint32_t kRdmTileLog2 = kSweepL + kRdmM;
const uint32_t kRdmTile = 1u << kRdmTileLog2;
const uint32_t kRdmColsLog2 = 6;   // kept bits inside the tile
const int kRdmThreads = 256;
const int kRdmPer = kRdmTile / kRdmThreads;  // tile amplitudes staged per thread
const int kRdmGrid = 264;          // CTAs per sweep: two per SM of a 132-SM H100
static_assert(kRdmM <= kSweepMaxHi, "the high tile bits fit SweepTiles::hi_pos");

struct RdmArgs {
  SweepTiles geo;         // x_out = 0; the block bits are skipped
  uint64_t off_i, off_j;  // block bits of the tiles I and J
  uint32_t rows;          // rows per tile: 2^tb / C
  uint8_t slot[kRdmTileLog2];  // tile slot -> 0x80 | column bit, or row bit
};

// Register blocks: RB x RB entries per thread, Q x Q blocks, S threads per block splitting the rows.
template <int C>
struct RdmShape {
  static constexpr int RB = C < 4 ? C : 4;
  static constexpr int Q = C / RB;
  static constexpr int NB = Q * Q;
  static constexpr int S = kRdmThreads / NB;
  // C >= 32: X stored row by row, the threads of a warp read neighbouring columns of one row; C <= 16: column by
  // column, the threads of a warp read neighbouring rows of one column.  Either way a warp's loads are contiguous.
  static constexpr bool ROWMAJOR = C >= 32;
  static constexpr size_t RED_BYTES = S > 1 ? (size_t)RB * RB * kRdmThreads * sizeof(double2) : 0;
};

template <typename R, int C, bool SAME>
__global__ void __launch_bounds__(kRdmThreads, 2)
    k_rdm(const R *__restrict__ psi, const __grid_constant__ RdmArgs a, double2 *__restrict__ partials) {
  typedef typename SweepV<R>::type V;
  typedef RdmShape<C> SH;
  constexpr int RB = SH::RB, Q = SH::Q, NB = SH::NB, S = SH::S;
  constexpr bool ROWMAJOR = SH::ROWMAJOR;
  constexpr int NT = SAME ? 1 : 2;  // tiles per visit; single tiles are double-buffered, so 2 tiles of smem either way
  extern __shared__ __align__(16) unsigned char smem[];
  V *tiles = reinterpret_cast<V *>(smem);
  const int t = threadIdx.x;
  const uint32_t tsize = 1u << a.geo.tb, rows = a.rows;
  const int blk = ROWMAJOR ? t % NB : t / S, split = ROWMAJOR ? t / NB : t % S;
  const int ablk = blk / Q, bblk = blk % Q;
  // global offset and shared-memory slot of the tile elements this thread stages
  uint64_t off[kRdmPer];
  uint32_t dst[kRdmPer];
#pragma unroll
  for (int k = 0; k < kRdmPer; ++k) {
    const uint32_t e = t + kRdmThreads * k;
    // tile_offset(a.geo, e), fused with the slot loop: written as tile_offset plus a separate slot loop, each k_rdm
    // instantiation compiles to 96-112 more SASS instructions (e.g. k_rdm<double, 64, true>: 2000 -> 2096) and its
    // register count moves by -12..+8 (sm_90a, CUDA 12.9)
    uint64_t o = e & ((1u << a.geo.L) - 1);
    uint32_t c = 0, r = 0;
    for (uint32_t sl = 0; sl < a.geo.tb; ++sl) {
      const uint32_t bit = (e >> sl) & 1u;
      if (sl >= a.geo.L) o |= (uint64_t)bit << a.geo.hi_pos[sl - a.geo.L];
      const uint32_t code = a.slot[sl];
      if (code & 0x80)
        c |= bit << (code & 0x7f);
      else
        r |= bit << code;
    }
    off[k] = o;
    dst[k] = ROWMAJOR ? r * C + c : c * rows + r;
  }
  auto issue = [&](uint64_t v, int b) {
    const uint64_t base = visit_base(a.geo, v);
    V *sI = tiles + (size_t)b * tsize;
    V *sJ = sI + tsize;
#pragma unroll
    for (int k = 0; k < kRdmPer; ++k) {
      if ((uint32_t)(t + kRdmThreads * k) >= tsize) continue;
      cp_async<sizeof(V)>(sI + dst[k], psi + 2 * (base | a.off_i | off[k]));
      if (!SAME) cp_async<sizeof(V)>(sJ + dst[k], psi + 2 * (base | a.off_j | off[k]));
    }
  };
  double2 acc[RB][RB];
#pragma unroll
  for (int i = 0; i < RB; ++i)
#pragma unroll
    for (int j = 0; j < RB; ++j) acc[i][j] = make_double2(0.0, 0.0);
  uint64_t v = blockIdx.x;
  if (v < a.geo.n_visits) issue(v, 0);
  cp_async_commit();
  int cur = 0;
  for (; v < a.geo.n_visits; v += gridDim.x) {
    const uint64_t nv = v + gridDim.x;
    if (SAME) {  // the next tile into the other buffer, then wait for the current one only
      if (nv < a.geo.n_visits) issue(nv, cur ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const V *XI = tiles + (size_t)cur * NT * tsize;
    const V *XJ = SAME ? XI : XI + tsize;
    for (uint32_t r = split; r < rows; r += S) {
      double2 xi[RB], xj[RB];
#pragma unroll
      for (int i = 0; i < RB; ++i) {
        const V u = XI[ROWMAJOR ? r * C + ablk + Q * i : (ablk + Q * i) * rows + r];
        xi[i] = make_double2((double)u.x, (double)u.y);
      }
#pragma unroll
      for (int j = 0; j < RB; ++j) {
        const V u = XJ[ROWMAJOR ? r * C + bblk + Q * j : (bblk + Q * j) * rows + r];
        xj[j] = make_double2((double)u.x, (double)u.y);
      }
#pragma unroll
      for (int i = 0; i < RB; ++i)
#pragma unroll
        for (int j = 0; j < RB; ++j) {
          if (SAME && i > j) continue;  // strictly below the diagonal: written by the host from the upper triangle
          // acc += xi * conj(xj)
          acc[i][j].x = fma(xi[i].x, xj[j].x, acc[i][j].x);
          acc[i][j].x = fma(xi[i].y, xj[j].y, acc[i][j].x);
          acc[i][j].y = fma(xi[i].y, xj[j].x, acc[i][j].y);
          acc[i][j].y = fma(-xi[i].x, xj[j].y, acc[i][j].y);
        }
    }
    __syncthreads();  // the readers of this buffer are done
    if (SAME) {
      cur ^= 1;
    } else {
      if (nv < a.geo.n_visits) issue(nv, 0);
      cp_async_commit();
    }
  }
  cp_async_wait<0>();
  double2 *col = partials + (size_t)blockIdx.x * C * C;  // this CTA's partials
  if (S == 1) {
#pragma unroll
    for (int i = 0; i < RB; ++i)
#pragma unroll
      for (int j = 0; j < RB; ++j) col[(ablk + Q * i) * C + bblk + Q * j] = acc[i][j];
    return;
  }
  // the S row splits of every register block, summed in split order
  __syncthreads();
  double2 *red = reinterpret_cast<double2 *>(smem);  // [entry of the register block][thread]
#pragma unroll
  for (int i = 0; i < RB; ++i)
#pragma unroll
    for (int j = 0; j < RB; ++j) red[(i * RB + j) * kRdmThreads + t] = acc[i][j];
  __syncthreads();
  for (int e = t; e < C * C; e += kRdmThreads) {
    const int ea = e / C, eb = e % C;
    const int slot = (ea / Q) * RB + eb / Q, bk = (ea % Q) * Q + eb % Q;
    double2 sum = make_double2(0.0, 0.0);
    for (int q = 0; q < S; ++q) {
      const double2 p = red[slot * kRdmThreads + (ROWMAJOR ? q * NB + bk : bk * S + q)];
      sum.x += p.x;
      sum.y += p.y;
    }
    col[e] = sum;
  }
}

// rho'[(I C + a) K + J C + b] = sum over the grid's partials, in CTA order.
__global__ void __launch_bounds__(256) k_rdm_reduce(const double2 *__restrict__ partials, uint32_t C, uint32_t grid,
                                                     double2 *__restrict__ rho, uint32_t K, uint32_t I, uint32_t J) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t E = C * C;
  if (e >= E) return;
  double2 s = make_double2(0.0, 0.0);
  for (uint32_t c = 0; c < grid; ++c) {
    const double2 p = partials[(uint64_t)c * E + e];
    s.x += p.x;
    s.y += p.y;
  }
  rho[(uint64_t)(I * C + e / C) * K + J * C + e % C] = s;
}

template <typename R, int C, bool SAME>
cudaError_t launch_rdm(const void *psi, const RdmArgs &a, double2 *partials, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  typedef RdmShape<C> SH;
  static_assert(2 * kRdmTile * sizeof(double2) <= 113 * 1024 && SH::RED_BYTES <= 113 * 1024,
                "two CTAs per SM: at most 113 KiB of shared memory each");
  const size_t smem = std::max(((size_t)2 << a.geo.tb) * sizeof(V), SH::RED_BYTES);
  const size_t smem_max = std::max((size_t)2 * kRdmTile * sizeof(V), SH::RED_BYTES);
  cudaError_t e = cudaFuncSetAttribute(k_rdm<R, C, SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
  if (e != cudaSuccess) return e;
  k_rdm<R, C, SAME><<<kRdmGrid, kRdmThreads, smem, s>>>((const R *)psi, a, partials);
  return cudaGetLastError();
}

template <typename R>
cudaError_t launch_sweep(const void *psi, const RdmArgs &a, uint32_t C, bool same, double2 *partials, cudaStream_t s) {
  if (!same) return launch_rdm<R, 64, false>(psi, a, partials, s);  // off-diagonal blocks: k > 6, so C = 64
  switch (C) {
    case 2: return launch_rdm<R, 2, true>(psi, a, partials, s);
    case 4: return launch_rdm<R, 4, true>(psi, a, partials, s);
    case 8: return launch_rdm<R, 8, true>(psi, a, partials, s);
    case 16: return launch_rdm<R, 16, true>(psi, a, partials, s);
    case 32: return launch_rdm<R, 32, true>(psi, a, partials, s);
    default: return launch_rdm<R, 64, true>(psi, a, partials, s);
  }
}

}  // namespace

uint64_t rdm_launch_count(uint32_t k) {
  const uint64_t nb = 1ull << (k > kRdmColsLog2 ? k - kRdmColsLog2 : 0);
  return nb * (nb + 1);
}

cudaError_t run_reduced_density(qip_prec prec, const void *psi, uint32_t n, const uint32_t *pos, uint32_t k,
                                double *out, cudaStream_t s, uint64_t *launches) {
  const uint32_t L = std::min(kSweepL, n);
  const uint32_t k_in = std::min(k, kRdmColsLog2), C = 1u << k_in, nB = 1u << (k - k_in), K = 1u << k;
  // columns: the kept bits among the L low bits (always in the tile) first, then the others in the given order; the
  // kept bits left over are block bits, all above the low bits
  std::vector<uint32_t> col, blk;
  uint64_t kept = 0;
  for (uint32_t i = 0; i < k; ++i) {
    kept |= 1ull << pos[i];
    if (pos[i] < L) col.push_back(i);
  }
  for (uint32_t i = 0; i < k; ++i)
    if (pos[i] >= L) (col.size() < k_in ? col : blk).push_back(i);
  // high tile bits: the columns above the low bits, then the lowest bits that are not kept
  uint64_t hi = 0, blk_mask = 0;
  for (uint32_t i : col)
    if (pos[i] >= L) hi |= 1ull << pos[i];
  const uint32_t m = std::min(kRdmM, n - L - (uint32_t)blk.size());
  for (uint32_t b = L; b < n && (uint32_t)__builtin_popcountll(hi) < m; ++b)
    if (!((kept >> b) & 1)) hi |= 1ull << b;
  for (uint32_t i : blk) blk_mask |= 1ull << pos[i];
  RdmArgs a;
  memset(&a, 0, sizeof(a));
  a.geo = sweep_tiles(n, L, hi, 0, blk_mask);
  uint32_t n_rows_bits = 0;
  for (uint32_t sl = 0; sl < a.geo.tb; ++sl) {
    const uint32_t p = sl < L ? sl : a.geo.hi_pos[sl - L];
    uint32_t code = 0xff;
    for (uint32_t ci = 0; ci < k_in; ++ci)
      if (pos[col[ci]] == p) code = 0x80 | ci;
    a.slot[sl] = (uint8_t)(code == 0xff ? n_rows_bits++ : code);
  }
  a.rows = 1u << n_rows_bits;

  const size_t part_bytes = (size_t)kRdmGrid * C * C * sizeof(double2);
  const size_t rho_bytes = (size_t)K * K * sizeof(double2);
  char *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, part_bytes + rho_bytes, s);
  if (e != cudaSuccess) return e;
  double2 *d_part = (double2 *)d;
  double2 *d_rho = (double2 *)(d + part_bytes);
  auto spread = [&](uint32_t I) {
    uint64_t o = 0;
    for (size_t bi = 0; bi < blk.size(); ++bi) o |= (uint64_t)((I >> bi) & 1u) << pos[blk[bi]];
    return o;
  };
  for (uint32_t I = 0; I < nB && e == cudaSuccess; ++I)
    for (uint32_t J = I; J < nB && e == cudaSuccess; ++J) {
      a.off_i = spread(I);
      a.off_j = spread(J);
      e = prec == QIP_F32 ? launch_sweep<float>(psi, a, C, I == J, d_part, s)
                          : launch_sweep<double>(psi, a, C, I == J, d_part, s);
      ++*launches;
      if (e != cudaSuccess) break;
      k_rdm_reduce<<<(C * C + 255) / 256, 256, 0, s>>>(d_part, C, kRdmGrid, d_rho, K, I, J);
      ++*launches;
      e = cudaGetLastError();
    }
  std::vector<std::complex<double>> h((size_t)K * K);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h.data(), d_rho, rho_bytes, cudaMemcpyDeviceToHost, s);
  const cudaError_t ef = cudaFreeAsync(d, s);
  if (e == cudaSuccess) e = ef;
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = es;
  if (e != cudaSuccess) return e;
  // internal index: bit ci < k_in <-> kept qubit col[ci], bit k_in + bi <-> blk[bi]; only its upper triangle is valid
  std::vector<uint32_t> map(K, 0);
  for (uint32_t x = 0; x < K; ++x)
    for (uint32_t i = 0; i < k; ++i) {
      if (!((x >> i) & 1)) continue;
      for (uint32_t ci = 0; ci < k_in; ++ci)
        if (col[ci] == i) map[x] |= 1u << ci;
      for (size_t bi = 0; bi < blk.size(); ++bi)
        if (blk[bi] == i) map[x] |= 1u << (k_in + bi);
    }
  for (uint32_t x = 0; x < K; ++x)
    for (uint32_t y = 0; y < K; ++y) {
      const uint32_t xi = map[x], yi = map[y];
      std::complex<double> v = xi <= yi ? h[(size_t)xi * K + yi] : std::conj(h[(size_t)yi * K + xi]);
      if (x == y) v.imag(0.0);
      out[2 * ((size_t)x * K + y)] = v.real();
      out[2 * ((size_t)x * K + y) + 1] = v.imag();
    }
  return cudaSuccess;
}

}  // namespace qipb200
