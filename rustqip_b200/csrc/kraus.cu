// kraus.cu -- one quantum-trajectory step of channels on k = 1..4 qubits each with any complete set of Kraus operators
// (qipb200_state_apply_kraus_channels): the host-side validation, grouping and choice, and the grouped apply sweep.
//
// Sampling.  For channels c on disjoint qubits the outcome tuple i has probability p(i) = Tr[(x)_c M_{i_c} rho] with
// M = K^dagger K and rho = |psi><psi|.  A general M is not diagonal, so the monomial argument of channel.cu (one sample
// draw decides every channel) does not apply; the tuple is drawn channel by channel instead, each choice conditioned
// on the earlier ones:
//   p(i_c | i_1 .. i_{c-1}) = Tr[(M_{i_1} (x) .. (x) M_{i_c}) rho] / Tr[(M_{i_1} (x) .. (x) M_{i_{c-1}}) rho]
// (completeness sums the later channels out), and the product of the conditionals is p(i).  Within a group the
// numerators only need the reduced density matrix of the group's qubits.  Across groups, the state after the earlier
// groups' chosen operators, each scaled by 1/sqrt(cond), is the conditioned state renormalised: its reduced density
// matrix on the next group's qubits gives that group's conditionals.  So each group costs the sweep that applies the
// previous group's operators, which accumulates the next group's matrix from the amplitudes it stores.
//   - A state-independent channel (every M_i within 1e-12 of w_i I) has p(i_c | ...) = w_i whatever the state: it is
//     drawn on the host and its operator K / sqrt(w_i), unitary, goes through the fused schedule after the groups
//     (its qubits are disjoint from the groups', so it commutes with them).
//   - Each group's choice is made on the host in double from its matrix (kraus_draw_group).
//
// Sweep (k_kraus_apply_rdm<R, C, KMAX>): tiles of the sweep.cuh geometry, the 4 low bits plus the physical bits of the
// current group (A) and of the next one (B) above them, filled up with the lowest free bits to kSweepMaxHi high bits:
// 2^12 amplitudes, 64 KiB in f64.  A CTA stages a tile with cp.async, applies A's operators in channel order, each as
// a 2^k matvec on every fibre of its bits, stores the tile back, and accumulates the C x C matrix of B (C = 2^|B|)
// from the stored values, widened to double.  With no next group C = 0 and the accumulation is compiled out.
//
// Arithmetic of the apply (fixed, so that a host emulation reproduces it bit for bit): the scaled operator
// K' = RN_prec(K_re s) + i RN_prec(K_im s), s = 1 / sqrt(cond) in double (sqrt and the division each rounded once),
// and for every fibre (x_0 .. x_{2^k - 1}) of the channel's bits (the column index in the matrix convention)
//   y_r = ((t_r0 + t_r1) + t_r2) + ...,   t_rb = (RN(RN(K'_re x_re) - RN(K'_im x_im)), RN(RN(K'_re x_im) + RN(K'_im x_re)))
// in the state's precision without FMA, columns in ascending order, one channel after the other.
//
// Accumulation (C > 0): the register-block scheme of rdm.cu.  Thread t owns a RB x RB block of entries and a share
// of the rows; per thread the terms are added in tile order, then row order, with explicit fma; the S row splits of
// a block are added in split order; one partial per CTA on a fixed grid of kKrausGrid CTAs, summed in CTA order by
// k_kraus_reduce.  No floating-point atomics, so the matrix is the same bits on every run and every device.  Entries
// strictly below the diagonal are not accumulated: the host writes them as the conjugates of the upper ones.
#include "kraus.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "sweep.cuh"

namespace qipb200 {

namespace {

typedef std::complex<double> cd;

const uint32_t kKrausHi = kSweepMaxHi;              // chosen high bits of a tile
const uint32_t kKrausTileLog2 = kSweepL + kKrausHi;
const uint32_t kKrausTile = 1u << kKrausTileLog2;   // 4096 amplitudes
const int kKrausThreads = 256;
const int kKrausPer = kKrausTile / kKrausThreads;   // tile amplitudes staged per thread
const int kKrausGrid = 264;                         // fixed: two CTAs per SM of a 132-SM H100
const uint32_t kKrausMatEntries = 256;              // complex entries of a group's scaled operators (sum of 4^k <= 4^4)

struct KrausArgs {
  SweepTiles geo;
  uint32_t n_ch;                              // channels of group A
  uint32_t k[kKrausGroupBits];                // their arities
  uint32_t mat_off[kKrausGroupBits];          // their matrices' first entry
  uint8_t slot[kKrausGroupBits][kKrausMaxArity];  // their tile slots, ascending
  uint16_t off[kKrausGroupBits][16];          // tile-local offset of matrix index b
  uint32_t nb;                                // bits of group B
  uint8_t bslot[kKrausGroupBits];             // B's tile slots, ascending
  uint16_t boff[16];                          // tile-local offset of column a of B
};

// Register blocks of the accumulation, as in rdm.cu: RB x RB entries per thread, Q x Q blocks, S row splits.
template <int C>
struct KrausShape {
  static constexpr int RB = C < 4 ? (C < 1 ? 1 : C) : 4;
  static constexpr int Q = C < 1 ? 1 : C / RB;
  static constexpr int NB = Q * Q;
  static constexpr int S = kKrausThreads / NB;
  static constexpr size_t RED_BYTES = C > 0 && S > 1 ? (size_t)RB * RB * kKrausThreads * sizeof(double2) : 0;
};

// f with a zero bit inserted at each of the k ascending slots s.
__device__ __forceinline__ uint32_t insert_zeros(uint32_t f, const uint8_t *s, uint32_t k) {
  for (uint32_t i = 0; i < k; ++i) f = ((f >> s[i]) << (s[i] + 1)) | (f & ((1u << s[i]) - 1));
  return f;
}

// k' x in the state's precision without FMA.
template <typename V>
__device__ __forceinline__ V cmul_prec(V k, V x) {
  V y;
  y.x = add_rn(mul_rn(k.x, x.x), -mul_rn(k.y, x.y));
  y.y = add_rn(mul_rn(k.x, x.y), mul_rn(k.y, x.x));
  return y;
}

// y = K' x on every fibre of one channel's K bits in the tile.
template <int K, typename V>
__device__ __forceinline__ void apply_fibres(V *tile, const V *M, const uint8_t *slot, const uint16_t *off,
                                             uint32_t tsize) {
  constexpr int D = 1 << K;
  const uint32_t nf = tsize >> K;
  for (uint32_t f = threadIdx.x; f < nf; f += kKrausThreads) {
    const uint32_t e0 = insert_zeros(f, slot, K);
    V x[D];
#pragma unroll
    for (int b = 0; b < D; ++b) x[b] = tile[e0 | off[b]];
#pragma unroll
    for (int r = 0; r < D; ++r) {
      V y = cmul_prec(M[r * D], x[0]);
#pragma unroll
      for (int b = 1; b < D; ++b) {
        const V t = cmul_prec(M[r * D + b], x[b]);
        y.x = add_rn(y.x, t.x);
        y.y = add_rn(y.y, t.y);
      }
      tile[e0 | off[r]] = y;
    }
  }
}

template <typename R, int C, int KMAX>
__global__ void __launch_bounds__(kKrausThreads, 2)
    k_kraus_apply_rdm(R *__restrict__ psi, const __grid_constant__ KrausArgs a, const void *__restrict__ mat,
                      double2 *__restrict__ partials) {
  typedef typename SweepV<R>::type V;
  typedef KrausShape<C> SH;
  constexpr int RB = SH::RB, Q = SH::Q, NB = SH::NB, S = SH::S;
  extern __shared__ __align__(16) unsigned char smem[];
  V *tile = reinterpret_cast<V *>(smem);
  V *M = tile + kKrausTile;
  __shared__ uint64_t hi_off[kKrausPer];  // offset of tile element 256 j beyond the visit's base
  const int t = threadIdx.x;
  const uint32_t tsize = 1u << a.geo.tb;
  for (uint32_t i = t; i < kKrausMatEntries; i += kKrausThreads) M[i] = reinterpret_cast<const V *>(mat)[i];
  if (t < kKrausPer) hi_off[t] = tile_offset(a.geo, ((uint32_t)t * kKrausThreads) & (kKrausTile - 1));
  const uint64_t lo_off = tile_offset(a.geo, (uint32_t)t & (tsize - 1));
  const int blk = t % NB, split = t / NB;
  const int ablk = blk / Q, bblk = blk % Q;
  const uint32_t rows = tsize >> a.nb;
  double2 acc[RB][RB];
#pragma unroll
  for (int i = 0; i < RB; ++i)
#pragma unroll
    for (int j = 0; j < RB; ++j) acc[i][j] = make_double2(0.0, 0.0);
  __syncthreads();
  for (uint64_t v = blockIdx.x; v < a.geo.n_visits; v += gridDim.x) {
    const uint64_t base = visit_base(a.geo, v) | lo_off;
#pragma unroll
    for (int j = 0; j < kKrausPer; ++j) {
      const uint32_t e = t + kKrausThreads * j;
      if (e < tsize) cp_async<sizeof(V)>(tile + e, psi + 2 * (base | hi_off[j]));
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    for (uint32_t c = 0; c < a.n_ch; ++c) {
      const V *Mc = M + a.mat_off[c];
      if (KMAX <= 2) {
        if (a.k[c] == 1)
          apply_fibres<1>(tile, Mc, a.slot[c], a.off[c], tsize);
        else
          apply_fibres<2>(tile, Mc, a.slot[c], a.off[c], tsize);
      } else {
        switch (a.k[c]) {
          case 1: apply_fibres<1>(tile, Mc, a.slot[c], a.off[c], tsize); break;
          case 2: apply_fibres<2>(tile, Mc, a.slot[c], a.off[c], tsize); break;
          case 3: apply_fibres<3>(tile, Mc, a.slot[c], a.off[c], tsize); break;
          default: apply_fibres<4>(tile, Mc, a.slot[c], a.off[c], tsize); break;
        }
      }
      __syncthreads();
    }
    V *P = reinterpret_cast<V *>(psi);
#pragma unroll 2
    for (int j = 0; j < kKrausPer; ++j) {
      const uint32_t e = t + kKrausThreads * j;
      if (e < tsize) P[base | hi_off[j]] = tile[e];
    }
    if (C > 0) {
      uint32_t ao[RB], bo[RB];
#pragma unroll
      for (int i = 0; i < RB; ++i) {
        ao[i] = a.boff[ablk + Q * i];
        bo[i] = a.boff[bblk + Q * i];
      }
      for (uint32_t r = split; r < rows; r += S) {
        const uint32_t e0 = insert_zeros(r, a.bslot, a.nb);
        double2 xi[RB], xj[RB];
#pragma unroll
        for (int i = 0; i < RB; ++i) {
          const V u = tile[e0 | ao[i]];
          xi[i] = make_double2((double)u.x, (double)u.y);
        }
#pragma unroll
        for (int j = 0; j < RB; ++j) {
          const V u = tile[e0 | bo[j]];
          xj[j] = make_double2((double)u.x, (double)u.y);
        }
#pragma unroll
        for (int i = 0; i < RB; ++i)
#pragma unroll
          for (int j = 0; j < RB; ++j) {
            if (i > j) continue;  // strictly below the diagonal (a > b): written by the host
            acc[i][j].x = fma(xi[i].x, xj[j].x, acc[i][j].x);
            acc[i][j].x = fma(xi[i].y, xj[j].y, acc[i][j].x);
            acc[i][j].y = fma(xi[i].y, xj[j].x, acc[i][j].y);
            acc[i][j].y = fma(-xi[i].x, xj[j].y, acc[i][j].y);
          }
      }
    }
    __syncthreads();  // every reader of the tile is done before the next one lands
  }
  if (C == 0) return;
  constexpr int CC = C > 0 ? C : 1;  // C itself below, where C > 0
  double2 *col = partials + (size_t)blockIdx.x * CC * CC;
  if (S == 1) {
#pragma unroll
    for (int i = 0; i < RB; ++i)
#pragma unroll
      for (int j = 0; j < RB; ++j) col[(ablk + Q * i) * CC + bblk + Q * j] = acc[i][j];
    return;
  }
  double2 *red = reinterpret_cast<double2 *>(smem);  // [entry of the register block][thread]
#pragma unroll
  for (int i = 0; i < RB; ++i)
#pragma unroll
    for (int j = 0; j < RB; ++j) red[(i * RB + j) * kKrausThreads + t] = acc[i][j];
  __syncthreads();
  for (int e = t; e < CC * CC; e += kKrausThreads) {
    const int ea = e / CC, eb = e % CC;
    const int slot = (ea / Q) * RB + eb / Q, bk = (ea % Q) * Q + eb % Q;
    double2 sum = make_double2(0.0, 0.0);
    for (int q = 0; q < S; ++q) {
      const double2 p = red[slot * kKrausThreads + q * NB + bk];
      sum.x += p.x;
      sum.y += p.y;
    }
    col[e] = sum;
  }
}

// rho[e] = the grid's partials of entry e, added in CTA order.
__global__ void __launch_bounds__(256) k_kraus_reduce(const double2 *__restrict__ partials, uint32_t E,
                                                       double2 *__restrict__ rho) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double2 s = make_double2(0.0, 0.0);
  for (uint32_t c = 0; c < (uint32_t)kKrausGrid; ++c) {
    const double2 p = partials[(uint64_t)c * E + e];
    s.x += p.x;
    s.y += p.y;
  }
  rho[e] = s;
}

template <typename R, int C, int KMAX>
cudaError_t launch_kraus(void *psi, const KrausArgs &a, const void *mat, double2 *partials, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  const size_t smem = std::max((size_t)(kKrausTile + kKrausMatEntries) * sizeof(V), KrausShape<C>::RED_BYTES);
  static_assert((kKrausTile + kKrausMatEntries) * sizeof(double2) <= 113 * 1024, "two CTAs per SM");
  cudaError_t e = cudaFuncSetAttribute(k_kraus_apply_rdm<R, C, KMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_kraus_apply_rdm<R, C, KMAX><<<kKrausGrid, kKrausThreads, smem, s>>>((R *)psi, a, mat, partials);
  return cudaGetLastError();
}

template <typename R, int KMAX>
cudaError_t launch_kraus_c(void *psi, const KrausArgs &a, const void *mat, double2 *partials, cudaStream_t s) {
  switch (a.nb) {
    case 0: return launch_kraus<R, 0, KMAX>(psi, a, mat, partials, s);
    case 1: return launch_kraus<R, 2, KMAX>(psi, a, mat, partials, s);
    case 2: return launch_kraus<R, 4, KMAX>(psi, a, mat, partials, s);
    case 3: return launch_kraus<R, 8, KMAX>(psi, a, mat, partials, s);
    default: return launch_kraus<R, 16, KMAX>(psi, a, mat, partials, s);
  }
}

// KMAX: the largest arity the instantiation applies (2, or 4): the fibre of a 3- or 4-qubit operator holds 8 or 16
// amplitudes in registers, which the groups of one- and two-qubit channels need not reserve.
template <typename R>
cudaError_t launch_kraus_prec(void *psi, const KrausArgs &a, const void *mat, double2 *partials, cudaStream_t s) {
  uint32_t kmax = 0;
  for (uint32_t c = 0; c < a.n_ch; ++c) kmax = std::max(kmax, a.k[c]);
  return kmax <= 2 ? launch_kraus_c<R, 2>(psi, a, mat, partials, s) : launch_kraus_c<R, 4>(psi, a, mat, partials, s);
}

const size_t kPartBytes = (size_t)kKrausGrid * 256 * sizeof(double2);
const size_t kRhoBytes = 256 * sizeof(double2);
const size_t kMatBytes = kKrausMatEntries * sizeof(double2);

}  // namespace

int parse_kraus_channels(const std::string &who, uint32_t n, size_t n_channels, const uint32_t *arity,
                         const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, KrausSet *out,
                         std::string *err, bool sequential) {
  if (n_channels && (!arity || !qubits || !n_kraus || !kraus)) {
    *err = who + ": NULL arity, qubits, n_kraus or kraus";
    return QIPB200_ERR_INVALID_ARG;
  }
  KrausSet &ks = *out;
  ks = KrausSet();
  uint64_t seen = 0;
  size_t off = 0;
  for (size_t c = 0; c < n_channels; ++c) {
    const std::string ch = who + ": channel " + std::to_string(c);
    const uint32_t k = arity[c];
    if (k == 0 || k > kKrausMaxArity) {
      *err = ch + ": arity must be 1..4, got " + std::to_string(k);
      return QIPB200_ERR_INVALID_ARG;
    }
    ks.qfirst.push_back((uint32_t)ks.qubits.size());
    if (sequential) seen = 0;
    for (uint32_t i = 0; i < k; ++i) {
      const uint64_t q = qubits[ks.qubits.size()];
      if (q >= n) {
        *err = ch + ": qubit " + std::to_string(q) + " out of range for " + std::to_string(n) + " qubits";
        return QIPB200_ERR_BAD_INDEX;
      }
      if ((seen >> q) & 1) {
        *err = ch + ": qubit " + std::to_string(q) + " repeated";
        return QIPB200_ERR_BAD_INDEX;
      }
      seen |= 1ull << q;
      ks.qubits.push_back(q);
    }
    const uint32_t m = n_kraus[c];
    if (m == 0 || m > kKrausMaxOps) {
      *err = ch + ": n_kraus must be 1..256, got " + std::to_string(m);
      return QIPB200_ERR_INVALID_ARG;
    }
    ks.first.push_back((uint32_t)ks.mat.size());
    const uint32_t D = 1u << k;
    std::vector<cd> sum((size_t)D * D, cd(0.0, 0.0));
    bool indep = true;
    for (uint32_t i = 0; i < m; ++i, off += 2 * D * D) {
      const double *K = kraus + off;  // entry (r, col) at K[2 (r D + col)]
      const std::string op = ch + ", operator " + std::to_string(i);
      bool zero = true;
      for (uint32_t v = 0; v < 2 * D * D; ++v) {
        if (!std::isfinite(K[v])) {
          *err = op + ": an entry is not finite";
          return QIPB200_ERR_INVALID_ARG;
        }
        zero = zero && K[v] == 0.0;
      }
      if (zero) {
        *err = op + ": the zero matrix";
        return QIPB200_ERR_INVALID_ARG;
      }
      // M = K^dagger K: M[r][col] = sum_a conj(K[a][r]) K[a][col], a ascending
      std::vector<cd> M((size_t)D * D);
      for (uint32_t r = 0; r < D; ++r)
        for (uint32_t col = 0; col < D; ++col) {
          double re = 0.0, im = 0.0;
          for (uint32_t a = 0; a < D; ++a) {
            const double *x = K + 2 * (a * D + r), *y = K + 2 * (a * D + col);
            const double p1 = x[0] * y[0], p2 = x[1] * y[1], p3 = x[0] * y[1], p4 = x[1] * y[0];
            re += p1 + p2;
            im += p3 - p4;
          }
          M[(size_t)r * D + col] = cd(re, im);
        }
      double tr = 0.0;
      for (uint32_t r = 0; r < D; ++r) tr += M[(size_t)r * D + r].real();
      const double w = tr / D;
      for (uint32_t r = 0; r < D; ++r)
        for (uint32_t col = 0; col < D; ++col) {
          const cd x = M[(size_t)r * D + col] - (r == col ? cd(w, 0.0) : cd(0.0, 0.0));
          indep = indep && std::fabs(x.real()) <= kKrausTol && std::fabs(x.imag()) <= kKrausTol;
          sum[(size_t)r * D + col] += M[(size_t)r * D + col];
        }
      ks.mat.push_back(K);
      ks.gram.push_back(std::move(M));
      ks.w.push_back(w);
    }
    for (uint32_t r = 0; r < D; ++r)
      for (uint32_t col = 0; col < D; ++col) {
        const cd x = sum[(size_t)r * D + col] - (r == col ? cd(1.0, 0.0) : cd(0.0, 0.0));
        if (!(std::fabs(x.real()) <= kKrausTol && std::fabs(x.imag()) <= kKrausTol)) {
          char buf[96];
          snprintf(buf, sizeof(buf), "entry (%u, %u) of sum K^dagger K - I is %.3g%+.3gi", r, col, x.real(),
                   x.imag());
          *err = ch + ": the operators are not complete (" + buf + ")";
          return QIPB200_ERR_INVALID_ARG;
        }
      }
    ks.indep.push_back(indep ? 1 : 0);
  }
  ks.qfirst.push_back((uint32_t)ks.qubits.size());
  ks.first.push_back((uint32_t)ks.mat.size());
  return QIPB200_OK;
}

std::vector<std::vector<size_t>> kraus_groups(const KrausSet &ks) {
  std::vector<std::vector<size_t>> g;
  uint32_t bits = 0;
  for (size_t c = 0; c < ks.size(); ++c) {
    if (ks.indep[c]) continue;
    if (g.empty() || bits + ks.arity(c) > kKrausGroupBits) {
      g.emplace_back();
      bits = 0;
    }
    g.back().push_back(c);
    bits += ks.arity(c);
  }
  return g;
}

void plan_kraus_channels(const KrausSet &ks, uint32_t out4[4]) {
  const uint32_t r = (uint32_t)kraus_groups(ks).size();
  out4[0] = r;
  out4[1] = r ? 1 : 0;
  out4[2] = r;
  out4[3] = r ? 2 * r + 1 : 0;
}

uint32_t kraus_choose(const double *e, uint32_t m, double u) {
  double S = 0.0;
  for (uint32_t i = 0; i < m; ++i) S += e[i];
  const double t = u * S;
  double acc = 0.0;
  for (uint32_t i = 0; i < m; ++i) {
    acc += e[i];
    if (t < acc) return i;
  }
  for (uint32_t i = m; i-- > 0;)  // rounding left no such i
    if (e[i] > 0.0) return i;
  return 0;
}

bool kraus_draw_group(const KrausSet &ks, const std::vector<size_t> &g, const double *rho, const double *draws,
                      uint32_t *chosen, double *cond) {
  uint32_t m = 0;
  for (size_t c : g) m += ks.arity(c);
  const uint32_t Dg = 1u << m;
  std::vector<cd> L(1, cd(1.0, 0.0));  // the chosen M of the earlier channels, (x) in order
  uint32_t s = 0;                     // their qubits
  for (size_t c : g) {
    const uint32_t k = ks.arity(c), rest = m - s - k, Dx = 1u << (s + k), Dk = 1u << k, Ds = 1u << s;
    // rho' = rho with the later channels' qubits (the low bits) traced out
    std::vector<cd> rp((size_t)Dx * Dx, cd(0.0, 0.0));
    for (uint32_t x = 0; x < Dx; ++x)
      for (uint32_t y = 0; y < Dx; ++y)
        for (uint32_t t = 0; t < (1u << rest); ++t) {
          const size_t at = (size_t)((x << rest) | t) * Dg + ((y << rest) | t);
          rp[(size_t)x * Dx + y] += cd(rho[2 * at], rho[2 * at + 1]);
        }
    const uint32_t f = ks.first[c], n_ops = ks.first[c + 1] - f;
    std::vector<double> num(n_ops);
    for (uint32_t i = 0; i < n_ops; ++i) {
      const std::vector<cd> &Mi = ks.gram[f + i];
      cd tr(0.0, 0.0);  // Tr[(L (x) M_i) rho'] = sum_{x, y} (L (x) M_i)[x][y] rho'[y][x]
      for (uint32_t x = 0; x < Dx; ++x)
        for (uint32_t y = 0; y < Dx; ++y)
          tr += L[(size_t)(x / Dk) * Ds + y / Dk] * Mi[(size_t)(x % Dk) * Dk + y % Dk] * rp[(size_t)y * Dx + x];
      num[i] = tr.real() > 0.0 ? tr.real() : 0.0;  // a negative rounding residue counts as 0
    }
    double S = 0.0;
    for (uint32_t i = 0; i < n_ops; ++i) S += num[i];
    if (!(S > 0.0)) return false;
    const uint32_t i = kraus_choose(num.data(), n_ops, draws[c]);
    chosen[c] = i;
    cond[c] = num[i] / S;
    const std::vector<cd> &Mi = ks.gram[f + i];
    std::vector<cd> L2((size_t)Dx * Dx);
    for (uint32_t x = 0; x < Dx; ++x)
      for (uint32_t y = 0; y < Dx; ++y)
        L2[(size_t)x * Dx + y] = L[(size_t)(x / Dk) * Ds + y / Dk] * Mi[(size_t)(x % Dk) * Dk + y % Dk];
    L.swap(L2);
    s += k;
  }
  return true;
}

bool kraus_is_scaled_identity(const double *K, uint32_t k) {
  const uint32_t D = 1u << k;
  if (!(K[0] > 0.0)) return false;
  for (uint32_t r = 0; r < D; ++r)
    for (uint32_t col = 0; col < D; ++col) {
      const double *x = K + 2 * (r * D + col);
      if (x[1] != 0.0 || x[0] != (r == col ? K[0] : 0.0)) return false;
    }
  return true;
}

size_t kraus_scratch_bytes() { return kPartBytes + kRhoBytes + kMatBytes; }

cudaError_t run_kraus_sweep(qip_prec prec, void *psi, uint32_t n, const std::vector<KrausApplyOp> &ops,
                            const uint32_t *bpos, uint32_t nb, double *rho, void *d_scratch, cudaStream_t s,
                            uint64_t *launches) {
  const uint32_t L = std::min(kSweepL, n);
  uint64_t hi = 0;
  for (const KrausApplyOp &o : ops)
    for (uint32_t i = 0; i < o.k; ++i)
      if (o.pos[i] >= L) hi |= 1ull << o.pos[i];
  for (uint32_t i = 0; i < nb; ++i)
    if (bpos[i] >= L) hi |= 1ull << bpos[i];
  for (uint32_t b = L; b < n && (uint32_t)__builtin_popcountll(hi) < kKrausHi; ++b) hi |= 1ull << b;
  KrausArgs a;
  memset(&a, 0, sizeof(a));
  a.geo = sweep_tiles(n, L, hi, 0);
  a.n_ch = (uint32_t)ops.size();
  const size_t esz = prec == QIP_F32 ? 8 : 16;
  std::vector<unsigned char> mat(kMatBytes, 0);
  uint32_t at = 0;
  auto slot_of = [&](uint32_t p) { return (uint32_t)__builtin_ctz(tile_local(a.geo, 1ull << p)); };
  for (uint32_t c = 0; c < a.n_ch; ++c) {
    const KrausApplyOp &o = ops[c];
    a.k[c] = o.k;
    a.mat_off[c] = at;
    memcpy(mat.data() + at * esz, o.mat.data(), o.mat.size());
    at += 1u << (2 * o.k);
    uint32_t sl[kKrausMaxArity];
    for (uint32_t i = 0; i < o.k; ++i) sl[i] = slot_of(o.pos[i]);
    for (uint32_t b = 0; b < (1u << o.k); ++b) {
      uint32_t e = 0;
      for (uint32_t i = 0; i < o.k; ++i) e |= ((b >> (o.k - 1 - i)) & 1u) << sl[i];
      a.off[c][b] = (uint16_t)e;
    }
    std::sort(sl, sl + o.k);
    for (uint32_t i = 0; i < o.k; ++i) a.slot[c][i] = (uint8_t)sl[i];
  }
  a.nb = nb;
  uint32_t bs[kKrausGroupBits];
  for (uint32_t i = 0; i < nb; ++i) bs[i] = slot_of(bpos[i]);
  for (uint32_t v = 0; v < (1u << nb); ++v) {
    uint32_t e = 0;
    for (uint32_t i = 0; i < nb; ++i) e |= ((v >> i) & 1u) << bs[i];
    a.boff[v] = (uint16_t)e;
  }
  std::sort(bs, bs + nb);
  for (uint32_t i = 0; i < nb; ++i) a.bslot[i] = (uint8_t)bs[i];

  double2 *d_part = (double2 *)d_scratch;
  double2 *d_rho = (double2 *)((char *)d_scratch + kPartBytes);
  void *d_mat = (char *)d_scratch + kPartBytes + kRhoBytes;
  cudaError_t e = cudaMemcpyAsync(d_mat, mat.data(), kMatBytes, cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return e;
  e = prec == QIP_F32 ? launch_kraus_prec<float>(psi, a, d_mat, d_part, s)
                      : launch_kraus_prec<double>(psi, a, d_mat, d_part, s);
  ++*launches;
  // the host copy of mat must outlive the copy above
  if (e != cudaSuccess || nb == 0) {
    const cudaError_t es = cudaStreamSynchronize(s);
    return e != cudaSuccess ? e : es;
  }
  const uint32_t C = 1u << nb, E = C * C;
  k_kraus_reduce<<<(E + 255) / 256, 256, 0, s>>>(d_part, E, d_rho);
  ++*launches;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  std::vector<cd> h(E);
  if ((e = cudaMemcpyAsync(h.data(), d_rho, E * sizeof(double2), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
  for (uint32_t x = 0; x < C; ++x)
    for (uint32_t y = 0; y < C; ++y) {
      cd v = x <= y ? h[(size_t)x * C + y] : std::conj(h[(size_t)y * C + x]);
      if (x == y) v.imag(0.0);
      rho[2 * ((size_t)x * C + y)] = v.real();
      rho[2 * ((size_t)x * C + y) + 1] = v.imag();
    }
  return cudaSuccess;
}

}  // namespace qipb200
