// channel.cu -- one quantum-trajectory step of noise channels on distinct qubits, each on k = 1..4 qubits, whose Kraus
// operators have at most one nonzero entry per column, all on one XOR-shifted diagonal: K|b> = d(b)|b ^ f>
// (qipb200_state_apply_channels, k = 1, and qipb200_state_apply_multiqubit_channels): the host-side validation, choice
// and tables, and the weight and apply sweeps.
//
// Sampling.  Such an operator has K^dagger K = diag_b |d(b)|^2.  For channels c on disjoint qubit sets the outcome
// tuple i has probability
//   p(i) = <psi| (x)_c E_{i_c} |psi> = sum_x P(x) prod_c |d_{i_c}(x_c)|^2,
// with P(x) the distribution of the channel qubits in the computational basis and x_c channel c's value.  Completeness
// makes sum_i |d_i(b)|^2 = 1 for each b, so drawing x from P (launch_sample, one draw) and then each i_c independently
// from the weights |d_i(x_c)|^2 draws i with probability exactly p(i).  A channel whose operators each have one |d(b)|^2
// for every b does not need x_c (its weights do not depend on it), so only the state-dependent channels' qubits are
// sampled.
//
// Weight (k_channel_weight, when some chosen operator has |d(b)|^2 depending on b): S = sum_j |psi_j|^2 w(j) and
// N = sum_j |psi_j|^2, w(j) = the product of the real tables (byte tables in table order, then the gathered tables in
// operator order), on a fixed grid of kChanWeightGrid CTAs.  Order: chunks of C = min(2^n, 2048) consecutive amplitudes
// go to CTA c mod G; a thread adds its terms in chunk order, its 8 elements per chunk in order; each warp sums by an
// xor-shuffle tree (5 levels), the CTA's 8 warp sums are added in warp order, and the host adds the G partials in CTA
// order.  No floating-point atomics.
// Rounding: |psi_j|^2 = RN(RN(a^2) + RN(b^2)) (f32 amplitudes are exact in double) costs gamma_2; w(j), a product of
// one weight |d_c(b_c)|^2 (a double) per remaining operator, costs gamma_{k-1} for k operators, whatever their arity
// (host tables and device products alike); the product |psi_j|^2 w(j) one more u.  The longest chain of additions is
// D = 8 ceil(V / G) + 5 + 7 + (G - 1) for V = 2^n / C chunks.  So, to first order in u = 2^-53, with the sums taken
// exactly over the per-operator weights,
//   |S_got - S| <= (k + 2 + D) u S,  |N_got - N| <= (2 + D) u N,  and q = S / N to (k + 5 + 2 D) u relative.
//
// Apply (k_channel_apply): psi'_{j ^ F} = W(j) psi_j with W(j) = RN_prec(((T_0[i_0(j)] T_1[i_1(j)]) ...) (1/sqrt q)):
// the byte tables indexed by their index byte, then the gathered tables indexed by their operators' physical bits (in
// the matrix convention), the complex products in double without FMA (the last one by a real: each part times
// 1/sqrt q), then the update of function ops, (RN(RN(Wr a) - RN(Wi b)), RN(RN(Wr b) + RN(Wi a))) in the state's
// precision without FMA.  A warp owns rows of 32 consecutive amplitudes: row R and its partner row R ^ (F & ~31) when F
// has bits above 4, else two independent rows (R and R | 32).  Every lane loads its amplitude of both rows (whole
// sectors), computes the values they send, and takes the value its own index receives from lane ^ (F & 31) of the
// source row by a shuffle, so the stores cover the same whole sectors.  The two rows' loads precede their stores inside
// the warp and no other warp touches them, so the sweep is race-free in place; every amplitude is read and written
// once.
#include "channel.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "function_dev.cuh"
#include "kernels.cuh"
#include "sweep_dev.cuh"

namespace qipb200 {

namespace {

const uint32_t kChanChunk = kChanThreads * kChanPer;

const uint32_t kChanTabEntries = kChanMaxTables * 256 + kChanMaxGatherEntries;

struct ChanArgs {
  uint32_t n, n_tab, n_gat, n_ent;  // n_ent: table entries in all
  uint32_t shift[kChanMaxTables];  // 8 x the index byte of table t
  uint32_t gat[kChanMaxGather];    // ChannelTables::gat
  uint32_t h;                      // apply: the bit that tells a unit's two rows apart
  uint32_t rows;                   // apply: 2, or 1 when the state has at most 32 amplitudes
  uint64_t n_units;                // apply: warp work units
  uint64_t F;
  double inv;
};

// (a.x + i a.y)(b.x + i b.y) in double, each product and sum rounded once.
__host__ __device__ __forceinline__ double2 cmul_rn(double2 a, double2 b) {
#ifdef __CUDA_ARCH__
  return make_double2(__dsub_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)),
                      __dadd_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)));
#else
  const double p1 = a.x * b.x, p2 = a.y * b.y, p3 = a.x * b.y, p4 = a.y * b.x;  // x86-64 SSE2: no contraction
  return make_double2(p1 - p2, p3 + p4);
#endif
}

// The index of gathered table g for amplitude j: the bits at the 6-bit positions of g, the first the most significant.
__device__ __forceinline__ uint32_t chan_gather(uint32_t g, uint64_t j) {
  const uint32_t k = (g >> 24) + 1;
  uint32_t b = 0;
  for (uint32_t i = 0; i < k; ++i) b = (b << 1) | (uint32_t)((j >> ((g >> (6 * i)) & 63u)) & 1ull);
  return b;
}

// The product of the tables for amplitude j: byte tables in order, then gathered tables in order (the first factor
// taken as it is).  T is the shared copy, G the gathered tables' descriptors.
template <typename D, typename Mul>
__device__ __forceinline__ D chan_product(const ChanArgs &a, const D *T, const uint32_t *G, uint64_t j, Mul mul) {
  D w = a.n_tab ? T[(j >> a.shift[0]) & 255] : T[chan_gather(G[0], j)];
#pragma unroll
  for (uint32_t u = 1; u < kChanMaxTables; ++u)
    if (u < a.n_tab) w = mul(w, T[u * 256 + ((j >> a.shift[u]) & 255)]);
  uint32_t off = a.n_tab * 256;
  for (uint32_t u = 0; u < a.n_gat; ++u) {
    const uint32_t g = G[u];
    if (u || a.n_tab) w = mul(w, T[off + chan_gather(g, j)]);
    off += 2u << (g >> 24);
  }
  return w;
}

// chan_product for a warp that owns the row of j (j & 31 == lane): a gathered table's index is the OR of its bits
// below 5, Lo[u * 32 + lane], and its bits above, the same for the whole row and computed by lane u into hi.
__device__ __forceinline__ double2 chan_product_row(const ChanArgs &a, const double2 *T, const uint32_t *G,
                                                    const uint8_t *Lo, uint32_t hi, uint32_t lane, uint64_t j) {
  double2 w = a.n_tab ? T[(j >> a.shift[0]) & 255] : make_double2(0.0, 0.0);
#pragma unroll
  for (uint32_t u = 1; u < kChanMaxTables; ++u)
    if (u < a.n_tab) w = cmul_rn(w, T[u * 256 + ((j >> a.shift[u]) & 255)]);
  uint32_t off = a.n_tab * 256;
  for (uint32_t u = 0; u < a.n_gat; ++u) {
    const double2 t = T[off + (__shfl_sync(0xffffffffu, hi, u) | Lo[u * 32 + lane])];
    w = (u || a.n_tab) ? cmul_rn(w, t) : t;
    off += 2u << (G[u] >> 24);
  }
  return w;
}

template <typename R>
__global__ void __launch_bounds__(kChanThreads)
    k_channel_weight(const R *__restrict__ psi, const __grid_constant__ ChanArgs a, const double *__restrict__ tab,
                     double *__restrict__ partial) {
  typedef typename SweepV<R>::type V;
  __shared__ double T[kChanTabEntries];
  __shared__ uint32_t G[kChanMaxGather];
  __shared__ double ws[2][kChanThreads / 32];
  for (uint32_t i = threadIdx.x; i < a.n_ent; i += kChanThreads) T[i] = tab[i];
  if (threadIdx.x < a.n_gat) G[threadIdx.x] = a.gat[threadIdx.x];
  __syncthreads();
  const V *P = reinterpret_cast<const V *>(psi);
  const uint64_t N = 1ull << a.n;
  const uint32_t C = N < (uint64_t)kChanChunk ? (uint32_t)N : kChanChunk;
  const uint64_t n_chunks = N / C;
  const uint32_t t = threadIdx.x;
  double accS = 0.0, accN = 0.0;
  for (uint64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const uint64_t b = c * C;
    V p[kChanPer];
#pragma unroll
    for (int k = 0; k < kChanPer; ++k)
      if (t + kChanThreads * k < C) p[k] = __ldg(P + b + t + kChanThreads * k);
#pragma unroll
    for (int k = 0; k < kChanPer; ++k)
      if (t + kChanThreads * k < C) {
        const uint64_t j = b + t + kChanThreads * k;
        const double re = p[k].x, im = p[k].y;
        const double pj = __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im));
        const double w = chan_product(a, T, G, j, [](double x, double y) { return __dmul_rn(x, y); });
        accN = __dadd_rn(accN, pj);
        accS = __dadd_rn(accS, __dmul_rn(pj, w));
      }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    accS = __dadd_rn(accS, __shfl_xor_sync(0xffffffffu, accS, o));
    accN = __dadd_rn(accN, __shfl_xor_sync(0xffffffffu, accN, o));
  }
  if ((t & 31) == 0) {
    ws[0][t >> 5] = accS;
    ws[1][t >> 5] = accN;
  }
  __syncthreads();
  if (t == 0) {
    double s = ws[0][0], m = ws[1][0];
    for (int w = 1; w < kChanThreads / 32; ++w) {
      s = __dadd_rn(s, ws[0][w]);
      m = __dadd_rn(m, ws[1][w]);
    }
    partial[2 * blockIdx.x] = s;
    partial[2 * blockIdx.x + 1] = m;
  }
}

// RN_prec(w / sqrt q) psi_j in the state's precision.
template <typename R, typename V>
__device__ __forceinline__ V chan_scale(const ChanArgs &a, double2 w, V p) {
  V wr;
  wr.x = (R)__dmul_rn(w.x, a.inv);
  wr.y = (R)__dmul_rn(w.y, a.inv);
  return fn_phase<R, V, true>(p, wr);
}

template <typename R, typename V>
__device__ __forceinline__ V chan_value(const ChanArgs &a, const double2 *T, const uint32_t *G, uint64_t j, V p) {
  return chan_scale<R, V>(a, chan_product(a, T, G, j, [](double2 x, double2 y) { return cmul_rn(x, y); }), p);
}

template <typename V>
__device__ __forceinline__ V shfl_v(V v, uint32_t src) {
  V o;
  o.x = __shfl_sync(0xffffffffu, v.x, src);
  o.y = __shfl_sync(0xffffffffu, v.y, src);
  return o;
}

template <typename R>
__global__ void __launch_bounds__(kChanThreads)
    k_channel_apply(R *__restrict__ psi, const __grid_constant__ ChanArgs a, const double2 *__restrict__ tab) {
  typedef typename SweepV<R>::type V;
  __shared__ double2 T[kChanTabEntries];
  __shared__ uint32_t G[kChanMaxGather];
  __shared__ uint8_t Lo[kChanMaxGather * 32];
  for (uint32_t i = threadIdx.x; i < a.n_ent; i += kChanThreads) T[i] = tab[i];
  if (threadIdx.x < a.n_gat) G[threadIdx.x] = a.gat[threadIdx.x];
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < a.n_gat * 32; i += kChanThreads) Lo[i] = (uint8_t)chan_gather(G[i >> 5], i & 31);
  __syncthreads();
  V *P = reinterpret_cast<V *>(psi);
  const uint32_t lane = threadIdx.x & 31, src = lane ^ ((uint32_t)a.F & 31u);
  const uint64_t fhi = a.F & ~31ull, N = 1ull << a.n, low = (1ull << a.h) - 1;
  const uint64_t warps = ((uint64_t)gridDim.x * kChanThreads) >> 5;
  for (uint64_t u = ((uint64_t)blockIdx.x * kChanThreads + threadIdx.x) >> 5; u < a.n_units; u += warps) {
    const uint64_t r = u << 5;
    V zero;
    zero.x = zero.y = (R)0;
    if (a.rows == 1) {  // at most 32 amplitudes: one row, lanes past the state idle
      const bool ok = lane < N;
      const V y = ok ? chan_value<R, V>(a, T, G, lane, P[lane]) : zero;
      const V o = shfl_v(y, src);
      if (ok) P[lane] = o;
      continue;
    }
    const uint64_t j0 = ((r & ~low) << 1) | (r & low) | lane;  // bit h clear
    const uint64_t j1 = fhi ? j0 ^ fhi : j0 | (1ull << a.h);
    const V p0 = P[j0], p1 = P[j1];
    // lane u < n_gat gathers table u's bits above 4 for both rows
    const uint32_t g = lane < a.n_gat ? G[lane] : 0u;
    const uint32_t hi0 = lane < a.n_gat ? chan_gather(g, j0 & ~31ull) : 0u;
    const uint32_t hi1 = lane < a.n_gat ? chan_gather(g, j1 & ~31ull) : 0u;
    const V y0 = chan_scale<R, V>(a, chan_product_row(a, T, G, Lo, hi0, lane, j0), p0);
    const V y1 = chan_scale<R, V>(a, chan_product_row(a, T, G, Lo, hi1, lane, j1), p1);
    // index j receives W(j ^ F) psi_{j ^ F}: from the partner row when F leaves the row, lane ^ (F & 31) either way
    const V o0 = shfl_v(fhi ? y1 : y0, src), o1 = shfl_v(fhi ? y0 : y1, src);
    P[j0] = o0;
    P[j1] = o1;
  }
}

ChanArgs chan_args(uint32_t n, const ChannelTables &t, double inv) {
  ChanArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n;
  a.n_tab = t.n_tab;
  a.n_gat = t.n_gat;
  a.n_ent = (uint32_t)t.e.size();
  for (uint32_t i = 0; i < t.n_tab; ++i) a.shift[i] = 8 * t.byte[i];
  for (uint32_t i = 0; i < t.n_gat; ++i) a.gat[i] = t.gat[i];
  a.F = t.flip;
  a.inv = inv;
  a.h = (t.flip >> 5) ? 63 - (uint32_t)__builtin_clzll(t.flip) : 5;
  a.rows = n >= 6 ? 2 : 1;
  a.n_units = n >= 6 ? 1ull << (n - 6) : 1;
  return a;
}

const size_t kTabBytes = kChanTabEntries * sizeof(double2);

}  // namespace

int parse_channels(const std::string &who, uint32_t n, size_t n_channels, const uint32_t *arity,
                   const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, uint32_t max_kraus,
                   ChannelSet *out, std::string *err) {
  if (n_channels && (!qubits || !n_kraus || !kraus)) {
    *err = who + (arity ? ": NULL arity, qubits, n_kraus or kraus" : ": NULL qubits, n_kraus or kraus");
    return QIPB200_ERR_INVALID_ARG;
  }
  ChannelSet &cs = *out;
  cs = ChannelSet();
  uint64_t seen = 0;
  size_t off = 0;
  for (size_t c = 0; c < n_channels; ++c) {
    const std::string ch = who + ": channel " + std::to_string(c);
    const uint32_t k = arity ? arity[c] : 1;
    if (k == 0 || k > kChanMaxArity) {
      *err = ch + ": arity must be 1..4, got " + std::to_string(k);
      return QIPB200_ERR_INVALID_ARG;
    }
    cs.qfirst.push_back((uint32_t)cs.qubits.size());
    for (uint32_t i = 0; i < k; ++i) {
      const uint64_t q = qubits[cs.qubits.size()];
      if (q >= n) {
        *err = ch + ": qubit " + std::to_string(q) + " out of range for " + std::to_string(n) + " qubits";
        return QIPB200_ERR_BAD_INDEX;
      }
      if ((seen >> q) & 1) {
        *err = ch + ": qubit " + std::to_string(q) + " repeated";
        return QIPB200_ERR_BAD_INDEX;
      }
      seen |= 1ull << q;
      cs.qubits.push_back(q);
    }
    const uint32_t m = n_kraus[c];
    if (m == 0 || m > max_kraus) {
      *err = ch + ": n_kraus must be 1.." + std::to_string(max_kraus) + ", got " + std::to_string(m);
      return QIPB200_ERR_INVALID_ARG;
    }
    cs.first.push_back((uint32_t)cs.ops.size());
    const uint32_t D = 1u << k;
    double sum[16] = {0.0};
    bool dep = false;
    for (uint32_t i = 0; i < m; ++i, off += 2 * D * D) {
      const double *K = kraus + off;  // entry (r, col) at K[2 (r D + col)]
      const std::string op = ch + ", operator " + std::to_string(i);
      for (uint32_t v = 0; v < 2 * D * D; ++v)
        if (!std::isfinite(K[v])) {
          *err = op + ": an entry is not finite";
          return QIPB200_ERR_INVALID_ARG;
        }
      ChannelOp o;
      memset(&o, 0, sizeof(o));
      o.k = k;
      int f = -1;  // the mask shared by the nonzero columns
      bool form = true;
      for (uint32_t col = 0; col < D; ++col)
        for (uint32_t r = 0; r < D; ++r) {
          const double *x = K + 2 * (r * D + col);
          if (x[0] == 0.0 && x[1] == 0.0) continue;
          form = form && (f < 0 || (uint32_t)f == (r ^ col));
          if (f < 0) f = (int)(r ^ col);
        }
      if (f < 0) {
        *err = op + ": the zero matrix";
        return QIPB200_ERR_INVALID_ARG;
      }
      if (!form) {
        *err = op + (arity ? ": not of the form K|b> = d(b)|b ^ f> (one nonzero entry per column, one f)"
                           : ": neither diagonal nor anti-diagonal");
        return QIPB200_ERR_INVALID_ARG;
      }
      o.f = (uint32_t)f;
      for (uint32_t col = 0; col < D; ++col) {  // d(b) = K[b ^ f][b]
        const double *x = K + 2 * ((col ^ o.f) * D + col);
        o.d[col][0] = x[0];
        o.d[col][1] = x[1];
        const double re2 = x[0] * x[0], im2 = x[1] * x[1];
        o.e[col] = re2 + im2;
        sum[col] += o.e[col];
        dep = dep || o.e[col] != o.e[0];
      }
      cs.ops.push_back(o);
    }
    for (uint32_t b = 0; b < D; ++b)
      if (!(std::fabs(sum[b] - 1.0) <= kChanCompleteTol)) {
        char buf[64];
        snprintf(buf, sizeof(buf), "%.3g", sum[b] - 1.0);
        *err = ch + ": the operators are not complete (sum of |d_i(" + std::to_string(b) + ")|^2 - 1 = " + buf + ")";
        return QIPB200_ERR_INVALID_ARG;
      }
    cs.dep.push_back(dep ? 1 : 0);
    cs.n_dep += dep ? 1 : 0;
  }
  cs.qfirst.push_back((uint32_t)cs.qubits.size());
  cs.first.push_back((uint32_t)cs.ops.size());
  return QIPB200_OK;
}

uint32_t channel_choose(const ChannelSet &cs, size_t c, uint32_t b, double u) {
  const uint32_t f = cs.first[c], m = cs.first[c + 1] - f;
  double S = 0.0;
  for (uint32_t i = 0; i < m; ++i) S += cs.ops[f + i].e[b];
  const double t = u * S;
  double acc = 0.0;
  for (uint32_t i = 0; i < m; ++i) {
    acc += cs.ops[f + i].e[b];
    if (t < acc) return i;
  }
  for (uint32_t i = m; i-- > 0;)  // rounding left no such i
    if (cs.ops[f + i].e[b] > 0.0) return i;
  return 0;  // unreachable for a complete channel
}

bool channel_op_is_scaled_identity(const ChannelOp &k) {
  if (k.f || !(k.d[0][0] > 0.0)) return false;
  for (uint32_t b = 0; b < (1u << k.k); ++b)
    if (k.d[b][0] != k.d[0][0] || k.d[b][1] != 0.0) return false;
  return true;
}

void plan_channels(const ChannelSet &cs, uint32_t out4[4]) {
  bool rw = false;
  for (const ChannelOp &k : cs.ops) rw = rw || !channel_op_is_scaled_identity(k);
  out4[0] = cs.n_dep;
  out4[1] = cs.n_dep ? 3 : 0;  // the sample's two reads (the second only of the chunk the draw landed in), the weight
  out4[2] = rw ? 1 : 0;
  out4[3] = (cs.n_dep ? kSampleLaunches + 1 : 0) + (rw ? 1 : 0);
}

void build_channel_tables(const uint32_t *pos, const ChannelOp *const *ops, size_t m, ChannelTables *t) {
  t->n_tab = 0;
  t->n_gat = 0;
  t->flip = 0;
  t->d.clear();
  t->e.clear();
  std::vector<const uint32_t *> p(m);  // operator i's physical bits, its first qubit first
  std::vector<uint32_t> lo(m), byte(m);  // its lowest bit, and its byte (kChanMaxTables: gathered)
  for (size_t i = 0, o = 0; i < m; o += ops[i]->k, ++i) {
    const uint32_t k = ops[i]->k;
    p[i] = pos + o;
    lo[i] = *std::min_element(p[i], p[i] + k);
    byte[i] = lo[i] / 8;
    for (uint32_t q = 0; q < k; ++q) {
      if (p[i][q] / 8 != byte[i]) byte[i] = kChanMaxTables;
      if ((ops[i]->f >> (k - 1 - q)) & 1) t->flip |= 1ull << p[i][q];
    }
  }
  std::vector<size_t> order(m);
  for (size_t i = 0; i < m; ++i) order[i] = i;
  std::sort(order.begin(), order.end(), [&](size_t x, size_t y) { return lo[x] < lo[y]; });
  for (uint32_t by = 0; by < kChanMaxTables; ++by) {
    std::vector<size_t> in;  // the operators in this byte, in the order of their lowest bit
    for (size_t i : order)
      if (byte[i] == by) in.push_back(i);
    if (in.empty()) continue;
    t->byte[t->n_tab++] = by;
    for (uint32_t v = 0; v < 256; ++v) {
      double2 d = make_double2(0.0, 0.0);
      double e = 0.0;
      for (size_t r = 0; r < in.size(); ++r) {
        const ChannelOp &K = *ops[in[r]];
        uint32_t b = 0;
        for (uint32_t q = 0; q < K.k; ++q) b = (b << 1) | ((v >> (p[in[r]][q] % 8)) & 1);
        const double2 f = make_double2(K.d[b][0], K.d[b][1]);
        d = r ? cmul_rn(d, f) : f;
        e = r ? e * K.e[b] : K.e[b];
      }
      t->d.push_back(d);
      t->e.push_back(e);
    }
  }
  for (size_t i = 0; i < m; ++i) {
    if (byte[i] != kChanMaxTables) continue;
    const ChannelOp &K = *ops[i];
    uint32_t g = (K.k - 1) << 24;
    for (uint32_t q = 0; q < K.k; ++q) g |= p[i][q] << (6 * q);
    t->gat[t->n_gat++] = g;
    for (uint32_t b = 0; b < (1u << K.k); ++b) {
      t->d.push_back(make_double2(K.d[b][0], K.d[b][1]));
      t->e.push_back(K.e[b]);
    }
  }
}

size_t channel_scratch_bytes() { return kTabBytes + 2 * kChanWeightGrid * sizeof(double); }

cudaError_t run_channel_weight(qip_prec prec, const void *psi, uint32_t n, const ChannelTables &t, void *d_scratch,
                               cudaStream_t s, uint64_t *launches, double *S, double *N) {
  double *d_tab = (double *)d_scratch, *d_part = (double *)((char *)d_scratch + kTabBytes);
  cudaError_t e = cudaMemcpyAsync(d_tab, t.e.data(), t.e.size() * sizeof(double), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return e;
  const ChanArgs a = chan_args(n, t, 0.0);
  if (prec == QIP_F32)
    k_channel_weight<float><<<kChanWeightGrid, kChanThreads, 0, s>>>((const float *)psi, a, d_tab, d_part);
  else
    k_channel_weight<double><<<kChanWeightGrid, kChanThreads, 0, s>>>((const double *)psi, a, d_tab, d_part);
  ++*launches;
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  double part[2 * kChanWeightGrid];
  if ((e = cudaMemcpyAsync(part, d_part, sizeof(part), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
  double sS = 0.0, sN = 0.0;
  for (int g = 0; g < kChanWeightGrid; ++g) {  // CTA order
    sS += part[2 * g];
    sN += part[2 * g + 1];
  }
  *S = sS;
  *N = sN;
  return cudaSuccess;
}

cudaError_t run_channel_apply(qip_prec prec, void *psi, uint32_t n, const ChannelTables &t, double inv,
                              void *d_scratch, int sm_count, cudaStream_t s, uint64_t *launches) {
  double2 *d_tab = (double2 *)d_scratch;
  cudaError_t e = cudaMemcpyAsync(d_tab, t.d.data(), t.d.size() * sizeof(double2), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return e;
  const ChanArgs a = chan_args(n, t, inv);
  const uint64_t blocks = (a.n_units + kChanThreads / 32 - 1) / (kChanThreads / 32);
  const int grid = (int)std::min<uint64_t>(blocks, (uint64_t)std::max(8 * sm_count, 1));
  if (prec == QIP_F32)
    k_channel_apply<float><<<grid, kChanThreads, 0, s>>>((float *)psi, a, d_tab);
  else
    k_channel_apply<double><<<grid, kChanThreads, 0, s>>>((double *)psi, a, d_tab);
  ++*launches;
  return cudaGetLastError();
}

}  // namespace qipb200
