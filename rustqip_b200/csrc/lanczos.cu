// lanczos.cu -- the lowest eigenvalue of a real Pauli sum H = sum_h c_h P_h reachable from a start state, by plain
// Lanczos (no reorthogonalisation) on the device, in the three states of the Chebyshev evolution
// (qipb200_state_lanczos_pauli_sum), and the tridiagonal solve the host runs after every step (qipb200_lanczos_ritz).
//
// The recurrence.  The identity terms sum to a and the others give the scale b = sum |c_h| (both in list order, in
// double, from +0.0); the sum plan runs over every term, identity terms included.  The Lanczos vectors are kept
// unnormalised, u_j = beta_j v_j with beta_j = |u_j|, so that each scaling folds into a host-rounded scalar:
//   u_0 = psi (the state as passed), beta_0 = |u_0|;
//   step j:  w_j = sum_h RN(c_h RN(1 / beta_j)) P_h u_j + RN(sigma_j u_j-1),  sigma_j = -RN(beta_j / beta_(j-1))
//            (no start term at j = 0), the sum sweeps of k_pauli_sum in Lanczos mode (gradient.cu: the accumulator
//            start RN(start from), and in the last sweep the partials of Re(conj(u_j) w_j) over the stored w_j);
//            alpha_j = RN(dot_j / beta_j), dot_j the fixed-order sum of those partials;
//            u_(j+1) = w_j - RN(mu_j u_j), mu_j = RN(alpha_j / beta_j), in place over w_j (k_lanczos_vec, update), and
//            beta_(j+1) = sqrt(the fixed-order sum of |u_(j+1)|^2 over the stored u_(j+1)).
// In exact arithmetic these are the textbook alpha_j = <v_j|H v_j> and beta_(j+1) = |H v_j - alpha_j v_j - beta_j
// v_(j-1)|.  u_0 is the state, u_j is in work_a for odd j and work_b for even j >= 2, and w_j is written over u_(j-1)
// (at j = 1 to work_b, the start read from the state): src = u_j is the only operand read at partner indices and it is
// not written in the step.  After step j (m = j + 1) the host solves the tridiagonal T_m (lanczos_ritz) for its lowest
// eigenvalue theta and unit eigenvector y, and stops when the estimate rho_m = beta_m |y_(m-1)| <= tol b or m ==
// max_steps.  beta_m = 0 (the Krylov space is exhausted) gives rho_m = 0: a convergence.  Since rho_m <= beta_m, no
// step divides by a beta_j <= tol b.
//
// Vector mode.  A second pass reruns steps 0 .. m-2 with the alpha and beta of the first: the kernels and scalars are
// the same, so u_1 .. u_(m-1) come out bit-identical.  With the weights c_j = RN(y_j / beta_j), its update sweeps
// accumulate x = sum_j c_j u_j into the state once u_0 is no longer read (after the sum sweeps of step 1):
//   step 0, m = 2:  S <- RN(RN(RN(c_0 S) + RN(0 u_0)) + RN(c_1 u_1))
//   step 1:         S <- RN(RN(RN(c_0 S) + RN(c_1 u_1)) + RN(c_2 u_2))
//   step j >= 2:    S <- RN(RN(RN(1 S) + RN(0 u_j)) + RN(c_(j+1) u_(j+1)))
// per component in double, rounded to the state's precision at the store.  (m = 1: x = u_0 / beta_0 = v_0, so the
// state is left as u_0 and |x| is reported as |u_0| / beta_0.)  Then three kernels around one application of H:
// |x| (a read sweep), S <- RN(RN(1 / |x|) S) (the normalisation), work_a <- H S (run_pauli_sum, exactly
// qipb200_state_apply_pauli_sum), and one read sweep for <x|Hx>, |Hx - theta x|^2 and |x|^2, from which
// E = <x|Hx> / |x|^2 and |Hx - E x| = sqrt(|Hx - theta x|^2 - (E - theta)^2 |x|^2) / |x| (shifting by theta, which is
// within rho of E, avoids the cancellation of |Hx|^2 - E^2).  In exact arithmetic some eigenvalue of H lies within
// that residual of E.  Everything is double with no FMA where the state is written, f32 amplitudes widened; the
// reductions use FMA.  tests/lanczos_ref.py emulates u_j, x and the normalised state bit for bit given alpha, beta and
// |x|.
//
// Reductions.  Every thread adds its amplitudes in a fixed order in double, the 32 lanes of a warp reduce by butterfly
// shuffles, the 8 warps of a CTA add in warp order into scratch[row][CTA], and the host adds the CTAs in order (the
// update kernel adds the sum sweep's partials itself, in the same order, to form mu_j on the device).  The grids are
// fixed functions of n and the plan, so the same inputs give the same bits with no atomics.  Bounds, to first order,
// for the stored vectors (D = 2 ceil(2^n / 256) + 1069 bounds the depth of every such sum: per-thread elements, 5
// shuffle levels, 8 warps and at most 1056 CTAs):
//   |alpha_j - Re<u_j|w_j> / beta_j| <= gamma_(D+2)(2^-53) |u_j| |w_j| / beta_j,
//   |beta_(j+1) - |u_(j+1)||         <= gamma_(D+2)(2^-53) |u_(j+1)|
// (the sums err by gamma_D times the sum of the magnitudes, <= |u| |w| by Cauchy-Schwarz; the division and the square
// root add one rounding each).  tests/lanczos_ref.py: alpha_beta_bound().
//
// The tridiagonal solve.  Sturm counts with LAPACK's pivot guard bisect the Gershgorin interval to the last bit (or to
// 2^-60 of |T|); inverse iteration (three solves from a constant vector) with a partially pivoted LU of T - theta, a
// zero pivot replaced by 2^-52 |T|, gives y.
#include "lanczos.h"

#include <algorithm>
#include <cfloat>
#include <cmath>

#include "../../include/qipb200.h"
#include "gradient.h"
#include "sweep.cuh"

namespace qipb200 {

namespace {

const int kLanThreads = 256;
const int kLanWarps = kLanThreads / 32;
const uint64_t kLanGrid = 1056;  // 8 CTAs per SM of an H100 SXM
const int kLanUnroll = 4;        // amplitudes in flight per thread

enum VecMode { kVecNorm, kVecScale, kVecUpdate, kVecResid };

struct VecArgs {
  void *p0;              // norm, scale: the state; update: w_j (becomes u_(j+1)); resid: x
  const void *p1;        // update: u_j; resid: H x
  void *state;           // update with acc: the state
  const double *dot;     // update, first pass: the sum sweep's partials (mu from them); NULL: mu as given
  uint32_t dot_grid, acc;
  double beta, mu;       // update: beta_j, or mu_j when dot is NULL
  double s;              // scale: the factor; resid: theta
  double w0, w1, w2;     // update with acc: S <- (w0 S + w1 u_j) + w2 u_(j+1)
  double *red;           // [row][CTA]
  uint64_t n_amp;
};

__device__ __forceinline__ double2 widen(float2 v) { return make_double2(v.x, v.y); }
__device__ __forceinline__ double2 widen(double2 v) { return v; }
__device__ __forceinline__ float2 narrow_to(double2 a, float2 *) { return make_float2((float)a.x, (float)a.y); }
__device__ __forceinline__ double2 narrow_to(double2 a, double2 *) { return a; }

template <typename R, int MODE>
__global__ void __launch_bounds__(kLanThreads) k_lanczos_vec(const __grid_constant__ VecArgs a) {
  typedef typename SweepV<R>::type V;
  __shared__ double wsum[3][kLanWarps];
  __shared__ double mu_s;
  const int t = threadIdx.x;
  V *p0 = (V *)a.p0;
  const V *p1 = (const V *)a.p1;
  V *S = (V *)a.state;  // may be p1 (step 0 of the second pass): read before written, by the same thread
  double mu = a.mu;
  if (MODE == kVecUpdate && a.dot) {  // alpha_j and mu_j exactly as the host forms them
    if (t == 0) {
      double d = 0.0;
      for (uint32_t c = 0; c < a.dot_grid; ++c) d += a.dot[c];
      mu_s = __ddiv_rn(__ddiv_rn(d, a.beta), a.beta);
    }
    __syncthreads();
    mu = mu_s;
  }
  double r0 = 0.0, r1 = 0.0, r2 = 0.0;
  const uint64_t stride = (uint64_t)gridDim.x * kLanThreads;
  for (uint64_t i0 = (uint64_t)blockIdx.x * kLanThreads + t; i0 < a.n_amp; i0 += kLanUnroll * stride) {
    V x[kLanUnroll], y[kLanUnroll], z[kLanUnroll];
#pragma unroll
    for (int k = 0; k < kLanUnroll; ++k) {
      const uint64_t i = i0 + k * stride;
      if (i >= a.n_amp) continue;
      x[k] = p0[i];
      if (MODE == kVecUpdate || MODE == kVecResid) y[k] = p1[i];
      if (MODE == kVecUpdate && a.acc) z[k] = S[i];
    }
#pragma unroll
    for (int k = 0; k < kLanUnroll; ++k) {
      const uint64_t i = i0 + k * stride;
      if (i >= a.n_amp) continue;
      const double2 xv = widen(x[k]);
      if (MODE == kVecNorm) {
        r0 = fma(xv.x, xv.x, fma(xv.y, xv.y, r0));
      } else if (MODE == kVecScale) {
        p0[i] = narrow_to(make_double2(__dmul_rn(a.s, xv.x), __dmul_rn(a.s, xv.y)), (V *)nullptr);
      } else if (MODE == kVecUpdate) {
        const double2 uj = widen(y[k]);
        const V un = narrow_to(make_double2(__dadd_rn(xv.x, -__dmul_rn(mu, uj.x)), __dadd_rn(xv.y, -__dmul_rn(mu, uj.y))),
                               (V *)nullptr);
        p0[i] = un;
        const double2 u = widen(un);
        r0 = fma(u.x, u.x, fma(u.y, u.y, r0));
        if (a.acc) {
          const double2 sv = widen(z[k]);
          const double rx = __dadd_rn(__dadd_rn(__dmul_rn(a.w0, sv.x), __dmul_rn(a.w1, uj.x)), __dmul_rn(a.w2, u.x));
          const double ry = __dadd_rn(__dadd_rn(__dmul_rn(a.w0, sv.y), __dmul_rn(a.w1, uj.y)), __dmul_rn(a.w2, u.y));
          S[i] = narrow_to(make_double2(rx, ry), (V *)nullptr);
        }
      } else {  // kVecResid
        const double2 h = widen(y[k]);
        const double dx = h.x - a.s * xv.x, dy = h.y - a.s * xv.y;
        r0 = fma(xv.x, h.x, fma(xv.y, h.y, r0));
        r1 = fma(dx, dx, fma(dy, dy, r1));
        r2 = fma(xv.x, xv.x, fma(xv.y, xv.y, r2));
      }
    }
  }
  if (MODE == kVecScale) return;
  const int rows = MODE == kVecResid ? 3 : 1;
  double r[3] = {r0, r1, r2};
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    if (q >= rows) break;
#pragma unroll
    for (int o = 16; o; o >>= 1) r[q] += __shfl_xor_sync(0xffffffffu, r[q], o);
    if ((t & 31) == 0) wsum[q][t >> 5] = r[q];
  }
  __syncthreads();
  if (t < rows) {
    double s = 0.0;
    for (int w = 0; w < kLanWarps; ++w) s += wsum[t][w];
    a.red[(uint64_t)t * gridDim.x + blockIdx.x] = s;
  }
}

template <int MODE>
cudaError_t launch_vec(qip_prec prec, const VecArgs &a, uint32_t grid, cudaStream_t s) {
  if (prec == QIP_F32)
    k_lanczos_vec<float, MODE><<<grid, kLanThreads, 0, s>>>(a);
  else
    k_lanczos_vec<double, MODE><<<grid, kLanThreads, 0, s>>>(a);
  return cudaGetLastError();
}

double ordered_sum(const double *v, uint32_t n) {
  double s = 0.0;
  for (uint32_t i = 0; i < n; ++i) s += v[i];
  return s;
}

// Sturm count: eigenvalues of T below x, with LAPACK's guard against tiny pivots.
uint32_t sturm_below(const double *alpha, const double *beta, uint32_t m, double x, double pivmin) {
  uint32_t c = 0;
  double d = 1.0;
  for (uint32_t i = 0; i < m; ++i) {
    d = (alpha[i] - x) - (i ? beta[i] * beta[i] / d : 0.0);
    if (std::fabs(d) < pivmin) d = -pivmin;
    if (d < 0) ++c;
  }
  return c;
}

}  // namespace

void lanczos_ritz(const double *alpha, const double *beta, uint32_t m, double *theta, double *y, double *estimate) {
  double lo = HUGE_VAL, hi = -HUGE_VAL, e2max = 1.0;
  for (uint32_t i = 0; i < m; ++i) {
    const double r = (i ? std::fabs(beta[i]) : 0.0) + (i + 1 < m ? std::fabs(beta[i + 1]) : 0.0);
    lo = std::min(lo, alpha[i] - r);
    hi = std::max(hi, alpha[i] + r);
    if (i) e2max = std::max(e2max, beta[i] * beta[i]);
  }
  const double tnorm = std::max(std::fabs(lo), std::fabs(hi));
  const double pivmin = DBL_MIN * e2max;
  lo -= 2 * DBL_EPSILON * tnorm + 2 * pivmin;
  hi += 2 * DBL_EPSILON * tnorm + 2 * pivmin;
  // invariant: no eigenvalue below lo, at least one below hi
  for (int it = 0; it < 2200; ++it) {
    const double mid = lo + 0.5 * (hi - lo);
    if (mid <= lo || mid >= hi || hi - lo <= 0x1p-60 * tnorm) break;
    if (sturm_below(alpha, beta, m, mid, pivmin) >= 1)
      hi = mid;
    else
      lo = mid;
  }
  const double th = lo + 0.5 * (hi - lo);
  *theta = th;
  std::vector<double> v(m, 1.0);
  if (m > 1) {
    // LU with partial pivoting of T - theta (LAPACK dgttrf's scheme), then three solves
    std::vector<double> dl(m - 1), d(m), du(m - 1), du2(m > 2 ? m - 2 : 0, 0.0);
    std::vector<uint8_t> swapped(m - 1, 0);
    for (uint32_t i = 0; i < m; ++i) d[i] = alpha[i] - th;
    for (uint32_t i = 0; i + 1 < m; ++i) dl[i] = du[i] = beta[i + 1];
    for (uint32_t i = 0; i + 1 < m; ++i) {
      if (std::fabs(d[i]) >= std::fabs(dl[i])) {
        if (d[i] != 0.0) {
          const double f = dl[i] / d[i];
          dl[i] = f;
          d[i + 1] -= f * du[i];
        }
      } else {
        const double f = d[i] / dl[i];
        d[i] = dl[i];
        dl[i] = f;
        const double tmp = du[i];
        du[i] = d[i + 1];
        d[i + 1] = tmp - f * d[i + 1];
        if (i + 2 < m) {
          du2[i] = du[i + 1];
          du[i + 1] = -f * du[i + 1];
        }
        swapped[i] = 1;
      }
    }
    const double tiny = std::max(0x1p-52 * tnorm, DBL_MIN);
    for (uint32_t i = 0; i < m; ++i)
      if (d[i] == 0.0) d[i] = tiny;
    for (int it = 0; it < 3; ++it) {
      for (uint32_t i = 0; i + 1 < m; ++i) {
        if (!swapped[i]) {
          v[i + 1] -= dl[i] * v[i];
        } else {
          const double tmp = v[i];
          v[i] = v[i + 1];
          v[i + 1] = tmp - dl[i] * v[i];
        }
      }
      v[m - 1] /= d[m - 1];
      v[m - 2] = (v[m - 2] - du[m - 2] * v[m - 1]) / d[m - 2];
      for (uint32_t i = m - 2; i-- > 0;) v[i] = (v[i] - du[i] * v[i + 1] - du2[i] * v[i + 2]) / d[i];
      double mx = 0.0;
      for (double q : v) mx = std::max(mx, std::fabs(q));
      if (!(mx > 0.0) || !std::isfinite(mx)) break;
      double nrm = 0.0;
      for (double &q : v) {
        q /= mx;
        nrm += q * q;
      }
      nrm = std::sqrt(nrm);
      for (double &q : v) q /= nrm;
    }
    if (v[0] < 0)
      for (double &q : v) q = -q;
  }
  if (y) std::copy(v.begin(), v.end(), y);
  *estimate = std::fabs(beta[m]) * std::fabs(v[m - 1]);
}

void lanczos_plan_counts(uint32_t n, const std::vector<PauliTerm> &terms, uint32_t out4[4]) {
  bool identity_only = true;
  for (const PauliTerm &t : terms) identity_only = identity_only && t.x == 0 && t.z == 0;
  if (identity_only) {
    out4[0] = out4[1] = out4[2] = 0;
    out4[3] = 2;
    return;
  }
  const uint32_t s = pauli_sum_sweep_count(n, terms);
  out4[0] = s;
  out4[1] = out4[2] = s + 1;
  out4[3] = s + 4;
}

cudaError_t run_lanczos(qip_prec prec, void *state, void *work_a, void *work_b, uint32_t n,
                        const std::vector<PauliTerm> &terms, const double *coeffs, double a, double b,
                        uint32_t max_steps, double tol, bool vector, cudaStream_t s, uint64_t *launches,
                        LanczosResult *r) {
  const uint64_t N = 1ull << n;
  const uint32_t vgrid = (uint32_t)std::min<uint64_t>(kLanGrid, (N + kLanThreads - 1) / kLanThreads);
  double *scratch = nullptr;  // [3][kLanGrid] vector-kernel rows, then kGradGrid dot partials
  const size_t rows = 3 * kLanGrid + kGradGrid;
  cudaError_t e = cudaMallocAsync((void **)&scratch, rows * sizeof(double), s);
  if (e != cudaSuccess) return e;
  double *red = scratch, *dot = scratch + 3 * kLanGrid;
  std::vector<double> host(rows);
  auto fetch = [&](const double *p, uint32_t cnt, double *out) {
    cudaError_t ec = cudaMemcpyAsync(out, p, cnt * sizeof(double), cudaMemcpyDeviceToHost, s);
    return ec != cudaSuccess ? ec : cudaStreamSynchronize(s);
  };
  auto vec = [&](int mode, VecArgs v) {
    v.red = red;
    v.n_amp = N;
    ++*launches;
    switch (mode) {
      case kVecNorm: return launch_vec<kVecNorm>(prec, v, vgrid, s);
      case kVecScale: return launch_vec<kVecScale>(prec, v, vgrid, s);
      case kVecUpdate: return launch_vec<kVecUpdate>(prec, v, vgrid, s);
      default: return launch_vec<kVecResid>(prec, v, vgrid, s);
    }
  };
  auto buf = [&](uint32_t j) { return j == 0 ? state : (j & 1) ? work_a : work_b; };
  *r = LanczosResult();
  std::vector<double> &al = r->alpha, &be = r->beta;
  std::vector<double> y;
  double theta = 0.0, est = 0.0;
  // one Lanczos step: w_j (sum sweeps) into buf(j + 1), then u_(j+1) in place; second pass: the weights of x
  auto step = [&](uint32_t j, bool first, uint32_t m) -> cudaError_t {
    uint32_t dg = 0;
    const double start = j == 0 ? 1.0 : -(be[j] / be[j - 1]);
    cudaError_t es = run_lanczos_sum(prec, buf(j + 1), buf(j), j == 0 ? nullptr : buf(j - 1), start, n, terms, coeffs,
                                     1.0 / be[j], first ? dot : nullptr, &dg, s, launches);
    if (es != cudaSuccess) return es;
    VecArgs v = {};
    v.p0 = buf(j + 1);
    v.p1 = buf(j);
    v.beta = be[j];
    if (first) {
      v.dot = dot;
      v.dot_grid = dg;
    } else {
      v.mu = al[j] / be[j];
      v.state = state;
      v.acc = j >= 1 || m == 2;
      v.w0 = j >= 2 ? 1.0 : y[0] / be[0];
      v.w1 = j == 1 ? y[1] / be[1] : 0.0;
      v.w2 = y[j + 1] / be[j + 1];
    }
    es = vec(kVecUpdate, v);
    if (es != cudaSuccess || !first) return es;
    es = fetch(scratch, (uint32_t)rows, host.data());
    if (es != cudaSuccess) return es;
    al.push_back(ordered_sum(host.data() + 3 * kLanGrid, dg) / be[j]);
    be.push_back(std::sqrt(ordered_sum(host.data(), vgrid)));
    return cudaSuccess;
  };
  VecArgs v = {};
  v.p0 = state;
  e = vec(kVecNorm, v);
  if (e == cudaSuccess) e = fetch(red, vgrid, host.data());
  if (e == cudaSuccess) {
    be.push_back(std::sqrt(ordered_sum(host.data(), vgrid)));
    if (!(be[0] > 0.0) || !std::isfinite(be[0])) r->zero_norm = true;
  }
  if (e == cudaSuccess && !r->zero_norm && b == 0.0) {  // every vector is an eigenvector, with eigenvalue a
    r->energy = a;
    r->converged = 1;
    if (vector) {
      v.s = 1.0 / be[0];
      e = vec(kVecScale, v);
      r->xnorm = 1.0;
    }
  } else if (e == cudaSuccess && !r->zero_norm) {
    y.assign(max_steps, 0.0);
    for (uint32_t j = 0; j < max_steps && e == cudaSuccess; ++j) {
      e = step(j, true, 0);
      if (e != cudaSuccess) break;
      const uint32_t m = j + 1;
      lanczos_ritz(al.data(), be.data(), m, &theta, y.data(), &est);
      r->steps = m;
      if (est <= tol * b) {
        r->converged = 1;
        break;
      }
    }
    r->energy = theta;
    r->residual = est;
    const uint32_t m = r->steps;
    if (e == cudaSuccess && vector) {
      for (uint32_t j = 0; j + 1 < m && e == cudaSuccess; ++j) e = step(j, false, m);
      v = VecArgs();
      v.p0 = state;
      if (e == cudaSuccess) e = vec(kVecNorm, v);
      if (e == cudaSuccess) e = fetch(red, vgrid, host.data());
      if (e == cudaSuccess) {
        const double nx = std::sqrt(ordered_sum(host.data(), vgrid));
        r->xnorm = m == 1 ? nx / be[0] : nx;
        v.s = 1.0 / nx;
        e = vec(kVecScale, v);
      }
      if (e == cudaSuccess) e = run_pauli_sum(prec, work_a, state, n, terms, coeffs, s, launches);
      v = VecArgs();
      v.p0 = state;
      v.p1 = work_a;
      v.s = theta;
      if (e == cudaSuccess) e = vec(kVecResid, v);
      if (e == cudaSuccess) e = fetch(red, 3 * vgrid, host.data());
      if (e == cudaSuccess) {
        const double xhx = ordered_sum(host.data(), vgrid), rt = ordered_sum(host.data() + vgrid, vgrid);
        const double xx = ordered_sum(host.data() + 2 * vgrid, vgrid);
        const double E = xhx / xx, d = E - theta;
        r->energy = E;
        r->residual = std::sqrt(std::max(0.0, rt - d * d * xx) / xx);
      }
    }
  }
  const cudaError_t ef = cudaFreeAsync(scratch, s);
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  return ef != cudaSuccess ? ef : es;
}

}  // namespace qipb200
