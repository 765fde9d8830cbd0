// function_dev.cuh -- the device side of function ops (function.cu): the bodies of the two apply kernels, of the
// diagonal expectation value, of the range and phase checks and of the tabulation.  Each body is templated on the
// source S of f and theta, which provides
//   typedef X             the type of x (uint32_t for tables, uint64_t for code: n_in may exceed 32);
//   bool has_f()          whether there is an out register;
//   f(x)                  f(x) (an integer; only called when has_f());
//   double2 cs(x)         (cos theta(x), sin theta(x)) in double;
//   double theta(x)       theta(x) in double (code sources only: a table keeps cos and sin, not theta).
// function.cu instantiates the bodies with nvcc for tables.  The text of this header and of sweep_dev.cuh is also
// embedded in the library and compiled with NVRTC ahead of the user's source for code functions, whose entry points
// (function.cu: code_program) call the same bodies.  So the apply of a table and of code differ only in where f and
// (c, s) come from.
#pragma once

#include "sweep_dev.cuh"

namespace qipb200 {

const uint32_t kFnTileF64 = 11;  // T_max: 2^11 x 16 B = 32 KiB per tile buffer
const uint32_t kFnTileF32 = 12;  // 2^12 x 8 B = 32 KiB
const int kFnPer = 8;            // tile amplitudes per thread
const int kFnPairThreads = 256;
const int kFnExpThreads = 256;                  // expect: CTA size
const int kFnExpGrid = 264;                     // expect: fixed grid, so the sum order does not depend on the device
const int kFnExpChunk = kFnExpThreads * kFnPer; // expect: amplitudes per chunk
const int kFnCheckThreads = 256;                // range/phase checks and tabulation

struct FnArgs {
  SweepTiles geo;      // tile path (x_out = 0)
  uint32_t n;          // index bits of the state
  uint32_t xbytes;     // bytes of the index that hold in bits
  uint32_t n_out, fbytes;
  uint8_t xbit[40];    // physical index bit -> bit of x, or 0xFF
  uint8_t dpos[32];    // bit i of f(x) -> index bit (pair path) or tile-local bit (tile path)
};

template <typename X>
struct FnTables {
  X x[5][256];         // byte k of the physical index -> its bits of x
  uint64_t d[4][256];  // byte k of f(x) -> its bits of d
};

namespace {

template <typename X>
__device__ void build_x_tables(FnTables<X> *T, const FnArgs &a) {
  for (uint32_t i = threadIdx.x; i < 5 * 256; i += blockDim.x) {
    const uint32_t k = i >> 8, v = i & 255;
    X x = 0;
    for (uint32_t b = 0; b < 8; ++b) {
      const uint32_t p = 8 * k + b;
      if (p < a.n && ((v >> b) & 1) && a.xbit[p] != 0xFF) x |= (X)1 << a.xbit[p];
    }
    T->x[k][v] = x;
  }
}

template <typename X>
__device__ void build_tables(FnTables<X> *T, const FnArgs &a) {
  build_x_tables(T, a);
  for (uint32_t i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
    const uint32_t k = i >> 8, v = i & 255;
    uint64_t d = 0;
    for (uint32_t b = 0; b < 8; ++b) {
      const uint32_t q = 8 * k + b;
      if (q < a.n_out && ((v >> b) & 1)) d |= 1ull << a.dpos[q];
    }
    T->d[k][v] = d;
  }
}

// x(j): the in bits of physical index j.  The bits map one by one, so x(j | j') = x(j) | x(j') for disjoint j, j'.
template <typename X>
__device__ __forceinline__ X x_of(const FnTables<X> &T, uint64_t j, uint32_t xbytes) {
  X x = 0;
#pragma unroll
  for (uint32_t k = 0; k < 5; ++k)
    if (k < xbytes) x |= T.x[k][(j >> (8 * k)) & 255];
  return x;
}

template <typename X>
__device__ __forceinline__ uint64_t d_of(const FnTables<X> &T, uint32_t fx, uint32_t fbytes) {
  uint64_t d = 0;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k)
    if (k < fbytes) d |= T.d[k][(fx >> (8 * k)) & 255];
  return d;
}

// (cos, sin) of theta(x) rounded once to R.
template <typename R, typename V>
__device__ __forceinline__ V fn_cs(double2 w) {
  V r;
  r.x = (R)w.x;
  r.y = (R)w.y;
  return r;
}

// e^{i theta} p: (RN(RN(c a) - RN(s b)), RN(RN(c b) + RN(s a))) with (c, s) = w.
template <typename R, typename V, bool THETA>
__device__ __forceinline__ V fn_phase(V p, V w) {
  if (!THETA) return p;
  const R c = w.x, s = w.y;
  V o;
  o.x = add_rn(mul_rn(c, p.x), -mul_rn(s, p.y));
  o.y = add_rn(mul_rn(c, p.y), mul_rn(s, p.x));
  return o;
}

template <typename R, typename V, bool THETA, typename S>
__device__ __forceinline__ V fn_value(V p, const S &src, typename S::X x) {
  return THETA ? fn_phase<R, V, THETA>(p, fn_cs<R, V>(src.cs(x))) : p;
}

template <typename R>
struct FnTile;
template <>
struct FnTile<double> {
  static const int kBits = kFnTileF64;
};
template <>
struct FnTile<float> {
  static const int kBits = kFnTileF32;
};

// The staged tile path: (1 << FnTile<R>::kBits) / kFnPer threads, 2 tile buffers and FnTables<S::X> of dynamic shared
// memory.
template <typename R, bool THETA, typename S>
__device__ __forceinline__ void fn_tile(R *__restrict__ psi, const FnArgs &a, const S &src) {
  typedef typename SweepV<R>::type V;
  typedef typename S::X X;
  constexpr int kTile = 1 << FnTile<R>::kBits, kThreads = kTile / kFnPer;
  extern __shared__ __align__(16) unsigned char smem[];
  V *tiles = reinterpret_cast<V *>(smem);  // [2][kTile]: double buffer
  FnTables<X> *T = reinterpret_cast<FnTables<X> *>(smem + 2 * kTile * sizeof(V));
  build_tables(T, a);
  const int t = threadIdx.x;
  const uint32_t tsize = 1u << a.geo.tb;  // below kTile only when the whole state is one tile
  uint64_t off[kFnPer];
#pragma unroll
  for (int k = 0; k < kFnPer; ++k) off[k] = tile_offset(a.geo, t + kThreads * k);
  auto issue = [&](uint64_t v, V *dst) {
    const uint64_t b = visit_base(a.geo, v);
#pragma unroll
    for (int k = 0; k < kFnPer; ++k) {
      const uint32_t e = t + kThreads * k;
      if (e < tsize) cp_async<sizeof(V)>(dst + e, psi + 2 * (b | off[k]));
    }
  };
  uint64_t v = blockIdx.x;
  if (v < a.geo.n_visits) issue(v, tiles);
  cp_async_commit();
  __syncthreads();  // the tables
  X xo[kFnPer];
#pragma unroll
  for (int k = 0; k < kFnPer; ++k) xo[k] = x_of(*T, off[k], a.xbytes);
  int cur = 0;
  for (; v < a.geo.n_visits; v += gridDim.x) {
    // the visit's f and (c, s) first: a table's L2 latency (or the code's arithmetic) overlaps the wait for the tile
    const uint64_t b = visit_base(a.geo, v);
    const X xb = x_of(*T, b, a.xbytes);
    uint32_t de[kFnPer];
    V w[kFnPer];
#pragma unroll
    for (int k = 0; k < kFnPer; ++k) {
      const X x = xb | xo[k];
      const bool mine = t + kThreads * k < tsize;
      de[k] = src.has_f() && mine ? (uint32_t)d_of(*T, (uint32_t)src.f(x), a.fbytes) : 0u;
      if (THETA && mine) w[k] = fn_cs<R, V>(src.cs(x));
    }
    const uint64_t nv = v + gridDim.x;  // the next tile into the other buffer, then wait for the current one only
    if (nv < a.geo.n_visits) issue(nv, tiles + (cur ^ 1) * kTile);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const V *A = tiles + cur * kTile;
#pragma unroll
    for (int k = 0; k < kFnPer; ++k) {
      const uint32_t e = t + kThreads * k;
      if (e >= tsize) continue;
      *reinterpret_cast<V *>(psi + 2 * (b | off[k])) = fn_phase<R, V, THETA>(A[e ^ de[k]], w[k]);
    }
    __syncthreads();  // every thread has read this buffer before the next cp.async writes it
    cur ^= 1;
  }
  cp_async_wait<0>();
}

// The pair path: kFnPairThreads threads, static shared memory only.
template <typename R, bool THETA, typename S>
__device__ __forceinline__ void fn_pair(R *__restrict__ psi, const FnArgs &a, const S &src) {
  typedef typename SweepV<R>::type V;
  typedef typename S::X X;
  __shared__ FnTables<X> T;
  build_tables(&T, a);
  __syncthreads();
  V *P = reinterpret_cast<V *>(psi);
  const uint64_t N = 1ull << a.n, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += stride) {
    const X x = x_of(T, j, a.xbytes);
    const uint64_t d = d_of(T, (uint32_t)src.f(x), a.fbytes);
    if (d == 0) {
      if (THETA) P[j] = fn_value<R, V, THETA>(P[j], src, x);
    } else if (!((j >> (63 - __clzll(d))) & 1)) {
      const V u = P[j], w = P[j ^ d];
      P[j] = fn_value<R, V, THETA>(w, src, x);
      P[j ^ d] = fn_value<R, V, THETA>(u, src, x);
    }
  }
}

// Per-CTA partial of sum_j |psi_j|^2 theta(x(j)) (kFnExpThreads threads, kFnExpGrid CTAs).  The state is cut into
// chunks of C = min(2^n, kFnExpChunk) consecutive amplitudes; chunk c goes to CTA c mod grid, and thread t owns the
// chunk's elements t + kFnExpThreads k, k < kFnPer, so x = x(chunk base) | x(element).  A thread adds its terms in
// chunk order, then k order; a CTA sums its threads by a fixed xor-shuffle tree per warp and the warps in order.
template <typename R, typename S>
__device__ __forceinline__ void fn_expect(const R *__restrict__ psi, const FnArgs &a, const S &src,
                                          double *__restrict__ partial) {
  typedef typename SweepV<R>::type V;
  typedef typename S::X X;
  __shared__ FnTables<X> T;
  __shared__ double warp_sum[kFnExpThreads / 32];
  build_x_tables(&T, a);
  __syncthreads();
  const V *P = reinterpret_cast<const V *>(psi);
  const uint64_t N = 1ull << a.n;
  const uint32_t C = N < (uint64_t)kFnExpChunk ? (uint32_t)N : (uint32_t)kFnExpChunk;
  const uint64_t n_chunks = N / C;
  const uint32_t t = threadIdx.x;
  X xo[kFnPer];
#pragma unroll
  for (int k = 0; k < kFnPer; ++k) xo[k] = x_of(T, t + kFnExpThreads * k, a.xbytes);
  double acc = 0.0;
  for (uint64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const uint64_t b = c * C;
    const X xb = x_of(T, b, a.xbytes);
    V p[kFnPer];
#pragma unroll
    for (int k = 0; k < kFnPer; ++k)
      if (t + kFnExpThreads * k < C) p[k] = __ldg(P + b + t + kFnExpThreads * k);
#pragma unroll
    for (int k = 0; k < kFnPer; ++k)
      if (t + kFnExpThreads * k < C) {
        const double re = p[k].x, im = p[k].y;
        const double w = __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im));
        acc = __dadd_rn(acc, __dmul_rn(w, src.theta(xb | xo[k])));
      }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if ((t & 31) == 0) warp_sum[t >> 5] = acc;
  __syncthreads();
  if (t == 0) {
    double s = warp_sum[0];
    for (int w = 1; w < kFnExpThreads / 32; ++w) s = __dadd_rn(s, warp_sum[w]);
    partial[blockIdx.x] = s;
  }
}

// *first = min(*first, x) over the x < 2^n_in with f(x) >= 2^n_out (RANGE) or a non-finite theta(x) (!RANGE).
template <bool RANGE, typename S>
__device__ __forceinline__ void fn_check(const S &src, uint32_t n_in, uint32_t n_out, unsigned long long *first) {
  const uint64_t N = 1ull << n_in, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < N; x += stride) {
    bool bad;
    if (RANGE) {
      bad = ((uint64_t)src.f((typename S::X)x) >> n_out) != 0;
    } else {
      const double th = src.theta((typename S::X)x);
      bad = !(fabs(th) <= 1.7976931348623157e308);  // NaN or +-inf
    }
    if (bad) atomicMin(first, (unsigned long long)x);
  }
}

// f(x) and (cos theta(x), sin theta(x)) for x in [x0, x0 + count); either output may be NULL.
template <typename S>
__device__ __forceinline__ void fn_tabulate(const S &src, uint64_t x0, uint64_t count, uint64_t *f_out,
                                            double2 *cs_out) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
    const typename S::X x = (typename S::X)(x0 + i);
    if (f_out) f_out[i] = src.has_f() ? (uint64_t)src.f(x) : 0ull;
    if (cs_out) cs_out[i] = src.cs(x);
  }
}

}  // namespace

}  // namespace qipb200
