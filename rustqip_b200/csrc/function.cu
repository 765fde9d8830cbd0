// function.cu -- psi <- U psi for a classical function given as a table, U|x>|y> = e^{i theta(x)} |x>|y ^ f(x)>
// (qipb200_state_apply_function).
//
// With x(j) the in-register value of index j and d(x) the out-register bits of f(x) scattered to their index bits,
//   (U psi)_j = e^{i theta(x(j))} psi_{j ^ d(x(j))}.
// The registers are disjoint, so x(j ^ d) = x(j): U pairs j with j ^ d, an involution whose partner and phase are the
// same from both sides.  One read-write sweep in place, whatever f is.
//
// Arithmetic.  Without theta the op moves amplitudes and is exact (-0 stays -0).  With theta, c and s are cos and sin
// of theta(x) computed in double on the host (qipb200_function_new) and rounded once here to the state's precision,
// and for the partner amplitude (a, b) = psi_{j ^ d}
//   out_j = (RN(RN(c a) - RN(s b)), RN(RN(c b) + RN(s a)))
// with explicit __dmul_rn / __dadd_rn (__fmul_rn / __fadd_rn), no FMA.  Neither the path, the tile geometry nor the
// layout changes a bit of the result.
//
// Index maps.  x(j) and d(f) are read from shared-memory chunk tables built per CTA: byte k of the physical index
// gives its bits of x (5 tables of 256), byte k of f(x) gives its bits of d (4 tables of 256).
//
// Staged tile path (k_function_tile; plan in function.h, tile geometry of sweep.cuh).  Every out bit lies in the tile,
// so every partner does too.
// A CTA visits tiles in turn: the next tile is loaded with cp.async into the second buffer while the current one is
// processed (as k_pauli_rot does).  A thread's elements e = t + threads k sit at fixed offsets off[k] in every tile, so
// x = x(base) | x(off[k]): the CTA-uniform part costs five table reads per visit and the per-thread parts are computed
// once.  A thread reads its f and (cos, sin) entries for a visit before it waits for the visit's tile, so their L2
// latency overlaps the tile's.  Each thread reads the old partner values from the staged tile and stores its new values
// straight to the state; the tile buffer is reused only after the next barrier.  d is scattered to tile-local bits by the f tables.
//
// Pair path (k_function_pair).  One thread per index j: d == 0 applies the phase (nothing without theta); otherwise
// the thread with the highest bit of d clear in j swaps psi_j and psi_{j ^ d} with the phase.  Each pair has exactly
// one owner, so the path is race-free in place, and every amplitude is read and written once.
#include "function.h"
#include "sweep.cuh"

#include <algorithm>
#include <cstring>

namespace qipb200 {

namespace {

const uint32_t kFnTileF64 = 11;  // T_max: 2^11 x 16 B = 32 KiB per tile buffer
const uint32_t kFnTileF32 = 12;  // 2^12 x 8 B = 32 KiB
static_assert(kFnTileF32 - kSweepL <= kSweepMaxHi && kFnTileF64 <= kFnTileF32,
              "the high tile bits fit SweepTiles::hi_pos");
const int kFnPer = 8;            // tile amplitudes per thread
const int kFnPairThreads = 256;

struct FnArgs {
  const uint32_t *f;   // f[x], or NULL (no out register)
  const double2 *cs;   // (cos, sin) of theta[x], or NULL (no phase)
  SweepTiles geo;      // tile path (x_out = 0)
  uint32_t n;          // index bits of the state
  uint32_t xbytes;     // bytes of the index that hold in bits
  uint32_t n_out, fbytes;
  uint8_t xbit[40];    // physical index bit -> bit of x, or 0xFF
  uint8_t dpos[32];    // bit i of f(x) -> index bit (pair path) or tile-local bit (tile path)
};

struct FnTables {
  uint32_t x[5][256];  // byte k of the physical index -> its bits of x
  uint64_t d[4][256];  // byte k of f(x) -> its bits of d
};

__device__ void build_tables(FnTables *T, const FnArgs &a) {
  for (uint32_t i = threadIdx.x; i < 5 * 256; i += blockDim.x) {
    const uint32_t k = i >> 8, v = i & 255;
    uint32_t x = 0;
    for (uint32_t b = 0; b < 8; ++b) {
      const uint32_t p = 8 * k + b;
      if (p < a.n && ((v >> b) & 1) && a.xbit[p] != 0xFF) x |= 1u << a.xbit[p];
    }
    T->x[k][v] = x;
  }
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

__device__ __forceinline__ uint32_t x_of(const FnTables &T, uint64_t j, uint32_t xbytes) {
  uint32_t x = 0;
#pragma unroll
  for (uint32_t k = 0; k < 5; ++k)
    if (k < xbytes) x |= T.x[k][(j >> (8 * k)) & 255];
  return x;
}

__device__ __forceinline__ uint64_t d_of(const FnTables &T, uint32_t fx, uint32_t fbytes) {
  uint64_t d = 0;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k)
    if (k < fbytes) d |= T.d[k][(fx >> (8 * k)) & 255];
  return d;
}

// (cos, sin) of theta(x) rounded once to R.
template <typename R, typename V>
__device__ __forceinline__ V fn_cs(const double2 *cs, uint32_t x) {
  const double2 w = __ldg(cs + x);
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

template <typename R, typename V, bool THETA>
__device__ __forceinline__ V fn_value(V p, const double2 *cs, uint32_t x) {
  return THETA ? fn_phase<R, V, THETA>(p, fn_cs<R, V>(cs, x)) : p;
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

template <typename R, bool THETA>
__global__ void __launch_bounds__((1 << FnTile<R>::kBits) / kFnPer, 2)
    k_function_tile(R *__restrict__ psi, const __grid_constant__ FnArgs a) {
  typedef typename SweepV<R>::type V;
  constexpr int kTile = 1 << FnTile<R>::kBits, kThreads = kTile / kFnPer;
  extern __shared__ __align__(16) unsigned char smem[];
  V *tiles = reinterpret_cast<V *>(smem);  // [2][kTile]: double buffer
  FnTables *T = reinterpret_cast<FnTables *>(smem + 2 * kTile * sizeof(V));
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
  uint32_t xo[kFnPer];
#pragma unroll
  for (int k = 0; k < kFnPer; ++k) xo[k] = x_of(*T, off[k], a.xbytes);
  int cur = 0;
  for (; v < a.geo.n_visits; v += gridDim.x) {
    // the visit's table entries first: their L2 latency overlaps the wait for the tile
    const uint64_t b = visit_base(a.geo, v);
    const uint32_t xb = x_of(*T, b, a.xbytes);
    uint32_t de[kFnPer];
    V w[kFnPer];
#pragma unroll
    for (int k = 0; k < kFnPer; ++k) {
      const uint32_t x = xb | xo[k];
      const bool mine = t + kThreads * k < tsize;
      de[k] = a.f && mine ? (uint32_t)d_of(*T, __ldg(a.f + x), a.fbytes) : 0u;
      if (THETA && mine) w[k] = fn_cs<R, V>(a.cs, x);
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

template <typename R, bool THETA>
__global__ void __launch_bounds__(kFnPairThreads) k_function_pair(R *__restrict__ psi, const __grid_constant__ FnArgs a) {
  typedef typename SweepV<R>::type V;
  __shared__ FnTables T;
  build_tables(&T, a);
  __syncthreads();
  V *P = reinterpret_cast<V *>(psi);
  const uint64_t N = 1ull << a.n, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += stride) {
    const uint32_t x = x_of(T, j, a.xbytes);
    const uint64_t d = d_of(T, __ldg(a.f + x), a.fbytes);
    if (d == 0) {
      if (THETA) P[j] = fn_value<R, V, THETA>(P[j], a.cs, x);
    } else if (!((j >> (63 - __clzll(d))) & 1)) {
      const V u = P[j], w = P[j ^ d];
      P[j] = fn_value<R, V, THETA>(w, a.cs, x);
      P[j ^ d] = fn_value<R, V, THETA>(u, a.cs, x);
    }
  }
}

template <typename R, bool THETA>
cudaError_t launch_tile(void *psi, const FnArgs &a, int sm_count, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  constexpr int kTile = 1 << FnTile<R>::kBits, kThreads = kTile / kFnPer;
  const size_t smem = 2 * kTile * sizeof(V) + sizeof(FnTables);
  static_assert(2 * (1 << kFnTileF64) * sizeof(double2) + sizeof(FnTables) <= 113 * 1024,
                "two CTAs per SM: at most 113 KiB of shared memory each");
  cudaError_t e = cudaFuncSetAttribute(k_function_tile<R, THETA>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  const int grid = (int)std::min<uint64_t>(a.geo.n_visits, (uint64_t)std::max(2 * sm_count, 1));
  k_function_tile<R, THETA><<<grid, kThreads, smem, s>>>((R *)psi, a);
  return cudaGetLastError();
}

template <typename R, bool THETA>
cudaError_t launch_pair(void *psi, const FnArgs &a, int sm_count, cudaStream_t s) {
  const uint64_t blocks = ((1ull << a.n) + kFnPairThreads - 1) / kFnPairThreads;
  const int grid = (int)std::min<uint64_t>(blocks, (uint64_t)std::max(8 * sm_count, 1));
  k_function_pair<R, THETA><<<grid, kFnPairThreads, 0, s>>>((R *)psi, a);
  return cudaGetLastError();
}

}  // namespace

FnPlan plan_function(qip_prec prec, uint32_t n, const uint32_t *out_pos, uint32_t n_out) {
  const uint32_t L = std::min(kSweepL, n), T = std::min(prec == QIP_F32 ? kFnTileF32 : kFnTileF64, n);
  FnPlan p;
  for (uint32_t i = 0; i < n_out; ++i)
    if (out_pos[i] >= L) p.hi |= 1ull << out_pos[i];
  if (L + (uint32_t)__builtin_popcountll(p.hi) > T) {
    p.path = 1;
    p.hi = 0;
    return p;
  }
  for (uint32_t b = L; b < n && L + (uint32_t)__builtin_popcountll(p.hi) < T; ++b) p.hi |= 1ull << b;
  p.tile_bits = T;
  return p;
}

cudaError_t run_function(qip_prec prec, void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                         const uint32_t *out_pos, uint32_t n_out, const uint32_t *f, const double2 *cs, int sm_count,
                         cudaStream_t s, uint64_t *launches) {
  FnArgs a;
  memset(&a, 0, sizeof(a));
  a.f = n_out ? f : nullptr;
  a.cs = cs;
  a.n = n;
  a.n_out = n_out;
  a.fbytes = (n_out + 7) / 8;
  memset(a.xbit, 0xFF, sizeof(a.xbit));
  uint32_t top = 0;
  for (uint32_t i = 0; i < n_in; ++i) {
    a.xbit[in_pos[i]] = (uint8_t)i;
    top = std::max(top, in_pos[i] + 1);
  }
  a.xbytes = (top + 7) / 8;
  const FnPlan p = plan_function(prec, n, out_pos, n_out);
  if (p.path == 1) {
    for (uint32_t i = 0; i < n_out; ++i) a.dpos[i] = (uint8_t)out_pos[i];
  } else {
    a.geo = sweep_tiles(n, std::min(kSweepL, n), p.hi, 0);
    for (uint32_t i = 0; i < n_out; ++i) a.dpos[i] = (uint8_t)__builtin_ctz(tile_local(a.geo, 1ull << out_pos[i]));
  }
  cudaError_t e;
  const bool th = cs != nullptr;
  if (p.path == 1) {
    if (prec == QIP_F32)
      e = th ? launch_pair<float, true>(psi, a, sm_count, s) : launch_pair<float, false>(psi, a, sm_count, s);
    else
      e = th ? launch_pair<double, true>(psi, a, sm_count, s) : launch_pair<double, false>(psi, a, sm_count, s);
  } else {
    if (prec == QIP_F32)
      e = th ? launch_tile<float, true>(psi, a, sm_count, s) : launch_tile<float, false>(psi, a, sm_count, s);
    else
      e = th ? launch_tile<double, true>(psi, a, sm_count, s) : launch_tile<double, false>(psi, a, sm_count, s);
  }
  ++*launches;
  return e;
}

}  // namespace qipb200
