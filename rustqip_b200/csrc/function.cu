// function.cu -- psi <- U psi for a classical function given as a table or as code, U|x>|y> = e^{i theta(x)} |x>|y ^ f(x)>
// (qipb200_state_apply_function), and the diagonal expectation value sum_j |psi_j|^2 theta(x(j)) of a code function
// (qipb200_state_expect_function).  The kernel bodies are in function_dev.cuh.
//
// With x(j) the in-register value of index j and d(x) the out-register bits of f(x) scattered to their index bits,
//   (U psi)_j = e^{i theta(x(j))} psi_{j ^ d(x(j))}.
// The registers are disjoint, so x(j ^ d) = x(j): U pairs j with j ^ d, an involution whose partner and phase are the
// same from both sides.  One read-write sweep in place, whatever f is.
//
// Arithmetic.  Without theta the op moves amplitudes and is exact (-0 stays -0).  With theta, c and s are cos and sin
// of theta(x) computed in double (on the host by qipb200_function_new for a table, on the device with sincos for code)
// and rounded once here to the state's precision, and for the partner amplitude (a, b) = psi_{j ^ d}
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
//
// Code functions (qipb200_function_new_code).  The user's source defines qip_f and, with a phase, qip_theta.
// code_program builds one NVRTC program: the text of sweep_dev.cuh and function_dev.cuh (embedded at build time), the
// user's source, and entry points that run the same bodies as the table kernels with a source QipCode that calls the
// user's functions, (c, s) = sincos(theta(x, p)) in double.  It is compiled with the generated pass kernels' options
// (jit_runtime: sm_90a SASS, --fmad=false) through jit_request, so the process cache and QIPB200_JIT_CACHE_DIR apply.
// x is a u64 there (n_in up to 34): a CTA's x tables take 10 KiB instead of 5.  The parameters p ride in the kernel
// arguments, so set_params never races with a queued apply.
//
// Diagonal expectation value (fn_expect; qipb200_state_expect_function): sum_j |psi_j|^2 theta(x(j)) in double on a
// fixed grid of kFnExpGrid CTAs.  Order: chunks of C = min(2^n, 2048) consecutive amplitudes go to CTA c mod G; a
// thread adds its terms sequentially in chunk order, its 8 elements per chunk in order; each warp sums by an xor-shuffle
// tree (5 levels), the CTA's 8 warp sums are added in warp order, and the host adds the G partials in CTA order.  No
// floating-point atomics: the same state and parameters give the same bits.
// Rounding: |psi_j|^2 = RN(RN(a^2) + RN(b^2)) (f32 amplitudes are exact in double) and its product with theta cost
// gamma_3 relative per term; the longest chain of additions is D = 8 ceil(V / G) + 5 + 7 + (G - 1) for V = 2^n / C
// chunks.  So, to first order in u = 2^-53, |got - sum_j |psi_j|^2 theta_j| <= (3 + D) u sum_j |psi_j|^2 |theta_j|,
// with theta_j the double theta(x(j), p) the device computes.
#include "function.h"

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/qipb200.h"
#include "function_dev.cuh"
#include "jit_runtime.h"
#include "sweep.cuh"

namespace qipb200 {

namespace {

static_assert(kFnTileF32 - kSweepL <= kSweepMaxHi && kFnTileF64 <= kFnTileF32,
              "the high tile bits fit SweepTiles::hi_pos");
static_assert(kFnExpGrid == kFnExpPartials, "function.h sizes the expect partials");

// sweep_dev.cuh and function_dev.cuh as text, without their #pragma once and #include lines (Makefile)
const char kFnDevText[] =
#include "function_dev_text.inc"
    ;

// f and (cos, sin) of theta from the device tables of qipb200_function_new.
struct FnTableSrc {
  typedef uint32_t X;
  const uint32_t *tf;  // f[x], or NULL (no out register)
  const double2 *tcs;  // (cos, sin) of theta[x], or NULL (no phase)
  __device__ __forceinline__ bool has_f() const { return tf != nullptr; }
  __device__ __forceinline__ uint32_t f(uint32_t x) const { return __ldg(tf + x); }
  __device__ __forceinline__ double2 cs(uint32_t x) const { return __ldg(tcs + x); }
};

// The host image of the program's QipCode: its parameters.
struct FnCodeArgs {
  double p[kFnCodeMaxParams];
};

template <typename R, bool THETA>
__global__ void __launch_bounds__((1 << FnTile<R>::kBits) / kFnPer, 2)
    k_function_tile(R *__restrict__ psi, const __grid_constant__ FnArgs a, const __grid_constant__ FnTableSrc src) {
  fn_tile<R, THETA>(psi, a, src);
}

template <typename R, bool THETA>
__global__ void __launch_bounds__(kFnPairThreads)
    k_function_pair(R *__restrict__ psi, const __grid_constant__ FnArgs a, const __grid_constant__ FnTableSrc src) {
  fn_pair<R, THETA>(psi, a, src);
}

__global__ void __launch_bounds__(kFnCheckThreads)
    k_function_tabulate(const __grid_constant__ FnTableSrc src, uint64_t x0, uint64_t count, uint64_t *f_out,
                        double2 *cs_out) {
  fn_tabulate(src, x0, count, f_out, cs_out);
}

template <typename R, typename X>
size_t tile_smem() {
  return 2 * (1 << FnTile<R>::kBits) * sizeof(typename SweepV<R>::type) + sizeof(FnTables<X>);
}
static_assert(2 * (1 << kFnTileF64) * sizeof(double2) + sizeof(FnTables<uint64_t>) <= 113 * 1024,
              "two CTAs per SM: at most 113 KiB of shared memory each");

int tile_grid(const FnArgs &a, int sm_count) {
  return (int)std::min<uint64_t>(a.geo.n_visits, (uint64_t)std::max(2 * sm_count, 1));
}

int pair_grid(const FnArgs &a, int sm_count) {
  const uint64_t blocks = ((1ull << a.n) + kFnPairThreads - 1) / kFnPairThreads;
  return (int)std::min<uint64_t>(blocks, (uint64_t)std::max(8 * sm_count, 1));
}

int check_grid(uint64_t count, int sm_count) {
  return (int)std::min<uint64_t>((count + kFnCheckThreads - 1) / kFnCheckThreads, (uint64_t)std::max(8 * sm_count, 1));
}

template <typename R, bool THETA>
cudaError_t launch_tile(void *psi, const FnArgs &a, const FnTableSrc &src, int sm_count, cudaStream_t s) {
  constexpr int kThreads = (1 << FnTile<R>::kBits) / kFnPer;
  const size_t smem = tile_smem<R, uint32_t>();
  cudaError_t e = cudaFuncSetAttribute(k_function_tile<R, THETA>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  k_function_tile<R, THETA><<<tile_grid(a, sm_count), kThreads, smem, s>>>((R *)psi, a, src);
  return cudaGetLastError();
}

template <typename R, bool THETA>
cudaError_t launch_pair(void *psi, const FnArgs &a, const FnTableSrc &src, int sm_count, cudaStream_t s) {
  k_function_pair<R, THETA><<<pair_grid(a, sm_count), kFnPairThreads, 0, s>>>((R *)psi, a, src);
  return cudaGetLastError();
}

// The arguments of every kernel of an op on in_pos / out_pos of a 2^n state, and its plan.
FnArgs fn_args(qip_prec prec, uint32_t n, const uint32_t *in_pos, uint32_t n_in, const uint32_t *out_pos,
               uint32_t n_out, FnPlan *plan) {
  FnArgs a;
  memset(&a, 0, sizeof(a));
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
  if (plan) *plan = p;
  return a;
}

// The entry points of a code function's program; QIP_FN_THETA and QIP_FN_NOUT are defined ahead of them.
const char kFnCodeEntries[] = R"QIPSRC(
struct QipCode {
  typedef uint64_t X;
  double p[16];
  __device__ __forceinline__ bool has_f() const { return QIP_FN_NOUT > 0; }
  __device__ __forceinline__ uint64_t f(uint64_t x) const {
#if QIP_FN_NOUT > 0
    return qip_f(x);
#else
    return 0;
#endif
  }
  __device__ __forceinline__ double theta(uint64_t x) const {
#if QIP_FN_THETA
    return qip_theta(x, p);
#else
    return 0.0;
#endif
  }
  __device__ __forceinline__ double2 cs(uint64_t x) const {
    double s, c;
    sincos(theta(x), &s, &c);
    return make_double2(c, s);
  }
};

#define QIP_FN_APPLY(R, NAME)                                                                                        \
  extern "C" __global__ void __launch_bounds__((1 << qipb200::FnTile<R>::kBits) / qipb200::kFnPer, 2)                \
      qip_fn_tile_##NAME(R *__restrict__ psi, const __grid_constant__ qipb200::FnArgs a,                             \
                         const __grid_constant__ QipCode src) {                                                      \
    qipb200::fn_tile<R, QIP_FN_THETA>(psi, a, src);                                                                  \
  }                                                                                                                  \
  extern "C" __global__ void __launch_bounds__(qipb200::kFnPairThreads)                                              \
      qip_fn_pair_##NAME(R *__restrict__ psi, const __grid_constant__ qipb200::FnArgs a,                             \
                         const __grid_constant__ QipCode src) {                                                      \
    qipb200::fn_pair<R, QIP_FN_THETA>(psi, a, src);                                                                  \
  }
QIP_FN_APPLY(float, f32)
QIP_FN_APPLY(double, f64)

#if QIP_FN_THETA
#define QIP_FN_EXPECT(R, NAME)                                                                                       \
  extern "C" __global__ void __launch_bounds__(qipb200::kFnExpThreads)                                               \
      qip_fn_expect_##NAME(const R *__restrict__ psi, const __grid_constant__ qipb200::FnArgs a,                     \
                           const __grid_constant__ QipCode src, double *__restrict__ partial) {                      \
    qipb200::fn_expect<R>(psi, a, src, partial);                                                                     \
  }
QIP_FN_EXPECT(float, f32)
QIP_FN_EXPECT(double, f64)

extern "C" __global__ void __launch_bounds__(qipb200::kFnCheckThreads)
    qip_fn_check_theta(const __grid_constant__ QipCode src, uint32_t n_in, uint32_t n_out, unsigned long long *first) {
  qipb200::fn_check<false>(src, n_in, n_out, first);
}
#endif

#if QIP_FN_NOUT > 0
extern "C" __global__ void __launch_bounds__(qipb200::kFnCheckThreads)
    qip_fn_check_f(const __grid_constant__ QipCode src, uint32_t n_in, uint32_t n_out, unsigned long long *first) {
  qipb200::fn_check<true>(src, n_in, n_out, first);
}
#endif

extern "C" __global__ void __launch_bounds__(qipb200::kFnCheckThreads)
    qip_fn_tabulate(const __grid_constant__ QipCode src, uint64_t x0, uint64_t count, uint64_t *f_out,
                    double2 *cs_out) {
  qipb200::fn_tabulate(src, x0, count, f_out, cs_out);
}
)QIPSRC";

std::string code_program(uint32_t n_out, const char *source, bool theta) {
  // the library's unreferenced constants and helpers do not warn; the user's source does
  std::string s = "#pragma nv_diag_suppress 177\n";
  s += kFnDevText;
  s += "\n#pragma nv_diag_default 177\n#line 1 \"qip_function\"\n";
  s += source;
  s += "\n#line 1 \"qip_function_entries\"\n#define QIP_FN_THETA ";
  s += theta ? "1" : "0";
  s += "\n#define QIP_FN_NOUT " + std::to_string(n_out) + "\n";
  s += kFnCodeEntries;
  return s;
}

// Compile (or find in a cache) the program of a code function; need_driver: it is to be launched.
int compile_code(uint32_t n_out, const char *source, bool theta, bool need_driver,
                 std::shared_ptr<const JitCubin> *out, std::string *msg) {
  std::string why;
  if (!jit_available(&why) && (need_driver || why.find("driver") == std::string::npos)) {
    *msg = why;
    return QIPB200_ERR_UNSUPPORTED;
  }
  std::shared_ptr<const JitCubin> c = jit_request(code_program(n_out, source, theta), true);
  if (!c || !c->ok) {
    *msg = c && !c->log.empty() ? c->log : std::string("NVRTC produced no cubin");
    return QIPB200_ERR_INVALID_ARG;
  }
  *msg = c->log;  // warnings, if any
  *out = c;
  return QIPB200_OK;
}

}  // namespace

struct FnCode {
  CUmodule mod = nullptr;
  CUfunction tile[2] = {}, pair[2] = {}, expect[2] = {};  // [0]: f32, [1]: f64
  CUfunction check_f = nullptr, check_theta = nullptr, tabulate = nullptr;
  bool theta = false;
  uint32_t n_out = 0;
};

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
  FnPlan p;
  const FnArgs a = fn_args(prec, n, in_pos, n_in, out_pos, n_out, &p);
  FnTableSrc src;
  src.tf = n_out ? f : nullptr;
  src.tcs = cs;
  cudaError_t e;
  const bool th = cs != nullptr;
  if (p.path == 1) {
    if (prec == QIP_F32)
      e = th ? launch_pair<float, true>(psi, a, src, sm_count, s) : launch_pair<float, false>(psi, a, src, sm_count, s);
    else
      e = th ? launch_pair<double, true>(psi, a, src, sm_count, s)
             : launch_pair<double, false>(psi, a, src, sm_count, s);
  } else {
    if (prec == QIP_F32)
      e = th ? launch_tile<float, true>(psi, a, src, sm_count, s) : launch_tile<float, false>(psi, a, src, sm_count, s);
    else
      e = th ? launch_tile<double, true>(psi, a, src, sm_count, s)
             : launch_tile<double, false>(psi, a, src, sm_count, s);
  }
  ++*launches;
  return e;
}

int function_code_compile(uint32_t n_out, const char *source, bool theta, std::string *msg) {
  std::shared_ptr<const JitCubin> c;
  return compile_code(n_out, source, theta, false, &c, msg);
}

int function_code_load(uint32_t n_out, const char *source, bool theta, FnCode **out, std::string *msg) {
  std::shared_ptr<const JitCubin> cubin;
  int st = compile_code(n_out, source, theta, true, &cubin, msg);
  if (st != QIPB200_OK) return st;
  FnCode *c = new FnCode();
  c->theta = theta;
  c->n_out = n_out;
  cudaError_t e = jit_module_load(*cubin, &c->mod, msg);
  auto kernel = [&](const char *name, unsigned smem, CUfunction *fn) {
    if (e == cudaSuccess) e = jit_module_kernel(c->mod, name, smem, fn, msg);
  };
  kernel("qip_fn_tile_f32", (unsigned)tile_smem<float, uint64_t>(), &c->tile[0]);
  kernel("qip_fn_tile_f64", (unsigned)tile_smem<double, uint64_t>(), &c->tile[1]);
  kernel("qip_fn_pair_f32", 0, &c->pair[0]);
  kernel("qip_fn_pair_f64", 0, &c->pair[1]);
  kernel("qip_fn_tabulate", 0, &c->tabulate);
  if (theta) {
    kernel("qip_fn_expect_f32", 0, &c->expect[0]);
    kernel("qip_fn_expect_f64", 0, &c->expect[1]);
    kernel("qip_fn_check_theta", 0, &c->check_theta);
  }
  if (n_out) kernel("qip_fn_check_f", 0, &c->check_f);
  if (e != cudaSuccess) {
    function_code_free(c);
    return QIPB200_ERR_CUDA;
  }
  *out = c;
  return QIPB200_OK;
}

void function_code_free(FnCode *c) {
  if (!c) return;
  jit_module_unload(c->mod);
  delete c;
}

cudaError_t function_code_first_bad(const FnCode *c, bool range, uint32_t n_in, uint32_t n_out, const double *params,
                                    uint64_t *d_word, int sm_count, cudaStream_t s, uint64_t *first,
                                    std::string *err) {
  FnCodeArgs src;
  memset(&src, 0, sizeof(src));
  if (params) memcpy(src.p, params, sizeof(src.p));
  cudaError_t e = cudaMemsetAsync(d_word, 0xFF, sizeof(uint64_t), s);
  if (e != cudaSuccess) return e;
  void *args[] = {&src, &n_in, &n_out, &d_word};
  if ((e = jit_kernel_launch(range ? c->check_f : c->check_theta, check_grid(1ull << n_in, sm_count),
                             kFnCheckThreads, 0, s, args, err)) != cudaSuccess)
    return e;
  if ((e = cudaMemcpyAsync(first, d_word, sizeof(uint64_t), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
  return cudaStreamSynchronize(s);
}

cudaError_t run_function_code(qip_prec prec, void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                              const uint32_t *out_pos, uint32_t n_out, const FnCode *c, const double *params,
                              int sm_count, cudaStream_t s, uint64_t *launches, std::string *err) {
  FnPlan p;
  FnArgs a = fn_args(prec, n, in_pos, n_in, out_pos, n_out, &p);
  FnCodeArgs src;
  memcpy(src.p, params, sizeof(src.p));
  void *args[] = {&psi, &a, &src};
  const int k = prec == QIP_F64;
  cudaError_t e;
  if (p.path == 1) {
    e = jit_kernel_launch(c->pair[k], pair_grid(a, sm_count), kFnPairThreads, 0, s, args, err);
  } else {
    const unsigned threads = (1u << (k ? kFnTileF64 : kFnTileF32)) / kFnPer;
    const size_t smem = k ? tile_smem<double, uint64_t>() : tile_smem<float, uint64_t>();
    e = jit_kernel_launch(c->tile[k], tile_grid(a, sm_count), threads, (unsigned)smem, s, args, err);
  }
  ++*launches;
  return e;
}

cudaError_t expect_function_code(qip_prec prec, const void *psi, uint32_t n, const uint32_t *in_pos, uint32_t n_in,
                                 const FnCode *c, const double *params, double *d_partials, cudaStream_t s,
                                 uint64_t *launches, double *out, std::string *err) {
  FnArgs a = fn_args(prec, n, in_pos, n_in, nullptr, 0, nullptr);
  FnCodeArgs src;
  memcpy(src.p, params, sizeof(src.p));
  void *args[] = {&psi, &a, &src, &d_partials};
  cudaError_t e = jit_kernel_launch(c->expect[prec == QIP_F64], kFnExpGrid, kFnExpThreads, 0, s, args, err);
  ++*launches;
  if (e != cudaSuccess) return e;
  double part[kFnExpGrid];
  if ((e = cudaMemcpyAsync(part, d_partials, sizeof(part), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
  double sum = 0.0;
  for (int g = 0; g < kFnExpGrid; ++g) sum += part[g];  // CTA order
  *out = sum;
  return cudaSuccess;
}

cudaError_t tabulate_function(const FnCode *c, const double *params, const uint32_t *f, const double2 *cs,
                              uint64_t x0, uint64_t count, uint64_t *f_out, double *cs_out, int sm_count,
                              cudaStream_t s, std::string *err) {
  const uint64_t chunk = std::min<uint64_t>(count, 1ull << 20);
  if (!chunk) return cudaSuccess;
  uint64_t *d_f = nullptr;
  double2 *d_cs = nullptr;
  cudaError_t e = cudaSuccess;
  if (f_out) e = cudaMallocAsync((void **)&d_f, chunk * sizeof(uint64_t), s);
  if (e == cudaSuccess && cs_out) e = cudaMallocAsync((void **)&d_cs, chunk * sizeof(double2), s);
  FnTableSrc tsrc;
  tsrc.tf = f;
  tsrc.tcs = cs;
  FnCodeArgs csrc;
  memset(&csrc, 0, sizeof(csrc));
  if (params) memcpy(csrc.p, params, sizeof(csrc.p));
  for (uint64_t i = 0; i < count && e == cudaSuccess; i += chunk) {
    uint64_t m = std::min(chunk, count - i), x = x0 + i;
    const int grid = check_grid(m, sm_count);
    if (c) {
      void *args[] = {&csrc, &x, &m, &d_f, &d_cs};
      e = jit_kernel_launch(c->tabulate, grid, kFnCheckThreads, 0, s, args, err);
    } else {
      k_function_tabulate<<<grid, kFnCheckThreads, 0, s>>>(tsrc, x, m, d_f, d_cs);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess && f_out)
      e = cudaMemcpyAsync(f_out + i, d_f, m * sizeof(uint64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && cs_out)
      e = cudaMemcpyAsync(cs_out + 2 * i, d_cs, m * sizeof(double2), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  }
  if (d_f) cudaFreeAsync(d_f, s);
  if (d_cs) cudaFreeAsync(d_cs, s);
  const cudaError_t e2 = cudaStreamSynchronize(s);
  return e != cudaSuccess ? e : e2;
}

}  // namespace qipb200
