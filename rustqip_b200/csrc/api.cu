// api.cu -- the extern "C" boundary of libqipb200 (include/qipb200.h).
//
// Host runtime above the kernels: owns the device amplitude buffer and the gate
// schedule, exactly the role of the fold in LocalBuilder::calculate_state_with_init
// (qip/src/builder.rs:400-519).  No CPU fallback: every compute entry needs a
// context, and a context needs a CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <exception>
#include <memory>
#include <new>
#include <thread>
#include <string>
#include <vector>

#include "../../include/qipb200.h"
#include "channel.h"
#include "density.h"
#include "dist.cuh"
#include "expect.h"
#include "kernels.cuh"
#include "kraus.h"
#include "opcompile.h"
#include "evolve.h"
#include "lanczos.h"
#include "function.h"
#include "gradient.h"
#include "pauli_rot.h"
#include "purity.h"
#include "rdm.h"
#include "schedule.h"
#include "spectrum.h"
#include "tile.cuh"
#include "jit_codegen.h"
#include "state.h"

using namespace qipb200;

namespace {

thread_local std::string g_tls_err = "";

int set_err(const qipb200_ctx *ctx, int status, const std::string &msg) {
  if (ctx)
    const_cast<qipb200_ctx *>(ctx)->err = msg;
  else
    g_tls_err = msg;
  return status;
}

int cuda_fail(const qipb200_ctx *ctx, cudaError_t e, const char *what) {
  std::string m = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  cudaGetLastError();  // clear sticky-free errors
  return set_err(ctx, e == cudaErrorMemoryAllocation ? QIPB200_ERR_OOM : QIPB200_ERR_CUDA, m);
}

#define CU(ctx, call)                                          \
  do {                                                         \
    cudaError_t e__ = (call);                                  \
    if (e__ != cudaSuccess) return cuda_fail(ctx, e__, #call); \
  } while (0)

int grow(qipb200_ctx *ctx, void **p, size_t *have, size_t need) {
  if (*have >= need) return QIPB200_OK;
  if (*p) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(*p);
    *p = nullptr;
    *have = 0;
  }
  cudaError_t e = cudaMalloc(p, need);
  if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaMalloc(staging)");
  *have = need;
  return QIPB200_OK;
}

// No C++ exception may cross the C boundary (the library allocates through std::vector / std::string):
// an allocation failure becomes QIPB200_ERR_OOM, anything else QIPB200_ERR_INVALID_ARG with its message.
template <typename F>
int guarded(const qipb200_ctx *ctx, F f) {
  try {
    return f();
  } catch (const std::bad_alloc &) {
    return set_err(ctx, QIPB200_ERR_OOM, "out of host memory");
  } catch (const std::exception &e) {
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, std::string("internal error: ") + e.what());
  }
}

// Run f(shard, rank) on every shard of a multi-device state, one host thread per device (the shards are
// ordinary sharded states: their exchange kernels wait for each other on the GPUs, so they must be driven
// concurrently, exactly as the one-process-per-GPU model drives them).  First failing status wins.
template <typename F>
int each_shard(qipb200_state *p, F f) {
  const size_t G = p->shards.size();
  std::vector<int> st(G, QIPB200_OK);
  auto run = [&](size_t r) {
    try {
      st[r] = f(p->shards[r], (int)r);
    } catch (const std::bad_alloc &) {
      st[r] = set_err(p->shards[r]->ctx, QIPB200_ERR_OOM, "out of host memory");
    } catch (const std::exception &e) {
      st[r] = set_err(p->shards[r]->ctx, QIPB200_ERR_INVALID_ARG, std::string("internal error: ") + e.what());
    }
  };
  std::vector<std::thread> th;
  bool spawn_failed = false;
  try {
    th.reserve(G);
    for (size_t r = 1; r < G; ++r) th.emplace_back(run, r);
  } catch (const std::exception &) {  // no thread for some device: the started ones run into the flag barriers' timeout
    spawn_failed = true;
  }
  if (!spawn_failed) run(0);
  for (std::thread &t : th) t.join();
  if (spawn_failed) return set_err(p->ctx, QIPB200_ERR_OOM, "could not start one host thread per device");
  for (size_t r = 0; r < G; ++r)
    if (st[r] != QIPB200_OK) return set_err(p->ctx, st[r], p->shards[r]->ctx->err);
  return QIPB200_OK;
}

bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }
int ilog2(int x) {
  int l = 0;
  while ((1 << l) < x) ++l;
  return l;
}

}  // namespace

// ===================================================================================
// library / context
// ===================================================================================

extern "C" int qipb200_abi_version(void) { return 1000; }

static int init_device_ctx(qipb200_ctx **out, int device_id);

extern "C" int qipb200_init(qipb200_ctx **out, int device_id) {
  if (!out) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "qipb200_init: ctx out-pointer is NULL");
  *out = nullptr;
  return guarded(nullptr, [&]() { return init_device_ctx(out, device_id); });
}

extern "C" int qipb200_init_multi(qipb200_ctx **out, int n_devices, const int *device_ids) {
  if (!out) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "qipb200_init_multi: ctx out-pointer is NULL");
  *out = nullptr;
  if (!is_pow2(n_devices) || n_devices > kMaxWorld)
    return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "qipb200_init_multi: n_devices must be a power of two <= 16");
  return guarded(nullptr, [&]() {
    qipb200_ctx *parent = new qipb200_ctx();
    for (int i = 0; i < n_devices; ++i) {
      const int dev = device_ids ? device_ids[i] : i;
      for (int j = 0; j < i; ++j)
        if (parent->children[j]->device == dev) {
          qipb200_shutdown(parent);
          return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "qipb200_init_multi: a device is listed twice");
        }
      qipb200_ctx *c = nullptr;
      int st = init_device_ctx(&c, dev);
      if (st != QIPB200_OK) {
        qipb200_shutdown(parent);
        return st;  // message already in the thread-local slot
      }
      c->parent = parent;
      parent->children.push_back(c);
    }
    // every device maps every other one (NVLink / NVSwitch peer access: the exchange kernels load and store
    // the partner's shard directly)
    for (int i = 0; i < n_devices; ++i) {
      cudaSetDevice(parent->children[i]->device);
      for (int j = 0; j < n_devices; ++j) {
        if (i == j) continue;
        int can = 0;
        cudaDeviceCanAccessPeer(&can, parent->children[i]->device, parent->children[j]->device);
        cudaError_t e = can ? cudaDeviceEnablePeerAccess(parent->children[j]->device, 0) : cudaErrorPeerAccessUnsupported;
        if (e == cudaErrorPeerAccessAlreadyEnabled) {
          cudaGetLastError();
          e = cudaSuccess;
        }
        if (e != cudaSuccess) {
          int st = cuda_fail(nullptr, e, "cudaDeviceEnablePeerAccess");
          qipb200_shutdown(parent);
          return st == QIPB200_ERR_CUDA ? QIPB200_ERR_COMM : st;
        }
      }
    }
    parent->device = parent->children[0]->device;
    parent->sm_count = parent->children[0]->sm_count;
    *out = parent;
    return (int)QIPB200_OK;
  });
}

static int init_device_ctx(qipb200_ctx **out, int device_id) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    cudaGetLastError();
    return set_err(nullptr, QIPB200_ERR_CUDA,
                   std::string("qipb200_init: no CUDA device (") + cudaGetErrorString(e) +
                       "); libqipb200 has no CPU path");
  }
  if (device_id < 0 || device_id >= count)
    return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "qipb200_init: device_id out of range");
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device_id);
  if (e != cudaSuccess) return cuda_fail(nullptr, e, "cudaGetDeviceProperties");
  if (prop.major != 9 || prop.minor != 0)
    return set_err(nullptr, QIPB200_ERR_CUDA,
                   std::string("qipb200_init: device '") + prop.name +
                       "' is not sm_90 (Hopper H100); this library ships sm_90a code only");
  e = cudaSetDevice(device_id);
  if (e != cudaSuccess) return cuda_fail(nullptr, e, "cudaSetDevice");
  qipb200_ctx *ctx = new (std::nothrow) qipb200_ctx();
  if (!ctx) return set_err(nullptr, QIPB200_ERR_OOM, "qipb200_init: out of host memory");
  ctx->device = device_id;
  ctx->sm_count = prop.multiProcessorCount;
  e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc((void **)&ctx->d_scalar, 64);
  if (e != cudaSuccess) {
    int st = cuda_fail(nullptr, e, "qipb200_init");
    delete ctx;
    return st;
  }
  *out = ctx;
  return QIPB200_OK;
}

extern "C" void qipb200_shutdown(qipb200_ctx *ctx) {
  if (!ctx) return;
  if (!ctx->children.empty() || (!ctx->stream && !ctx->d_scalar)) {  // multi-device parent: owns its children
    for (size_t i = 0; i < ctx->children.size(); ++i) qipb200_shutdown(ctx->children[i]);
    delete ctx;
    return;
  }
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->d_in) cudaFree(ctx->d_in);
  if (ctx->d_out) cudaFree(ctx->d_out);
  if (ctx->d_scalar) cudaFree(ctx->d_scalar);
  if (ctx->pool_buf) cudaFree(ctx->pool_buf);
  if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
  for (int cat = 0; cat < 2; ++cat)
    for (size_t i = 0; i < ctx->prof_events[cat].size(); ++i) {
      cudaEventDestroy(ctx->prof_events[cat][i].first);
      cudaEventDestroy(ctx->prof_events[cat][i].second);
    }
  for (size_t i = 0; i < ctx->prof_pool.size(); ++i) cudaEventDestroy(ctx->prof_pool[i]);
  jit_unload(&ctx->jit_loaded);
  eig_handle_destroy(ctx->eig_solver);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

extern "C" const char *qipb200_last_error(const qipb200_ctx *ctx) {
  return ctx ? ctx->err.c_str() : g_tls_err.c_str();
}

extern "C" int qipb200_stream_handle(const qipb200_ctx *ctx, void **stream) {
  if (!ctx || !stream) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "stream_handle: NULL argument");
  *stream = (void *)(ctx->children.empty() ? ctx->stream : ctx->children[0]->stream);
  return QIPB200_OK;
}

extern "C" uint64_t qipb200_kernel_launches(const qipb200_ctx *ctx) {
  if (!ctx) return 0;
  uint64_t n = ctx->launches;
  for (size_t i = 0; i < ctx->children.size(); ++i) n += ctx->children[i]->launches;
  return n;
}

extern "C" int qipb200_launch_stats(const qipb200_ctx *ctx, uint64_t *out4) {
  if (!ctx || !out4) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "launch_stats: NULL argument");
  out4[0] = ctx->launches;
  out4[1] = ctx->tile_launches;
  out4[2] = ctx->exchange_launches;
  out4[3] = ctx->fused_gates;
  for (size_t i = 0; i < ctx->children.size(); ++i) {  // multi-device context: summed over the devices
    const qipb200_ctx *c = ctx->children[i];
    out4[0] += c->launches;
    out4[1] += c->tile_launches;
    out4[2] += c->exchange_launches;
    out4[3] += i == 0 ? c->fused_gates : 0;  // every device folds the same gates: count them once
  }
  return QIPB200_OK;
}

extern "C" int qipb200_kernel_counts(const qipb200_ctx *ctx, uint64_t *out, size_t n) {
  if (!ctx || (!out && n)) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "kernel_counts: NULL argument");
  for (size_t k = 0; k < n && k < (size_t)QIPB200_KC_COUNT; ++k) {
    out[k] = ctx->kernel_counts[k];
    for (size_t i = 0; i < ctx->children.size(); ++i) out[k] += ctx->children[i]->kernel_counts[k];
  }
  return QIPB200_OK;
}

extern "C" int qipb200_release_pool(qipb200_ctx *ctx) {
  if (!ctx) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "release_pool: NULL context");
  for (size_t i = 0; i < ctx->children.size(); ++i) qipb200_release_pool(ctx->children[i]);
  if (ctx->pool_buf) {
    CU(ctx, cudaSetDevice(ctx->device));
    CU(ctx, cudaFree(ctx->pool_buf));
    ctx->pool_buf = nullptr;
    ctx->pool_bytes = 0;
  }
  return QIPB200_OK;
}

// Host-only (no GPU, no context): plan `ops` for an n-qubit single-device state (sharded states plan with their own
// geometry, f64 L = 5 instead of 4, so their passes are not among these programs), generate the specialised source
// of every fused pass and compile it with NVRTC for sm_90a.  out[0] = passes planned, out[1] = passes the
// generator covered, out[2] = of those compiled without error, out[3] = total NVRTC wall time (ms, all passes in
// parallel on the worker pool), out[4] = sum of the per-program compile times (ms).
extern "C" int qipb200_jit_precompile(qip_prec prec, uint32_t n_qubits, const qip_op *ops, size_t n_ops, double *out5,
                                      char *log, size_t log_len) {
  if (!out5 || (!ops && n_ops)) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "jit_precompile: NULL argument");
  for (int i = 0; i < 5; ++i) out5[i] = 0.0;
  if (log && log_len) log[0] = 0;
  std::string why;
  if (!jit_available(&why) && why.find("driver") == std::string::npos) {  // the driver is only needed to LAUNCH
    if (log && log_len) snprintf(log, log_len, "%s", why.c_str());
    return set_err(nullptr, QIPB200_ERR_UNSUPPORTED, why);
  }
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], prec, n_qubits, &flat[i], &err);
    if (st != QIPB200_OK) return set_err(nullptr, st, err);
  }
  const PlanConfig cfg = default_plan_config(prec, n_qubits);
  std::vector<PlanStep> steps;
  plan_passes(flat, n_qubits, prec, cfg, &steps);
  std::vector<std::string> sources;
  for (size_t i = 0; i < steps.size(); ++i) {
    if (!steps[i].is_pass) continue;
    out5[0] += 1;
    JitProgram prog;
    if (!jit_generate(steps[i].pass, prec, &prog, &why)) {
      if (log && log_len) snprintf(log, log_len, "declined: %s", why.c_str());
      continue;
    }
    out5[1] += 1;
    sources.push_back(prog.source);
  }
  const auto t0 = std::chrono::steady_clock::now();
  for (size_t i = 0; i < sources.size(); ++i) (void)jit_request(sources[i], false);
  for (size_t i = 0; i < sources.size(); ++i) {
    std::shared_ptr<const JitCubin> c = jit_request(sources[i], true);
    if (c && c->ok) {
      out5[2] += 1;
      out5[4] += c->compile_ms;
    } else if (log && log_len && c) {
      snprintf(log, log_len, "%s", c->log.c_str());
    }
  }
  out5[3] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (getenv("QIPB200_JIT_CACHE_DIR") && log && log_len && !log[0]) {
    uint64_t n_disk = 0;
    jit_wait_all(nullptr, nullptr, &n_disk);
    snprintf(log, log_len, "disk cache: %llu programs loaded from QIPB200_JIT_CACHE_DIR so far in this process", (unsigned long long)n_disk);
  }
  return QIPB200_OK;
}

extern "C" int qipb200_jit_stats(qipb200_ctx *ctx, int wait, double *out4, char *note, size_t note_len) {
  if (!ctx || !out4) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "jit_stats: NULL argument");
  uint64_t n = 0;
  double ms = 0.0;
  if (wait) jit_wait_all(&n, &ms);
  out4[0] = (double)ctx->jit_launches;
  out4[1] = (double)ctx->tile_launches;
  for (size_t i = 0; i < ctx->children.size(); ++i) {
    out4[0] += (double)ctx->children[i]->jit_launches;
    out4[1] += (double)ctx->children[i]->tile_launches;
    if (!ctx->children[i]->jit_note.empty()) ctx->jit_note = ctx->children[i]->jit_note;
  }
  out4[2] = (double)n;
  out4[3] = ms;
  if (note && note_len) snprintf(note, note_len, "%s", ctx->jit_note.c_str());
  return QIPB200_OK;
}

extern "C" int qipb200_profile_enable(qipb200_ctx *ctx, int on) {
  if (!ctx) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "profile_enable: ctx is NULL");
  ctx->profile = on != 0;
  for (size_t i = 0; i < ctx->children.size(); ++i) ctx->children[i]->profile = on != 0;
  return QIPB200_OK;
}

extern "C" int qipb200_profile_read(qipb200_ctx *ctx, double *out4) {
  if (!ctx || !out4) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "profile_read: NULL argument");
  if (!ctx->children.empty()) {  // multi-device context: the first device's timings (all devices run the same steps)
    for (size_t i = 1; i < ctx->children.size(); ++i) {
      double drop[4];
      qipb200_profile_read(ctx->children[i], drop);
    }
    return qipb200_profile_read(ctx->children[0], out4);
  }
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  for (int cat = 0; cat < 2; ++cat) {
    double ms = 0.0;
    for (size_t i = 0; i < ctx->prof_events[cat].size(); ++i) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, ctx->prof_events[cat][i].first, ctx->prof_events[cat][i].second) == cudaSuccess) ms += t;
      ctx->prof_pool.push_back(ctx->prof_events[cat][i].first);
      ctx->prof_pool.push_back(ctx->prof_events[cat][i].second);
    }
    out4[2 * cat] = ms;
    out4[2 * cat + 1] = (double)ctx->prof_events[cat].size();
    ctx->prof_events[cat].clear();
  }
  return QIPB200_OK;
}

extern "C" int qipb200_validate_op(const qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, const qip_op *op) {
  return guarded(ctx, [&]() -> int {
    std::string err;
    int st = validate_op(op, prec, n_qubits, &err);
    if (st != QIPB200_OK) return set_err(ctx, st, err);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// stateless drop-ins (host buffers)
// ===================================================================================

namespace {

int host_apply(qipb200_ctx *ctx, qip_prec prec, uint32_t n, const qip_op *op, const void *input,
               uint64_t input_len, void *output, uint64_t output_len, uint64_t input_offset,
               uint64_t output_offset, bool accumulate) {
  if (!ctx) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "ctx is NULL (call qipb200_init first; there is no CPU path)");
  if (!ctx->children.empty()) {  // a multi-device context serves the host-buffer drop-ins on its first device
    qipb200_ctx *parent = ctx;
    int st = host_apply(parent->children[0], prec, n, op, input, input_len, output, output_len, input_offset, output_offset, accumulate);
    if (st != QIPB200_OK) parent->err = parent->children[0]->err;
    return st;
  }
  if ((!input && input_len) || (!output && output_len))
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, "apply_op: NULL amplitude buffer");
  if (n > 40 || input_len > (1ull << 40) || output_len > (1ull << 40))  // keeps len * amp_bytes far from wrapping
    return set_err(ctx, QIPB200_ERR_SIZE_MISMATCH, "apply_op: buffer length out of range");
  FlatOp f;
  std::string err;
  int st = compile_op(op, prec, n, &f, &err);
  if (st != QIPB200_OK) return set_err(ctx, st, err);
  CU(ctx, cudaSetDevice(ctx->device));
  const size_t ab = amp_bytes(prec);
  if ((st = grow(ctx, &ctx->d_in, &ctx->d_in_bytes, std::max<size_t>(input_len * ab, 16))) != QIPB200_OK) return st;
  if ((st = grow(ctx, &ctx->d_out, &ctx->d_out_bytes, std::max<size_t>(output_len * ab, 16))) != QIPB200_OK) return st;
  if (input_len) CU(ctx, cudaMemcpyAsync(ctx->d_in, input, input_len * ab, cudaMemcpyHostToDevice, ctx->stream));
  if (accumulate && output_len)
    CU(ctx, cudaMemcpyAsync(ctx->d_out, output, output_len * ab, cudaMemcpyHostToDevice, ctx->stream));
  CU(ctx, launch_gather(prec, f, n, ctx->d_in, input_len, input_offset, ctx->d_out, output_len, output_offset,
                        accumulate, ctx->stream, &ctx->launches));
  if (output_len) CU(ctx, cudaMemcpyAsync(output, ctx->d_out, output_len * ab, cudaMemcpyDeviceToHost, ctx->stream));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_apply_op(qipb200_ctx *ctx, qip_prec prec, uint32_t n, const qip_op *op, const void *input,
                                uint64_t input_len, void *output, uint64_t output_len, uint64_t input_offset,
                                uint64_t output_offset) {
  return guarded(ctx, [&]() { return host_apply(ctx, prec, n, op, input, input_len, output, output_len, input_offset, output_offset, true); });
}

extern "C" int qipb200_apply_op_overwrite(qipb200_ctx *ctx, qip_prec prec, uint32_t n, const qip_op *op,
                                          const void *input, uint64_t input_len, void *output,
                                          uint64_t output_len, uint64_t input_offset, uint64_t output_offset) {
  return guarded(ctx, [&]() { return host_apply(ctx, prec, n, op, input, input_len, output, output_len, input_offset, output_offset, false); });
}

// ===================================================================================
// device-resident state
// ===================================================================================

namespace {

int state_alloc(qipb200_ctx *ctx, qip_prec prec, uint32_t n, int rank, int world, qipb200_state **out) {
  if (!ctx) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "ctx is NULL (call qipb200_init first; there is no CPU path)");
  if (!out) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "state out-pointer is NULL");
  *out = nullptr;
  if (prec != QIP_F32 && prec != QIP_F64) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "precision must be QIP_F32 or QIP_F64");
  if (!is_pow2(world) || world > kMaxWorld || rank < 0 || rank >= world)
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, "world_size must be a power of two <= 16 and 0 <= rank < world_size");
  const int g = ilog2(world);
  if (n == 0 || n > 40 || (int)n - g < 2 * (world > 1))
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, "n_qubits out of range for this world size");
  CU(ctx, cudaSetDevice(ctx->device));
  qipb200_state *s = new (std::nothrow) qipb200_state();
  if (!s) return set_err(ctx, QIPB200_ERR_OOM, "out of host memory");
  s->ctx = ctx;
  s->prec = prec;
  s->n = n;
  s->n_local = n - g;
  s->rank = rank;
  s->world = world;
  s->bytes = amp_bytes(prec) << s->n_local;
  s->phys_of_logical.resize(n);
  for (uint32_t b = 0; b < n; ++b) s->phys_of_logical[b] = b;
  cudaError_t e = cudaSuccess;
  if (world == 1 && ctx->pool_buf && ctx->pool_bytes == s->bytes) {  // the buffer a freed state of this size left behind
    s->buf = ctx->pool_buf;
    ctx->pool_buf = nullptr;
    ctx->pool_bytes = 0;
  } else {
    e = cudaMalloc(&s->buf, s->bytes);
  }
  if (e == cudaSuccess) e = cudaMemsetAsync(s->buf, 0, s->bytes, ctx->stream);
  if (e == cudaSuccess && world > 1) {
    e = cudaMalloc((void **)&s->flags, kFlagAllocBytes);  // flag page + reduction slot (dist.cuh)
    if (e == cudaSuccess) e = cudaMemsetAsync(s->flags, 0, kFlagAllocBytes, ctx->stream);
  }
  if (e != cudaSuccess) {
    int st = cuda_fail(ctx, e, "qipb200_state_new");
    if (s->buf) cudaFree(s->buf);
    if (s->flags) cudaFree(s->flags);
    delete s;
    return st;
  }
  *out = s;
  return QIPB200_OK;
}

bool layout_is_identity(const qipb200_state *s) {
  for (uint32_t b = 0; b < s->n; ++b)
    if (s->phys_of_logical[b] != b) return false;
  return true;
}

// P::one() / measured_prob.sqrt() evaluated in the state's precision (measurement_ops.rs:231)
double collapse_multiplier(qip_prec prec, double measured_prob) {
  if (prec == QIP_F32) return (double)(1.0f / sqrtf((float)measured_prob));
  return 1.0 / sqrt(measured_prob);
}

// The index bit of s that holds each of k qubits under the current layout: qubit q is logical bit n - 1 - q.
void phys_positions(const qipb200_state *s, const uint64_t *qubits, uint32_t k, uint32_t *pos) {
  for (uint32_t i = 0; i < k; ++i) pos[i] = s->phys_of_logical[s->n - 1 - (uint32_t)qubits[i]];
}

// measure_state with a known multiplier over this rank's amplitudes, under the current layout.
int launch_collapse_on(qipb200_state *s, const uint64_t *qubits, uint32_t n_qubits, uint64_t measured, double p_mult) {
  qipb200_ctx *ctx = s->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  uint32_t pos[64];  // distinct qubits of at most 40
  phys_positions(s, qubits, n_qubits, pos);
  uint64_t row_mask = 0, measured_mask = 0;
  for (uint32_t i = 0; i < n_qubits; ++i) {
    row_mask |= 1ull << pos[i];
    measured_mask |= ((measured >> i) & 1ull) << pos[i];
  }
  CU(ctx, launch_collapse(s->prec, s->buf, 1ull << s->n_local, (uint64_t)s->rank << s->n_local, row_mask,
                          measured_mask, p_mult, ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

// Apply the collapse qipb200_state_measure left pending, before anything reads or writes the amplitudes.
int materialise_collapse(qipb200_state *s) {
  if (!s->collapse_pending) return QIPB200_OK;
  s->collapse_pending = false;
  return launch_collapse_on(s, s->pend_qubits.data(), (uint32_t)s->pend_qubits.size(), s->pend_measured,
                            s->pend_p_mult);
}

}  // namespace
namespace qipb200 {

// Write the basis state qipb200_state_set_basis left pending: one write sweep, memsets only.  No kernel is launched,
// so the call that triggers it launches exactly the kernels it launches on a state set_basis wrote at once.
int materialise_init(qipb200_state *s) {
  if (!s->init_pending) return QIPB200_OK;
  qipb200_ctx *ctx = s->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, write_basis_state(s->prec, s->buf, 1ull << s->n_local, s->init_index, ctx->stream));
  s->init_pending = false;
  return QIPB200_OK;
}

}  // namespace qipb200
namespace {

// Whatever qipb200_state_set_basis or qipb200_state_measure left pending, applied to the amplitudes.
int materialise_pending(qipb200_state *s) {
  int st = qipb200::materialise_init(s);
  return st != QIPB200_OK ? st : materialise_collapse(s);
}

// s's device made current and its pending work applied: the start of every call that reads s.
int begin_device_work(qipb200_state *s) {
  CU(s->ctx, cudaSetDevice(s->ctx->device));
  return materialise_pending(s);
}

int check_barrier_error(qipb200_state *s) {
  uint32_t flag = 0;
  CU(s->ctx, cudaMemcpyAsync(&flag, s->flags + kFlagErrorSlot, sizeof(flag), cudaMemcpyDeviceToHost, s->ctx->stream));
  CU(s->ctx, cudaStreamSynchronize(s->ctx->stream));
  if (flag) return set_err(s->ctx, QIPB200_ERR_COMM, "multi-GPU flag barrier timed out (a peer rank is not participating)");
  return QIPB200_OK;
}

// After a migration of physical rank bit R and local bit l: count the bytes this rank sent and let the logical bits
// living at R and l trade places in the map.
void record_migration(qipb200_state *s, uint32_t R, uint32_t l) {
  s->exchange_bytes += (uint64_t)amp_bytes(s->prec) << (s->n_local - 1);
  for (uint32_t b = 0; b < s->n; ++b) {
    if (s->phys_of_logical[b] == R)
      s->phys_of_logical[b] = l;
    else if (s->phys_of_logical[b] == l)
      s->phys_of_logical[b] = R;
  }
}

// Swap physical rank bit R (>= n_local) with local bit l: the in-place pair exchange (dist.cu: k_pair_exchange)
// between two flag barriers.
int exchange_bits(qipb200_state *s, uint32_t R, uint32_t l) {
  qipb200_ctx *ctx = s->ctx;
  if (!s->ipc_ready)
    return set_err(ctx, QIPB200_ERR_COMM, "sharded state: peers not mapped (call qipb200_state_ipc_import)");
  const uint32_t r = R - s->n_local;
  const int partner = s->rank ^ (1 << r);
  const int rb = (s->rank >> r) & 1;
  {
    ProfileScope prof(ctx, 1);
    uint32_t s_bit = s->n_local - 1;
    if (s_bit == l) s_bit = s->n_local - 2;
    CU(ctx, launch_flag_barrier(s->peer_flags.data(), s->flags, s->rank, s->world, ++s->epoch,
                                s->flags + kFlagErrorSlot, ctx->stream, &ctx->launches));
    CU(ctx, launch_pair_exchange(s->prec, s->buf, s->peer_buf[partner], s->n_local, l, s_bit, rb, ctx->stream,
                                 &ctx->launches));
    CU(ctx, launch_flag_barrier(s->peer_flags.data(), s->flags, s->rank, s->world, ++s->epoch,
                                s->flags + kFlagErrorSlot, ctx->stream, &ctx->launches));
    ++ctx->exchange_launches;
  }
  record_migration(s, R, l);
  return QIPB200_OK;
}

// Swap two physical bits (any kind) so that the layout can be restored.
int swap_physical_bits(qipb200_state *s, uint32_t p, uint32_t q) {
  qipb200_ctx *ctx = s->ctx;
  if (p == q) return QIPB200_OK;
  if (p < q) std::swap(p, q);  // p > q
  const uint32_t nl = s->n_local;
  if (p < nl) {
    CU(ctx, launch_bitswap(s->prec, s->buf, nl, 0, q, p, ctx->stream, &ctx->launches));
    for (uint32_t b = 0; b < s->n; ++b) {
      if (s->phys_of_logical[b] == p)
        s->phys_of_logical[b] = q;
      else if (s->phys_of_logical[b] == q)
        s->phys_of_logical[b] = p;
    }
    return QIPB200_OK;
  }
  if (q < nl) return exchange_bits(s, p, q);
  // both rank bits: route through a local bit
  const uint32_t l = nl - 1;
  int st;
  if ((st = exchange_bits(s, p, l)) != QIPB200_OK) return st;
  if ((st = exchange_bits(s, q, l)) != QIPB200_OK) return st;
  return exchange_bits(s, p, l);
}

int restore_layout(qipb200_state *s) {
  // an unsharded state whose qubits were rotated through the low positions (schedule.cu: run_rotating): many displaced
  // bits -- swap-only tile passes instead of one half-sweep per transposition
  if (s->world == 1 && s->n_local >= 6 && rotate_enabled()) return restore_layout_planned(s);
  for (int p = (int)s->n - 1; p >= 0; --p) {
    const uint32_t where = s->phys_of_logical[p];
    if (where == (uint32_t)p) continue;
    int st = swap_physical_bits(s, (uint32_t)p, where);
    if (st != QIPB200_OK) return st;
  }
  return QIPB200_OK;
}

}  // namespace

namespace qipb200 {

// Non-diagonal target bits of a compiled op (the ones that must be local).
static void nondiag_bits(const FlatOp &f, std::vector<uint32_t> *out) {
  out->clear();
  switch (f.cls) {
    case CLASS_DENSE:
    case CLASS_FLIP:
      *out = f.tgt_sorted;
      break;
    case CLASS_BITSWAP:
      for (size_t i = 0; i < f.swaps.size(); ++i) {
        out->push_back(f.swaps[i].first);
        out->push_back(f.swaps[i].second);
      }
      break;
    case CLASS_GENERAL:
      for (uint32_t j = f.nc; j < f.k; ++j) out->push_back(f.idx_bits[j]);
      break;
    default:
      break;
  }
}

// Restrict a compiled op (physical bits, non-diagonal targets all local) to this rank:
// controls held by the rank index either vanish or switch the op off; diagonal bits held
// by the rank index select a slice of the diagonal.  No communication.  *skip = true when
// the op is the identity on this rank.
int restrict_to_rank(const qipb200_state *s, const FlatOp &f_in, FlatOp *out, bool *skip) {
  return restrict_to_rank_as(s, s->rank, f_in, out, skip);
}

// ... as rank `rank` of this state's world would see the op (rank == world - 1: every rank-held bit is 1)
int restrict_to_rank_as(const qipb200_state *s, int rank, const FlatOp &f_in, FlatOp *out, bool *skip) {
  restrict_flat_op(f_in, s->n_local, rank, out, skip);  // opcompile.cpp
  return QIPB200_OK;
}

// Launch the per-gate kernel of an op whose bits are all local (after restrict_to_rank).
int launch_local_op(qipb200_state *s, const FlatOp &f) {
  qipb200_ctx *ctx = s->ctx;
  const uint32_t nl = s->n_local;
  const uint64_t cm = f.ctrl_mask;
  switch (f.cls) {
    case CLASS_IDENTITY:
      return QIPB200_OK;
    case CLASS_DIAGONAL:
      if (__builtin_popcountll(cm) > kMaxIns) break;
      if (f.diag_bits.size() <= (size_t)kMaxDiagParamK) {
        CU(ctx, launch_diag(s->prec, s->buf, nl, cm, f.diag_bits, f.diag, ctx->stream, &ctx->launches));
        ++ctx->kernel_counts[QIPB200_KC_DIAG];
        return QIPB200_OK;
      }
      if (f.diag_bits.size() <= 10) {
        CU(ctx, launch_diag_wide(s->prec, s->buf, nl, cm, f.diag_bits, f.diag, ctx->stream, &ctx->launches));
        ++ctx->kernel_counts[QIPB200_KC_DIAG_WIDE];
        return QIPB200_OK;
      }
      break;
    case CLASS_FLIP:
      CU(ctx, launch_flip(s->prec, s->buf, nl, cm, f.tgt_sorted[0], ctx->stream, &ctx->launches));
      ++ctx->kernel_counts[QIPB200_KC_EXCHANGE];
      return QIPB200_OK;
    case CLASS_BITSWAP:
      for (size_t i = 0; i < f.swaps.size(); ++i) {
        CU(ctx, launch_bitswap(s->prec, s->buf, nl, cm, f.swaps[i].first, f.swaps[i].second, ctx->stream,
                               &ctx->launches));
        ++ctx->kernel_counts[QIPB200_KC_EXCHANGE];
      }
      return QIPB200_OK;
    case CLASS_DENSE:
      if (f.tgt_sorted.size() <= (size_t)kMaxRegK &&
          __builtin_popcountll(cm) + f.tgt_sorted.size() <= (size_t)kMaxIns) {
        CU(ctx, launch_dense(s->prec, s->buf, nl, f, ctx->stream, &ctx->launches));
        ++ctx->kernel_counts[QIPB200_KC_DENSE];
        return QIPB200_OK;
      }
      // k = 5..10 in place (the reference applies any k through the same row loop, qubit_iterators.rs:23-55)
      if (f.tgt_sorted.size() >= 5 && f.tgt_sorted.size() <= 10 &&
          __builtin_popcountll(cm) + f.tgt_sorted.size() <= (size_t)kMaxIns && nl >= f.tgt_sorted.size() + __builtin_popcountll(cm) &&
          (f.tgt_sorted.size() == 5 || nl - (uint32_t)__builtin_popcountll(cm) >= 8)) {
        CU(ctx, launch_dense_wide(s->prec, s->buf, nl, f, ctx->stream, &ctx->launches));
        const DenseWideKind kind = dense_wide_kind(s->prec, nl, f);
        ++ctx->kernel_counts[kind == DENSE_WIDE_DMMA ? QIPB200_KC_DENSE_DMMA
                             : kind == DENSE_WIDE_5  ? QIPB200_KC_DENSE5
                                                     : QIPB200_KC_DENSE_BIG];
        return QIPB200_OK;
      }
      break;
    default:
      break;
  }
  // Fallback: out-of-place row kernel with the reference's gather semantics.
  if (s->world > 1)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED,
                   "this op needs the out-of-place row kernel, which is not available on a sharded state");
  if (!s->scratch) {
    cudaError_t e = cudaMalloc(&s->scratch, s->bytes);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaMalloc(scratch arena)");
  }
  const uint64_t len = 1ull << nl;
  CU(ctx, launch_gather(s->prec, f, s->n, s->buf, len, 0, s->scratch, len, 0, false, ctx->stream, &ctx->launches));
  ++ctx->kernel_counts[QIPB200_KC_GATHER];
  std::swap(s->buf, s->scratch);  // `Ok((arena, state, ..))`, builder.rs:514
  return QIPB200_OK;
}

int apply_flat_local(qipb200_state *s, const FlatOp &f_in) {
  FlatOp f;
  bool skip = false;
  int st = restrict_to_rank(s, f_in, &f, &skip);
  if (st != QIPB200_OK || skip) return st;
  return launch_local_op(s, f);
}

int report_error(qipb200_state *s, int status, const std::string &msg) { return set_err(s->ctx, status, msg); }
int report_cuda_error(qipb200_state *s, cudaError_t e, const char *what) { return cuda_fail(s->ctx, e, what); }

// The local bit a migration evicts: not used by this op, next non-diagonal use furthest away.
static int choose_victim(const qipb200_state *s, const FlatOp &f, const uint64_t *next_use) {
  uint64_t used = f.ctrl_mask;
  for (uint32_t j = 0; j < f.k; ++j) used |= 1ull << f.idx_bits[j];
  int best = -1;
  uint64_t best_key = 0;
  for (uint32_t l = 0; l < s->n_local; ++l) {
    if ((used >> l) & 1ull) continue;
    uint64_t key = 1;
    if (next_use) {
      uint32_t logical = 0;
      for (uint32_t b = 0; b < s->n; ++b)
        if (s->phys_of_logical[b] == l) logical = b;
      key = next_use[logical] + 1;
    }
    // prefer high bits on ties: low bits give the exchange its coalescing
    if (best < 0 || key > best_key || (key == best_key && l > (uint32_t)best)) {
      best = (int)l;
      best_key = key;
    }
  }
  return best;
}

// The first exchange compile_and_localize(op) would perform under the current layout (none: returns false).
bool peek_first_exchange(const qipb200_state *s, const qip_op *op, const uint64_t *next_use, uint32_t *R, uint32_t *l) {
  if (s->world == 1) return false;
  FlatOp f;
  std::string err;
  if (compile_op(op, s->prec, s->n, &f, &err, s->phys_of_logical.data()) != QIPB200_OK) return false;
  if (f.cls == CLASS_BITSWAP && f.ctrl_mask == 0) return false;  // a relabelling: nothing moves
  std::vector<uint32_t> nd;
  nondiag_bits(f, &nd);
  for (size_t i = 0; i < nd.size(); ++i) {
    if (nd[i] < s->n_local) continue;
    const int v = choose_victim(s, f, next_use);
    if (v < 0) return false;
    *R = nd[i];
    *l = (uint32_t)v;
    return true;
  }
  return false;
}

// ---- migration fused into a tile pass, in place (paired send) ----
void paired_partner(const qipb200_state *s, uint32_t R, int *partner, int *give) {
  const uint32_t r = R - s->n_local;
  *partner = s->rank ^ (1 << r);
  *give = 1 - ((s->rank >> r) & 1);
}

// The rank's part of the per-tile protocol by a stand-alone kernel (its last pass ran without the send).
int paired_send_standin(qipb200_state *s, uint32_t R, uint32_t l, uint32_t cbit, uint32_t seq, const PassHeader &hdr) {
  qipb200_ctx *ctx = s->ctx;
  int partner = 0, give = 0;
  paired_partner(s, R, &partner, &give);
  PairedSendArgs a;
  memset(&a, 0, sizeof(a));
  a.mine = s->buf;
  a.peer = s->peer_buf[partner];
  a.my_flags = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(s->flags) + kPairFlagOffsetBytes);
  a.peer_flags = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(s->peer_flags[partner]) + kPairFlagOffsetBytes);
  a.error_word = s->flags + kFlagErrorSlot;
  a.seq = seq;
  a.n_local = s->n_local;
  a.T = hdr.T;
  a.L = hdr.L;
  a.m = hdr.m;
  a.l = l;
  a.cbit = cbit;
  a.give = (uint32_t)give;
  for (uint32_t i = 0; i < 8; ++i) a.hi_pos[i] = hdr.hi_pos[i];
  ProfileScope prof(ctx, 1);
  CU(ctx, launch_paired_send(s->prec, a, ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

int finish_paired_exchange(qipb200_state *s, uint32_t R, uint32_t l) {
  qipb200_ctx *ctx = s->ctx;
  {
    ProfileScope prof(ctx, 1);
    CU(ctx, launch_flag_barrier(s->peer_flags.data(), s->flags, s->rank, s->world, ++s->epoch, s->flags + kFlagErrorSlot,
                                ctx->stream, &ctx->launches));
  }
  ++ctx->exchange_launches;
  record_migration(s, R, l);
  return QIPB200_OK;
}

// Compile `op` against the current layout and migrate rank-held target bits to
// local bits if needed.  `next_use` (optional, n entries indexed by logical bit):
// position in the schedule of the next non-diagonal use, used to pick the victim.
int compile_and_localize(qipb200_state *s, const qip_op *op, FlatOp *f, const uint64_t *next_use) {
  qipb200_ctx *ctx = s->ctx;
  std::string err;
  int st = compile_op(op, s->prec, s->n, f, &err, s->phys_of_logical.data());
  if (st != QIPB200_OK) return set_err(ctx, st, err);
  if (s->world == 1) return QIPB200_OK;
  if (f->cls == CLASS_BITSWAP && f->ctrl_mask == 0) {
    // An uncontrolled Swap is a relabelling of index bits: update the map, move nothing.
    for (size_t i = 0; i < f->swaps.size(); ++i) {
      const uint32_t p = f->swaps[i].first, q = f->swaps[i].second;
      for (uint32_t b = 0; b < s->n; ++b) {
        if (s->phys_of_logical[b] == p)
          s->phys_of_logical[b] = q;
        else if (s->phys_of_logical[b] == q)
          s->phys_of_logical[b] = p;
      }
    }
    f->cls = CLASS_IDENTITY;
    return QIPB200_OK;
  }
  std::vector<uint32_t> nd;
  nondiag_bits(*f, &nd);
  for (size_t i = 0; i < nd.size(); ++i) {
    if (nd[i] < s->n_local) continue;
    const int best = choose_victim(s, *f, next_use);
    if (best < 0) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "op touches every local bit: cannot migrate a rank bit");
    if ((st = exchange_bits(s, nd[i], (uint32_t)best)) != QIPB200_OK) return st;
    // recompile after every move so later decisions see the new layout
    st = compile_op(op, s->prec, s->n, f, &err, s->phys_of_logical.data());
    if (st != QIPB200_OK) return set_err(ctx, st, err);
    nondiag_bits(*f, &nd);
    i = (size_t)-1;  // restart scan
  }
  return QIPB200_OK;
}

}  // namespace qipb200

// ---- multi-device (single process) states ---------------------------------------------------
namespace {

double *comm_of(uint32_t *flags) { return reinterpret_cast<double *>(reinterpret_cast<char *>(flags) + kCommOffsetBytes); }

int multi_state_new(qipb200_ctx *parent, qip_prec prec, uint32_t n, qipb200_state **out) {
  const int G = (int)parent->children.size();
  qipb200_state *p = new qipb200_state();
  p->ctx = parent;
  p->prec = prec;
  p->n = n;
  p->world = 1;
  p->n_local = n;
  for (int r = 0; r < G; ++r) {
    qipb200_state *sh = nullptr;
    int st = state_alloc(parent->children[r], prec, n, r, G, &sh);
    if (st != QIPB200_OK) {
      set_err(parent, st, parent->children[r]->err);
      for (size_t i = 0; i < p->shards.size(); ++i) qipb200_state_free(p->shards[i]);
      delete p;
      return st;
    }
    p->shards.push_back(sh);
  }
  for (int r = 0; r < G; ++r) {  // peers are plain device pointers here: peer access was enabled by init_multi
    qipb200_state *sh = p->shards[r];
    sh->peer_buf.assign(G, nullptr);
    sh->peer_flags.assign(G, nullptr);
    sh->peer_comm.assign(G, nullptr);
    for (int t = 0; t < G; ++t) {
      sh->peer_buf[t] = p->shards[t]->buf;
      sh->peer_flags[t] = p->shards[t]->flags;
      sh->peer_comm[t] = comm_of(p->shards[t]->flags);
    }
    sh->ipc_ready = true;
    cudaSetDevice(sh->ctx->device);
    cudaStreamSynchronize(sh->ctx->stream);  // the zero fill of buffer and flag page, before any peer touches them
  }
  *out = p;
  return QIPB200_OK;
}

// out[0..count) (device, on the rank's stream) <- sum over all ranks of their out[]; collective.
int allreduce_sum(qipb200_state *s, double *d_vec, uint32_t count) {
  qipb200_ctx *ctx = s->ctx;
  if (s->world == 1) return QIPB200_OK;
  if (!s->ipc_ready) return set_err(ctx, QIPB200_ERR_COMM, "sharded state: peers not mapped (call qipb200_state_ipc_import)");
  if (count > (uint32_t)kCommDoubles) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "cross-rank reduction larger than the reduction slot");
  CU(ctx, cudaMemcpyAsync(comm_of(s->flags), d_vec, count * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  CU(ctx, launch_flag_barrier(s->peer_flags.data(), s->flags, s->rank, s->world, ++s->epoch, s->flags + kFlagErrorSlot,
                              ctx->stream, &ctx->launches));
  CU(ctx, launch_comm_sum(s->peer_comm.data(), s->world, d_vec, count, ctx->stream, &ctx->launches));
  CU(ctx, launch_flag_barrier(s->peer_flags.data(), s->flags, s->rank, s->world, ++s->epoch, s->flags + kFlagErrorSlot,
                              ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_new(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, qipb200_state **state) {
  return guarded(ctx, [&]() -> int {
    if (ctx && !ctx->children.empty()) {
      if (!state) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "state out-pointer is NULL");
      *state = nullptr;
      if (ctx->children.size() == 1) return state_alloc(ctx->children[0], prec, n_qubits, 0, 1, state);
      return multi_state_new(ctx, prec, n_qubits, state);
    }
    return state_alloc(ctx, prec, n_qubits, 0, 1, state);
  });
}

extern "C" int qipb200_state_new_sharded(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, int rank,
                                         int world_size, qipb200_state **state) {
  if (ctx && !ctx->children.empty())
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, "state_new_sharded: a multi-device context shards its states itself (use qipb200_state_new)");
  return guarded(ctx, [&]() { return state_alloc(ctx, prec, n_qubits, rank, world_size, state); });
}

extern "C" void qipb200_state_free(qipb200_state *s) {
  if (!s) return;
  if (!s->shards.empty()) {
    for (size_t i = 0; i < s->shards.size(); ++i) {  // all work must have drained before any buffer goes away
      cudaSetDevice(s->shards[i]->ctx->device);
      cudaStreamSynchronize(s->shards[i]->ctx->stream);
    }
    for (size_t i = 0; i < s->shards.size(); ++i) qipb200_state_free(s->shards[i]);
    delete s;
    return;
  }
  qipb200_ctx *ctx = s->ctx;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (s->ipc_mapped)
    for (int t = 0; t < (int)s->peer_buf.size(); ++t) {
      if (t == s->rank) continue;
      if (s->peer_buf[t]) cudaIpcCloseMemHandle(s->peer_buf[t]);
      if (s->peer_flags[t]) cudaIpcCloseMemHandle(s->peer_flags[t]);
    }
  if (s->buf) {
    if (s->world == 1 && !ctx->pool_buf) {  // keep one buffer for the next state of this size
      ctx->pool_buf = s->buf;
      ctx->pool_bytes = s->bytes;
    } else {
      cudaFree(s->buf);
    }
  }
  if (s->scratch) cudaFree(s->scratch);
  if (s->flags) cudaFree(s->flags);
  delete s;
}

// QIPB200_NO_INIT_FOLD=1: set_basis writes the state at once (read per call, so one process can compare both paths).
static bool init_fold_enabled() {
  const char *e = getenv("QIPB200_NO_INIT_FOLD");
  return !(e && atoi(e) != 0);
}

static int set_basis_impl(qipb200_state *s, uint64_t index) {
  qipb200_ctx *ctx = s->ctx;
  if (index >> s->n) return set_err(ctx, QIPB200_ERR_BAD_INDEX, "initial index out of range");
  CU(ctx, cudaSetDevice(ctx->device));
  s->collapse_pending = false;  // every amplitude is overwritten
  s->init_pending = false;
  for (uint32_t b = 0; b < s->n; ++b) s->phys_of_logical[b] = b;  // a fresh state has the canonical layout
  if (s->world == 1 && init_fold_enabled()) {  // written by the next schedule's first tile pass, or before the next read
    s->init_pending = true;
    s->init_index = index;
    return QIPB200_OK;
  }
  const uint64_t len = 1ull << s->n_local;
  const bool owns = (index >> s->n_local) == (uint64_t)s->rank;
  CU(ctx, launch_set_basis(s->prec, s->buf, len, index & (len - 1), owns, ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

extern "C" int qipb200_state_set_basis(qipb200_state *s, uint64_t index) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) {
      if (index >> s->n) return set_err(s->ctx, QIPB200_ERR_BAD_INDEX, "initial index out of range");
      return each_shard(s, [&](qipb200_state *sh, int) { return set_basis_impl(sh, index); });
    }
    return set_basis_impl(s, index);
  });
}

static int transfer_impl(qipb200_state *s, void *host, uint64_t offset, uint64_t len, bool upload) {
  qipb200_ctx *ctx = s->ctx;
  const char *what = upload ? "upload" : "download";
  if (!host && len) return set_err(ctx, QIPB200_ERR_INVALID_ARG, std::string(what) + ": host pointer is NULL");
  if (len > (1ull << s->n_local) || offset > (1ull << s->n_local) - len)
    return set_err(ctx, QIPB200_ERR_SIZE_MISMATCH, std::string(what) + ": range exceeds the local state");
  if (upload && len == (1ull << s->n_local)) s->init_pending = false;  // every amplitude is overwritten
  int st = begin_device_work(s);  // a partial upload keeps the other amplitudes
  if (st != QIPB200_OK) return st;
  if (!layout_is_identity(s)) {
    st = restore_layout(s);
    if (st != QIPB200_OK) return st;
  }
  const size_t ab = amp_bytes(s->prec);
  if (len) {
    if (upload)
      CU(ctx, cudaMemcpyAsync((char *)s->buf + offset * ab, host, len * ab, cudaMemcpyHostToDevice, ctx->stream));
    else
      CU(ctx, cudaMemcpyAsync(host, (const char *)s->buf + offset * ab, len * ab, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  if (s->world > 1 && s->ipc_ready) return check_barrier_error(s);
  return QIPB200_OK;
}

// A multi-device state is addressed as ONE 2^n vector: the range is cut at the shard boundaries.  Every shard
// takes part even when its piece is empty (restoring the canonical layout is a collective exchange).
static int multi_transfer(qipb200_state *p, void *host, uint64_t offset, uint64_t len, bool upload) {
  if (!host && len) return set_err(p->ctx, QIPB200_ERR_INVALID_ARG, "upload/download: host pointer is NULL");
  if (len > (1ull << p->n) || offset > (1ull << p->n) - len)
    return set_err(p->ctx, QIPB200_ERR_SIZE_MISMATCH, "upload/download: range exceeds the state");
  const size_t ab = amp_bytes(p->prec);
  return each_shard(p, [&](qipb200_state *sh, int r) {
    const uint64_t lo = (uint64_t)r << sh->n_local, hi = lo + (1ull << sh->n_local);
    const uint64_t a = std::max(lo, offset), b = std::min(hi, offset + len);
    if (b <= a) return transfer_impl(sh, host, 0, 0, upload);
    return transfer_impl(sh, (char *)host + (a - offset) * ab, a - lo, b - a, upload);
  });
}

extern "C" int qipb200_state_upload(qipb200_state *s, const void *host, uint64_t offset, uint64_t len) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) return multi_transfer(s, const_cast<void *>(host), offset, len, true);
    return transfer_impl(s, const_cast<void *>(host), offset, len, true);
  });
}

extern "C" int qipb200_state_download(qipb200_state *s, void *host, uint64_t offset, uint64_t len) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) return multi_transfer(s, host, offset, len, false);
    return transfer_impl(s, host, offset, len, false);
  });
}

static int apply_op_impl(qipb200_state *s, const qip_op *op) {
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  FlatOp f;
  st = compile_and_localize(s, op, &f, nullptr);
  if (st != QIPB200_OK) return st;
  return apply_flat_local(s, f);
}

extern "C" int qipb200_state_apply_op(qipb200_state *s, const qip_op *op) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) return each_shard(s, [&](qipb200_state *sh, int) { return apply_op_impl(sh, op); });
    return apply_op_impl(s, op);
  });
}

// A schedule on a state with a pending collapse.  Fused: the collapse goes in front of the schedule as one-qubit
// diagonal gates (qipb200_collapse_ops), which the planner folds into the first tile pass.  A schedule that fails
// validation keeps the collapse pending when none of its ops runs; when the ops before the bad one run, the collapse
// is applied first.  QIPB200_SCHED_NO_FUSION keeps one sweep per entry: the collapse runs as its own sweep.
static int schedule_after_measure(qipb200_state *s, const qip_op *ops, size_t n_ops, uint32_t flags) {
  CU(s->ctx, cudaSetDevice(s->ctx->device));
  size_t bad = n_ops;
  for (size_t i = 0; i < n_ops && bad == n_ops; ++i) {
    FlatOp f;
    std::string err;
    if (compile_op(&ops[i], s->prec, s->n, &f, &err) != QIPB200_OK) bad = i;
  }
  if ((flags & QIPB200_SCHED_NO_FUSION) || bad != n_ops) {
    if (bad != 0) {
      int st = materialise_collapse(s);
      if (st != QIPB200_OK) return st;
    }
    return run_schedule(s, ops, n_ops, flags);
  }
  const uint32_t k = (uint32_t)s->pend_qubits.size();
  std::vector<qip_op> all(k + n_ops);
  std::vector<double> dense(8 * (size_t)k);  // 4 complex<prec> per op
  qipb200_collapse_ops(s->prec, s->pend_qubits.data(), k, s->pend_measured, s->pend_p_mult, all.data(), dense.data());
  std::copy(ops, ops + n_ops, all.begin() + k);
  s->collapse_pending = false;
  return run_schedule(s, all.data(), all.size(), flags);
}

extern "C" int qipb200_state_apply_schedule(qipb200_state *s, const qip_op *ops, size_t n_ops, uint32_t flags) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  if (!ops && n_ops) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "schedule: ops is NULL");
  return guarded(s->ctx, [&]() -> int {
    auto one = [&](qipb200_state *sh, int) -> int {
      CU(sh->ctx, cudaSetDevice(sh->ctx->device));
      return run_schedule(sh, ops, n_ops, flags);
    };
    if (!s->shards.empty()) return each_shard(s, one);
    if (s->collapse_pending) return schedule_after_measure(s, ops, n_ops, flags);
    return one(s, 0);
  });
}

// sum |a|^2 of the WHOLE state: on a sharded state the per-rank sums are all-reduced (collective call).
static int norm2_impl(qipb200_state *s, double *out) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  CU(ctx, launch_norm2(s->prec, s->buf, 1ull << s->n_local, ctx->d_scalar, ctx->stream, &ctx->launches));
  st = allreduce_sum(s, ctx->d_scalar, 1);
  if (st != QIPB200_OK) return st;
  CU(ctx, cudaMemcpyAsync(out, ctx->d_scalar, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

extern "C" int qipb200_state_norm2(qipb200_state *s, double *out) {
  if (!s || !out) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "norm2: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) {
      std::vector<double> v(s->shards.size(), 0.0);
      int st = each_shard(s, [&](qipb200_state *sh, int r) { return norm2_impl(sh, &v[r]); });
      *out = v[0];
      return st;
    }
    return norm2_impl(s, out);
  });
}

static int max_abs_diff_impl(qipb200_state *a, qipb200_state *b, double *out) {
  qipb200_ctx *ctx = a->ctx;
  if (a->ctx != b->ctx || a->prec != b->prec || a->n != b->n || a->world != b->world || a->rank != b->rank)
    return set_err(ctx, QIPB200_ERR_SIZE_MISMATCH, "max_abs_diff: the two states differ in context, precision or shape");
  if (a->phys_of_logical != b->phys_of_logical)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "max_abs_diff: the two sharded states hold different qubit layouts");
  int st = begin_device_work(a);
  if (st == QIPB200_OK) st = materialise_pending(b);
  if (st != QIPB200_OK) return st;
  CU(ctx, launch_max_abs_diff(a->prec, a->buf, b->buf, 1ull << a->n_local, ctx->d_scalar, ctx->stream, &ctx->launches));
  CU(ctx, cudaMemcpyAsync(out, ctx->d_scalar, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

extern "C" int qipb200_state_max_abs_diff(qipb200_state *a, qipb200_state *b, double *out) {
  if (!a || !b || !out) return set_err(a ? a->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "max_abs_diff: NULL argument");
  return guarded(a->ctx, [&]() -> int {
    if (a->shards.size() != b->shards.size())
      return set_err(a->ctx, QIPB200_ERR_SIZE_MISMATCH, "max_abs_diff: the two states differ in context, precision or shape");
    if (!a->shards.empty()) {
      std::vector<double> v(a->shards.size(), 0.0);
      int st = each_shard(a, [&](qipb200_state *sh, int r) { return max_abs_diff_impl(sh, b->shards[r], &v[r]); });
      *out = *std::max_element(v.begin(), v.end());
      return st;
    }
    return max_abs_diff_impl(a, b, out);
  });
}

static int sync_impl(qipb200_state *s) {
  CU(s->ctx, cudaSetDevice(s->ctx->device));
  CU(s->ctx, cudaStreamSynchronize(s->ctx->stream));
  if (s->world > 1 && s->ipc_ready) return check_barrier_error(s);
  return QIPB200_OK;
}

extern "C" int qipb200_state_sync(qipb200_state *s) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty()) return each_shard(s, [&](qipb200_state *sh, int) { return sync_impl(sh); });
    return sync_impl(s);
  });
}

extern "C" int qipb200_calculate_state(qipb200_ctx *ctx, qip_prec prec, uint32_t n_qubits, uint64_t init_index,
                                       const qip_op *ops, size_t n_ops, uint32_t flags, void *host_out) {
  if (!ctx) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "ctx is NULL (call qipb200_init first; there is no CPU path)");
  if (!host_out) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "calculate_state: host_out is NULL");
  qipb200_state *s = nullptr;
  int st = qipb200_state_new(ctx, prec, n_qubits, &s);
  if (st != QIPB200_OK) return st;
  st = qipb200_state_set_basis(s, init_index);
  if (st == QIPB200_OK) st = qipb200_state_apply_schedule(s, ops, n_ops, flags);
  if (st == QIPB200_OK) st = qipb200_state_download(s, host_out, 0, 1ull << n_qubits);
  qipb200_state_free(s);
  return st;
}

extern "C" int qipb200_apply_ops(qipb200_ctx *ctx, qip_prec prec, uint32_t n, const qip_op *ops, size_t n_ops,
                                 const void *input, uint64_t input_len, void *output, uint64_t output_len,
                                 uint64_t input_offset, uint64_t output_offset) {
  if (!ctx) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "ctx is NULL (call qipb200_init first; there is no CPU path)");
  const size_t ab = amp_bytes(prec);
  if (n_ops == 0) {
    // matrix_ops.rs:170-183: copy of the overlapping index range
    const uint64_t lower = std::max(input_offset, output_offset);
    const uint64_t upper = std::min(input_offset + input_len, output_offset + output_len);
    if (upper > lower) {
      if (!input || !output) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "apply_ops: NULL amplitude buffer");
      memcpy((char *)output + (lower - output_offset) * ab, (const char *)input + (lower - input_offset) * ab,
             (upper - lower) * ab);
    }
    return QIPB200_OK;
  }
  if (n_ops == 1)  // matrix_ops.rs:167
    return qipb200_apply_op(ctx, prec, n, ops, input, input_len, output, output_len, input_offset, output_offset);
  // Several ops: the reference's multi-op row iterator (matrix_ops.rs:184-217), restated as it is -- including
  // SURVEY.md quirk Q5 -- by k_multi_gather; accumulates into `output` like the reference (:212).
  return guarded(ctx, [&]() -> int {
    qipb200_ctx *c = ctx->children.empty() ? ctx : ctx->children[0];
    if ((!input && input_len) || (!output && output_len)) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "apply_ops: NULL amplitude buffer");
    if (n > 40 || input_len > (1ull << 40) || output_len > (1ull << 40))
      return set_err(ctx, QIPB200_ERR_SIZE_MISMATCH, "apply_ops: buffer length out of range");
    if (n_ops > 8) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "apply_ops: more than 8 ops in one multi-op sweep");
    std::vector<FlatOp> fs(n_ops);
    uint32_t ktot = 0;
    for (size_t i = 0; i < n_ops; ++i) {
      std::string err;
      int st = compile_op(&ops[i], prec, n, &fs[i], &err);
      if (st != QIPB200_OK) return set_err(ctx, st, err);
      ktot += fs[i].k;
    }
    if (ktot > 40) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "apply_ops: more than 40 indices over all ops");
    if (cudaSetDevice(c->device) != cudaSuccess) return set_err(ctx, QIPB200_ERR_CUDA, "cudaSetDevice");
    int st;
    if ((st = grow(c, &c->d_in, &c->d_in_bytes, std::max<size_t>(input_len * ab, 16))) != QIPB200_OK ||
        (st = grow(c, &c->d_out, &c->d_out_bytes, std::max<size_t>(output_len * ab, 16))) != QIPB200_OK) {
      if (c != ctx) ctx->err = c->err;
      return st;
    }
    cudaError_t e = cudaSuccess;
    if (input_len) e = cudaMemcpyAsync(c->d_in, input, input_len * ab, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess && output_len) e = cudaMemcpyAsync(c->d_out, output, output_len * ab, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess)
      e = launch_multi_gather(prec, fs, c->d_in, input_len, input_offset, c->d_out, output_len, output_offset, c->stream, &c->launches);
    if (e == cudaSuccess && output_len) e = cudaMemcpyAsync(output, c->d_out, output_len * ab, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return set_err(ctx, QIPB200_ERR_CUDA, std::string("apply_ops: ") + cudaGetErrorString(e));
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// N3: state files ("QIPA" v1, one file per shard; layout in rustqip_b200/wire.py) -- checkpoint / resume
// ===================================================================================

namespace {

struct QipaHeader {
  uint32_t magic, version, prec, n_qubits, rank, world;
  uint64_t first_index, n_amplitudes;
};
static_assert(sizeof(QipaHeader) == 40, "QIPA header is 40 bytes");
const uint32_t kQipaMagic = 0x41504951u;
const size_t kFileChunkBytes = 64u << 20;  // host bounce buffer: the shard never sits in host memory as a whole

int state_file_impl(qipb200_state *s, const char *path, bool save) {
  qipb200_ctx *ctx = s->ctx;
  CU(ctx, cudaSetDevice(ctx->device));
  if (save) {
    int st = materialise_pending(s);
    if (st != QIPB200_OK) return st;
  }
  if (!layout_is_identity(s)) {  // files hold the canonical layout (collective on a sharded state)
    int st = restore_layout(s);
    if (st != QIPB200_OK) return st;
  }
  const size_t ab = amp_bytes(s->prec);
  const uint64_t len = 1ull << s->n_local;
  FILE *f = fopen(path, save ? "wb" : "rb");
  if (!f) return set_err(ctx, QIPB200_ERR_INVALID_ARG, std::string("state file: cannot open ") + path);
  QipaHeader h;
  int st = QIPB200_OK;
  if (save) {
    h.magic = kQipaMagic, h.version = 1, h.prec = (uint32_t)s->prec, h.n_qubits = s->n, h.rank = (uint32_t)s->rank;
    h.world = (uint32_t)s->world, h.first_index = (uint64_t)s->rank << s->n_local, h.n_amplitudes = len;
    if (fwrite(&h, sizeof(h), 1, f) != 1) st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "state file: write failed");
  } else {
    if (fread(&h, sizeof(h), 1, f) != 1 || h.magic != kQipaMagic || h.version != 1)
      st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "not a QIPA version-1 state file");
    else if (h.prec != (uint32_t)s->prec || h.n_qubits != s->n || h.rank != (uint32_t)s->rank || h.world != (uint32_t)s->world ||
             h.n_amplitudes != len)
      st = set_err(ctx, QIPB200_ERR_SIZE_MISMATCH, "state file does not match the target state (prec/n/rank/world/length)");
    if (st == QIPB200_OK) s->collapse_pending = s->init_pending = false;  // every amplitude is overwritten
  }
  std::vector<char> bounce;
  if (st == QIPB200_OK) bounce.resize((size_t)std::min<uint64_t>(kFileChunkBytes, len * ab));
  for (uint64_t done = 0; st == QIPB200_OK && done < len * ab;) {
    const size_t n = (size_t)std::min<uint64_t>(bounce.size(), len * ab - done);
    cudaError_t e;
    if (save) {
      e = cudaMemcpyAsync(bounce.data(), (const char *)s->buf + done, n, cudaMemcpyDeviceToHost, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      if (e != cudaSuccess) st = cuda_fail(ctx, e, "state file: device -> host");
      else if (fwrite(bounce.data(), 1, n, f) != n) st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "state file: write failed");
    } else {
      if (fread(bounce.data(), 1, n, f) != n) {
        st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "state file truncated");
        break;
      }
      e = cudaMemcpyAsync((char *)s->buf + done, bounce.data(), n, cudaMemcpyHostToDevice, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      if (e != cudaSuccess) st = cuda_fail(ctx, e, "state file: host -> device");
    }
    done += n;
  }
  if (st == QIPB200_OK && !save && fgetc(f) != EOF) st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "state file: trailing bytes");
  if (fclose(f) != 0 && st == QIPB200_OK && save) st = set_err(ctx, QIPB200_ERR_INVALID_ARG, "state file: close failed");
  return st;
}

int state_file(qipb200_state *s, const char *path, bool save) {
  if (!s || !path) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "state file: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    if (!s->shards.empty())  // multi-device state: one file per shard, "<path>.<rank>"
      return each_shard(s, [&](qipb200_state *sh, int r) { return state_file_impl(sh, (std::string(path) + "." + std::to_string(r)).c_str(), save); });
    return state_file_impl(s, path, save);
  });
}

}  // namespace

extern "C" int qipb200_state_save(qipb200_state *s, const char *path) { return state_file(s, path, true); }
extern "C" int qipb200_state_load(qipb200_state *s, const char *path) { return state_file(s, path, false); }

// ===================================================================================
// measurement (collective on a sharded state: every rank calls, every rank gets the answer)
// ===================================================================================

namespace {

int check_indices(qipb200_state *s, const uint64_t *indices, uint32_t n_indices) {
  if (!indices || n_indices == 0 || n_indices > s->n)
    return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "measurement: bad index list");
  uint64_t seen = 0;
  for (uint32_t i = 0; i < n_indices; ++i) {
    if (indices[i] >= s->n) return set_err(s->ctx, QIPB200_ERR_BAD_INDEX, "measurement: qubit index out of range");
    if ((seen >> indices[i]) & 1) return set_err(s->ctx, QIPB200_ERR_BAD_INDEX, "measurement: repeated qubit index");
    seen |= 1ull << indices[i];
  }
  return QIPB200_OK;
}

int measure_probs_impl(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double *out) {
  qipb200_ctx *ctx = s->ctx;
  if (n_indices > 26) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "measure_probs: more than 26 measured qubits");
  if (s->world > 1 && (1u << n_indices) > (uint32_t)kCommDoubles)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "measure_probs on a sharded state: more than 16 measured qubits");
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  uint32_t bitpos[32];
  phys_positions(s, indices, n_indices, bitpos);
  double *d_hist = nullptr;
  CU(ctx, cudaMallocAsync((void **)&d_hist, sizeof(double) << n_indices, ctx->stream));
  CU(ctx, launch_measure_probs(s->prec, s->buf, 1ull << s->n_local, (uint64_t)s->rank << s->n_local, bitpos,
                               n_indices, d_hist, ctx->stream, &ctx->launches));
  // measurement_ops.rs:115-127 sums over the WHOLE vector: per-rank histograms are added across the ranks
  st = allreduce_sum(s, d_hist, 1u << n_indices);
  if (st == QIPB200_OK)
    CU(ctx, cudaMemcpyAsync(out, d_hist, sizeof(double) << n_indices, cudaMemcpyDeviceToHost, ctx->stream));
  CU(ctx, cudaFreeAsync(d_hist, ctx->stream));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return st;
}

// The serial scan of measurement_ops.rs:166-172 over this rank's amplitudes, starting with `rem` left of the
// draw: per-chunk sums on the device, chunk search on the host, then a scan of the chunk holding the crossing
// (and of the following ones when rounding leaves the chunk-level search one step short).
int local_scan(qipb200_state *s, double rem, bool *crossed, uint64_t *idx_out) {
  qipb200_ctx *ctx = s->ctx;
  const uint64_t len = 1ull << s->n_local;
  const uint32_t chunk_log2 = s->n_local > 12 ? 12 : s->n_local;
  const uint64_t chunks = len >> chunk_log2;
  double *d_sums = nullptr;
  CU(ctx, cudaMallocAsync((void **)&d_sums, chunks * sizeof(double), ctx->stream));
  CU(ctx, launch_chunk_sums(s->prec, s->buf, len, chunk_log2, d_sums, ctx->stream, &ctx->launches));
  std::vector<double> sums(chunks);
  CU(ctx, cudaMemcpyAsync(sums.data(), d_sums, chunks * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CU(ctx, cudaFreeAsync(d_sums, ctx->stream));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  uint64_t c = 0;
  for (; c + 1 < chunks; ++c) {
    if (rem - sums[c] <= 0.0) break;
    rem -= sums[c];
  }
  const uint64_t clen = 1ull << chunk_log2;
  const size_t ab = amp_bytes(s->prec);
  std::vector<char> host(clen * ab);
  *crossed = false;
  *idx_out = 0;
  for (; c < chunks && !*crossed; ++c) {
    CU(ctx, cudaMemcpyAsync(host.data(), (const char *)s->buf + c * clen * ab, clen * ab, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint64_t i = 0; i < clen; ++i) {
      double re, im;
      if (s->prec == QIP_F32) {
        re = ((const float *)host.data())[2 * i];
        im = ((const float *)host.data())[2 * i + 1];
      } else {
        re = ((const double *)host.data())[2 * i];
        im = ((const double *)host.data())[2 * i + 1];
      }
      rem -= re * re + im * im;
      if (rem <= 0.0) {
        *idx_out = c * clen + i;
        *crossed = true;
        break;
      }
    }
  }
  return QIPB200_OK;
}

int soft_measure_impl(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double r, uint64_t *measured) {
  qipb200_ctx *ctx = s->ctx;
  int st0 = begin_device_work(s);
  if (st0 != QIPB200_OK) return st0;
  uint64_t idx = 0;  // the reference leaves measured_indx = 0 when the scan never crosses
  if (s->world == 1) {
    bool crossed = false;
    int st = local_scan(s, r, &crossed, &idx);  // full-length input: r * 1 (measurement_ops.rs:160-165)
    if (st != QIPB200_OK) return st;
  } else {
    // The reference scans the whole vector in index order: restore the canonical layout (rank r then holds
    // indices [r 2^nl, (r+1) 2^nl)), all-gather the per-rank totals, let every rank scan its own shard with the
    // part of the draw the lower ranks left over, all-gather (crossed, index): the lowest crossing rank wins.
    if (!layout_is_identity(s)) {
      int st = restore_layout(s);
      if (st != QIPB200_OK) return st;
    }
    const int W = s->world;
    double *d_vec = nullptr;
    CU(ctx, cudaMallocAsync((void **)&d_vec, 2 * W * sizeof(double), ctx->stream));
    CU(ctx, cudaMemsetAsync(d_vec, 0, 2 * W * sizeof(double), ctx->stream));
    CU(ctx, launch_norm2(s->prec, s->buf, 1ull << s->n_local, ctx->d_scalar, ctx->stream, &ctx->launches));
    CU(ctx, cudaMemcpyAsync(d_vec + s->rank, ctx->d_scalar, sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    int st = allreduce_sum(s, d_vec, (uint32_t)W);
    std::vector<double> tot(2 * W, 0.0);
    if (st == QIPB200_OK) {
      CU(ctx, cudaMemcpyAsync(tot.data(), d_vec, W * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
      CU(ctx, cudaStreamSynchronize(ctx->stream));
      double rem = r;
      for (int t = 0; t < s->rank; ++t) rem -= tot[t];
      bool crossed = false;
      uint64_t li = 0;
      if (rem <= 0.0 && s->rank > 0) {
        crossed = true;  // the draw ran out below this rank: a serial scan arriving here stops at the first element
      } else {
        st = local_scan(s, rem, &crossed, &li);
      }
      std::vector<double> mine(2 * W, 0.0);
      mine[2 * s->rank] = crossed ? 1.0 : 0.0;
      mine[2 * s->rank + 1] = (double)(((uint64_t)s->rank << s->n_local) + li);  // < 2^40: exact in a double
      if (st == QIPB200_OK) {
        CU(ctx, cudaMemcpyAsync(d_vec, mine.data(), 2 * W * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        st = allreduce_sum(s, d_vec, (uint32_t)(2 * W));
      }
      if (st == QIPB200_OK) {
        CU(ctx, cudaMemcpyAsync(tot.data(), d_vec, 2 * W * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        for (int t = 0; t < W; ++t)
          if (tot[2 * t] != 0.0) {
            idx = (uint64_t)tot[2 * t + 1];
            break;
          }
      }
    }
    CU(ctx, cudaFreeAsync(d_vec, ctx->stream));
    if (st != QIPB200_OK) return st;
  }
  uint64_t m = 0;  // extract_bits(measured_indx, [n-1-index]) (measurement_ops.rs:174-175)
  for (uint32_t i = 0; i < n_indices; ++i) m |= ((idx >> (s->n - 1 - indices[i])) & 1ull) << i;
  *measured = m;
  return QIPB200_OK;
}

// n_draws soft_measure draws on one unsharded state (kernels.cu: launch_sample): one upload of the draws, a constant
// number of kernels, one download of the results.  The scan runs over canonical indices, so a permuted layout is
// restored first.
int sample_impl(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, const double *draws, uint64_t n_draws,
                uint64_t *measured) {
  qipb200_ctx *ctx = s->ctx;
  if (n_draws > 0xffffffffull) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, "sample: more than 2^32-1 draws in one call");
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  if (!layout_is_identity(s)) {
    st = restore_layout(s);
    if (st != QIPB200_OK) return st;
  }
  SampleBits bits;
  bits.n_bits = n_indices;
  for (uint32_t i = 0; i < n_indices; ++i) bits.bitpos[i] = s->n - 1 - (uint32_t)indices[i];  // measurement_ops.rs:174-175
  const size_t io = 16 * (size_t)n_draws;  // draws (double) + results (u64)
  char *d = nullptr;
  CU(ctx, cudaMallocAsync((void **)&d, io + sample_scratch_bytes(s->n_local, n_draws), ctx->stream));
  double *d_draws = (double *)d;
  uint64_t *d_out = (uint64_t *)(d + 8 * n_draws);
  cudaError_t e = cudaMemcpyAsync(d_draws, draws, 8 * n_draws, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess)
    e = launch_sample(s->prec, s->buf, s->n_local, d_draws, n_draws, bits, d + io, d_out, ctx->sm_count, ctx->stream,
                      &ctx->launches);
  if (e == cudaSuccess) e = cudaMemcpyAsync(measured, d_out, 8 * n_draws, cudaMemcpyDeviceToHost, ctx->stream);
  cudaError_t ef = cudaFreeAsync(d, ctx->stream);
  if (e != cudaSuccess) return cuda_fail(ctx, e, "sample");
  CU(ctx, ef);
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

int collapse_impl(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, uint64_t measured, double measured_prob) {
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  if (measured_prob == 0.0) return QIPB200_OK;  // measurement_ops.rs:230: untouched
  return launch_collapse_on(s, indices, n_indices, measured, collapse_multiplier(s->prec, measured_prob));
}

// measure on an unsharded single-device state (kernels.cu: launch_measure): one upload of the draw or the forced
// outcome, a fixed number of kernels, one download of {m, p}.  The collapse is left pending on the state.
int measure_impl(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double r, uint32_t flags,
                 uint64_t *measured, double *prob) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  MeasureRecord rec = {(flags & QIPB200_MEASURE_FORCED) ? *measured : 0, 0.0};
  if (flags & QIPB200_MEASURE_FORCED_PROB) {
    rec.p = *prob;
  } else if ((flags & QIPB200_MEASURE_FORCED) && n_indices < 64 && (rec.m >> n_indices)) {
    rec.p = 0.0;  // measure_prob of an outcome the index list cannot produce
  } else {
    if (!layout_is_identity(s)) {  // the scan and the chunk sums run over canonical indices
      st = restore_layout(s);
      if (st != QIPB200_OK) return st;
    }
    SampleBits bits;
    bits.n_bits = n_indices;
    for (uint32_t i = 0; i < n_indices; ++i) bits.bitpos[i] = s->n - 1 - (uint32_t)indices[i];  // measurement_ops.rs:174-175
    char *d = nullptr;
    CU(ctx, cudaMallocAsync((void **)&d, 32 + measure_scratch_bytes(s->n_local), ctx->stream));
    MeasureRecord *d_rec = (MeasureRecord *)d;
    double *d_draw = (double *)(d + 16);
    const bool forced = (flags & QIPB200_MEASURE_FORCED) != 0;
    cudaError_t e = forced ? cudaMemcpyAsync(d_rec, &rec, sizeof(rec), cudaMemcpyHostToDevice, ctx->stream)
                           : cudaMemcpyAsync(d_draw, &r, sizeof(r), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess)
      e = launch_measure(s->prec, s->buf, s->n_local, forced ? nullptr : d_draw, bits, d + 32, d_rec, ctx->sm_count,
                         ctx->stream, &ctx->launches);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&rec, d_rec, sizeof(rec), cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t ef = cudaFreeAsync(d, ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "measure");
    CU(ctx, ef);
  }
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  if (rec.p != 0.0) {  // measurement_ops.rs:230: a zero probability leaves the state untouched
    s->pend_qubits.assign(indices, indices + n_indices);
    s->pend_measured = rec.m;
    s->pend_p_mult = collapse_multiplier(s->prec, rec.p);
    s->collapse_pending = true;
  }
  *measured = rec.m;
  *prob = rec.p;
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_measure_probs(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double *out) {
  if (!s || !out) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "measure_probs: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (!s->shards.empty()) {
      if (n_indices > 16) return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, "measure_probs on a sharded state: more than 16 measured qubits");
      std::vector<std::vector<double>> v(s->shards.size(), std::vector<double>((size_t)1 << n_indices));
      st = each_shard(s, [&](qipb200_state *sh, int r) { return measure_probs_impl(sh, indices, n_indices, v[r].data()); });
      if (st == QIPB200_OK) memcpy(out, v[0].data(), sizeof(double) << n_indices);
      return st;
    }
    return measure_probs_impl(s, indices, n_indices, out);
  });
}

extern "C" int qipb200_state_measure_prob(qipb200_state *s, uint64_t measured, const uint64_t *indices,
                                          uint32_t n_indices, double *out) {
  if (!s || !out) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "measure_prob: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (n_indices > 26) return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, "measure_prob: more than 26 measured qubits");
    std::vector<double> probs(1ull << n_indices);
    st = qipb200_state_measure_probs(s, indices, n_indices, probs.data());
    if (st != QIPB200_OK) return st;
    *out = (measured >> n_indices) ? 0.0 : probs[measured];
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_soft_measure(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double r,
                                          uint64_t *measured) {
  if (!s || !measured) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "soft_measure: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (!s->shards.empty()) {
      std::vector<uint64_t> v(s->shards.size(), 0);
      st = each_shard(s, [&](qipb200_state *sh, int rk) { return soft_measure_impl(sh, indices, n_indices, r, &v[rk]); });
      *measured = v[0];
      return st;
    }
    return soft_measure_impl(s, indices, n_indices, r, measured);
  });
}

extern "C" int qipb200_state_sample(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, const double *draws,
                                    uint64_t n_draws, uint64_t *measured) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "sample: NULL state");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (s->world > 1 || !s->shards.empty())
      return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, "sample: sharded states are not supported (use soft_measure per draw)");
    if (n_draws == 0) return (int)QIPB200_OK;
    if (!draws || !measured) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "sample: NULL draws or measured");
    return sample_impl(s, indices, n_indices, draws, n_draws, measured);
  });
}

extern "C" int qipb200_state_measure(qipb200_state *s, const uint64_t *indices, uint32_t n_indices, double r,
                                     uint32_t flags, uint64_t *measured, double *prob) {
  if (!s || !measured || !prob)
    return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "measure: NULL argument");
  return guarded(s->ctx, [&]() -> int {
    if ((flags & ~(uint32_t)(QIPB200_MEASURE_FORCED | QIPB200_MEASURE_FORCED_PROB)) ||
        ((flags & QIPB200_MEASURE_FORCED_PROB) && !(flags & QIPB200_MEASURE_FORCED)))
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "measure: unknown flags, or FORCED_PROB without FORCED");
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (s->world == 1 && s->shards.empty()) return measure_impl(s, indices, n_indices, r, flags, measured, prob);
    // sharded and multi-device states: the collective calls in turn, collapsing at once
    uint64_t m = *measured;
    double p = *prob;
    if (!(flags & QIPB200_MEASURE_FORCED) && (st = qipb200_state_soft_measure(s, indices, n_indices, r, &m)) != QIPB200_OK)
      return st;
    if (!(flags & QIPB200_MEASURE_FORCED_PROB) && (st = qipb200_state_measure_prob(s, m, indices, n_indices, &p)) != QIPB200_OK)
      return st;
    if ((st = qipb200_state_collapse(s, indices, n_indices, m, p)) != QIPB200_OK) return st;
    if ((st = qipb200_state_sync(s)) != QIPB200_OK) return st;
    *measured = m;
    *prob = p;
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_collapse(qipb200_state *s, const uint64_t *indices, uint32_t n_indices,
                                      uint64_t measured, double measured_prob) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "state is NULL");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, indices, n_indices);
    if (st != QIPB200_OK) return st;
    if (!s->shards.empty())
      return each_shard(s, [&](qipb200_state *sh, int) { return collapse_impl(sh, indices, n_indices, measured, measured_prob); });
    return collapse_impl(s, indices, n_indices, measured, measured_prob);
  });
}

// ===================================================================================
// Pauli-string expectation values (expect.cu)
// ===================================================================================

namespace {

// The checks the feature entries below share: each returns QIPB200_OK or the status of the refusal it reported.

// The Pauli term list of an n-qubit state, or parse_pauli_terms' refusal reported on ctx.
int parse_terms(const qipb200_ctx *ctx, uint32_t n, const uint64_t *qubits, const char *paulis, const uint32_t *term_len,
                size_t n_terms, std::vector<PauliTerm> *terms) {
  std::string err;
  const int st = parse_pauli_terms(n, qubits, paulis, term_len, n_terms, terms, &err);
  return st == QIPB200_OK ? st : set_err(ctx, st, err);
}

// The preconditions of every host-only plan: its outputs (named outs) given, a known precision and 1..40 qubits.
int check_plan_args(const std::string &who, qip_prec prec, uint32_t n_qubits, bool outs_present, const char *outs) {
  if (outs_present && (prec == QIP_F32 || prec == QIP_F64) && n_qubits >= 1 && n_qubits <= 40) return QIPB200_OK;
  return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL " + outs + ", bad precision or n_qubits not in 1..40");
}

int require_unsharded(const qipb200_state *s, const std::string &who) {
  if (s->world > 1 || !s->shards.empty())
    return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, who + ": sharded states are not supported");
  return QIPB200_OK;
}

// Context, precision and size, then sharding: the checks every call on two states makes.
int check_compatible(const qipb200_state *a, const qipb200_state *b, const std::string &who) {
  if (a->ctx != b->ctx || a->prec != b->prec || a->n != b->n)
    return set_err(a->ctx, QIPB200_ERR_SIZE_MISMATCH, who + ": the states differ in context, precision or size");
  int st = require_unsharded(a, who);
  if (st == QIPB200_OK) st = require_unsharded(b, who);
  return st;
}

// dst == src first: an out-of-place call cannot read the state it writes.
int check_state_pair(const qipb200_state *dst, const qipb200_state *src, const std::string &who) {
  if (dst == src) return set_err(dst->ctx, QIPB200_ERR_INVALID_ARG, who + ": the two states must differ");
  return check_compatible(dst, src, who);
}

// A state and the two work states it is evolved through.
int check_three_states(const qipb200_state *state, const qipb200_state *work_a, const qipb200_state *work_b,
                       const std::string &who) {
  if (state == work_a || state == work_b || work_a == work_b)
    return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": the three states must differ");
  int st = check_compatible(work_a, state, who);
  if (st == QIPB200_OK) st = check_compatible(work_b, state, who);
  return st;
}

int check_finite(qipb200_ctx *ctx, const double *v, size_t n, const std::string &who, const char *what) {
  if (n && !v) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL " + what + "s");
  for (size_t t = 0; t < n; ++t)
    if (!std::isfinite(v[t]))
      return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": " + what + " " + std::to_string(t) + " is not finite");
  return QIPB200_OK;
}

// src's pending work runs, dst's is dropped (dst is overwritten), and dst takes src's layout.
int prepare_out_of_place(qipb200_state *dst, qipb200_state *src) {
  int st = materialise_pending(src);
  if (st != QIPB200_OK) return st;
  dst->collapse_pending = dst->init_pending = false;
  dst->phys_of_logical = src->phys_of_logical;
  return QIPB200_OK;
}

int prepare_work_states(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b) {
  int st = prepare_out_of_place(work_a, state);
  if (st == QIPB200_OK) st = prepare_out_of_place(work_b, state);
  return st;
}

// Logical masks -> physical index bits of s (a permuted layout needs no restore sweep: Pauli masks permute with bits).
std::vector<PauliTerm> phys_terms(const qipb200_state *s, const std::vector<PauliTerm> &terms) {
  std::vector<PauliTerm> phys(terms.size());
  for (size_t t = 0; t < terms.size(); ++t) {
    phys[t].n_y = terms[t].n_y;
    for (uint32_t b = 0; b < s->n; ++b) {
      const uint64_t p = 1ull << s->phys_of_logical[b];
      if ((terms[t].x >> b) & 1) phys[t].x |= p;
      if ((terms[t].z >> b) & 1) phys[t].z |= p;
    }
  }
  return phys;
}

int expect_impl(qipb200_state *s, const std::vector<PauliTerm> &terms, double *out) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  // A state left permuted (QIPB200_ROTATE) needs no restore_layout sweep: Pauli masks permute with the bits.
  const std::vector<PauliTerm> phys = phys_terms(s, terms);
  CU(ctx, run_expect(s->prec, s->buf, s->n_local, phys, out, ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_expect_paulis(qipb200_state *s, const uint64_t *qubits, const char *paulis,
                                           const uint32_t *term_len, size_t n_terms, double *out) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "expect_paulis: NULL state");
  return guarded(s->ctx, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = parse_terms(s->ctx, s->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = require_unsharded(s, "expect_paulis");
    if (st != QIPB200_OK) return st;
    if (n_terms == 0) return (int)QIPB200_OK;
    if (!out) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "expect_paulis: NULL out");
    return expect_impl(s, terms, out);
  });
}

extern "C" int qipb200_expect_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis,
                                   const uint32_t *term_len, size_t n_terms, uint32_t *sweeps) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args("expect_plan", prec, n_qubits, sweeps, "sweeps");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    *sweeps = expect_sweep_count(n_qubits, terms);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_transition_paulis(qipb200_state *bra, qipb200_state *ket, const uint64_t *qubits,
                                               const char *paulis, const uint32_t *term_len, size_t n_terms,
                                               double *out) {
  const std::string who = "transition_paulis";
  if (!bra || !ket) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(bra->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves both states (and a pending collapse) as they were
    std::vector<PauliTerm> terms;
    int st = parse_terms(bra->ctx, bra->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_compatible(bra, ket, who);  // bra == ket is allowed
    if (st != QIPB200_OK) return st;
    if (n_terms == 0) return (int)QIPB200_OK;
    if (!out) return set_err(bra->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL out");
    qipb200_ctx *ctx = bra->ctx;
    if ((st = begin_device_work(bra)) != QIPB200_OK) return st;
    if ((st = materialise_pending(ket)) != QIPB200_OK) return st;
    // One qubit map: the states are read where they are (Pauli masks permute with the bits).  Two maps: each permuted
    // state goes back to the canonical layout first, as before a download.
    if (bra->phys_of_logical != ket->phys_of_logical) {
      if ((st = restore_layout(bra)) != QIPB200_OK) return st;
      if ((st = restore_layout(ket)) != QIPB200_OK) return st;
    }
    CU(ctx, run_transition(bra->prec, bra->buf, ket->buf, bra->n_local, phys_terms(bra, terms), out, ctx->stream,
                           &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_transition_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis,
                                       const uint32_t *term_len, size_t n_terms, uint32_t *out2) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args("transition_plan", prec, n_qubits, out2, "out2");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    out2[0] = out2[1] = 0;
    if (!terms.empty()) transition_plan_counts(n_qubits, terms, out2);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// reduced density matrices (rdm.cu)
// ===================================================================================

namespace {

int rdm_impl(qipb200_state *s, const uint64_t *qubits, uint32_t k, double *out) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  // A state left permuted (QIPB200_ROTATE) needs no restore_layout sweep: the kept qubits are read where they are.
  uint32_t pos[kRdmMaxKept];
  phys_positions(s, qubits, k, pos);
  CU(ctx, run_reduced_density(s->prec, s->buf, s->n_local, pos, k, out, ctx->stream, &ctx->launches));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_reduced_density(qipb200_state *s, const uint64_t *qubits, uint32_t n_qubits_kept,
                                             double *out) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "reduced_density: NULL state");
  return guarded(s->ctx, [&]() -> int {
    int st = check_indices(s, qubits, n_qubits_kept);
    if (st != QIPB200_OK) return st;
    if (!out) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "reduced_density: NULL out");
    if (n_qubits_kept > kRdmMaxKept)
      return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED,
                     "reduced_density: at most 10 kept qubits (the output at 10 is already 16 MiB)");
    if ((st = require_unsharded(s, "reduced_density")) != QIPB200_OK) return st;
    return rdm_impl(s, qubits, n_qubits_kept, out);
  });
}

// ===================================================================================
// purity of a bipartition (purity.cu)
// ===================================================================================

namespace {

// The kept qubits of a host-only plan of a cut: 1..n distinct qubits below n.
int check_plan_cut(const std::string &who, uint32_t n_qubits, const uint64_t *qubits, uint32_t k) {
  if (!qubits || k == 0 || k > n_qubits) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": bad qubit list");
  uint64_t seen = 0;
  for (uint32_t i = 0; i < k; ++i) {
    if (qubits[i] >= n_qubits) return set_err(nullptr, QIPB200_ERR_BAD_INDEX, who + ": qubit index out of range");
    if ((seen >> qubits[i]) & 1) return set_err(nullptr, QIPB200_ERR_BAD_INDEX, who + ": repeated qubit index");
    seen |= 1ull << qubits[i];
  }
  return QIPB200_OK;
}

// The side of the cut: the kept qubits if they are at most half, else their complement (Tr rho_A^2 = Tr rho_B^2).
std::vector<uint64_t> purity_side(uint32_t n, const uint64_t *qubits, uint32_t k) {
  std::vector<uint64_t> side;
  if (k <= n - k) return std::vector<uint64_t>(qubits, qubits + k);
  uint64_t kept = 0;
  for (uint32_t i = 0; i < k; ++i) kept |= 1ull << qubits[i];
  for (uint32_t q = 0; q < n; ++q)
    if (!((kept >> q) & 1)) side.push_back(q);
  return side;
}

int purity_impl(qipb200_state *s, const uint64_t *qubits, uint32_t k, double *out2) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  // A state left permuted (QIPB200_ROTATE) is read where it is, as by reduced_density.
  const std::vector<uint64_t> side = purity_side(s->n, qubits, k);
  const uint32_t sb = (uint32_t)side.size();
  std::vector<uint32_t> pos(sb);
  phys_positions(s, side.data(), sb, pos.data());
  uint64_t mask = 0;
  for (uint32_t i = 0; i < sb; ++i) mask |= 1ull << pos[i];
  switch (purity_route(sb)) {
    case 0: {
      double v = 0.0;
      CU(ctx, run_purity_norm2(s->prec, s->buf, s->n_local, &v, ctx->stream, &ctx->launches));
      out2[0] = v * v;
      out2[1] = v;
      return QIPB200_OK;
    }
    case 1: {
      // ||rho||_F^2 in a fixed order: each row's |rho_ab|^2 in column order, then the rows in order
      const size_t K = (size_t)1 << sb;
      std::vector<double> rho(2 * K * K);
      CU(ctx, run_reduced_density(s->prec, s->buf, s->n_local, pos.data(), sb, rho.data(), ctx->stream,
                                  &ctx->launches));
      double p = 0.0, tr = 0.0;
      for (size_t a = 0; a < K; ++a) {
        double row = 0.0;
        for (size_t b = 0; b < K; ++b) {
          row = std::fma(rho[2 * (a * K + b)], rho[2 * (a * K + b)], row);
          row = std::fma(rho[2 * (a * K + b) + 1], rho[2 * (a * K + b) + 1], row);
        }
        p += row;
        tr += rho[2 * (a * K + a)];
      }
      out2[0] = p;
      out2[1] = tr;
      return QIPB200_OK;
    }
    default:
      CU(ctx, run_purity_gram(s->prec, s->buf, s->n_local, mask, out2, ctx->stream, &ctx->launches));
      return QIPB200_OK;
  }
}

}  // namespace

extern "C" int qipb200_state_purity(qipb200_state *s, const uint64_t *qubits, uint32_t k, double *out2) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "purity: NULL state");
  return guarded(s->ctx, [&]() -> int {
    if (!out2) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "purity: NULL out2");
    int st = check_indices(s, qubits, k);
    if (st == QIPB200_OK) st = require_unsharded(s, "purity");
    if (st != QIPB200_OK) return st;
    return purity_impl(s, qubits, k, out2);
  });
}

extern "C" int qipb200_purity_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, uint32_t k,
                                   uint32_t *out4) {
  return guarded(nullptr, [&]() -> int {
    int st = check_plan_args("purity_plan", prec, n_qubits, out4, "out4");
    if (st == QIPB200_OK) st = check_plan_cut("purity_plan", n_qubits, qubits, k);
    if (st != QIPB200_OK) return st;
    const uint32_t sb = std::min(k, n_qubits - k);
    out4[0] = purity_route(sb);
    out4[1] = sb;
    out4[2] = (uint32_t)purity_launch_count(sb);
    out4[3] = out4[0] == 2 ? (uint32_t)purity_gram_blocks(sb) : 0;
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// entanglement spectrum of a bipartition (purity.cu store epilogue + spectrum.cu)
// ===================================================================================

namespace {

// Device bytes of G for a side of s qubits (0 on the s = 0 route, which needs no matrix).
uint64_t spectrum_matrix_bytes(uint32_t s) { return s == 0 ? 0 : (16ull << (2 * s)); }

uint64_t spectrum_launch_count(uint32_t s) {
  switch (purity_route(s)) {
    case 0: return 1;
    case 1: return rdm_launch_count(s);
    default: return 1;
  }
}

int spectrum_side_too_large(const qipb200_ctx *ctx, const std::string &who, uint32_t sb) {
  return set_err(ctx, QIPB200_ERR_UNSUPPORTED,
                 who + ": the smaller side has " + std::to_string(sb) +
                     " qubits; at most 13 are supported (the matrix of 14 would be 4 GiB or more)");
}

// out2[0] = sum of the diagonal in index order; out2[1] = -sum p ln p over the eigenvalues > 0 in ascending order,
// p = lambda / T; eigs = the eigenvalues in descending order.  cuSOLVER's values are ascending only up to rounding
// among (nearly) equal ones, so they are sorted here first.
void spectrum_finish(std::vector<double> asc, double trace, double *eigs, double *out2) {
  std::sort(asc.begin(), asc.end());
  const size_t K = asc.size();
  double h = 0.0;
  if (trace != 0.0)
    for (size_t i = 0; i < K; ++i)
      if (asc[i] > 0.0) {
        const double p = asc[i] / trace;
        h -= p * std::log(p);
      }
  for (size_t i = 0; i < K; ++i) eigs[i] = asc[K - 1 - i];
  out2[0] = trace;
  out2[1] = h;
}

int spectrum_impl(qipb200_state *s, const uint64_t *qubits, uint32_t k, double *eigs, double *rho, double *out2) {
  qipb200_ctx *ctx = s->ctx;
  const std::vector<uint64_t> side = purity_side(s->n, qubits, k);
  const uint32_t sb = (uint32_t)side.size();
  const size_t K = (size_t)1 << sb;
  const uint32_t route = purity_route(sb);
  // The solver handle and every device buffer come before the state is touched: a refusal for memory leaves the
  // state and anything pending on it as they were.
  CU(ctx, cudaSetDevice(ctx->device));
  EigWork w;
  if (route != 0) {
    std::string err;
    const int st = eig_work_alloc(&ctx->eig_solver, (uint32_t)K, &w, ctx->stream, &err);
    if (st != QIPB200_OK) return set_err(ctx, st, "entanglement_spectrum: " + err);
  }
  struct Release {
    EigWork *w;
    cudaStream_t s;
    ~Release() {
      eig_work_free(w, s);
      cudaStreamSynchronize(s);
    }
  } release{&w, ctx->stream};
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  // A state left permuted (QIPB200_ROTATE) is read where it is, as by purity.
  std::vector<uint32_t> pos(sb);
  phys_positions(s, side.data(), sb, pos.data());
  double trace = 0.0;
  if (route == 0) {
    CU(ctx, run_purity_norm2(s->prec, s->buf, s->n_local, &trace, ctx->stream, &ctx->launches));
    spectrum_finish(std::vector<double>(1, trace), trace, eigs, out2);
    return QIPB200_OK;
  }
  std::vector<double> diag(K);
  if (route == 1) {
    std::unique_ptr<double[]> own(rho ? nullptr : new double[2 * K * K]);  // rho itself when given
    double *host = rho ? rho : own.get();
    CU(ctx, run_reduced_density(s->prec, s->buf, s->n_local, pos.data(), sb, host, ctx->stream, &ctx->launches));
    for (size_t a = 0; a < K; ++a) diag[a] = host[2 * (a * K + a)];
    CU(ctx, cudaMemcpyAsync(w.G, host, 16 * K * K, cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));  // own is released when this block ends
  } else {
    CU(ctx, run_gram_store(s->prec, s->buf, s->n_local, pos.data(), sb, w.G, ctx->stream, &ctx->launches));
    if (rho) CU(ctx, cudaMemcpyAsync(rho, w.G, 16 * K * K, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpy2DAsync(diag.data(), sizeof(double), w.G, (K + 1) * sizeof(double2), sizeof(double), K,
                              cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
  }
  for (size_t a = 0; a < K; ++a) trace += diag[a];
  std::vector<double> asc(K);
  std::string err;
  st = eig_solve(ctx->eig_solver, &w, ctx->stream, asc.data(), &err);
  if (st != QIPB200_OK) return set_err(ctx, st, "entanglement_spectrum: " + err);
  spectrum_finish(asc, trace, eigs, out2);
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_entanglement_spectrum(qipb200_state *s, const uint64_t *qubits, uint32_t k, double *eigs,
                                                   size_t eigs_cap, double *rho, double *out2) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "entanglement_spectrum: NULL state");
  return guarded(s->ctx, [&]() -> int {
    if (!eigs || !out2) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, "entanglement_spectrum: NULL eigs or out2");
    int st = check_indices(s, qubits, k);
    if (st == QIPB200_OK) st = require_unsharded(s, "entanglement_spectrum");
    if (st != QIPB200_OK) return st;
    const uint32_t sb = std::min(k, s->n - k);
    if (sb > kSpectrumMaxSide) return spectrum_side_too_large(s->ctx, "entanglement_spectrum", sb);
    if (eigs_cap < ((size_t)1 << sb))
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG,
                     "entanglement_spectrum: eigs_cap " + std::to_string(eigs_cap) + " is below the " +
                         std::to_string(1ull << sb) + " eigenvalues of the side");
    if (rho && k > s->n - k)
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG,
                     "entanglement_spectrum: rho is the matrix of the smaller side; k > n - k, so pass the "
                     "complement of these qubits to get it");
    std::string why;
    if (sb > 0 && !eig_solver_available(&why))
      return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, "entanglement_spectrum: the eigen-solver is unavailable: " + why);
    return spectrum_impl(s, qubits, k, eigs, rho, out2);
  });
}

extern "C" int qipb200_entanglement_spectrum_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, uint32_t k,
                                                  uint32_t *out5) {
  return guarded(nullptr, [&]() -> int {
    int st = check_plan_args("entanglement_spectrum_plan", prec, n_qubits, out5, "out5");
    if (st == QIPB200_OK) st = check_plan_cut("entanglement_spectrum_plan", n_qubits, qubits, k);
    if (st != QIPB200_OK) return st;
    const uint32_t sb = std::min(k, n_qubits - k);
    if (sb > kSpectrumMaxSide) return spectrum_side_too_large(nullptr, "entanglement_spectrum_plan", sb);
    out5[0] = purity_route(sb);
    out5[1] = sb;
    out5[2] = (uint32_t)spectrum_launch_count(sb);
    out5[3] = (uint32_t)spectrum_matrix_bytes(sb);
    out5[4] = eig_solver_available(nullptr) ? 1 : 0;
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// Pauli-string rotations (pauli_rot.cu)
// ===================================================================================

namespace {

int pauli_rot_impl(qipb200_state *s, const std::vector<PauliTerm> &terms, const double *angles) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  // A state left permuted (QIPB200_ROTATE) is rotated where it is: Pauli masks permute with the bits.
  const std::vector<PauliTerm> phys = phys_terms(s, terms);
  CU(ctx, run_pauli_rotations(s->prec, s->buf, s->n_local, phys, angles, 2 * ctx->sm_count, ctx->stream,
                              &ctx->launches));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_apply_pauli_rotations(qipb200_state *s, const uint64_t *qubits, const char *paulis,
                                                   const uint32_t *term_len, size_t n_terms, const double *angles) {
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "apply_pauli_rotations: NULL state");
  return guarded(s->ctx, [&]() -> int {
    // every term and angle is checked before any device work: a refused call leaves the state as it was
    const char *who = "apply_pauli_rotations";
    std::vector<PauliTerm> terms;
    int st = parse_terms(s->ctx, s->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_finite(s->ctx, angles, n_terms, who, "angle");
    if (st == QIPB200_OK) st = require_unsharded(s, who);
    if (st != QIPB200_OK) return st;
    if (n_terms == 0) return (int)QIPB200_OK;
    return pauli_rot_impl(s, terms, angles);
  });
}

extern "C" int qipb200_pauli_rotation_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits,
                                           const char *paulis, const uint32_t *term_len, size_t n_terms,
                                           uint32_t *sweeps) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args("pauli_rotation_plan", prec, n_qubits, sweeps, "sweeps");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    *sweeps = pauli_rotation_sweep_count(n_qubits, terms);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// noise channels along quantum trajectories (channel.cu)
// ===================================================================================

namespace {

int parse_channel_list(const qipb200_ctx *ctx, const std::string &who, uint32_t n, size_t n_channels,
                       const uint32_t *arity, const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus,
                       ChannelSet *cs) {
  std::string err;
  const uint32_t max_kraus = arity ? kChanMaxKrausMulti : kChanMaxKraus;
  const int st = parse_channels(who, n, n_channels, arity, qubits, n_kraus, kraus, max_kraus, cs, &err);
  return st == QIPB200_OK ? st : set_err(ctx, st, err);
}

// x over the state-dependent channels' qubits in channel order, each channel's in its qubit order:
// qipb200_state_sample's kernels with draws[0].
int channels_sample(qipb200_state *s, const std::string &who, const ChannelSet &cs, double draw, uint64_t *x) {
  qipb200_ctx *ctx = s->ctx;
  if (!layout_is_identity(s)) {  // the scan runs over canonical indices
    int st = restore_layout(s);
    if (st != QIPB200_OK) return st;
  }
  SampleBits bits;
  bits.n_bits = 0;
  for (size_t c = 0; c < cs.size(); ++c)
    for (uint32_t i = cs.qfirst[c]; cs.dep[c] && i < cs.qfirst[c + 1]; ++i)
      bits.bitpos[bits.n_bits++] = s->n - 1 - (uint32_t)cs.qubits[i];
  char *d = nullptr;
  CU(ctx, cudaMallocAsync((void **)&d, 16 + sample_scratch_bytes(s->n_local, 1), ctx->stream));
  cudaError_t e = cudaMemcpyAsync(d, &draw, sizeof(draw), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess)
    e = launch_sample(s->prec, s->buf, s->n_local, (const double *)d, 1, bits, d + 16, (uint64_t *)(d + 8),
                      ctx->sm_count, ctx->stream, &ctx->launches);
  if (e == cudaSuccess) e = cudaMemcpyAsync(x, d + 8, sizeof(*x), cudaMemcpyDeviceToHost, ctx->stream);
  cudaError_t ef = cudaFreeAsync(d, ctx->stream);
  if (e != cudaSuccess) return cuda_fail(ctx, e, (who + ": sample").c_str());
  CU(ctx, ef);
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

int channels_impl(qipb200_state *s, const std::string &who, const ChannelSet &cs, const double *draws,
                  uint32_t *chosen, double *prob) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  uint64_t x = 0;
  if (cs.n_dep && (st = channels_sample(s, who, cs, draws[0], &x)) != QIPB200_OK) return st;
  // the choices, then the chosen operators that are not positive multiples of the identity
  std::vector<const ChannelOp *> rest;
  std::vector<uint64_t> rest_q;
  double dropped = 1.0, uniform = 1.0;
  bool nonuniform = false;
  uint32_t k_dep = 0;  // the bit of x of the next state-dependent channel's first qubit
  for (size_t c = 0; c < cs.size(); ++c) {
    const uint32_t k = cs.qfirst[c + 1] - cs.qfirst[c];
    uint32_t b = 0;  // x's bits of the channel in the matrix convention: its first qubit the most significant
    for (uint32_t i = 0; cs.dep[c] && i < k; ++i) b = (b << 1) | (uint32_t)((x >> (k_dep + i)) & 1);
    k_dep += cs.dep[c] ? k : 0;
    chosen[c] = channel_choose(cs, c, b, draws[1 + c]);
    const ChannelOp &K = cs.ops[cs.first[c] + chosen[c]];
    if (channel_op_is_scaled_identity(K)) {
      dropped *= K.e[0];
      continue;
    }
    rest.push_back(&K);
    rest_q.insert(rest_q.end(), cs.qubits.begin() + cs.qfirst[c], cs.qubits.begin() + cs.qfirst[c + 1]);
    bool flat = true;
    for (uint32_t v = 1; v < (1u << k); ++v) flat = flat && K.e[v] == K.e[0];
    if (!flat)
      nonuniform = true;
    else
      uniform *= K.e[0];
  }
  if (rest.empty()) {
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    *prob = dropped;
    return QIPB200_OK;
  }
  // A permuted layout (QIPB200_ROTATE, no state-dependent channel) is worked on where it is.
  std::vector<uint32_t> pos(rest_q.size());
  phys_positions(s, rest_q.data(), (uint32_t)rest_q.size(), pos.data());
  ChannelTables t;
  build_channel_tables(pos.data(), rest.data(), rest.size(), &t);
  char *d = nullptr;
  CU(ctx, cudaMallocAsync((void **)&d, channel_scratch_bytes(), ctx->stream));
  double q = uniform;
  cudaError_t e = cudaSuccess;
  if (nonuniform) {
    double S = 0.0, N = 0.0;
    e = run_channel_weight(s->prec, s->buf, s->n_local, t, d, ctx->stream, &ctx->launches, &S, &N);
    q = N > 0.0 ? S / N : 0.0;
  }
  if (e == cudaSuccess && q > 0.0)  // q == 0 (a zero state): untouched
    e = run_channel_apply(s->prec, s->buf, s->n_local, t, 1.0 / std::sqrt(q), d, ctx->sm_count, ctx->stream,
                          &ctx->launches);
  cudaError_t ef = cudaFreeAsync(d, ctx->stream);
  if (e != cudaSuccess) return cuda_fail(ctx, e, who.c_str());
  CU(ctx, ef);
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  *prob = q * dropped;
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_apply_channels(qipb200_state *s, size_t n_channels, const uint64_t *qubits,
                                            const uint32_t *n_kraus, const double *kraus, const double *draws,
                                            uint32_t *chosen, double *prob) {
  const std::string who = "apply_channels";
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(s->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the state (and a pending collapse) as it was
    if (!prob) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL prob");
    if (n_channels && (!draws || !chosen))
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL draws or chosen");
    ChannelSet cs;
    int st = parse_channel_list(s->ctx, who, s->n, n_channels, nullptr, qubits, n_kraus, kraus, &cs);
    if (st != QIPB200_OK) return st;
    for (size_t k = 0; n_channels && k <= n_channels; ++k)
      if (!(draws[k] >= 0.0 && draws[k] < 1.0))
        return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": draw " + std::to_string(k) + " is not in [0, 1)");
    if ((st = require_unsharded(s, who)) != QIPB200_OK) return st;
    if (n_channels == 0) {
      *prob = 1.0;
      return (int)QIPB200_OK;
    }
    return channels_impl(s, who, cs, draws, chosen, prob);
  });
}

extern "C" int qipb200_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels, const uint64_t *qubits,
                                     const uint32_t *n_kraus, const double *kraus, uint32_t *out4) {
  const std::string who = "channels_plan";
  return guarded(nullptr, [&]() -> int {
    ChannelSet cs;
    int st = check_plan_args(who, prec, n_qubits, out4, "out4");
    if (st == QIPB200_OK)
      st = parse_channel_list(nullptr, who, n_qubits, n_channels, nullptr, qubits, n_kraus, kraus, &cs);
    if (st != QIPB200_OK) return st;
    plan_channels(cs, out4);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_apply_multiqubit_channels(qipb200_state *s, size_t n_channels, const uint32_t *arity,
                                                       const uint64_t *qubits, const uint32_t *n_kraus,
                                                       const double *kraus, const double *draws, uint32_t *chosen,
                                                       double *prob) {
  const std::string who = "apply_multiqubit_channels";
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(s->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the state (and a pending collapse) as it was
    if (!prob) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL prob");
    if (n_channels && (!draws || !chosen))
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL draws or chosen");
    if (n_channels && !arity)
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL arity, qubits, n_kraus or kraus");
    ChannelSet cs;
    int st = parse_channel_list(s->ctx, who, s->n, n_channels, arity, qubits, n_kraus, kraus, &cs);
    if (st != QIPB200_OK) return st;
    for (size_t k = 0; n_channels && k <= n_channels; ++k)
      if (!(draws[k] >= 0.0 && draws[k] < 1.0))
        return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": draw " + std::to_string(k) + " is not in [0, 1)");
    if ((st = require_unsharded(s, who)) != QIPB200_OK) return st;
    if (n_channels == 0) {
      *prob = 1.0;
      return (int)QIPB200_OK;
    }
    return channels_impl(s, who, cs, draws, chosen, prob);
  });
}

extern "C" int qipb200_multiqubit_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels,
                                                const uint32_t *arity, const uint64_t *qubits,
                                                const uint32_t *n_kraus, const double *kraus, uint32_t *out4) {
  const std::string who = "multiqubit_channels_plan";
  return guarded(nullptr, [&]() -> int {
    ChannelSet cs;
    int st = check_plan_args(who, prec, n_qubits, out4, "out4");
    if (st == QIPB200_OK && n_channels && !arity)
      st = set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL arity, qubits, n_kraus or kraus");
    if (st == QIPB200_OK)
      st = parse_channel_list(nullptr, who, n_qubits, n_channels, arity, qubits, n_kraus, kraus, &cs);
    if (st != QIPB200_OK) return st;
    plan_channels(cs, out4);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// general Kraus channels along quantum trajectories (kraus.cu)
// ===================================================================================

namespace {

// K * (1 / sqrt(p)) in double, each part rounded once to the state's precision: 4^k complex<prec>, row-major.
std::vector<unsigned char> kraus_scaled(qip_prec prec, const double *K, uint32_t k, double p) {
  const double inv = 1.0 / std::sqrt(p);
  const size_t E = 2ull << (2 * k);
  std::vector<unsigned char> out(E * (prec == QIP_F32 ? sizeof(float) : sizeof(double)));
  for (size_t i = 0; i < E; ++i) {
    const double v = K[i] * inv;
    if (prec == QIP_F32)
      ((float *)out.data())[i] = (float)v;
    else
      ((double *)out.data())[i] = v;
  }
  return out;
}

int kraus_impl(qipb200_state *s, const std::string &who, const KrausSet &ks, const double *draws, uint32_t *chosen,
               double *cond) {
  qipb200_ctx *ctx = s->ctx;
  int st = begin_device_work(s);
  if (st != QIPB200_OK) return st;
  const size_t nc = ks.size();
  std::fill(cond, cond + nc, 0.0);
  std::fill(chosen, chosen + nc, 0u);
  // the rdm positions of a group: bit i of the matrix index <-> its (m - 1 - i)-th qubit, so that the index is in
  // the matrix convention over the group's qubits in channel order
  auto group_pos = [&](const std::vector<size_t> &g, uint32_t *pos) {
    std::vector<uint64_t> q;
    for (size_t c : g) q.insert(q.end(), ks.qubits.begin() + ks.qfirst[c], ks.qubits.begin() + ks.qfirst[c + 1]);
    std::reverse(q.begin(), q.end());
    phys_positions(s, q.data(), (uint32_t)q.size(), pos);
    return (uint32_t)q.size();
  };
  const std::vector<std::vector<size_t>> groups = kraus_groups(ks);
  if (!groups.empty()) {
    std::vector<double> rho(2 << (2 * kKrausGroupBits));
    uint32_t pos[kKrausGroupBits];
    uint32_t m = group_pos(groups[0], pos);
    CU(ctx, run_reduced_density(s->prec, s->buf, s->n_local, pos, m, rho.data(), ctx->stream, &ctx->launches));
    char *d = nullptr;
    CU(ctx, cudaMallocAsync((void **)&d, kraus_scratch_bytes(), ctx->stream));
    cudaError_t e = cudaSuccess;
    bool zero = false;
    for (size_t gi = 0; gi < groups.size() && e == cudaSuccess; ++gi) {
      if (!kraus_draw_group(ks, groups[gi], rho.data(), draws, chosen, cond)) {  // Tr rho = 0: a zero state
        zero = true;
        break;
      }
      std::vector<KrausApplyOp> ops;
      for (size_t c : groups[gi]) {
        KrausApplyOp o;
        o.k = ks.arity(c);
        phys_positions(s, ks.qubits.data() + ks.qfirst[c], o.k, o.pos);
        o.mat = kraus_scaled(s->prec, ks.mat[ks.first[c] + chosen[c]], o.k, cond[c]);
        ops.push_back(std::move(o));
      }
      m = gi + 1 < groups.size() ? group_pos(groups[gi + 1], pos) : 0;
      e = run_kraus_sweep(s->prec, s->buf, s->n_local, ops, pos, m, rho.data(), d, ctx->stream, &ctx->launches);
    }
    const cudaError_t ef = cudaFreeAsync(d, ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, who.c_str());
    CU(ctx, ef);
    if (zero) {
      std::fill(cond, cond + nc, 0.0);
      std::fill(chosen, chosen + nc, 0u);
      CU(ctx, cudaStreamSynchronize(ctx->stream));
      return QIPB200_OK;
    }
  }
  // the state-independent channels: drawn from their weights, K / sqrt(w) through the fused schedule
  std::vector<qip_op> sched;
  std::vector<std::vector<unsigned char>> dense;
  dense.reserve(nc);
  for (size_t c = 0; c < nc; ++c) {
    if (!ks.indep[c]) continue;
    const uint32_t f = ks.first[c], k = ks.arity(c);
    chosen[c] = kraus_choose(ks.w.data() + f, ks.first[c + 1] - f, draws[c]);
    cond[c] = ks.w[f + chosen[c]];
    const double *K = ks.mat[f + chosen[c]];
    if (kraus_is_scaled_identity(K, k)) continue;
    dense.push_back(kraus_scaled(s->prec, K, k, cond[c]));
    qip_op op;
    memset(&op, 0, sizeof(op));
    op.kind = QIP_OP_MATRIX;
    op.n_indices = k;
    op.n_entries = 1ull << (2 * k);
    op.indices = ks.qubits.data() + ks.qfirst[c];
    op.dense = dense.back().data();
    sched.push_back(op);
  }
  if (!sched.empty() && (st = qipb200_state_apply_schedule(s, sched.data(), sched.size(), 0)) != QIPB200_OK)
    return st;
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_apply_kraus_channels(qipb200_state *s, size_t n_channels, const uint32_t *arity,
                                                  const uint64_t *qubits, const uint32_t *n_kraus,
                                                  const double *kraus, const double *draws, uint32_t *chosen,
                                                  double *cond, double *prob) {
  const std::string who = "apply_kraus_channels";
  if (!s) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(s->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the state (and a pending collapse) as it was
    if (!prob) return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL prob");
    if (n_channels && (!draws || !chosen))
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL draws or chosen");
    KrausSet ks;
    std::string err;
    int st = parse_kraus_channels(who, s->n, n_channels, arity, qubits, n_kraus, kraus, &ks, &err);
    if (st != QIPB200_OK) return set_err(s->ctx, st, err);
    for (size_t k = 0; k < n_channels; ++k)
      if (!(draws[k] >= 0.0 && draws[k] < 1.0))
        return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": draw " + std::to_string(k) + " is not in [0, 1)");
    if ((st = require_unsharded(s, who)) != QIPB200_OK) return st;
    if (n_channels == 0) {
      *prob = 1.0;
      return (int)QIPB200_OK;
    }
    std::vector<double> cd(n_channels, 0.0);
    if ((st = kraus_impl(s, who, ks, draws, chosen, cd.data())) != QIPB200_OK) return st;
    double p = 1.0;
    for (size_t c = 0; c < n_channels; ++c) p *= cd[c];
    *prob = p;
    if (cond) std::copy(cd.begin(), cd.end(), cond);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_kraus_channels_plan(qip_prec prec, uint32_t n_qubits, size_t n_channels,
                                           const uint32_t *arity, const uint64_t *qubits, const uint32_t *n_kraus,
                                           const double *kraus, uint32_t *out4) {
  const std::string who = "kraus_channels_plan";
  return guarded(nullptr, [&]() -> int {
    KrausSet ks;
    std::string err;
    int st = check_plan_args(who, prec, n_qubits, out4, "out4");
    if (st != QIPB200_OK) return st;
    if ((st = parse_kraus_channels(who, n_qubits, n_channels, arity, qubits, n_kraus, kraus, &ks, &err)) !=
        QIPB200_OK)
      return set_err(nullptr, st, err);
    plan_kraus_channels(ks, out4);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// density matrices (density.cu)
// ===================================================================================

namespace {

// The n of a density matrix held by rho (2n qubits), or the refusal: a sharded state, an odd qubit count.
int density_qubits(const qipb200_state *rho, const std::string &who, uint32_t *n) {
  int st = require_unsharded(rho, who);
  if (st != QIPB200_OK) return st;
  if (rho->n % 2)
    return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG,
                   who + ": a density matrix is a state of an even number of qubits, got " + std::to_string(rho->n));
  *n = rho->n / 2;
  return QIPB200_OK;
}

// psi of n qubits in rho's context and precision, unsharded.
int density_check_psi(const qipb200_state *rho, const qipb200_state *psi, uint32_t n, const std::string &who) {
  if (psi->ctx != rho->ctx || psi->prec != rho->prec || psi->n != n)
    return set_err(rho->ctx, QIPB200_ERR_SIZE_MISMATCH,
                   who + ": psi must have the density matrix's context and precision and " + std::to_string(n) +
                       " qubits");
  return require_unsharded(psi, who);
}

// psi's pending work applied and its qubits back in the canonical layout.
int density_prepare_psi(qipb200_state *psi) {
  int st = materialise_pending(psi);
  if (st == QIPB200_OK && !layout_is_identity(psi)) st = restore_layout(psi);
  return st;
}

// k distinct qubits below n (k == 0 allowed when zero_ok).
int density_check_qubits(const qipb200_state *rho, const std::string &who, uint32_t n, const uint64_t *qubits,
                         uint32_t k, bool zero_ok) {
  if ((k && !qubits) || (!zero_ok && k == 0) || k > n)
    return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": bad qubit list");
  uint64_t seen = 0;
  for (uint32_t i = 0; i < k; ++i) {
    if (qubits[i] >= n) return set_err(rho->ctx, QIPB200_ERR_BAD_INDEX, who + ": qubit index out of range");
    if ((seen >> qubits[i]) & 1) return set_err(rho->ctx, QIPB200_ERR_BAD_INDEX, who + ": repeated qubit index");
    seen |= 1ull << qubits[i];
  }
  return QIPB200_OK;
}

// Physical index bits of row qubit q (state qubit q) and of column qubit q (state qubit n + q).
uint64_t row_bit(const qipb200_state *rho, uint32_t n, uint64_t q) { return 1ull << rho->phys_of_logical[2 * n - 1 - q]; }
uint64_t col_bit(const qipb200_state *rho, uint32_t n, uint64_t q) { return 1ull << rho->phys_of_logical[n - 1 - q]; }

// The traced qubits (every qubit not in qubits[0..k)), ascending: the low key bits of run_density_sums.
std::vector<uint64_t> density_trace_masks(const qipb200_state *rho, uint32_t n, const uint64_t *qubits, uint32_t k) {
  uint64_t kept = 0;
  for (uint32_t i = 0; i < k; ++i) kept |= 1ull << qubits[i];
  std::vector<uint64_t> m;
  for (uint32_t q = 0; q < n; ++q)
    if (!((kept >> q) & 1)) m.push_back(row_bit(rho, n, q) | col_bit(rho, n, q));
  return m;
}

}  // namespace

extern "C" int qipb200_density_apply(qipb200_state *rho, const qip_op *ops, size_t n_ops, size_t n_channels,
                                     const uint64_t *channel_pos, const uint32_t *arity, const uint64_t *qubits,
                                     const uint32_t *n_kraus, const double *kraus, uint32_t flags) {
  const std::string who = "density_apply";
  if (!rho) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves rho (and anything pending) as it was
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st != QIPB200_OK) return st;
    DensitySchedule d;
    std::string err;
    st = build_density_schedule(who, rho->prec, n, ops, n_ops, n_channels, channel_pos, arity, qubits, n_kraus, kraus,
                                &d, &err);
    if (st != QIPB200_OK) return set_err(rho->ctx, st, err);
    return qipb200_state_apply_schedule(rho, d.ops.data(), d.ops.size(), flags);
  });
}

extern "C" int qipb200_density_schedule(qip_prec prec, uint32_t n, const qip_op *ops, size_t n_ops, size_t n_channels,
                                        const uint64_t *channel_pos, const uint32_t *arity, const uint64_t *qubits,
                                        const uint32_t *n_kraus, const double *kraus, void *buf, size_t cap,
                                        size_t *len) {
  const std::string who = "density_schedule";
  return guarded(nullptr, [&]() -> int {
    if (!len) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL len");
    DensitySchedule d;
    std::string err;
    int st = build_density_schedule(who, prec, n, ops, n_ops, n_channels, channel_pos, arity, qubits, n_kraus, kraus,
                                    &d, &err);
    if (st != QIPB200_OK) return set_err(nullptr, st, err);
    const size_t need = qipb200_schedule_serialise(prec, 2 * n, d.ops.data(), d.ops.size(), nullptr, 0);
    if (need == 0) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": the schedule could not be written");
    *len = need;
    if (!buf || cap < need)
      return set_err(nullptr, QIPB200_ERR_SIZE_MISMATCH,
                     who + ": the schedule needs " + std::to_string(need) + " bytes, cap is " + std::to_string(cap));
    qipb200_schedule_serialise(prec, 2 * n, d.ops.data(), d.ops.size(), buf, cap);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_from_state(qipb200_state *rho, qipb200_state *psi) {
  const std::string who = "density_from_state";
  if (!rho || !psi) return set_err(rho ? rho->ctx : nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st == QIPB200_OK) st = density_check_psi(rho, psi, n, who);
    if (st != QIPB200_OK) return st;
    qipb200_ctx *ctx = rho->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = density_prepare_psi(psi)) != QIPB200_OK) return st;
    // every amplitude of rho is written: its pending work is dropped and its layout becomes the canonical one
    rho->collapse_pending = rho->init_pending = false;
    for (uint32_t b = 0; b < rho->n; ++b) rho->phys_of_logical[b] = b;
    CU(ctx, run_density_from_state(rho->prec, rho->buf, psi->buf, n, ctx->stream, &ctx->launches));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_measure_probs(qipb200_state *rho, const uint64_t *indices, uint32_t n_indices,
                                             double *out) {
  const std::string who = "density_measure_probs";
  if (!rho) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st == QIPB200_OK) st = density_check_qubits(rho, who, n, indices, n_indices, true);
    if (st != QIPB200_OK) return st;
    if (!out) return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL out");
    qipb200_ctx *ctx = rho->ctx;
    if ((st = begin_device_work(rho)) != QIPB200_OK) return st;
    std::vector<uint64_t> masks = density_trace_masks(rho, n, indices, n_indices);
    const uint32_t nb = (uint32_t)masks.size();
    for (uint32_t i = 0; i < n_indices; ++i) masks.push_back(row_bit(rho, n, indices[i]) | col_bit(rho, n, indices[i]));
    std::vector<double> sums(2ull << n_indices);
    CU(ctx, run_density_sums(rho->prec, rho->buf, masks, nb, n_indices, 0, sums.data(), ctx->stream, &ctx->launches));
    for (size_t m = 0; m < (1ull << n_indices); ++m) out[m] = sums[2 * m];
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_expect_paulis(qipb200_state *rho, const uint64_t *qubits, const char *paulis,
                                             const uint32_t *term_len, size_t n_terms, double *out) {
  const std::string who = "density_expect_paulis";
  if (!rho) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    std::vector<PauliTerm> terms;
    if (st == QIPB200_OK) st = parse_terms(rho->ctx, n, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    if (n_terms == 0) return (int)QIPB200_OK;
    if (!out) return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL out");
    qipb200_ctx *ctx = rho->ctx;
    if ((st = begin_device_work(rho)) != QIPB200_OK) return st;
    CU(ctx, run_density_expect(rho->prec, rho->buf, n, rho->phys_of_logical, terms, out, ctx->stream, &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_reduced(qipb200_state *rho, const uint64_t *qubits, uint32_t k, double *out) {
  const std::string who = "density_reduced";
  if (!rho) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st == QIPB200_OK) st = density_check_qubits(rho, who, n, qubits, k, false);
    if (st != QIPB200_OK) return st;
    if (!out) return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL out");
    if (k > kRdmMaxKept)
      return set_err(rho->ctx, QIPB200_ERR_UNSUPPORTED, who + ": at most 10 kept qubits, got " + std::to_string(k));
    qipb200_ctx *ctx = rho->ctx;
    if ((st = begin_device_work(rho)) != QIPB200_OK) return st;
    // key = b | a << nb | a' << (nb + k): a on the kept row qubits, a' on the kept column qubits
    std::vector<uint64_t> masks = density_trace_masks(rho, n, qubits, k);
    const uint32_t nb = (uint32_t)masks.size();
    for (uint32_t i = 0; i < k; ++i) masks.push_back(row_bit(rho, n, qubits[i]));
    for (uint32_t i = 0; i < k; ++i) masks.push_back(col_bit(rho, n, qubits[i]));
    std::vector<double> sums(2ull << (2 * k));
    CU(ctx, run_density_sums(rho->prec, rho->buf, masks, nb, 2 * k, k, sums.data(), ctx->stream, &ctx->launches));
    const size_t K = 1ull << k;
    for (size_t a = 0; a < K; ++a)
      for (size_t b = a; b < K; ++b) {
        const double *v = &sums[2 * (a | (b << k))];
        out[2 * (a * K + b)] = v[0];
        out[2 * (a * K + b) + 1] = a == b ? 0.0 : v[1];
        out[2 * (b * K + a)] = v[0];
        out[2 * (b * K + a) + 1] = a == b ? 0.0 : -v[1];
      }
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_fidelity(qipb200_state *rho, qipb200_state *psi, double *out2) {
  const std::string who = "density_fidelity";
  if (!rho || !psi) return set_err(rho ? rho->ctx : nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st == QIPB200_OK) st = density_check_psi(rho, psi, n, who);
    if (st != QIPB200_OK) return st;
    if (!out2) return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL out2");
    qipb200_ctx *ctx = rho->ctx;
    if ((st = begin_device_work(rho)) != QIPB200_OK) return st;
    if ((st = density_prepare_psi(psi)) != QIPB200_OK) return st;
    CU(ctx, run_density_fidelity(rho->prec, rho->buf, psi->buf, n, rho->phys_of_logical, out2, ctx->stream,
                                 &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_density_spectrum(qipb200_state *rho, double *eigs) {
  const std::string who = "density_spectrum";
  if (!rho) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(rho->ctx, [&]() -> int {
    uint32_t n = 0;
    int st = density_qubits(rho, who, &n);
    if (st != QIPB200_OK) return st;
    if (!eigs) return set_err(rho->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL eigs");
    if (n > kDensitySpectrumMax)
      return set_err(rho->ctx, QIPB200_ERR_UNSUPPORTED,
                     who + ": " + std::to_string(n) + " qubits; at most 13 are supported (the matrix of 14 is 4 GiB)");
    std::string why;
    if (!eig_solver_available(&why))
      return set_err(rho->ctx, QIPB200_ERR_UNSUPPORTED, who + ": the eigen-solver is unavailable: " + why);
    qipb200_ctx *ctx = rho->ctx;
    const size_t K = 1ull << n;
    // the solver's buffers come before rho is touched: a refusal for memory leaves it and anything pending as it was
    CU(ctx, cudaSetDevice(ctx->device));
    EigWork w;
    std::string err;
    st = eig_work_alloc(&ctx->eig_solver, (uint32_t)K, &w, ctx->stream, &err);
    if (st != QIPB200_OK) return set_err(ctx, st, who + ": " + err);
    struct Release {
      EigWork *w;
      cudaStream_t s;
      ~Release() {
        eig_work_free(w, s);
        cudaStreamSynchronize(s);
      }
    } release{&w, ctx->stream};
    if ((st = begin_device_work(rho)) != QIPB200_OK) return st;
    CU(ctx, run_density_widen(rho->prec, rho->buf, n, rho->phys_of_logical, w.G, ctx->stream, &ctx->launches));
    std::vector<double> asc(K);
    st = eig_solve(ctx->eig_solver, &w, ctx->stream, asc.data(), &err);
    if (st != QIPB200_OK) return set_err(ctx, st, who + ": " + err);
    std::sort(asc.begin(), asc.end());
    for (size_t i = 0; i < K; ++i) eigs[i] = asc[K - 1 - i];
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// classical function ops (function.cu)
// ===================================================================================

namespace {

// The in and out registers of an n-qubit state: NULL arrays, then every qubit in range and none repeated within or
// across the two registers.
int check_function_registers(const qipb200_ctx *ctx, const std::string &who, uint32_t n, const uint64_t *in_q,
                             uint32_t n_in, const uint64_t *out_q, uint32_t n_out) {
  if ((n_in && !in_q) || (n_out && !out_q)) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL qubit array");
  uint64_t seen = 0;
  for (int r = 0; r < 2; ++r) {
    const uint64_t *q = r ? out_q : in_q;
    const uint32_t m = r ? n_out : n_in;
    for (uint32_t i = 0; i < m; ++i) {
      if (q[i] >= n)
        return set_err(ctx, QIPB200_ERR_BAD_INDEX, who + ": qubit " + std::to_string(q[i]) + " out of range for " +
                                                       std::to_string(n) + " qubits");
      if ((seen >> q[i]) & 1)
        return set_err(ctx, QIPB200_ERR_BAD_INDEX, who + ": qubit " + std::to_string(q[i]) + " repeated");
      seen |= 1ull << q[i];
    }
  }
  return QIPB200_OK;
}

// n_in and n_out of a function: the limits function_new and function_plan share.
int check_function_sizes(const qipb200_ctx *ctx, const std::string &who, uint32_t n_in, uint32_t n_out) {
  if (n_in == 0) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": n_in must be at least 1");
  if (n_in > kFnMaxIn)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED,
                   who + ": at most 26 input qubits (the table of 2^n_in entries would exceed 1.25 GiB)");
  if (n_out > kFnMaxOut) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, who + ": at most 32 output qubits");
  return QIPB200_OK;
}

void free_function_tables(qipb200_function *fn) {
  cudaSetDevice(fn->ctx->device);
  if (fn->d_f) cudaFreeAsync(fn->d_f, fn->ctx->stream);
  if (fn->d_cs) cudaFreeAsync(fn->d_cs, fn->ctx->stream);
  fn->d_f = nullptr;
  fn->d_cs = nullptr;
}

// A code function's module cannot be unloaded in stream order: the context's stream is drained first.
void free_function_code(qipb200_function *fn) {
  if (!fn->code && !fn->d_scratch) return;
  cudaSetDevice(fn->ctx->device);
  cudaStreamSynchronize(fn->ctx->stream);
  function_code_free(fn->code);
  if (fn->d_scratch) cudaFreeAsync(fn->d_scratch, fn->ctx->stream);
  fn->code = nullptr;
  fn->d_scratch = nullptr;
}

// n_in, n_out, flags, n_params and source of a code function: the checks function_new_code and function_code_compile
// share.
int check_code_args(const qipb200_ctx *ctx, const std::string &who, uint32_t n_in, uint32_t n_out, const char *source,
                    uint32_t flags, uint32_t n_params) {
  if (!source || !*source) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL or empty source");
  if (n_in == 0) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": n_in must be at least 1");
  if (flags & ~(uint32_t)QIPB200_FN_CODE_THETA)
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": unknown flags " + std::to_string(flags));
  const bool theta = flags & QIPB200_FN_CODE_THETA;
  if (!n_out && !theta)
    return set_err(ctx, QIPB200_ERR_INVALID_ARG,
                   who + ": no output qubits and no QIPB200_FN_CODE_THETA: nothing to apply");
  if (n_params > kFnCodeMaxParams)
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": at most 16 parameters, got " + std::to_string(n_params));
  if (n_out > kFnMaxOut) return set_err(ctx, QIPB200_ERR_UNSUPPORTED, who + ": at most 32 output qubits");
  if (n_in + n_out > kFnCodeMaxBits)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED,
                   who + ": n_in + n_out = " + std::to_string(n_in + n_out) +
                       " exceeds 34 (no state on one device is larger)");
  return QIPB200_OK;
}

void copy_log(char *log, size_t log_len, const std::string &msg) {
  if (log && log_len) snprintf(log, log_len, "%s", msg.c_str());
}

// A code function's status with msg (the NVRTC log for a compile error) in the last error and in log.
int code_fail(const qipb200_ctx *ctx, const std::string &who, int st, const std::string &msg, char *log,
              size_t log_len) {
  copy_log(log, log_len, msg);
  const char *what = st == QIPB200_ERR_INVALID_ARG    ? ": the source does not compile:\n"
                     : st == QIPB200_ERR_UNSUPPORTED ? ": code functions need NVRTC and the driver API: "
                                                      : ": ";
  return set_err(ctx, st, who + what + msg);
}

// A code-function call that failed with e: the driver's launch error in err when it gave one, else e of what.
int code_error(const qipb200_ctx *ctx, const std::string &who, cudaError_t e, const std::string &err, const char *what) {
  return err.empty() ? cuda_fail(ctx, e, what) : set_err(ctx, QIPB200_ERR_CUDA, who + ": " + err);
}

// theta(x, params) is finite for every x < 2^n_in, or the error that names the first x where it is not.
int check_code_theta(qipb200_function *fn, const double *params, const std::string &who) {
  qipb200_ctx *ctx = fn->ctx;
  uint64_t first = 0;
  std::string err;
  cudaError_t e = function_code_first_bad(fn->code, false, fn->n_in, fn->n_out, params, (uint64_t *)fn->d_scratch,
                                          ctx->sm_count, ctx->stream, &first, &err);
  ++ctx->launches;
  if (e != cudaSuccess) return code_error(ctx, who, e, err, "function_code_first_bad");
  if (first != ~0ull)
    return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": theta(" + std::to_string(first) + ") is not finite");
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_function_new(qipb200_ctx *ctx, uint32_t n_in, uint32_t n_out, const uint64_t *f,
                                    const double *theta, qipb200_function **out) {
  const std::string who = "function_new";
  if (!ctx || !out) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL context or out-pointer");
  *out = nullptr;
  return guarded(ctx, [&]() -> int {
    // the whole table is checked before anything is allocated
    int st = check_function_sizes(ctx, who, n_in, n_out);
    if (st != QIPB200_OK) return st;
    if (n_out && !f) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL f with n_out > 0");
    if (!n_out && !theta)
      return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": no output qubits and no theta: nothing to apply");
    const uint64_t N = 1ull << n_in;
    if (f)
      for (uint64_t x = 0; x < N; ++x)
        if (f[x] >> n_out)
          return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": f[" + std::to_string(x) + "] = " +
                                                           std::to_string(f[x]) + " does not fit in " +
                                                           std::to_string(n_out) + " output bits");
    if (theta)
      for (uint64_t x = 0; x < N; ++x)
        if (!std::isfinite(theta[x]))
          return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": theta[" + std::to_string(x) + "] is not finite");
    if (!ctx->children.empty())
      return set_err(ctx, QIPB200_ERR_UNSUPPORTED, who + ": multi-device contexts are not supported");
    // host copies first: an allocation failure here (std::bad_alloc) leaves nothing behind
    std::vector<uint32_t> hf(n_out ? N : 0);
    for (size_t x = 0; x < hf.size(); ++x) hf[x] = (uint32_t)f[x];
    std::vector<double2> hcs(theta ? N : 0);
    for (size_t x = 0; x < hcs.size(); ++x) hcs[x] = make_double2(cos(theta[x]), sin(theta[x]));
    qipb200_function *fn = new qipb200_function();
    fn->ctx = ctx;
    fn->n_in = n_in;
    fn->n_out = n_out;
    auto fail = [&](cudaError_t e, const char *what) {
      const int code = cuda_fail(ctx, e, what);
      free_function_tables(fn);
      delete fn;
      return code;
    };
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) return fail(e, "cudaSetDevice");
    if (n_out) {
      if ((e = cudaMallocAsync((void **)&fn->d_f, N * sizeof(uint32_t), ctx->stream)) != cudaSuccess)
        return fail(e, "cudaMallocAsync(function table)");
      if ((e = cudaMemcpyAsync(fn->d_f, hf.data(), N * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream)) !=
          cudaSuccess)
        return fail(e, "cudaMemcpyAsync(function table)");
    }
    if (theta) {
      if ((e = cudaMallocAsync((void **)&fn->d_cs, N * sizeof(double2), ctx->stream)) != cudaSuccess)
        return fail(e, "cudaMallocAsync(phase table)");
      if ((e = cudaMemcpyAsync(fn->d_cs, hcs.data(), N * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream)) !=
          cudaSuccess)
        return fail(e, "cudaMemcpyAsync(phase table)");
    }
    if ((e = cudaStreamSynchronize(ctx->stream)) != cudaSuccess) return fail(e, "cudaStreamSynchronize");
    *out = fn;
    return (int)QIPB200_OK;
  });
}

extern "C" void qipb200_function_free(qipb200_function *fn) {
  if (!fn) return;
  free_function_tables(fn);  // stream-ordered: an apply queued before runs first
  free_function_code(fn);
  delete fn;
}

extern "C" int qipb200_state_apply_function(qipb200_state *s, const qipb200_function *fn, const uint64_t *in_qubits,
                                            const uint64_t *out_qubits) {
  const std::string who = "apply_function";
  if (!s || !fn) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state or function");
  return guarded(s->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the state (and a pending collapse) as it was
    int st = check_function_registers(s->ctx, who, s->n, in_qubits, fn->n_in, out_qubits, fn->n_out);
    if (st == QIPB200_OK) st = require_unsharded(s, who);
    if (st != QIPB200_OK) return st;
    if (fn->ctx != s->ctx)
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": the function was made on another context");
    qipb200_ctx *ctx = s->ctx;
    if ((st = begin_device_work(s)) != QIPB200_OK) return st;
    // A permuted layout (QIPB200_ROTATE) needs no restore: the registers are read and written where their qubits are.
    uint32_t in_pos[kFnCodeMaxBits], out_pos[kFnMaxOut];
    phys_positions(s, in_qubits, fn->n_in, in_pos);
    phys_positions(s, out_qubits, fn->n_out, out_pos);
    if (fn->code) {
      std::string err;
      const cudaError_t e = run_function_code(s->prec, s->buf, s->n_local, in_pos, fn->n_in, out_pos, fn->n_out,
                                              fn->code, fn->params, ctx->sm_count, ctx->stream, &ctx->launches, &err);
      if (e != cudaSuccess) return code_error(ctx, who, e, err, "run_function_code");
      return (int)QIPB200_OK;
    }
    CU(ctx, run_function(s->prec, s->buf, s->n_local, in_pos, fn->n_in, out_pos, fn->n_out, fn->d_f, fn->d_cs,
                         ctx->sm_count, ctx->stream, &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_function_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *in_qubits, uint32_t n_in,
                                     const uint64_t *out_qubits, uint32_t n_out, uint32_t *out2) {
  const std::string who = "function_plan";
  return guarded(nullptr, [&]() -> int {
    int st = check_plan_args(who, prec, n_qubits, out2, "out2");
    if (st == QIPB200_OK) st = check_function_sizes(nullptr, who, n_in, n_out);
    if (st == QIPB200_OK) st = check_function_registers(nullptr, who, n_qubits, in_qubits, n_in, out_qubits, n_out);
    if (st != QIPB200_OK) return st;
    uint32_t out_pos[kFnMaxOut];
    for (uint32_t i = 0; i < n_out; ++i) out_pos[i] = n_qubits - 1 - (uint32_t)out_qubits[i];
    const FnPlan p = plan_function(prec, n_qubits, out_pos, n_out);
    out2[0] = p.path;
    out2[1] = p.tile_bits;
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_function_code_compile(uint32_t n_in, uint32_t n_out, const char *source, uint32_t flags,
                                             uint32_t n_params, char *log, size_t log_len) {
  const std::string who = "function_code_compile";
  copy_log(log, log_len, std::string());
  return guarded(nullptr, [&]() -> int {
    int st = check_code_args(nullptr, who, n_in, n_out, source, flags, n_params);
    if (st != QIPB200_OK) return st;
    std::string msg;
    if ((st = function_code_compile(n_out, source, flags & QIPB200_FN_CODE_THETA, &msg)) != QIPB200_OK)
      return code_fail(nullptr, who, st, msg, log, log_len);
    copy_log(log, log_len, msg);  // warnings, if any
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_function_new_code(qipb200_ctx *ctx, uint32_t n_in, uint32_t n_out, const char *source,
                                         uint32_t flags, uint32_t n_params, char *log, size_t log_len,
                                         qipb200_function **out) {
  const std::string who = "function_new_code";
  copy_log(log, log_len, std::string());
  if (!ctx || !out) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL context or out-pointer");
  *out = nullptr;
  return guarded(ctx, [&]() -> int {
    int st = check_code_args(ctx, who, n_in, n_out, source, flags, n_params);
    if (st != QIPB200_OK) return st;
    if (!ctx->children.empty())
      return set_err(ctx, QIPB200_ERR_UNSUPPORTED, who + ": multi-device contexts are not supported");
    CU(ctx, cudaSetDevice(ctx->device));
    const bool theta = flags & QIPB200_FN_CODE_THETA;
    std::string msg;
    FnCode *code = nullptr;
    if ((st = function_code_load(n_out, source, theta, &code, &msg)) != QIPB200_OK)
      return code_fail(ctx, who, st, msg, log, log_len);
    copy_log(log, log_len, msg);
    qipb200_function *fn = new qipb200_function();
    fn->ctx = ctx;
    fn->n_in = n_in;
    fn->n_out = n_out;
    fn->code = code;
    fn->theta = theta;
    fn->n_params = n_params;
    auto refuse = [&](int code_st) {
      free_function_code(fn);
      delete fn;
      return code_st;
    };
    cudaError_t e = cudaMallocAsync(&fn->d_scratch, (1 + kFnExpPartials) * sizeof(double), ctx->stream);
    if (e != cudaSuccess) return refuse(cuda_fail(ctx, e, "cudaMallocAsync(function scratch)"));
    std::string err;
    if (n_out) {  // every f(x) fits the out register
      uint64_t first = 0;
      e = function_code_first_bad(code, true, n_in, n_out, fn->params, (uint64_t *)fn->d_scratch, ctx->sm_count,
                                  ctx->stream, &first, &err);
      ++ctx->launches;
      uint64_t fx = 0;
      if (e == cudaSuccess && first != ~0ull)
        e = tabulate_function(code, fn->params, nullptr, nullptr, first, 1, &fx, nullptr, ctx->sm_count, ctx->stream,
                              &err);
      if (e != cudaSuccess) return refuse(code_error(ctx, who, e, err, "function_code_first_bad"));
      if (first != ~0ull)
        return refuse(set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": f(" + std::to_string(first) + ") = " +
                                                                std::to_string(fx) + " does not fit in " +
                                                                std::to_string(n_out) + " output bits"));
    }
    if (theta && (st = check_code_theta(fn, fn->params, who)) != QIPB200_OK) return refuse(st);
    *out = fn;
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_function_set_params(qipb200_function *fn, const double *params, uint32_t n_params) {
  const std::string who = "function_set_params";
  if (!fn) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL function");
  qipb200_ctx *ctx = fn->ctx;
  return guarded(ctx, [&]() -> int {
    if (!fn->code)
      return set_err(ctx, QIPB200_ERR_UNSUPPORTED, who + ": a table function has no parameters");
    if (n_params != fn->n_params)
      return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": the function takes " + std::to_string(fn->n_params) +
                                                       " parameters, got " + std::to_string(n_params));
    if (n_params && !params) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL params");
    double p[kFnCodeMaxParams] = {};
    for (uint32_t i = 0; i < n_params; ++i) p[i] = params[i];
    if (fn->theta) {
      CU(ctx, cudaSetDevice(ctx->device));
      const int st = check_code_theta(fn, p, who);
      if (st != QIPB200_OK) return st;  // the previous parameters stay
    }
    memcpy(fn->params, p, sizeof(p));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_function_tabulate(const qipb200_function *fn, uint64_t x0, uint64_t count, uint64_t *f_out,
                                         double *cs_out) {
  const std::string who = "function_tabulate";
  if (!fn) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL function");
  qipb200_ctx *ctx = fn->ctx;
  return guarded(ctx, [&]() -> int {
    const uint64_t N = 1ull << fn->n_in;
    if (x0 > N || count > N - x0)
      return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": [x0, x0 + count) exceeds 2^n_in = " + std::to_string(N));
    if (!count) return (int)QIPB200_OK;
    const bool phase = fn->code ? fn->theta : fn->d_cs != nullptr;
    if (cs_out && !phase)  // no phase: e^{i 0}
      for (uint64_t i = 0; i < count; ++i) {
        cs_out[2 * i] = 1.0;
        cs_out[2 * i + 1] = 0.0;
      }
    if (!f_out && !(cs_out && phase)) return (int)QIPB200_OK;
    CU(ctx, cudaSetDevice(ctx->device));
    std::string err;
    const cudaError_t e = tabulate_function(fn->code, fn->params, fn->d_f, fn->d_cs, x0, count, f_out,
                                            phase ? cs_out : nullptr, ctx->sm_count, ctx->stream, &err);
    ++ctx->launches;
    if (e != cudaSuccess) return code_error(ctx, who, e, err, "tabulate_function");
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_expect_function(qipb200_state *s, const qipb200_function *fn, const uint64_t *in_qubits,
                                             double *out) {
  const std::string who = "expect_function";
  if (!s || !fn || !out)
    return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state, function or out");
  return guarded(s->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the state (and a pending collapse) as it was
    if (!fn->code)
      return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED,
                     who + ": a table function keeps cos theta and sin theta, not theta: make it from code");
    if (!fn->theta)
      return set_err(s->ctx, QIPB200_ERR_UNSUPPORTED, who + ": the function has no theta (QIPB200_FN_CODE_THETA)");
    int st = check_function_registers(s->ctx, who, s->n, in_qubits, fn->n_in, nullptr, 0);
    if (st == QIPB200_OK) st = require_unsharded(s, who);
    if (st != QIPB200_OK) return st;
    if (fn->ctx != s->ctx)
      return set_err(s->ctx, QIPB200_ERR_INVALID_ARG, who + ": the function was made on another context");
    qipb200_ctx *ctx = s->ctx;
    if ((st = begin_device_work(s)) != QIPB200_OK) return st;
    uint32_t in_pos[kFnCodeMaxBits];
    phys_positions(s, in_qubits, fn->n_in, in_pos);
    std::string err;
    const cudaError_t e = expect_function_code(s->prec, s->buf, s->n_local, in_pos, fn->n_in, fn->code, fn->params,
                                               (double *)fn->d_scratch + 1, ctx->stream, &ctx->launches, out, &err);
    if (e != cudaSuccess) return code_error(ctx, who, e, err, "expect_function_code");
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// Pauli sums and the adjoint energy gradient (gradient.cu)
// ===================================================================================

extern "C" int qipb200_state_apply_pauli_sum(qipb200_state *dst, const qipb200_state *src, const uint64_t *qubits,
                                             const char *paulis, const uint32_t *term_len, size_t n_terms,
                                             const double *coeffs) {
  if (!dst || !src) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "apply_pauli_sum: NULL state");
  return guarded(dst->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves both states as they were
    std::vector<PauliTerm> terms;
    int st = check_state_pair(dst, src, "apply_pauli_sum");
    if (st == QIPB200_OK) st = parse_terms(dst->ctx, src->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_finite(dst->ctx, coeffs, n_terms, "apply_pauli_sum", "coefficient");
    if (st != QIPB200_OK) return st;
    qipb200_state *s = const_cast<qipb200_state *>(src);  // a pending collapse is applied: the state it stands for
    qipb200_ctx *ctx = dst->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = prepare_out_of_place(dst, s)) != QIPB200_OK) return st;
    CU(ctx, run_pauli_sum(src->prec, dst->buf, src->buf, src->n_local, phys_terms(src, terms), coeffs, ctx->stream,
                          &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_pauli_sum_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis,
                                      const uint32_t *term_len, size_t n_terms, uint32_t *sweeps) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args("pauli_sum_plan", prec, n_qubits, sweeps, "sweeps");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    *sweeps = pauli_sum_sweep_count(n_qubits, terms);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_pauli_energy_gradient(qipb200_state *state, qipb200_state *work, const uint64_t *qubits,
                                                   const char *paulis, const uint32_t *term_len, size_t n_terms,
                                                   const double *angles, const uint64_t *ham_qubits,
                                                   const char *ham_paulis, const uint32_t *ham_term_len, size_t n_ham,
                                                   const double *coeffs, double *energy, double *grad) {
  const char *who = "pauli_energy_gradient";
  if (!state || !work) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, std::string(who) + ": NULL state");
  return guarded(state->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves both states as they were
    std::vector<PauliTerm> ansatz, ham;
    int st = check_state_pair(work, state, who);
    if (st == QIPB200_OK) st = parse_terms(state->ctx, state->n, qubits, paulis, term_len, n_terms, &ansatz);
    if (st == QIPB200_OK) st = parse_terms(state->ctx, state->n, ham_qubits, ham_paulis, ham_term_len, n_ham, &ham);
    if (st == QIPB200_OK) st = check_finite(state->ctx, angles, n_terms, who, "angle");
    if (st == QIPB200_OK) st = check_finite(state->ctx, coeffs, n_ham, who, "coefficient");
    if (st != QIPB200_OK) return st;
    if (!energy) return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, std::string(who) + ": NULL energy");
    if (n_terms && !grad) return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, std::string(who) + ": NULL grad");
    qipb200_ctx *ctx = state->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = prepare_out_of_place(work, state)) != QIPB200_OK) return st;
    CU(ctx, run_pauli_gradient(state->prec, state->buf, work->buf, state->n_local, phys_terms(state, ansatz), angles,
                               phys_terms(state, ham), coeffs, 2 * ctx->sm_count, ctx->stream, &ctx->launches, energy,
                               grad));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_pauli_gradient_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits,
                                           const char *paulis, const uint32_t *term_len, size_t n_terms,
                                           const uint64_t *ham_qubits, const char *ham_paulis,
                                           const uint32_t *ham_term_len, size_t n_ham, uint32_t *out3) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> ansatz, ham;
    int st = check_plan_args("pauli_gradient_plan", prec, n_qubits, out3, "out3");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &ansatz);
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, ham_qubits, ham_paulis, ham_term_len, n_ham, &ham);
    if (st != QIPB200_OK) return st;
    out3[0] = pauli_rotation_sweep_count(n_qubits, ansatz);
    out3[1] = pauli_sum_sweep_count(n_qubits, ham);
    out3[2] = pauli_adjoint_sweep_count(n_qubits, ansatz);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// the quantum geometric tensor of a Pauli-rotation circuit (gradient.cu)
// ===================================================================================

namespace {

const size_t kQgtMaxTerms = 2048;  // the result alone is 2 T^2 doubles (64 MiB at this size)

int check_qgt_terms(qipb200_ctx *ctx, const std::string &who, size_t n_terms) {
  if (n_terms > kQgtMaxTerms)
    return set_err(ctx, QIPB200_ERR_UNSUPPORTED,
                   who + ": " + std::to_string(n_terms) + " terms, at most " + std::to_string(kQgtMaxTerms));
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_pauli_geometric_tensor(qipb200_state *state, qipb200_state *work_a,
                                                    qipb200_state *work_b, const uint64_t *qubits,
                                                    const char *paulis, const uint32_t *term_len, size_t n_terms,
                                                    const double *angles, double *qgt, double *expect) {
  const std::string who = "pauli_geometric_tensor";
  if (!state || !work_a || !work_b) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(state->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the three states (and a pending collapse) as
    // they were
    std::vector<PauliTerm> ansatz;
    int st = check_three_states(state, work_a, work_b, who);
    if (st == QIPB200_OK) st = parse_terms(state->ctx, state->n, qubits, paulis, term_len, n_terms, &ansatz);
    if (st == QIPB200_OK) st = check_finite(state->ctx, angles, n_terms, who, "angle");
    if (st != QIPB200_OK) return st;
    if (n_terms && !qgt) return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL qgt");
    if ((st = check_qgt_terms(state->ctx, who, n_terms)) != QIPB200_OK) return st;
    qipb200_ctx *ctx = state->ctx;
    if (n_terms == 0) return begin_device_work(state);  // the work states are not touched
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = prepare_work_states(state, work_a, work_b)) != QIPB200_OK) return st;
    CU(ctx, run_pauli_qgt(state->prec, state->buf, work_a->buf, work_b->buf, state->n_local,
                          phys_terms(state, ansatz), angles, ctx->stream, &ctx->launches, qgt, expect));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_pauli_geometric_tensor_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits,
                                                   const char *paulis, const uint32_t *term_len, size_t n_terms,
                                                   uint32_t *out3) {
  const std::string who = "pauli_geometric_tensor_plan";
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> ansatz;
    int st = check_plan_args(who, prec, n_qubits, out3, "out3");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &ansatz);
    if (st == QIPB200_OK) st = check_qgt_terms(nullptr, who, n_terms);
    if (st != QIPB200_OK) return st;
    const uint32_t T = (uint32_t)n_terms, S = pauli_qgt_sweep_count(n_qubits, ansatz);
    out3[0] = T;
    out3[1] = S;
    out3[2] = T ? T + 2 * S + 1 : 0;
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// exp(-iHt) for a real Pauli sum by a Chebyshev expansion (evolve.h, gradient.cu)
// ===================================================================================

namespace {

// The checks the evolution call and its plan share once the terms are parsed.
int check_evolution_args(qipb200_ctx *ctx, const std::string &who, const double *coeffs, size_t n_terms, double time,
                         double tol) {
  int st = check_finite(ctx, coeffs, n_terms, who, "coefficient");
  if (st != QIPB200_OK) return st;
  if (!std::isfinite(time)) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": time is not finite");
  if (!(tol > 0.0 && tol < 1.0)) return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": tol must be in (0, 1)");
  return QIPB200_OK;
}

}  // namespace

extern "C" int qipb200_state_evolve_pauli_sum(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b,
                                              const uint64_t *qubits, const char *paulis, const uint32_t *term_len,
                                              size_t n_terms, const double *coeffs, double time, double tol,
                                              uint32_t *degree, double *tail) {
  const std::string who = "evolve_pauli_sum";
  if (!state || !work_a || !work_b) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(state->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the three states (and a pending collapse) as
    // they were
    std::vector<PauliTerm> terms;
    int st = check_three_states(state, work_a, work_b, who);
    if (st == QIPB200_OK) st = parse_terms(state->ctx, state->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_evolution_args(state->ctx, who, coeffs, n_terms, time, tol);
    if (st != QIPB200_OK) return st;
    if (!degree || !tail) return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL degree or tail");
    EvolutionPlan p;
    std::string err;
    if ((st = plan_evolution(terms, coeffs, time, tol, &p, &err)) != QIPB200_OK) return set_err(state->ctx, st, err);
    *degree = p.degree;
    *tail = p.tail;
    if (p.kind == EvolutionPlan::kNoop) return (int)QIPB200_OK;
    qipb200_ctx *ctx = state->ctx;
    if (p.kind == EvolutionPlan::kPhase) {  // e^{-iat}: the empty-term rotation by 2 RN(a t)
      if ((st = begin_device_work(state)) != QIPB200_OK) return st;
      const double angle = 2.0 * (p.a * time);
      CU(ctx, run_pauli_rotations(state->prec, state->buf, state->n_local, std::vector<PauliTerm>(1), &angle,
                                  2 * ctx->sm_count, ctx->stream, &ctx->launches));
      return (int)QIPB200_OK;
    }
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = prepare_work_states(state, work_a, work_b)) != QIPB200_OK) return st;
    CU(ctx, run_pauli_evolution(state->prec, state->buf, work_a->buf, work_b->buf, state->n_local,
                                phys_terms(state, p.terms), p.coeffs.data(), p.b, p.C, ctx->stream, &ctx->launches));
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_pauli_evolution_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits,
                                            const char *paulis, const uint32_t *term_len, size_t n_terms,
                                            const double *coeffs, double time, double tol, uint32_t *out3,
                                            double *tail, double *coeffs_out, size_t coeffs_cap) {
  const std::string who = "pauli_evolution_plan";
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args(who, prec, n_qubits, out3 && tail, "out3 or tail");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_evolution_args(nullptr, who, coeffs, n_terms, time, tol);
    if (st != QIPB200_OK) return st;
    EvolutionPlan p;
    std::string err;
    if ((st = plan_evolution(terms, coeffs, time, tol, &p, &err)) != QIPB200_OK) return set_err(nullptr, st, err);
    const uint64_t s = p.kind == EvolutionPlan::kSeries ? pauli_sum_sweep_count(n_qubits, p.terms) : 0;
    out3[0] = p.degree;
    out3[1] = (uint32_t)s;
    out3[2] = p.kind == EvolutionPlan::kPhase ? 1u : (uint32_t)std::min<uint64_t>(p.degree * s, UINT32_MAX);
    *tail = p.tail;
    if (coeffs_out && coeffs_cap >= p.C.size()) std::copy(p.C.begin(), p.C.end(), coeffs_out);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// the lowest eigenvalue of a real Pauli sum by Lanczos (lanczos.cu)
// ===================================================================================

extern "C" int qipb200_state_lanczos_pauli_sum(qipb200_state *state, qipb200_state *work_a, qipb200_state *work_b,
                                               const uint64_t *qubits, const char *paulis, const uint32_t *term_len,
                                               size_t n_terms, const double *coeffs, uint32_t max_steps, double tol,
                                               uint32_t flags, uint32_t *steps, uint32_t *converged, double *alpha,
                                               double *beta, double *out3) {
  const std::string who = "lanczos_pauli_sum";
  if (!state || !work_a || !work_b) return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL state");
  return guarded(state->ctx, [&]() -> int {
    // every check runs before any device work: a refused call leaves the three states (and a pending collapse) as
    // they were
    std::vector<PauliTerm> terms;
    int st = check_three_states(state, work_a, work_b, who);
    if (st == QIPB200_OK) st = parse_terms(state->ctx, state->n, qubits, paulis, term_len, n_terms, &terms);
    if (st == QIPB200_OK) st = check_finite(state->ctx, coeffs, n_terms, who, "coefficient");
    if (st != QIPB200_OK) return st;
    if (max_steps == 0 || max_steps > kLanczosMaxSteps)
      return set_err(state->ctx, QIPB200_ERR_INVALID_ARG,
                     who + ": max_steps must be in 1.." + std::to_string(kLanczosMaxSteps));
    if (!(tol > 0.0 && tol < 1.0)) return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": tol must be in (0, 1)");
    if (flags & ~(uint32_t)QIPB200_LANCZOS_VECTOR)
      return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": unknown flags");
    if (!steps || !converged || !out3)
      return set_err(state->ctx, QIPB200_ERR_INVALID_ARG, who + ": NULL steps, converged or out3");
    double a = 0.0, b = 0.0;  // the identity terms' sum and the scale of the others, in list order
    for (size_t h = 0; h < n_terms; ++h) {
      if (terms[h].x == 0 && terms[h].z == 0)
        a += coeffs[h];
      else
        b += std::fabs(coeffs[h]);
    }
    qipb200_ctx *ctx = state->ctx;
    CU(ctx, cudaSetDevice(ctx->device));
    if ((st = prepare_work_states(state, work_a, work_b)) != QIPB200_OK) return st;
    LanczosResult r;
    CU(ctx, run_lanczos(state->prec, state->buf, work_a->buf, work_b->buf, state->n_local, phys_terms(state, terms),
                        coeffs, a, b, max_steps, tol, (flags & QIPB200_LANCZOS_VECTOR) != 0, ctx->stream,
                        &ctx->launches, &r));
    if (r.zero_norm)
      return set_err(ctx, QIPB200_ERR_INVALID_ARG, who + ": the start state has zero (or non-finite) norm");
    *steps = r.steps;
    *converged = r.converged;
    if (alpha) std::copy(r.alpha.begin(), r.alpha.end(), alpha);
    if (beta) std::copy(r.beta.begin(), r.beta.end(), beta);
    out3[0] = r.energy;
    out3[1] = r.residual;
    out3[2] = r.xnorm;
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_pauli_lanczos_plan(qip_prec prec, uint32_t n_qubits, const uint64_t *qubits, const char *paulis,
                                          const uint32_t *term_len, size_t n_terms, uint32_t *out4) {
  return guarded(nullptr, [&]() -> int {
    std::vector<PauliTerm> terms;
    int st = check_plan_args("pauli_lanczos_plan", prec, n_qubits, out4, "out4");
    if (st == QIPB200_OK) st = parse_terms(nullptr, n_qubits, qubits, paulis, term_len, n_terms, &terms);
    if (st != QIPB200_OK) return st;
    lanczos_plan_counts(n_qubits, terms, out4);
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_lanczos_ritz(const double *alpha, const double *beta, uint32_t m, double *theta, double *y,
                                    double *estimate) {
  const std::string who = "lanczos_ritz";
  if (!alpha || !beta || !theta || !estimate || m == 0)
    return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": NULL alpha, beta, theta or estimate, or m == 0");
  return guarded(nullptr, [&]() -> int {
    for (uint32_t i = 0; i < m; ++i)
      if (!std::isfinite(alpha[i]))
        return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": alpha " + std::to_string(i) + " is not finite");
    for (uint32_t i = 0; i <= m; ++i)
      if (!std::isfinite(beta[i]))
        return set_err(nullptr, QIPB200_ERR_INVALID_ARG, who + ": beta " + std::to_string(i) + " is not finite");
    lanczos_ritz(alpha, beta, m, theta, y, estimate);
    return (int)QIPB200_OK;
  });
}

// ===================================================================================
// multi-GPU plumbing (one process per GPU: CUDA IPC)
// ===================================================================================

extern "C" int qipb200_state_ipc_export(qipb200_state *s, void *amp_handle, void *flag_handle) {
  if (!s || !amp_handle || !flag_handle) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "ipc_export: NULL argument");
  qipb200_ctx *ctx = s->ctx;
  if (s->world == 1) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "ipc_export: not a sharded state");
  static_assert(sizeof(cudaIpcMemHandle_t) == QIPB200_IPC_HANDLE_BYTES, "IPC handle size");
  CU(ctx, cudaSetDevice(ctx->device));
  CU(ctx, cudaStreamSynchronize(ctx->stream));
  cudaIpcMemHandle_t h;
  CU(ctx, cudaIpcGetMemHandle(&h, s->buf));
  memcpy(amp_handle, &h, sizeof(h));
  CU(ctx, cudaIpcGetMemHandle(&h, s->flags));
  memcpy(flag_handle, &h, sizeof(h));
  return QIPB200_OK;
}

extern "C" int qipb200_state_ipc_import(qipb200_state *s, const void *amp_handles, const void *flag_handles) {
  if (!s || !amp_handles || !flag_handles) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "ipc_import: NULL argument");
  qipb200_ctx *ctx = s->ctx;
  if (s->world == 1) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "ipc_import: not a sharded state");
  if (s->ipc_ready) return set_err(ctx, QIPB200_ERR_INVALID_ARG, "ipc_import: peers are already mapped");
  return guarded(ctx, [&]() -> int {
    CU(ctx, cudaSetDevice(ctx->device));
    s->peer_buf.assign(s->world, nullptr);
    s->peer_flags.assign(s->world, nullptr);
    s->peer_comm.assign(s->world, nullptr);
    s->ipc_mapped = true;
    for (int t = 0; t < s->world; ++t) {
      if (t == s->rank) {
        s->peer_buf[t] = s->buf;
        s->peer_flags[t] = s->flags;
        s->peer_comm[t] = comm_of(s->flags);
        continue;
      }
      cudaIpcMemHandle_t h;
      memcpy(&h, (const char *)amp_handles + (size_t)t * QIPB200_IPC_HANDLE_BYTES, sizeof(h));
      cudaError_t e = cudaIpcOpenMemHandle(&s->peer_buf[t], h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        cuda_fail(ctx, e, "cudaIpcOpenMemHandle(amplitudes)");
        return (int)QIPB200_ERR_COMM;
      }
      memcpy(&h, (const char *)flag_handles + (size_t)t * QIPB200_IPC_HANDLE_BYTES, sizeof(h));
      void *fp = nullptr;
      e = cudaIpcOpenMemHandle(&fp, h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        cuda_fail(ctx, e, "cudaIpcOpenMemHandle(flags)");
        return (int)QIPB200_ERR_COMM;
      }
      s->peer_flags[t] = (uint32_t *)fp;
      s->peer_comm[t] = comm_of((uint32_t *)fp);
    }
    s->ipc_ready = true;
    return (int)QIPB200_OK;
  });
}

extern "C" int qipb200_state_qubit_map(qipb200_state *s, uint32_t *bit_of_qubit) {
  if (!s || !bit_of_qubit) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "qubit_map: NULL argument");
  const qipb200_state *src = s->shards.empty() ? s : s->shards[0];
  for (uint32_t q = 0; q < s->n; ++q) bit_of_qubit[q] = src->phys_of_logical[s->n - 1 - q];
  return QIPB200_OK;
}

extern "C" int qipb200_state_exchange_bytes(qipb200_state *s, uint64_t *bytes) {
  if (!s || !bytes) return set_err(s ? s->ctx : nullptr, QIPB200_ERR_INVALID_ARG, "exchange_bytes: NULL argument");
  *bytes = s->shards.empty() ? s->exchange_bytes : s->shards[0]->exchange_bytes;
  return QIPB200_OK;
}

extern "C" int qipb200_plan_exchanges(qip_prec prec, uint32_t n_qubits, int world_size, const qip_op *ops,
                                      size_t n_ops, uint32_t *needs_exchange) {
  if (!is_pow2(world_size) || (!ops && n_ops) || !needs_exchange)
    return set_err(nullptr, QIPB200_ERR_INVALID_ARG, "plan_exchanges: bad argument");
  return guarded(nullptr, [&]() -> int {
    const uint32_t n_local = n_qubits - (uint32_t)ilog2(world_size);
    for (size_t i = 0; i < n_ops; ++i) {
      FlatOp f;
      std::string err;
      int st = compile_op(&ops[i], prec, n_qubits, &f, &err);
      if (st != QIPB200_OK) return set_err(nullptr, st, err);
      std::vector<uint32_t> nd;
      nondiag_bits(f, &nd);
      uint32_t cnt = 0;
      for (size_t j = 0; j < nd.size(); ++j) cnt += nd[j] >= n_local;
      needs_exchange[i] = cnt;
    }
    return (int)QIPB200_OK;
  });
}
