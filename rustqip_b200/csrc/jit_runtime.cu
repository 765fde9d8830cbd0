// jit_runtime.cu -- see jit_runtime.h.
#include "jit_runtime.h"

#include <dlfcn.h>
#include <nvrtc.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <thread>
#include <unordered_map>

namespace qipb200 {

namespace {

// ---- NVRTC through dlopen: the library must load (and the interpreter path work) without it ----
struct Nvrtc {
  void *h = nullptr;
  nvrtcResult (*create)(nvrtcProgram *, const char *, const char *, int, const char *const *, const char *const *) = nullptr;
  nvrtcResult (*compile)(nvrtcProgram, int, const char *const *) = nullptr;
  nvrtcResult (*cubin_size)(nvrtcProgram, size_t *) = nullptr;
  nvrtcResult (*cubin)(nvrtcProgram, char *) = nullptr;
  nvrtcResult (*log_size)(nvrtcProgram, size_t *) = nullptr;
  nvrtcResult (*log)(nvrtcProgram, char *) = nullptr;
  nvrtcResult (*destroy)(nvrtcProgram *) = nullptr;
  nvrtcResult (*version)(int *, int *) = nullptr;  // optional
  std::string why;
  bool ok = false;
};

Nvrtc &nvrtc() {
  static Nvrtc n;
  static std::once_flag once;
  std::call_once(once, [&]() {
    const char *names[] = {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so"};
    for (const char *nm : names)
      if ((n.h = dlopen(nm, RTLD_NOW | RTLD_LOCAL))) break;
    if (!n.h) {
      n.why = std::string("libnvrtc not found: ") + dlerror();
      return;
    }
#define QIP_SYM(field, name)                                     \
  *(void **)(&n.field) = dlsym(n.h, name);                       \
  if (!n.field) {                                                \
    n.why = std::string("libnvrtc lacks ") + name;               \
    return;                                                      \
  }
    QIP_SYM(create, "nvrtcCreateProgram")
    QIP_SYM(compile, "nvrtcCompileProgram")
    QIP_SYM(cubin_size, "nvrtcGetCUBINSize")
    QIP_SYM(cubin, "nvrtcGetCUBIN")
    QIP_SYM(log_size, "nvrtcGetProgramLogSize")
    QIP_SYM(log, "nvrtcGetProgramLog")
    QIP_SYM(destroy, "nvrtcDestroyProgram")
#undef QIP_SYM
    *(void **)(&n.version) = dlsym(n.h, "nvrtcVersion");
    n.ok = true;
  });
  return n;
}

// ---- driver API through the runtime's entry-point query (no link-time dependency on libcuda) ----
struct Driver {
  CUresult (*module_load)(CUmodule *, const void *) = nullptr;
  CUresult (*module_get)(CUfunction *, CUmodule, const char *) = nullptr;
  CUresult (*module_unload)(CUmodule) = nullptr;
  CUresult (*func_set_attr)(CUfunction, CUfunction_attribute, int) = nullptr;
  CUresult (*launch)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void **, void **) = nullptr;
  CUresult (*err_name)(CUresult, const char **) = nullptr;
  bool ok = false;
  std::string why;
};

Driver &driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [&]() {
    auto get = [&](const char *name, void **fp) {
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint(name, fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !*fp) {
        (void)cudaGetLastError();
        d.why = std::string("driver entry point missing: ") + name;
        return false;
      }
      return true;
    };
    if (!get("cuModuleLoadData", (void **)&d.module_load) || !get("cuModuleGetFunction", (void **)&d.module_get) ||
        !get("cuModuleUnload", (void **)&d.module_unload) || !get("cuFuncSetAttribute", (void **)&d.func_set_attr) ||
        !get("cuLaunchKernel", (void **)&d.launch) || !get("cuGetErrorName", (void **)&d.err_name))
      return;
    d.ok = true;
  });
  return d;
}

std::shared_ptr<JitCubin> compile_now(const std::string &source) {
  std::shared_ptr<JitCubin> out = std::make_shared<JitCubin>();
  Nvrtc &n = nvrtc();
  if (!n.ok) {
    out->log = n.why;
    return out;
  }
  const auto t0 = std::chrono::steady_clock::now();
  nvrtcProgram prog;
  if (n.create(&prog, source.c_str(), "qip_pass.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) {
    out->log = "nvrtcCreateProgram failed";
    return out;
  }
  // sm_90a SASS directly (no PTX JIT by the driver); implicit mul+add contraction off: the generated source
  // spells every FMA out, in the interpreter kernel's order
  const char *opts[] = {"--gpu-architecture=sm_90a", "--std=c++17", "--fmad=false", "-lineinfo", "-default-device"};
  const nvrtcResult r = n.compile(prog, 5, opts);
  size_t ls = 0;
  if (n.log_size(prog, &ls) == NVRTC_SUCCESS && ls > 1) {
    out->log.resize(ls);
    n.log(prog, &out->log[0]);
  }
  if (r == NVRTC_SUCCESS) {
    size_t cs = 0;
    if (n.cubin_size(prog, &cs) == NVRTC_SUCCESS && cs) {
      out->image.resize(cs);
      out->ok = n.cubin(prog, out->image.data()) == NVRTC_SUCCESS;
    }
  }
  n.destroy(&prog);
  out->compile_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return out;
}

// ---- optional on-disk cache of cubins (QIPB200_JIT_CACHE_DIR) ---------------------------------------------
// A program is keyed by its source text (two independent 64-bit FNV-1a hashes + the length) and the compiler
// identity (NVRTC version, target, options).  Files are written to a temporary name and renamed, so concurrent
// processes sharing the directory never see a partial file; anything that does not check out is recompiled.
uint64_t fnv1a(const std::string &s, uint64_t seed) {
  uint64_t h = 1469598103934665603ull ^ seed;
  for (size_t i = 0; i < s.size(); ++i) {
    h ^= (unsigned char)s[i];
    h *= 1099511628211ull;
  }
  return h;
}

struct DiskHeader {
  char magic[8];
  uint64_t source_len, hash_a, hash_b, image_len;
};

std::string disk_path(const std::string &source, uint64_t *ha, uint64_t *hb) {
  const char *dir = getenv("QIPB200_JIT_CACHE_DIR");
  if (!dir || !*dir) return std::string();
  int major = 0, minor = 0;
  Nvrtc &n = nvrtc();
  if (n.ok && n.version) n.version(&major, &minor);
  const std::string ident = "nvrtc " + std::to_string(major) + "." + std::to_string(minor) + " sm_90a c++17 fmad=false lineinfo|";
  *ha = fnv1a(ident + source, 0);
  *hb = fnv1a(ident + source, 0x9E3779B97F4A7C15ull);
  char name[96];
  snprintf(name, sizeof(name), "/qip_%016llx_%zu.cubin", (unsigned long long)*ha, source.size());
  return std::string(dir) + name;
}

bool disk_load(const std::string &source, JitCubin *out) {
  uint64_t ha = 0, hb = 0;
  const std::string path = disk_path(source, &ha, &hb);
  if (path.empty()) return false;
  FILE *f = fopen(path.c_str(), "rb");
  if (!f) return false;
  DiskHeader h;
  bool ok = fread(&h, sizeof(h), 1, f) == 1 && !memcmp(h.magic, "QIPJIT1", 8) && h.source_len == source.size() && h.hash_a == ha &&
            h.hash_b == hb && h.image_len > 0 && h.image_len < (1ull << 28);
  if (ok) {
    out->image.resize(h.image_len);
    ok = fread(out->image.data(), 1, h.image_len, f) == h.image_len && fgetc(f) == EOF;
  }
  fclose(f);
  if (!ok) out->image.clear();
  return ok;
}

void disk_store(const std::string &source, const JitCubin &c) {
  uint64_t ha = 0, hb = 0;
  const std::string path = disk_path(source, &ha, &hb);
  if (path.empty() || !c.ok) return;
  char suffix[64];
  snprintf(suffix, sizeof(suffix), ".tmp.%ld.%llx", (long)getpid(), (unsigned long long)(uintptr_t)&c);
  const std::string tmp = path + suffix;
  FILE *f = fopen(tmp.c_str(), "wb");
  if (!f) return;  // an unwritable cache directory is not an error: the program was compiled anyway
  DiskHeader h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, "QIPJIT1", 8);
  h.source_len = source.size();
  h.hash_a = ha;
  h.hash_b = hb;
  h.image_len = c.image.size();
  const bool ok = fwrite(&h, sizeof(h), 1, f) == 1 && fwrite(c.image.data(), 1, c.image.size(), f) == c.image.size();
  if (fclose(f) != 0 || !ok || rename(tmp.c_str(), path.c_str()) != 0) remove(tmp.c_str());
}

std::shared_ptr<JitCubin> compile_or_load(const std::string &source, bool *from_disk) {
  *from_disk = false;
  if (getenv("QIPB200_JIT_CACHE_DIR")) {
    const auto t0 = std::chrono::steady_clock::now();
    std::shared_ptr<JitCubin> hit = std::make_shared<JitCubin>();
    if (disk_load(source, hit.get())) {
      hit->ok = true;
      hit->log = "loaded from QIPB200_JIT_CACHE_DIR";
      hit->compile_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      *from_disk = true;
      return hit;
    }
  }
  std::shared_ptr<JitCubin> c = compile_now(source);
  disk_store(source, *c);
  return c;
}

// ---- process-wide cache + background workers ----
struct Entry {
  std::shared_ptr<const JitCubin> cubin;  // null while pending
  bool pending = false;
};

struct Cache {
  std::mutex mu;
  std::condition_variable cv;
  std::unordered_map<std::string, Entry> map;  // keyed by the source text itself
  std::deque<std::string> queue;
  std::vector<std::thread> workers;
  unsigned in_flight = 0;
  uint64_t n_compiled = 0, n_from_disk = 0;
  double total_ms = 0.0;
  bool stop = false;

  void start_workers() {
    if (!workers.empty()) return;
    unsigned nthr = std::thread::hardware_concurrency();
    if (const char *e = getenv("QIPB200_JIT_THREADS")) nthr = (unsigned)std::max(1, atoi(e));
    nthr = std::max(1u, std::min(nthr, 32u));
    for (unsigned i = 0; i < nthr; ++i) workers.emplace_back([this]() { this->worker(); });
  }
  void worker() {
    for (;;) {
      std::string src;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&]() { return stop || !queue.empty(); });
        if (stop) return;
        src.swap(queue.front());
        queue.pop_front();
      }
      bool from_disk = false;
      std::shared_ptr<JitCubin> c = compile_or_load(src, &from_disk);
      {
        std::lock_guard<std::mutex> lk(mu);
        Entry &e = map[src];
        e.cubin = c;
        e.pending = false;
        --in_flight;
        if (from_disk) {
          ++n_from_disk;
        } else {
          ++n_compiled;
          total_ms += c->compile_ms;
        }
      }
      cv.notify_all();
    }
  }
  ~Cache() {
    {
      std::lock_guard<std::mutex> lk(mu);
      stop = true;
    }
    cv.notify_all();
    for (std::thread &t : workers) t.join();
  }
};

Cache &cache() {
  static Cache *c = new Cache();  // intentionally leaked at exit when workers are still compiling
  return *c;
}

}  // namespace

bool jit_available(std::string *why) {
  if (!nvrtc().ok) {
    if (why) *why = nvrtc().why;
    return false;
  }
  if (!driver().ok) {
    if (why) *why = driver().why;
    return false;
  }
  return true;
}

std::shared_ptr<const JitCubin> jit_request(const std::string &source, bool wait) {
  Cache &c = cache();
  std::unique_lock<std::mutex> lk(c.mu);
  Entry &e = c.map[source];
  if (e.cubin) return e.cubin;
  if (!e.pending) {
    e.pending = true;
    ++c.in_flight;
    c.queue.push_back(source);
    c.start_workers();
    c.cv.notify_all();
  }
  if (!wait) return nullptr;
  c.cv.wait(lk, [&]() { return c.map[source].cubin != nullptr; });
  return c.map[source].cubin;
}

void jit_wait_all(uint64_t *n_compiled, double *total_ms, uint64_t *n_from_disk) {
  Cache &c = cache();
  std::unique_lock<std::mutex> lk(c.mu);
  c.cv.wait(lk, [&]() { return c.in_flight == 0; });
  if (n_compiled) *n_compiled = c.n_compiled;
  if (total_ms) *total_ms = c.total_ms;
  if (n_from_disk) *n_from_disk = c.n_from_disk;
}

cudaError_t jit_launch(const std::shared_ptr<const JitCubin> &cubin, std::vector<std::pair<const JitCubin *, JitLoaded>> *loaded,
                       const JitProgram &prog, void *psi, uint32_t n_local, const CUtensorMap &tmap, cudaStream_t stream,
                       std::string *err, const CUtensorMap *tmap_out, uint32_t send_bit, uint32_t send_val,
                       const JitPair *pair) {
  Driver &d = driver();
  if (!d.ok || !cubin || !cubin->ok) {
    if (err) *err = !d.ok ? d.why : "no cubin";
    return cudaErrorNotSupported;
  }
  JitLoaded *L = nullptr;
  for (size_t i = 0; i < loaded->size(); ++i)
    if ((*loaded)[i].first == cubin.get()) L = &(*loaded)[i].second;
  auto fail = [&](CUresult r, const char *what) {
    const char *nm = nullptr;
    d.err_name(r, &nm);
    if (err) *err = std::string(what) + ": " + (nm ? nm : "?");
    return cudaErrorUnknown;
  };
  if (!L) {
    JitLoaded nl;
    CUresult r = d.module_load(&nl.mod, cubin->image.data());
    if (r != CUDA_SUCCESS) return fail(r, "cuModuleLoadData");
    r = d.module_get(&nl.fn, nl.mod, "qip_pass");
    if (r != CUDA_SUCCESS) return fail(r, "cuModuleGetFunction");
    r = d.func_set_attr(nl.fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)prog.smem_bytes);
    if (r != CUDA_SUCCESS) return fail(r, "cuFuncSetAttribute(max dynamic shared memory)");
    loaded->push_back(std::make_pair(cubin.get(), nl));
    L = &loaded->back().second;
  }
  alignas(64) CUtensorMap tm = tmap;
  alignas(64) CUtensorMap tm_out = tmap_out ? *tmap_out : tmap;
  std::vector<unsigned char> params = prog.params;  // the send fields are per launch
  if (tmap_out && prog.send_offset + 8 <= params.size()) {
    memcpy(params.data() + prog.send_offset, &send_bit, 4);
    memcpy(params.data() + prog.send_offset + 4, &send_val, 4);
  }
  void *args[4] = {&psi, params.data(), &tm, &tm_out};
  const uint64_t tiles = 1ull << (n_local - prog.tiles_log2_sub);
  if (prog.send_offset + 64 > params.size()) return cudaErrorInvalidValue;
  {
    const uint32_t w[4] = {0u, 0u, (uint32_t)tiles, (uint32_t)(tiles >> 32)};  // tile offset 0, every tile
    memcpy(params.data() + prog.send_offset + 8, w, 16);
  }
  // QIPB200_JIT_PERSISTENT=<CTAs>: a fixed grid of persistent CTAs walking the tile counter instead of one CTA per tile
  static const unsigned persistent_ctas = []() {
    const char *e = getenv("QIPB200_JIT_PERSISTENT");
    return e ? (unsigned)std::max(0, atoi(e)) : 0u;
  }();
  unsigned grid = (unsigned)std::min<uint64_t>(tiles, 0x7fffffffull);
  if (persistent_ctas && grid > persistent_ctas) grid = persistent_ctas;
  // QIPB200_JIT_PREFETCH=<tiles>: L2 prefetch distance in the tile counter (0 = off)
  static const unsigned prefetch_dist = []() {
    const char *e = getenv("QIPB200_JIT_PREFETCH");
    return e ? (unsigned)std::max(0, atoi(e)) : 0u;
  }();
  memcpy(params.data() + prog.send_offset + 24, &prefetch_dist, 4);
  if (pair && tmap_out) {
    const uint64_t mf = (uint64_t)(uintptr_t)pair->my_flags, pf = (uint64_t)(uintptr_t)pair->peer_flags,
                   ew = (uint64_t)(uintptr_t)pair->error_word;
    const uint32_t w[8] = {pair->cbit, pair->seq, (uint32_t)mf, (uint32_t)(mf >> 32), (uint32_t)pf, (uint32_t)(pf >> 32),
                           (uint32_t)ew, (uint32_t)(ew >> 32)};
    memcpy(params.data() + prog.send_offset + 32, w, 32);
  }
  const CUresult r = d.launch(L->fn, grid, 1, 1, prog.threads, 1, 1, prog.smem_bytes, (CUstream)stream, args, nullptr);
  if (r != CUDA_SUCCESS) return fail(r, "cuLaunchKernel");
  return cudaSuccess;
}

void jit_unload(std::vector<std::pair<const JitCubin *, JitLoaded>> *loaded) {
  Driver &d = driver();
  if (d.ok)
    for (size_t i = 0; i < loaded->size(); ++i)
      if ((*loaded)[i].second.mod) d.module_unload((*loaded)[i].second.mod);
  loaded->clear();
}

namespace {

cudaError_t driver_fail(CUresult r, const char *what, std::string *err) {
  const char *nm = nullptr;
  driver().err_name(r, &nm);
  if (err) *err = std::string(what) + ": " + (nm ? nm : "?");
  return cudaErrorUnknown;
}

}  // namespace

cudaError_t jit_module_load(const JitCubin &cubin, CUmodule *mod, std::string *err) {
  Driver &d = driver();
  if (!d.ok || !cubin.ok) {
    if (err) *err = !d.ok ? d.why : "no cubin";
    return cudaErrorNotSupported;
  }
  const CUresult r = d.module_load(mod, cubin.image.data());
  return r == CUDA_SUCCESS ? cudaSuccess : driver_fail(r, "cuModuleLoadData", err);
}

cudaError_t jit_module_kernel(CUmodule mod, const char *name, unsigned max_dyn_smem, CUfunction *fn, std::string *err) {
  Driver &d = driver();
  CUresult r = d.module_get(fn, mod, name);
  if (r != CUDA_SUCCESS) return driver_fail(r, "cuModuleGetFunction", err);
  if (max_dyn_smem && (r = d.func_set_attr(*fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)max_dyn_smem)) !=
                          CUDA_SUCCESS)
    return driver_fail(r, "cuFuncSetAttribute(max dynamic shared memory)", err);
  return cudaSuccess;
}

cudaError_t jit_kernel_launch(CUfunction fn, unsigned grid, unsigned threads, unsigned smem, cudaStream_t stream,
                              void **args, std::string *err) {
  const CUresult r = driver().launch(fn, grid, 1, 1, threads, 1, 1, smem, (CUstream)stream, args, nullptr);
  return r == CUDA_SUCCESS ? cudaSuccess : driver_fail(r, "cuLaunchKernel", err);
}

void jit_module_unload(CUmodule mod) {
  if (mod && driver().ok) driver().module_unload(mod);
}

JitMode jit_mode_from_env(uint32_t n_local) {
  if (const char *e = getenv("QIPB200_JIT")) {
    if (!strcmp(e, "off") || !strcmp(e, "0")) return JIT_OFF;
    if (!strcmp(e, "sync")) return JIT_SYNC;
    if (!strcmp(e, "async") || !strcmp(e, "1")) return JIT_ASYNC;
  }
  // below ~2^22 amplitudes a pass takes microseconds: compiling a kernel for it never pays off
  return n_local >= 22 ? JIT_ASYNC : JIT_OFF;
}

}  // namespace qipb200
