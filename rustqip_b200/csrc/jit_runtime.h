// jit_runtime.h -- compiles the generated pass kernels (jit_codegen) with NVRTC for sm_90a and launches them.
//
// Tiered execution: a pass whose specialised kernel is not compiled yet runs through the interpreter kernel
// (tile_kernel.cu) while a background worker pool compiles it; the next run of the same pass STRUCTURE (the
// numeric gate constants, tile geometry and conditions are kernel parameters, not part of the key) finds the
// cubin in the process-wide cache.  Both kernels issue the same arithmetic, so mixing them is invisible in the
// results.  QIPB200_JIT = off | async (default for big states) | sync (compile before launching; tests).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "jit_codegen.h"

namespace qipb200 {

enum JitMode { JIT_OFF = 0, JIT_ASYNC = 1, JIT_SYNC = 2 };

struct JitCubin {  // one compiled program (host memory, device independent)
  std::vector<char> image;
  std::string log;
  bool ok = false;
  double compile_ms = 0.0;
};

struct JitLoaded {  // per (context == device): a loaded module of one cubin
  CUmodule mod = nullptr;
  CUfunction fn = nullptr;
};

// NVRTC + the driver entry points could be resolved in this process.
bool jit_available(std::string *why);

// Ask for the cubin of `source`: returns it when ready, nullptr when it is (now) being compiled in the
// background; with wait = true blocks until the compilation finishes.  Thread-safe.
std::shared_ptr<const JitCubin> jit_request(const std::string &source, bool wait);

// Block until the background queue is empty; returns the number of programs compiled so far, the total compile
// time spent (sum over programs, ms) and the number of programs taken from the on-disk cache instead
// (QIPB200_JIT_CACHE_DIR: cubins keyed by source text + compiler identity, shared between processes).
void jit_wait_all(uint64_t *n_compiled, double *total_ms, uint64_t *n_from_disk = nullptr);

// Load (once per context) and launch.  `loaded` is the context's module cache keyed by the cubin pointer.
// `tmap_out` / `send_bit` / `send_val` / `pair` (optional, the paired send of a multi-GPU qubit migration): tiles whose
// index bit send_bit equals send_val are stored through tmap_out, a map over the partner's SHARD, at the index with that
// bit flipped; the migration is done in place, tile by tile, under a per-tile flag handshake with the partner's pass
// (jit_codegen.cpp: pair_*).
struct JitPair {
  uint32_t cbit = 0;              // position of index bit send_bit in the tile counter
  uint32_t seq = 0;               // value of this migration in the flag words
  uint32_t *my_flags = nullptr;   // this rank's per-tile flag words (polled locally)
  uint32_t *peer_flags = nullptr; // the partner's (written over NVLink)
  uint32_t *error_word = nullptr;
};
cudaError_t jit_launch(const std::shared_ptr<const JitCubin> &cubin, std::vector<std::pair<const JitCubin *, JitLoaded>> *loaded,
                       const JitProgram &prog, void *psi, uint32_t n_local, const CUtensorMap &tmap, cudaStream_t stream,
                       std::string *err, const CUtensorMap *tmap_out = nullptr, uint32_t send_bit = 64, uint32_t send_val = 0,
                       const JitPair *pair = nullptr);

void jit_unload(std::vector<std::pair<const JitCubin *, JitLoaded>> *loaded);

// A compiled program as a module of the current device's context whose kernels are looked up by name and launched on
// runtime streams (the code functions of function.cu).  The calls fail with cudaErrorNotSupported when the driver entry
// points are missing, with cudaErrorUnknown on a driver error; *err then says which.
cudaError_t jit_module_load(const JitCubin &cubin, CUmodule *mod, std::string *err);
// Kernel `name` of mod, allowed max_dyn_smem bytes of dynamic shared memory (0: the default).
cudaError_t jit_module_kernel(CUmodule mod, const char *name, unsigned max_dyn_smem, CUfunction *fn, std::string *err);
cudaError_t jit_kernel_launch(CUfunction fn, unsigned grid, unsigned threads, unsigned smem, cudaStream_t stream,
                              void **args, std::string *err);
void jit_module_unload(CUmodule mod);

JitMode jit_mode_from_env(uint32_t n_local);

}  // namespace qipb200
