// state.h -- context and device-resident state objects behind the C ABI.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "../../include/qipb200.h"
#include "jit_runtime.h"
#include "opcompile.h"

struct qipb200_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  uint64_t tile_launches = 0;      // fused tile passes among `launches`
  uint64_t exchange_launches = 0;  // NVLink pair-exchange kernels among `launches`
  uint64_t fused_gates = 0;        // reference ops folded into tile passes
  uint64_t jit_launches = 0;       // tile passes among `tile_launches` that ran a generated (specialised) kernel
  std::vector<std::pair<const qipb200::JitCubin *, qipb200::JitLoaded>> jit_loaded;  // modules loaded on this device
  std::string jit_note;            // why the generated-kernel path was not taken last time (diagnostics)
  // multi-device context (qipb200_init_multi): one child context per device, owned by the parent; states created
  // on the parent are sharded over the children inside this one process (peer access instead of CUDA IPC)
  std::vector<qipb200_ctx *> children;
  qipb200_ctx *parent = nullptr;
  // one released state buffer kept for the next state of the same size (qipb200_calculate_state re-allocates
  // 2^n amplitudes per call otherwise)
  void *pool_buf = nullptr;
  size_t pool_bytes = 0;
  // per-gate kernel launches by kernel (qipb200_kernel_counts; index = QIPB200_KC_*)
  uint64_t kernel_counts[QIPB200_KC_COUNT] = {};
  bool tile_configured = false;    // the tile kernels' > 48 KiB shared-memory opt-in was done on this device
  // optional per-category device timing (qipb200_profile_enable): CUDA-event pairs recorded on `stream`
  // around every fused tile pass [0] and every NVLink exchange incl. its two flag barriers [1]
  bool profile = false;
  struct ProfEvent {
    cudaEvent_t first, second;
  };
  std::vector<ProfEvent> prof_events[2];
  std::vector<cudaEvent_t> prof_pool;
  // staging buffers of the host-buffer drop-ins (qipb200_apply_op*)
  void *d_in = nullptr, *d_out = nullptr;
  size_t d_in_bytes = 0, d_out_bytes = 0;
  double *d_scalar = nullptr;   // one device double for reductions
  void *eig_solver = nullptr;   // cuSOLVER handle of qipb200_state_entanglement_spectrum, created on first use
  void *h_pinned = nullptr;     // pinned bounce buffer for downloads/uploads
  size_t h_pinned_bytes = 0;
};

struct qipb200_state {
  qipb200_ctx *ctx = nullptr;
  qip_prec prec = QIP_F64;
  uint32_t n = 0;        // qubits of the whole state
  uint32_t n_local = 0;  // index bits held by this rank
  int rank = 0, world = 1;
  void *buf = nullptr;      // 2^n_local amplitudes
  uint32_t pair_seq = 0;    // migrations fused into a tile pass so far (value written into the per-tile flag words)
  void *scratch = nullptr;  // same size, lazily allocated (out-of-place row kernel only)
  size_t bytes = 0;
  // logical index bit b (= n-1-q) -> physical index bit.  Physical bits >= n_local are
  // rank bits.  Identity unless an exchange migrated a qubit (multi-GPU only).
  std::vector<uint32_t> phys_of_logical;
  // CUDA-IPC peer mappings (multi-GPU)
  std::vector<void *> peer_buf;
  uint32_t *flags = nullptr;  // world slots, written by peers
  std::vector<uint32_t *> peer_flags;
  std::vector<const double *> peer_comm;  // every rank's reduction slot (behind its flag page, dist.cuh)
  std::vector<qipb200_state *> shards;    // parent state of a multi-device context: one sharded state per device
  bool ipc_mapped = false;                // peers were mapped with cudaIpcOpenMemHandle (to be closed on free)
  uint32_t epoch = 0;
  uint64_t exchange_bytes = 0;
  bool ipc_ready = false;
  // Collapse left pending by qipb200_state_measure (unsharded single-device states only): measure_state over the
  // logical qubits pend_qubits with outcome pend_measured and multiplier pend_p_mult.  The next fused schedule runs
  // it as diagonal gates in its first tile pass; every other access to the amplitudes applies it first (api.cu).
  bool collapse_pending = false;
  std::vector<uint64_t> pend_qubits;
  uint64_t pend_measured = 0;
  double pend_p_mult = 1.0;
  // Basis state left pending by qipb200_state_set_basis (unsharded single-device states only): the amplitudes are
  // |init_index>, but nothing has been written yet.  The next fused schedule whose first step is a generated tile pass
  // builds its tiles from the index instead of loading them; every other access to the amplitudes writes the basis
  // state first (api.cu: materialise_init).  Never set together with collapse_pending.
  bool init_pending = false;
  uint64_t init_index = 0;
};

namespace qipb200 {
struct FnCode;
}

// A classical function of an n_in-bit register, given as tables (qipb200_function_new: they live on ctx's device and
// are freed on ctx's stream) or as code (qipb200_function_new_code: a compiled program loaded on ctx's device).
struct qipb200_function {
  qipb200_ctx *ctx = nullptr;
  uint32_t n_in = 0, n_out = 0;
  uint32_t *d_f = nullptr;    // f[x] for x < 2^n_in, NULL when n_out == 0
  double2 *d_cs = nullptr;    // (cos, sin) of theta[x] in double, NULL without phases
  // code functions only
  qipb200::FnCode *code = nullptr;
  bool theta = false;         // the source defines qip_theta
  uint32_t n_params = 0;
  double params[16] = {};     // the parameters theta is evaluated with (unused entries 0)
  void *d_scratch = nullptr;  // one u64 for the checks, then the expect partials
};

namespace qipb200 {

// RAII bracket of one profiled region (no-op unless ctx->profile).
struct ProfileScope {
  qipb200_ctx *ctx;
  int cat;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ProfileScope(qipb200_ctx *c, int category) : ctx(c), cat(category) {
    if (!ctx->profile) return;
    auto take = [&]() {
      cudaEvent_t e = nullptr;
      if (!ctx->prof_pool.empty()) {
        e = ctx->prof_pool.back();
        ctx->prof_pool.pop_back();
      } else if (cudaEventCreate(&e) != cudaSuccess) {
        e = nullptr;
      }
      return e;
    };
    e0 = take();
    e1 = take();
    if (e0) cudaEventRecord(e0, ctx->stream);
  }
  ~ProfileScope() {
    if (!e0 || !e1) return;
    cudaEventRecord(e1, ctx->stream);
    qipb200_ctx::ProfEvent pe = {e0, e1};
    ctx->prof_events[cat].push_back(pe);
  }
};

inline size_t amp_bytes(qip_prec p) { return p == QIP_F32 ? 8 : 16; }

}  // namespace qipb200
