// schedule.cu -- executes a list of ops on a device-resident state.
//
// Reference: the sequential fold over the pipeline in
// LocalBuilder::calculate_state_with_init (qip/src/builder.rs:423-514): one
// apply_op_overwrite sweep per entry.  Here
//   * QIPB200_SCHED_NO_FUSION: every entry is compiled to one in-place per-gate kernel;
//   * default: runs of entries are planned into fused shared-memory tile passes
//     (planner.cpp / tile_kernel.cu), each pass one HBM sweep for many gates.
// On a sharded state a look-ahead over the schedule picks which local qubit to evict
// when a rank-held qubit has to be migrated; an exchange is a fusion barrier.
#include "schedule.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/qipb200.h"
#include "dist.cuh"
#include "jit_codegen.h"
#include "jit_runtime.h"
#include "tile.cuh"
#include "tile_launch.cuh"

namespace qipb200 {

static const uint64_t kNever = ~0ull >> 1;

namespace {

bool needs_exchange(const qipb200_state *s, const FlatOp &f) {
  if (s->world == 1) return false;
  const uint32_t nl = s->n_local;
  if (f.cls == CLASS_DENSE || f.cls == CLASS_FLIP) {
    for (size_t j = 0; j < f.tgt_sorted.size(); ++j)
      if (f.tgt_sorted[j] >= nl) return true;
  } else if (f.cls == CLASS_BITSWAP) {
    for (size_t j = 0; j < f.swaps.size(); ++j)
      if (f.swaps[j].first >= nl || f.swaps[j].second >= nl) return true;
  } else if (f.cls == CLASS_GENERAL) {
    for (uint32_t j = f.nc; j < f.k; ++j)
      if (f.idx_bits[j] >= nl) return true;
  }
  return false;
}

// The qubit migration that follows this epoch, to be done by the epoch's last tile pass.
struct SendPlan {
  bool pair = false;     // in-place protocol fused into the last pass (paired send): tiles of the give-half go straight into
                         // the partner's shard under a per-tile flag handshake; a rank whose last pass cannot do it runs
                         // the pass normally and then the stand-in kernel -- the partner does not see the difference
  uint32_t R = 0, l = 0;
};

int execute_steps(qipb200_state *s, const std::vector<PlanStep> &steps, const std::vector<FlatOp> &local,
                  const PlanConfig &cfg, const SendPlan &send = SendPlan()) {
  qipb200_ctx *ctx = s->ctx;
  int st = QIPB200_OK;
  PassParams *pp = new PassParams();
  // Generated kernels (jit_codegen / jit_runtime): every pass is turned into specialised source; a pass whose
  // cubin is ready runs it, the others run the interpreter kernel while the background workers compile.
  bool paired_done = false;
  uint32_t pair_cbit = 0, pair_seq = 0;
  if (send.pair && !steps.empty() && steps.back().is_pass) {
    const PassHeader &lh = steps.back().pass.hdr;
    pair_cbit = send.l - lh.L;
    for (uint32_t k = 0; k < lh.m; ++k)
      if (lh.hi_pos[k] < send.l) --pair_cbit;
    pair_seq = ++s->pair_seq;  // one value per migration, the same on every rank
  }
  const JitMode jmode = cfg.use_tma && cfg.groups_per_thread == 1 ? jit_mode_from_env(s->n_local) : JIT_OFF;
  std::vector<JitProgram> progs(steps.size());
  std::vector<char> have_prog(steps.size(), 0);
  if (jmode != JIT_OFF && jit_available(&ctx->jit_note)) {
    for (size_t i = 0; i < steps.size(); ++i) {
      if (!steps[i].is_pass) continue;
      std::string why;
      // a state still pending as a basis state (unsharded only) is built by its first pass instead of being loaded
      const uint64_t *synth = i == 0 && s->init_pending && s->world == 1 ? &s->init_index : nullptr;
      if (jit_generate(steps[i].pass, s->prec, &progs[i], &why, send.pair && i + 1 == steps.size(), synth)) {
        have_prog[i] = 1;
        (void)jit_request(progs[i].source, false);  // all compilations of this schedule start now, in parallel
      } else {
        ctx->jit_note = why;
      }
    }
  }
  for (size_t i = 0; i < steps.size() && st == QIPB200_OK; ++i) {
    if (steps[i].is_pass && have_prog[i]) {
      alignas(64) CUtensorMap tmap;
      memset(&tmap, 0, sizeof(tmap));
      if (make_tile_map(&tmap, s->prec, s->buf, s->n_local, steps[i].pass.hdr)) {
        std::shared_ptr<const JitCubin> cubin = jit_request(progs[i].source, jmode == JIT_SYNC);
        if (cubin && !cubin->ok) ctx->jit_note = "NVRTC: " + cubin->log;
        if (cubin && cubin->ok) {
          // Paired send: the give-half tiles go into the partner's shard, tile by tile under the flag handshake.
          alignas(64) CUtensorMap tmap_out;
          const CUtensorMap *tmo = nullptr;
          uint32_t send_bit = 64, send_val = 0;
          const PassHeader &ph = steps[i].pass.hdr;
          JitPair pair;
          // (test hook QIPB200_PAIRED_STANDIN_RANK=<rank | -1 for all>: that rank never fuses the send into its pass)
          static const int standin_rank = getenv("QIPB200_PAIRED_STANDIN_RANK") ? atoi(getenv("QIPB200_PAIRED_STANDIN_RANK")) : -2;
          const bool pair_here = send.pair && i + 1 == steps.size() && standin_rank != -1 && standin_rank != s->rank;
          if (pair_here) {
            int partner = 0, give = 0;
            paired_partner(s, send.R, &partner, &give);
            memset(&tmap_out, 0, sizeof(tmap_out));
            if (make_tile_map(&tmap_out, s->prec, s->peer_buf[partner], s->n_local, ph)) {
              tmo = &tmap_out;
              send_bit = send.l;
              send_val = (uint32_t)give;
              pair.cbit = pair_cbit;
              pair.seq = pair_seq;
              pair.my_flags = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(s->flags) + kPairFlagOffsetBytes);
              pair.peer_flags = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(s->peer_flags[partner]) + kPairFlagOffsetBytes);
              pair.error_word = s->flags + kFlagErrorSlot;
            }
          }
          std::string err;
          cudaError_t e;
          {
            ProfileScope prof(ctx, 0);
            e = jit_launch(cubin, &ctx->jit_loaded, progs[i], s->buf, s->n_local, tmap, ctx->stream, &err, tmo, send_bit, send_val,
                           tmo ? &pair : nullptr);
          }
          if (e == cudaSuccess) {
            if (progs[i].synthesised) s->init_pending = false;
            if (tmo) paired_done = true;
            ++ctx->launches;
            ++ctx->tile_launches;
            ++ctx->jit_launches;
            ctx->fused_gates += steps[i].pass.n_gates;
            continue;
          }
          ctx->jit_note = err;  // fall through to the interpreter kernel
          (void)cudaGetLastError();
        }
      }
    }
    // a step that reads the amplitudes: a pending basis state is written first (no generated synthesising pass ran)
    if (s->init_pending && (st = materialise_init(s)) != QIPB200_OK) break;
    if (steps[i].is_pass) {
      if (!serialise_pass(steps[i].pass, pp)) {
        st = report_error(s, QIPB200_ERR_UNSUPPORTED, "internal: fused pass exceeds the kernel parameter space");
        break;
      }
      ProfileScope prof(ctx, 0);
      cudaError_t e = launch_tile_pass(s->prec, s->buf, s->n_local, *pp, cfg.groups_per_thread, cfg.use_tma, ctx->stream,
                                       &ctx->launches);
      if (e != cudaSuccess) st = report_cuda_error(s, e, "launch_tile_pass");
      ++ctx->tile_launches;
      ctx->fused_gates += steps[i].pass.n_gates;
    } else {
      st = launch_local_op(s, local[steps[i].op_index]);
    }
  }
  delete pp;
  if (st == QIPB200_OK && send.pair && !paired_done)  // the last pass ran without the send: play the protocol separately
    st = paired_send_standin(s, send.R, send.l, pair_cbit, pair_seq, steps.back().pass.hdr);
  if (send.pair && getenv("QIPB200_PAIRED_DEBUG"))
    fprintf(stderr, "paired send: rank %d migration %u (R=%u l=%u) %s\n", s->rank, pair_seq, send.R, send.l,
            paired_done ? "fused into the pass" : "stand-in kernel");
  return st;
}

// Fused execution.  The schedule is consumed in EPOCHS: under the current layout every op whose
// non-diagonal targets are local is planned into tile passes (ops needing a rank-held qubit are
// "blocked"; later ops may overtake them only when they commute); when nothing more can run, the
// first blocked op's qubit is migrated over NVLink (one exchange) and the next epoch starts.
int run_fused(qipb200_state *s, const qip_op *ops, size_t n_ops, const std::vector<uint64_t> &next_use) {
  // cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-DEVICE setting and a process may hold contexts on
  // several GPUs: the opt-in is tracked per context (a context is bound to one device and driven by one thread).
  if (!s->ctx->tile_configured) {
    cudaError_t e = tile_pass_configure();
    if (e != cudaSuccess) return report_cuda_error(s, e, "cudaFuncSetAttribute(tile pass)");
    s->ctx->tile_configured = true;
  }
  const PlanConfig cfg = default_plan_config(s->prec, s->n_local, s->world > 1);
  // Paired send (QIPB200_PAIRED_SEND=1): the migration that ends an epoch is fused into the epoch's last tile pass and done
  // in place, tile by tile, against the partner's copy of the same pass.  Tiles pair up across GPUs, so every rank must
  // choose the same tile bits: the planner then selects from rank-independent data only (op_uniform_info).
  static const bool paired_env = getenv("QIPB200_PAIRED_SEND") != nullptr && atoi(getenv("QIPB200_PAIRED_SEND")) != 0;
  const bool paired_mode = paired_env && s->world > 1 && cfg.use_tma &&
                           cfg.groups_per_thread == 1 && jit_mode_from_env(s->n_local) != JIT_OFF &&
                           cfg.T == (s->prec == QIP_F32 ? 13u : 12u) && s->n_local > cfg.T && s->n_local - cfg.T <= kPairFlagLog2;
  std::vector<size_t> remaining(n_ops);
  for (size_t i = 0; i < n_ops; ++i) remaining[i] = i;
  while (!remaining.empty()) {
    // compile what is left under the current layout
    std::vector<FlatOp> local(remaining.size());
    std::vector<char> blocked(remaining.size(), 0);
    std::vector<DepMasks> dep(remaining.size());
    for (size_t r = 0; r < remaining.size(); ++r) {
      FlatOp f;
      std::string err;
      int st = compile_op(&ops[remaining[r]], s->prec, s->n, &f, &err, s->phys_of_logical.data());
      if (st != QIPB200_OK) {
        // run everything before the bad op, then report (sequential semantics)
        local.resize(r);
        blocked.resize(r);
        dep.resize(r);
        std::vector<PlanStep> steps;
        std::vector<size_t> left;
        plan_passes(local, s->n_local, s->prec, cfg, &steps, &blocked, &left, &dep);
        execute_steps(s, steps, local, cfg);
        return report_error(s, st, err);
      }
      op_dependency_masks(f, &dep[r]);
      if (paired_mode) {  // what the op looks like on the rank whose rank-held bits are all 1: the same on every rank
        FlatOp fv;
        bool skipv = false;
        if ((st = restrict_to_rank_as(s, s->world - 1, f, &fv, &skipv)) != QIPB200_OK) return st;
        if (skipv) {
          fv = FlatOp();
          fv.cls = CLASS_IDENTITY;
        }
        op_uniform_info(fv, &dep[r]);
      }
      if (needs_exchange(s, f)) {
        blocked[r] = 1;
        local[r] = f;
        continue;
      }
      bool skip = false;
      if ((st = restrict_to_rank(s, f, &local[r], &skip)) != QIPB200_OK) return st;
      if (skip) {
        local[r] = FlatOp();
        local[r].cls = CLASS_IDENTITY;
      }
    }
    std::vector<PlanStep> steps;
    std::vector<size_t> left;  // indices into `local`
    plan_passes(local, s->n_local, s->prec, cfg, &steps, &blocked, &left, &dep);
    // the first blocked op (program order) decides the migration; identical on every rank
    size_t first_blocked = left.size();
    for (size_t i = 0; i < left.size(); ++i)
      if (blocked[left[i]]) {
        first_blocked = i;
        break;
      }
    // The migration that ends this epoch is known before the epoch runs: under the paired send the epoch's last tile
    // pass does it.
    SendPlan send;
    if (paired_mode && first_blocked != left.size()) {
      const size_t op_idx = remaining[left[first_blocked]];
      const uint64_t *nu = next_use.empty() ? nullptr : &next_use[(op_idx + 1) * s->n];
      if (!steps.empty() && steps.back().is_pass && peek_first_exchange(s, &ops[op_idx], nu, &send.R, &send.l)) {
        const PassHeader &ph = steps.back().pass.hdr;  // rank-independent geometry: bit l must be constant within a tile
        bool ok = send.l >= ph.L && ph.T == cfg.T;
        for (uint32_t k = 0; k < ph.m; ++k) ok = ok && ph.hi_pos[k] != send.l;
        send.pair = ok;
      }
    }
    int st = execute_steps(s, steps, local, cfg, send);
    if (st != QIPB200_OK) return st;
    if (send.pair && (st = finish_paired_exchange(s, send.R, send.l)) != QIPB200_OK) return st;
    if (left.empty()) break;
    if (first_blocked == left.size())
      return report_error(s, QIPB200_ERR_UNSUPPORTED, "internal: schedule made no progress");
    // Migrate the first blocked op's qubit only.  (Migrating the qubits of the other waiting
    // blocked ops at the same boundary as well evicts qubits that are needed again soon, which
    // costs further exchanges.)
    std::vector<char> consumed(left.size(), 0);
    {
      const size_t op_idx = remaining[left[first_blocked]];
      FlatOp f;
      const uint64_t *nu = next_use.empty() ? nullptr : &next_use[(op_idx + 1) * s->n];
      if ((st = compile_and_localize(s, &ops[op_idx], &f, nu)) != QIPB200_OK) return st;  // exchange(s) happen here
      // an uncontrolled Swap on a rank-held qubit is consumed as a relabelling of the bit map (it is
      // the first leftover op: nothing earlier can still depend on the old labels)
      if (f.cls == CLASS_IDENTITY) consumed[first_blocked] = 1;
    }
    std::vector<size_t> next;
    for (size_t i = 0; i < left.size(); ++i)
      if (!consumed[i]) next.push_back(remaining[left[i]]);
    remaining.swap(next);
  }
  return QIPB200_OK;
}

}  // namespace

bool rotate_enabled() {
  static const bool on = getenv("QIPB200_ROTATE") != nullptr && atoi(getenv("QIPB200_ROTATE")) != 0;
  return on;
}

// Unsharded state, qubit rotation: the whole schedule planned in one go over LOGICAL qubits; the state keeps the layout
// of the last pass (restored lazily by the API).  Returns false when the plan could not be made (the caller then takes the
// plain path, which also owns the error reporting for malformed ops).
static bool run_rotating(qipb200_state *s, const qip_op *ops, size_t n_ops, int *status) {
  if (!s->ctx->tile_configured) {
    if (tile_pass_configure() != cudaSuccess) return false;
    s->ctx->tile_configured = true;
  }
  const PlanConfig cfg = default_plan_config(s->prec, s->n_local);
  RotatePlan plan;
  std::string err;
  std::vector<uint32_t> layout = s->phys_of_logical;
  if ((*status = materialise_init(s)) != QIPB200_OK) return true;  // the rotating passes always load their tiles
  if (plan_rotating(ops, n_ops, s->prec, s->n_local, cfg, &plan, &err, layout.data(), false) != QIPB200_OK) return false;
  s->phys_of_logical = layout;
  *status = execute_steps(s, plan.steps, plan.singles, cfg);
  return true;
}

int restore_layout_planned(qipb200_state *s) {
  if (!s->ctx->tile_configured) {
    cudaError_t e = tile_pass_configure();
    if (e != cudaSuccess) return report_cuda_error(s, e, "cudaFuncSetAttribute(tile pass)");
    s->ctx->tile_configured = true;
  }
  const PlanConfig cfg = default_plan_config(s->prec, s->n_local);
  RotatePlan plan;
  std::string err;
  std::vector<uint32_t> layout = s->phys_of_logical;
  int st = plan_layout_restore(s->prec, s->n_local, cfg, layout.data(), &plan, &err);
  if (st != QIPB200_OK) return report_error(s, st, err);
  st = execute_steps(s, plan.steps, plan.singles, cfg);
  if (st == QIPB200_OK) s->phys_of_logical = layout;
  return st;
}

int run_schedule(qipb200_state *s, const qip_op *ops, size_t n_ops, uint32_t flags) {
  std::vector<uint64_t> next_use;  // [i * n + logical_bit]
  if (s->world > 1 && n_ops) {
    // next non-diagonal use of every logical bit after op i (backward scan)
    next_use.assign((n_ops + 1) * s->n, kNever);
    for (size_t i = n_ops; i-- > 0;) {
      for (uint32_t b = 0; b < s->n; ++b) next_use[i * s->n + b] = next_use[(i + 1) * s->n + b];
      FlatOp f;
      std::string err;
      if (compile_op(&ops[i], s->prec, s->n, &f, &err) != QIPB200_OK) continue;  // reported when executed
      if (f.cls == CLASS_DENSE || f.cls == CLASS_FLIP)
        for (size_t j = 0; j < f.tgt_sorted.size(); ++j) next_use[i * s->n + f.tgt_sorted[j]] = i;
      else if (f.cls == CLASS_GENERAL)
        for (uint32_t j = f.nc; j < f.k; ++j) next_use[i * s->n + f.idx_bits[j]] = i;
    }
  }
  const bool fuse = !(flags & QIPB200_SCHED_NO_FUSION) && s->n_local >= 6;
  if (fuse && s->world == 1 && rotate_enabled() && n_ops) {
    int st = QIPB200_OK;
    if (run_rotating(s, ops, n_ops, &st)) return st;
  }
  if (fuse) return run_fused(s, ops, n_ops, next_use);
  if (n_ops) {  // one sweep per entry: the pending basis state is written first
    const int st = materialise_init(s);
    if (st != QIPB200_OK) return st;
  }
  for (size_t i = 0; i < n_ops; ++i) {
    FlatOp f;
    const uint64_t *nu = next_use.empty() ? nullptr : &next_use[(i + 1) * s->n];
    int st = compile_and_localize(s, &ops[i], &f, nu);
    if (st != QIPB200_OK) return st;
    st = apply_flat_local(s, f);
    if (st != QIPB200_OK) return st;
  }
  return QIPB200_OK;
}

}  // namespace qipb200
