// plan_emulator.cpp -- TEST INFRASTRUCTURE: executes the fusion planner's output on the CPU
// exactly as the tile kernel would (same serialised blob, same micro-op semantics), so the
// host logic (planner.cpp, opcompile.cpp, serialisation) is validated without a GPU.
// Built by tests/test_planner_cpu.py into tests/native/_build/; never part of libqipb200.
#include <algorithm>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../rustqip_b200/csrc/opcompile.h"
#include "../../rustqip_b200/csrc/jit_codegen.h"
#include "../../rustqip_b200/csrc/tile.cuh"

#include <dlfcn.h>
#include <unistd.h>

using namespace qipb200;
typedef std::complex<double> cd;

// reference-semantics application of one compiled op on the full state (gather form)
static void apply_single(const FlatOp &f, uint32_t n, std::vector<cd> &psi) {
  const uint64_t N = 1ull << n;
  std::vector<cd> out(N);
  const uint64_t thr = f.nc ? ((1ull << f.k) - (1ull << f.kop)) : 0;
  for (uint64_t row = 0; row < N; ++row) {
    uint64_t matrow = 0;
    for (uint32_t j = 0; j < f.k; ++j) matrow |= ((row >> f.idx_bits[j]) & 1ull) << (f.k - 1 - j);
    auto full = [&](uint64_t col) {
      uint64_t c = row;
      for (uint32_t j = 0; j < f.k; ++j) {
        c &= ~(1ull << f.idx_bits[j]);
        c |= ((col >> (f.k - 1 - j)) & 1ull) << f.idx_bits[j];
      }
      return c;
    };
    cd acc(0, 0);
    if (matrow < thr) {
      acc = psi[row];
    } else {
      const uint64_t r = matrow - thr, side = 1ull << f.kop;
      if (f.base_kind == QIP_OP_SWAP) {
        const uint32_t half = f.kop >> 1;
        const uint64_t lm = ~(~0ull << half);
        acc = psi[full((((r & lm) << half) + (r >> half)) + thr)];
      } else if (f.has_dense) {
        for (uint64_t c = 0; c < side; ++c) acc += f.dense[r * side + c] * psi[full(c + thr)];
      } else {
        for (uint64_t e = f.sp_rowptr[r]; e < f.sp_rowptr[r + 1]; ++e) acc += f.sp_val[e] * psi[full(f.sp_col[e] + thr)];
      }
    }
    out[row] = acc;
  }
  psi.swap(out);
}

// elementary op on the 8 register-resident amplitudes of one group (mirrors tile_kernel.cu:
// the specialised case ids do NOT read the mask field, so the emulator derives the mask from the
// id as the kernel's straight-line code does and flags a record whose stored mask disagrees)
static int g_decode_errors = 0;

template <typename R>
static void run_elem(const Elem<R> &e, const R *mat8, cd a[8], uint64_t base, const CondTerm *conds, uint32_t n_conds) {
  if (e.op & kElemHasCond) {
    const uint32_t slot = elem_cond_slot(e.op);
    bool on = (base & e.gmask) == e.gval;
    if (slot != kCondOverflow) {
      if (slot >= n_conds || conds[slot].gmask != e.gmask || conds[slot].gval != e.gval) ++g_decode_errors;
      else on = (base & conds[slot].gmask) == conds[slot].gval;
    }
    if (!on) return;
  }
  const uint32_t id = elem_case(e.op);
  uint32_t mask = (e.op >> 12) & 0xff;
  enum { K_D1, K_X, K_PH, K_PHN, K_D3 } kind;
  bool real = false, had = false;
  uint32_t j = 0;
  if (id >= EC_D1R_FULL && id < EC_PHASE) {
    kind = K_D1;
    real = (id < EC_D1C_FULL) || (id >= EC_D1R_MASK && id < EC_D1C_MASK);
    j = (id - 1) % 3;
    if ((id < EC_D1R_MASK) != (mask == 0xf)) ++g_decode_errors;
  } else if (id >= EC_D1R_C1 && id < EC_D1R_C2) {
    kind = K_D1;
    real = true;
    j = (id - EC_D1R_C1) / 2;
    const uint32_t want = kPairMaskC1[(id - EC_D1R_C1) % 2];
    if (mask != want) ++g_decode_errors;
    mask = want;
  } else if (id >= EC_D1R_C2 && id < EC_PHASE_2) {
    kind = K_D1;
    real = true;
    j = id - EC_D1R_C2;
    if (mask != kPairMaskC2) ++g_decode_errors;
    mask = kPairMaskC2;
  } else if (id >= EC_X_FULL && id < EC_PHASEN) {
    kind = K_X;
    j = (id - EC_X_FULL) % 3;
    if ((id < EC_X_MASK) != (mask == 0xf)) ++g_decode_errors;
  } else if (id == EC_PHASEN) {
    kind = K_PHN;
  } else if (id == EC_PHASE) {
    kind = K_PH;
  } else if (id >= EC_PHASE_J && id < EC_D1R_C1) {
    kind = K_PH;
    if (mask != kPhaseMaskJ[id - EC_PHASE_J]) ++g_decode_errors;
    mask = kPhaseMaskJ[id - EC_PHASE_J];
  } else if (id >= EC_PHASE_2 && id < EC_HAD) {
    kind = K_PH;
    if (mask != kPhaseMask2[id - EC_PHASE_2]) ++g_decode_errors;
    mask = kPhaseMask2[id - EC_PHASE_2];
  } else if (id >= EC_HAD && id < EC_N_CASES) {
    kind = K_D1;
    real = true;
    j = id - EC_HAD;
    if (mask != 0xf || (e.op & kElemHasCond)) ++g_decode_errors;
    had = true;
  } else if (id == EC_DENSE3) {
    kind = K_D3;
  } else {
    ++g_decode_errors;
    return;
  }
  if (kind == K_D1) {
    uint32_t p = 0;
    for (uint32_t c = 0; c < 8; ++c) {
      if ((c >> j) & 1) continue;
      const bool on = (mask >> p) & 1;
      ++p;
      if (!on) continue;
      const uint32_t i0 = c, i1 = c | (1u << j);
      const cd x = a[i0], y = a[i1];
      if (had) {  // un-normalised butterfly: the record's matrix is not read
        a[i0] = x + y;
        a[i1] = x - y;
      } else if (real) {
        a[i0] = (double)e.m[0] * x + (double)e.m[1] * y;
        a[i1] = (double)e.m[2] * x + (double)e.m[3] * y;
      } else {
        a[i0] = cd(e.m[0], e.m[1]) * x + cd(e.m[2], e.m[3]) * y;
        a[i1] = cd(e.m[4], e.m[5]) * x + cd(e.m[6], e.m[7]) * y;
      }
    }
  } else if (kind == K_X) {
    uint32_t p = 0;
    for (uint32_t c = 0; c < 8; ++c) {
      if ((c >> j) & 1) continue;
      const bool on = (mask >> p) & 1;
      ++p;
      if (on) std::swap(a[c], a[c | (1u << j)]);
    }
  } else if (kind == K_PHN) {
    cd w(e.m[0], e.m[1]);
    const PhaseTerm<R> *t = reinterpret_cast<const PhaseTerm<R> *>(mat8);
    const uint32_t nt = (elem_size_bytes(e.op) - (uint32_t)sizeof(Elem<R>)) / (uint32_t)sizeof(PhaseTerm<R>);
    for (uint32_t k = 0; k < nt; ++k)
      if ((base & t[k].gmask) == t[k].gval) w *= cd(t[k].re, t[k].im);
    for (uint32_t c = 0; c < 8; ++c)
      if ((mask >> c) & 1) a[c] *= w;
  } else if (kind == K_PH) {
    for (uint32_t c = 0; c < 8; ++c)
      if ((mask >> c) & 1) a[c] *= cd(e.m[0], e.m[1]);
  } else {  // EC_DENSE3
    cd out[8];
    for (uint32_t u = 0; u < 8; ++u) {
      cd acc(0, 0);
      for (uint32_t v = 0; v < 8; ++v) acc += cd(mat8[2 * (u * 8 + v)], mat8[2 * (u * 8 + v) + 1]) * a[v];
      out[u] = acc;
    }
    for (uint32_t u = 0; u < 8; ++u) a[u] = out[u];
  }
}

template <typename R>
static void run_pass_params(const PassParams &pp, uint32_t n, std::vector<cd> &psi) {
  const PassHeader &h = pp.h;
  const uint32_t T = h.T, L = h.L, m = h.m;
  const uint64_t tiles = 1ull << (n - T);
  std::vector<cd> tile(1ull << T);
  for (uint64_t tau = 0; tau < tiles; ++tau) {
    uint64_t base = tau << L;  // expand: insert zeros at the high tile bits (ascending)
    for (uint32_t i = 0; i < m; ++i) {
      const uint32_t p = h.hi_pos[i];
      base = ((base >> p) << (p + 1)) | (base & ((1ull << p) - 1));
    }
    for (uint64_t t = 0; t < (1ull << T); ++t) tile[t] = psi[base + h.chunk_off[t >> L] + (t & ((1ull << L) - 1))];
    const unsigned char *rp = pp.recs;
    const CondTerm *conds = reinterpret_cast<const CondTerm *>(pp.recs + h.cond_off);
    for (uint32_t oi = 0; oi < h.n_ops; ++oi) {
      MicroOp mo;
      memcpy(&mo, rp, sizeof(mo));
      const unsigned char *data = rp + sizeof(mo);
      rp += sizeof(mo) + mo.data_bytes;
      if ((base & mo.gmask) != mo.gmask) continue;
      if (mo.kind == MK_DIAG) {
        const DiagTerm<R> *terms = reinterpret_cast<const DiagTerm<R> *>(data);
        for (uint64_t t = 0; t < (1ull << T); ++t)
          for (uint32_t k = 0; k < mo.nterms; ++k)
            if ((base & terms[k].gmask) == terms[k].gval && ((uint32_t)t & terms[k].lmask) == terms[k].lval)
              tile[t] *= cd(terms[k].re, terms[k].im);
        continue;
      }
      const uint64_t groups = 1ull << mo.groups_log2;
      for (uint64_t g = 0; g < groups; ++g) {
        uint64_t t0 = g;
        for (uint32_t i = 0; i < mo.ins_n; ++i) {
          const uint32_t p = mo.ins_pos[i];
          t0 = ((t0 >> p) << (p + 1)) | (t0 & ((1ull << p) - 1));
        }
        t0 |= mo.lor_mask;
        if (mo.kind == MK_EXCH) {
          std::swap(tile[t0 + mo.off[0]], tile[t0 + mo.off[1]]);
        } else if (mo.kind == MK_SUPER) {
          cd a[8];
          for (uint32_t u = 0; u < 8; ++u) {
            const uint32_t off = mo.off[u];
            const uint32_t want = sizeof(R) == 8 ? (off ^ ((off >> 3) & 7u)) << 4 : (off ^ (((off >> 4) & 7u) << 1)) << 3;
            if (g == 0 && mo.soff[u] != want) ++g_decode_errors;
            a[u] = tile[t0 + off];
          }
          {  // the kernel expands the group counter with t += t & (~0 << p): must equal the bit insertion
            uint32_t t = (uint32_t)g;
            for (uint32_t i = 0; i < 3; ++i) t += t & (~0u << mo.ins_pos[i]);
            if (mo.ins_n != 3 || mo.lor_mask != 0 || t != (uint32_t)t0) ++g_decode_errors;
          }
          const unsigned char *ep = data;
          for (;;) {
            Elem<R> e;
            memcpy(&e, ep, sizeof(e));
            if (elem_case(e.op) == EC_END) break;
            const R *mat8 = reinterpret_cast<const R *>(ep + sizeof(e));
            ep += elem_size_bytes(e.op);
            run_elem<R>(e, mat8, a, base, conds, h.n_conds);
          }
          for (uint32_t u = 0; u < 8; ++u) tile[t0 + mo.off[u]] = a[u];
        } else {
          const uint32_t S = 1u << mo.k;
          const R *mat = reinterpret_cast<const R *>(data);
          cd in[8], out[8];
          for (uint32_t u = 0; u < S; ++u) in[u] = tile[t0 + mo.off[u]];
          for (uint32_t u = 0; u < S; ++u) {
            cd acc(0, 0);
            for (uint32_t v = 0; v < S; ++v) acc += cd(mat[2 * (u * S + v)], mat[2 * (u * S + v) + 1]) * in[v];
            out[u] = acc;
          }
          for (uint32_t u = 0; u < S; ++u) tile[t0 + mo.off[u]] = out[u];
        }
      }
    }
    // CTA-uniform phase terms, applied once at store time
    cd gp(1, 0);
    const GlobalTerm<R> *gt = reinterpret_cast<const GlobalTerm<R> *>(pp.recs + h.gterm_off);
    for (uint32_t k = 0; k < h.n_gterms; ++k)
      if ((base & gt[k].gmask) == gt[k].gval) gp *= cd(gt[k].re, gt[k].im);
    for (uint64_t t = 0; t < (1ull << T); ++t) psi[base + h.chunk_off[t >> L] + (t & ((1ull << L) - 1))] = tile[t] * gp;
  }
}

// number of elementary records whose condition did not get a slot of the pass's condition table
template <typename R>
static uint64_t count_overflow_conditions(const PassParams &pp) {
  uint64_t n = 0;
  const unsigned char *rp = pp.recs;
  for (uint32_t oi = 0; oi < pp.h.n_ops; ++oi) {
    MicroOp mo;
    memcpy(&mo, rp, sizeof(mo));
    const unsigned char *ep = rp + sizeof(mo);
    rp += sizeof(mo) + mo.data_bytes;
    if (mo.kind != MK_SUPER) continue;
    for (;;) {
      Elem<R> e;
      memcpy(&e, ep, sizeof(e));
      if (elem_case(e.op) == EC_END) break;
      if ((e.op & kElemHasCond) && elem_cond_slot(e.op) == kCondOverflow) ++n;
      ep += elem_size_bytes(e.op);
    }
  }
  return n;
}

extern "C" int emul_schedule(int prec, uint32_t n, const qip_op *ops, size_t n_ops, double *state, uint32_t T,
                             uint32_t L, int fuse_blocks, uint32_t max_k, uint64_t *stats, char *errbuf,
                             size_t errlen) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err);
    if (st != QIPB200_OK) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
      return st;
    }
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  cfg.fuse_blocks = fuse_blocks != 0;
  if (max_k) cfg.compose_threshold = max_k;
  std::vector<PlanStep> steps;
  plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  g_decode_errors = 0;
  std::vector<cd> psi(1ull << n);
  for (uint64_t i = 0; i < (1ull << n); ++i) psi[i] = cd(state[2 * i], state[2 * i + 1]);
  uint64_t n_pass = 0, n_single = 0, n_micro = 0, n_gates_in_pass = 0, n_overflow = 0, max_conds = 0;
  for (size_t s = 0; s < steps.size(); ++s) {
    if (steps[s].is_pass) {
      PassParams pp;
      if (!serialise_pass(steps[s].pass, &pp)) {
        if (errbuf && errlen) snprintf(errbuf, errlen, "pass does not fit the parameter space");
        return -2;
      }
      n_overflow += prec == QIP_F32 ? count_overflow_conditions<float>(pp) : count_overflow_conditions<double>(pp);
      if (pp.h.n_conds > max_conds) max_conds = pp.h.n_conds;
      if (prec == QIP_F32)
        run_pass_params<float>(pp, n, psi);
      else
        run_pass_params<double>(pp, n, psi);
      ++n_pass;
      n_micro += steps[s].pass.ops.size();
      n_gates_in_pass += steps[s].pass.n_gates;
    } else {
      apply_single(flat[steps[s].op_index], n, psi);
      ++n_single;
    }
  }
  for (uint64_t i = 0; i < (1ull << n); ++i) {
    state[2 * i] = psi[i].real();
    state[2 * i + 1] = psi[i].imag();
  }
  if (stats) {
    stats[0] = n_pass;
    stats[1] = n_single;
    stats[2] = n_micro;
    stats[3] = n_gates_in_pass;
    stats[4] = n_overflow;
    stats[5] = max_conds;
  }
  if (g_decode_errors) {
    if (errbuf && errlen) snprintf(errbuf, errlen, "%d records disagree with their case id / condition slot / offsets", g_decode_errors);
    return -3;
  }
  return 0;
}

// The epoch loop of a sharded state (schedule.cu: run_fused) without the sharding: ops whose non-diagonal bits
// touch `remote_bits` are BLOCKED (as if a rank index held those qubits); each epoch plans and runs what may
// run, then "migrates" for the first blocked op that is left (here: simply unblocks it) and starts over.
// Validates the commutation rules of plan_passes(blocked, leftover, dep) on one address space.
extern "C" int emul_schedule_blocked(int prec, uint32_t n, const qip_op *ops, size_t n_ops, double *state, uint32_t T,
                                     uint32_t L, uint64_t remote_bits, uint64_t *stats, char *errbuf, size_t errlen) {
  std::vector<FlatOp> flat(n_ops);
  std::vector<DepMasks> dep_all(n_ops);
  std::vector<char> blocked_all(n_ops, 0);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err);
    if (st != QIPB200_OK) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
      return st;
    }
    op_dependency_masks(flat[i], &dep_all[i]);
    blocked_all[i] = (dep_all[i].nd & remote_bits) ? 1 : 0;
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  g_decode_errors = 0;
  std::vector<cd> psi(1ull << n);
  for (uint64_t i = 0; i < (1ull << n); ++i) psi[i] = cd(state[2 * i], state[2 * i + 1]);
  std::vector<size_t> remaining(n_ops);
  for (size_t i = 0; i < n_ops; ++i) remaining[i] = i;
  uint64_t epochs = 0, n_pass = 0;
  while (!remaining.empty()) {
    ++epochs;
    std::vector<FlatOp> local(remaining.size());
    std::vector<char> blocked(remaining.size());
    std::vector<DepMasks> dep(remaining.size());
    for (size_t r = 0; r < remaining.size(); ++r) {
      local[r] = flat[remaining[r]];
      blocked[r] = blocked_all[remaining[r]];
      dep[r] = dep_all[remaining[r]];
    }
    std::vector<PlanStep> steps;
    std::vector<size_t> left;
    plan_passes(local, n, (qip_prec)prec, cfg, &steps, &blocked, &left, &dep);
    for (size_t s = 0; s < steps.size(); ++s) {
      if (steps[s].is_pass) {
        PassParams pp;
        if (!serialise_pass(steps[s].pass, &pp)) return -2;
        if (prec == QIP_F32)
          run_pass_params<float>(pp, n, psi);
        else
          run_pass_params<double>(pp, n, psi);
        ++n_pass;
      } else {
        if (blocked[steps[s].op_index]) return -4;  // a blocked op must never be scheduled
        apply_single(local[steps[s].op_index], n, psi);
      }
    }
    if (left.empty()) break;
    size_t first_blocked = left.size();
    for (size_t i = 0; i < left.size(); ++i)
      if (blocked[left[i]]) {
        first_blocked = i;
        break;
      }
    if (first_blocked == left.size()) return -5;  // no progress and nothing to migrate for
    blocked_all[remaining[left[first_blocked]]] = 0;
    std::vector<size_t> next;
    for (size_t i = 0; i < left.size(); ++i) next.push_back(remaining[left[i]]);
    remaining.swap(next);
  }
  for (uint64_t i = 0; i < (1ull << n); ++i) {
    state[2 * i] = psi[i].real();
    state[2 * i + 1] = psi[i].imag();
  }
  if (stats) {
    stats[0] = n_pass;
    stats[1] = epochs;
  }
  if (g_decode_errors) return -3;
  return 0;
}

// A 2^g-way SHARDED state with rank-independent planning (schedule.cu: run_fused in paired-send mode): every epoch,
// every virtual rank restricts the remaining ops to itself (opcompile.cpp: restrict_flat_op), plans with the uniform
// selection data (op_uniform_info of the all-ones rank) and must arrive at the SAME steps -- same tile bits, same ops
// taken, same single steps, same leftovers -- because a migration fused into a pass pairs up tiles across GPUs.  The
// passes are then executed per rank on its shard (what each rank emitted for ITSELF, ops that are the identity on a rank
// included), single steps and migrations on the whole vector.  Returns -10 when two ranks plan differently.
// stats: [0] passes, [1] epochs, [2] migrations, [3] ops that were the identity on at least one rank but not on all.
static void swap_index_bits(std::vector<cd> &psi, uint32_t a, uint32_t b) {
  if (a == b) return;
  for (uint64_t i = 0; i < psi.size(); ++i)
    if (((i >> a) & 1ull) == 0 && ((i >> b) & 1ull) == 1) std::swap(psi[i], psi[i ^ (1ull << a) ^ (1ull << b)]);
}

extern "C" int emul_sharded_uniform(int prec, uint32_t n, uint32_t g, const qip_op *ops, size_t n_ops, double *state, uint32_t T,
                                    uint32_t L, uint64_t *stats, char *errbuf, size_t errlen) {
  const uint32_t nl = n - g, world = 1u << g;
  std::vector<uint32_t> phys(n);
  for (uint32_t b = 0; b < n; ++b) phys[b] = b;
  PlanConfig cfg = default_plan_config((qip_prec)prec, nl);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  g_decode_errors = 0;
  std::vector<cd> psi(1ull << n);
  for (uint64_t i = 0; i < (1ull << n); ++i) psi[i] = cd(state[2 * i], state[2 * i + 1]);
  std::vector<size_t> remaining(n_ops);
  for (size_t i = 0; i < n_ops; ++i) remaining[i] = i;
  uint64_t epochs = 0, n_pass = 0, n_mig = 0, n_mixed = 0;
  auto fail = [&](int code, const std::string &msg) {
    if (errbuf && errlen) snprintf(errbuf, errlen, "%s", msg.c_str());
    return code;
  };
  while (!remaining.empty()) {
    ++epochs;
    std::vector<FlatOp> flat(remaining.size());
    std::vector<char> blocked(remaining.size(), 0);
    std::vector<DepMasks> dep(remaining.size());
    for (size_t r = 0; r < remaining.size(); ++r) {
      std::string err;
      int st = compile_op(&ops[remaining[r]], (qip_prec)prec, n, &flat[r], &err, phys.data());
      if (st != QIPB200_OK) return fail(st, err);
      op_dependency_masks(flat[r], &dep[r]);
      blocked[r] = (dep[r].nd >> nl) ? 1 : 0;
      FlatOp fv;
      bool skipv = false;
      restrict_flat_op(flat[r], nl, (int)world - 1, &fv, &skipv);
      if (skipv) {
        fv = FlatOp();
        fv.cls = CLASS_IDENTITY;
      }
      if (!getenv("EMUL_NO_UNIFORM")) op_uniform_info(fv, &dep[r]);
    }
    std::vector<std::vector<PlanStep>> steps(world);
    std::vector<std::vector<FlatOp>> local(world, std::vector<FlatOp>(remaining.size()));
    std::vector<size_t> left0;
    for (uint32_t rk = 0; rk < world; ++rk) {
      std::vector<size_t> left;
      for (size_t r = 0; r < remaining.size(); ++r) {
        if (blocked[r]) {
          local[rk][r] = flat[r];
          continue;
        }
        bool skip = false;
        restrict_flat_op(flat[r], nl, (int)rk, &local[rk][r], &skip);
        if (skip) {
          local[rk][r] = FlatOp();
          local[rk][r].cls = CLASS_IDENTITY;
        }
      }
      plan_passes(local[rk], nl, (qip_prec)prec, cfg, &steps[rk], &blocked, &left, &dep);
      if (rk == 0) {
        left0 = left;
      } else {
        if (left != left0 || steps[rk].size() != steps[0].size()) return fail(-10, "ranks disagree on the number of steps / leftovers");
        for (size_t s = 0; s < steps[0].size(); ++s) {
          const PlanStep &a = steps[0][s], &b = steps[rk][s];
          if (a.is_pass != b.is_pass) return fail(-10, "ranks disagree on the kind of a step");
          if (!a.is_pass && a.op_index != b.op_index) return fail(-10, "ranks disagree on a single step");
          if (a.is_pass && (memcmp(a.pass.hdr.hi_pos, b.pass.hdr.hi_pos, sizeof(a.pass.hdr.hi_pos)) != 0 || a.pass.hdr.T != b.pass.hdr.T ||
                            a.pass.hdr.L != b.pass.hdr.L || a.pass.n_gates != b.pass.n_gates))
            return fail(-10, "ranks disagree on the tile bits / the gates of a pass");
        }
      }
    }
    for (size_t r = 0; r < remaining.size(); ++r) {
      if (blocked[r]) continue;
      bool any = false, all = true;
      for (uint32_t rk = 0; rk < world; ++rk) {
        const bool id = local[rk][r].cls == CLASS_IDENTITY;
        any = any || id;
        all = all && id;
      }
      if (any && !all) ++n_mixed;
    }
    for (size_t s = 0; s < steps[0].size(); ++s) {
      if (!steps[0][s].is_pass) {
        if (blocked[steps[0][s].op_index]) return fail(-4, "a blocked op was scheduled");
        apply_single(flat[steps[0][s].op_index], n, psi);  // == every rank applying its restriction to its shard
        continue;
      }
      for (uint32_t rk = 0; rk < world; ++rk) {
        PassParams pp;
        if (!serialise_pass(steps[rk][s].pass, &pp)) return fail(-2, "pass exceeds the parameter space");
        std::vector<cd> shard(psi.begin() + ((uint64_t)rk << nl), psi.begin() + ((uint64_t)(rk + 1) << nl));
        if (prec == QIP_F32)
          run_pass_params<float>(pp, nl, shard);
        else
          run_pass_params<double>(pp, nl, shard);
        std::copy(shard.begin(), shard.end(), psi.begin() + ((uint64_t)rk << nl));
      }
      ++n_pass;
    }
    if (left0.empty()) break;
    size_t fb = left0.size();
    for (size_t i = 0; i < left0.size(); ++i)
      if (blocked[left0[i]]) {
        fb = i;
        break;
      }
    if (fb == left0.size()) return fail(-5, "no progress and nothing to migrate for");
    // migrate: every rank-held non-diagonal bit of the first blocked op trades places with the highest free local bit
    const FlatOp &f = flat[left0[fb]];
    uint64_t used = dep[left0[fb]].nd | dep[left0[fb]].dg;
    for (uint32_t R = nl; R < n; ++R) {
      if (!((dep[left0[fb]].nd >> R) & 1ull)) continue;
      int l = -1;
      for (int b = (int)nl - 1; b >= 0; --b)
        if (!((used >> b) & 1ull)) {
          l = b;
          break;
        }
      if (l < 0) return fail(-6, "op touches every local bit");
      swap_index_bits(psi, R, (uint32_t)l);
      for (uint32_t b = 0; b < n; ++b) {
        if (phys[b] == R)
          phys[b] = (uint32_t)l;
        else if (phys[b] == (uint32_t)l)
          phys[b] = R;
      }
      used |= 1ull << l;
      ++n_mig;
    }
    (void)f;
    std::vector<size_t> next;
    for (size_t i = 0; i < left0.size(); ++i) next.push_back(remaining[left0[i]]);
    remaining.swap(next);
  }
  // restore the canonical layout: logical bit b back at physical bit b
  for (uint32_t b = 0; b < n; ++b) {
    if (phys[b] == b) continue;
    const uint32_t where = phys[b];
    swap_index_bits(psi, b, where);
    for (uint32_t c = 0; c < n; ++c) {
      if (phys[c] == b)
        phys[c] = where;
      else if (phys[c] == where)
        phys[c] = b;
    }
  }
  for (uint64_t i = 0; i < (1ull << n); ++i) {
    state[2 * i] = psi[i].real();
    state[2 * i + 1] = psi[i].imag();
  }
  if (stats) {
    stats[0] = n_pass;
    stats[1] = epochs;
    stats[2] = n_mig;
    stats[3] = n_mixed;
  }
  if (g_decode_errors) return fail(-3, "decode errors");
  return 0;
}

// Planning with qubit rotation (planner.cpp: plan_rotating): passes that end with a permutation of their tile bits, tracked
// layout, restore folded into the last pass / swap-only passes (restore != 0) or left to the caller (restore == 0: the
// layout the state is left in comes back in `layout`, n entries logical -> physical, also the layout it starts in;
// unpermute != 0 brings the amplitudes back to the canonical order here, for the comparison with the oracle).
// Executed on the CPU; the result must be the plain schedule's.  state == NULL: plan only.
// stats: [0] passes, [1] single steps, [2] relabelling swaps, [3] restore steps, [4] gates in passes
extern "C" int emul_schedule_rotate(int prec, uint32_t n, const qip_op *ops, size_t n_ops, double *state, uint32_t T, uint32_t L,
                                    int restore, uint32_t *layout, int unpermute, uint64_t *stats, char *errbuf, size_t errlen) {
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  RotatePlan plan;
  std::string err;
  std::vector<uint32_t> lay(n);
  for (uint32_t b = 0; b < n; ++b) lay[b] = layout ? layout[b] : b;
  int st = plan_rotating(ops, n_ops, (qip_prec)prec, n, cfg, &plan, &err, lay.data(), restore != 0);
  if (st != QIPB200_OK) {
    if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
    return st;
  }
  uint64_t n_pass = 0, n_single = 0, n_gates = 0;
  if (state) {
    g_decode_errors = 0;
    std::vector<cd> psi(1ull << n);
    for (uint64_t i = 0; i < (1ull << n); ++i) psi[i] = cd(state[2 * i], state[2 * i + 1]);
    auto run_steps = [&](const RotatePlan &pl) -> int {
      for (size_t s = 0; s < pl.steps.size(); ++s) {
        if (pl.steps[s].is_pass) {
          PassParams pp;
          if (!serialise_pass(pl.steps[s].pass, &pp)) return -2;
          if (prec == QIP_F32)
            run_pass_params<float>(pp, n, psi);
          else
            run_pass_params<double>(pp, n, psi);
        } else {
          apply_single(pl.singles[pl.steps[s].op_index], n, psi);
        }
      }
      return 0;
    };
    int rc = run_steps(plan);
    if (rc) return rc;
    if (unpermute) {  // what the API does before a download: planned swap-only steps (planner.cpp: plan_layout_restore)
      RotatePlan back;
      st = plan_layout_restore((qip_prec)prec, n, cfg, lay.data(), &back, &err);
      if (st != QIPB200_OK) return st;
      rc = run_steps(back);
      if (rc) return rc;
      plan.n_restore_steps += back.n_restore_steps;
    }
    for (uint64_t i = 0; i < (1ull << n); ++i) {
      state[2 * i] = psi[i].real();
      state[2 * i + 1] = psi[i].imag();
    }
    if (g_decode_errors) return -3;
  }
  if (layout)
    for (uint32_t b = 0; b < n; ++b) layout[b] = lay[b];
  for (size_t s = 0; s < plan.steps.size(); ++s) {
    if (plan.steps[s].is_pass) {
      ++n_pass;
      n_gates += plan.steps[s].pass.n_gates;
    } else {
      ++n_single;
    }
  }
  if (stats) {
    stats[0] = n_pass;
    stats[1] = n_single;
    stats[2] = plan.n_swaps;
    stats[3] = plan.n_restore_steps;
    stats[4] = n_gates;
  }
  return 0;
}

// Generated-kernel statistics of a whole plan (no amplitudes): rotate != 0: the rotating planner (lazy layout).
// stats: [0] passes, [1] passes the generator declined, [2] super-ops (shared-memory round trips), [3] elementary ops,
//        [4] CTA barriers, [5] warp syncs, [6] renamed (instruction-free) ops
extern "C" int emul_jit_plan_stats(int prec, uint32_t n, const qip_op *ops, size_t n_ops, int rotate, uint64_t *stats) {
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  std::vector<PlanStep> steps;
  RotatePlan rplan;
  if (rotate) {
    std::string err;
    if (plan_rotating(ops, n_ops, (qip_prec)prec, n, cfg, &rplan, &err, nullptr, false) != QIPB200_OK) return -1;
    steps = rplan.steps;
  } else {
    std::vector<FlatOp> flat(n_ops);
    for (size_t i = 0; i < n_ops; ++i) {
      std::string err;
      if (compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err) != QIPB200_OK) return -1;
    }
    plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  }
  for (int i = 0; i < 8; ++i) stats[i] = 0;
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) continue;
    ++stats[0];
    JitProgram prog;
    std::string why;
    if (!jit_generate(steps[s].pass, (qip_prec)prec, &prog, &why)) {
      ++stats[1];
      continue;
    }
    stats[2] += prog.n_super;
    stats[3] += prog.n_elems;
    stats[4] += prog.n_cta_barriers;
    stats[5] += prog.n_warp_syncs;
    stats[6] += prog.n_renamed;
  }
  return 0;
}

// Coverage histogram of a plan (no amplitudes): which shapes the planner and the generator emitted for a circuit, so a
// test can assert that a circuit family reaches every one of them.
// hist: [0..39] interpreter case ids (EC_*) of the serialised records; [40..44] JElem kinds of the generated-kernel view
//       (D1, X, PH, DK, HAD); [45] JElem phases with a thread predicate (pm != 0); [46] JElem phases with thread-term
//       factors; [47] JElem phases with CTA-uniform factor terms; [48] JElems under a CTA-uniform condition;
//       [49] / [50] conditional exchanges folded into a load / store address of the generated source;
//       [51] records on the condition-table overflow path; [52] passes; [53] passes the generator declined;
//       [54] single steps; [55] CTA-uniform store-time phase terms; [56] MK_DENSE, [57] MK_DIAG, [58] MK_EXCH micro-ops;
//       [59] most distinct CTA-uniform conditions of the generated-kernel view in one pass; [60] fewest tiles of a pass
//       (2^(n-T)); [61] passes the generator declined although they hold register-group work and every op fits a group;
//       [62] passes holding an op wider than a register group; [63] passes with no register-group work at all (only
//       CTA-uniform store-time phases) -- [62] and [63] run the interpreter kernel by design
static uint64_t count_substr(const std::string &s, const char *what) {
  uint64_t n = 0;
  for (size_t at = s.find(what); at != std::string::npos; at = s.find(what, at + 1)) ++n;
  return n;
}

extern "C" int emul_plan_coverage(int prec, uint32_t n, const qip_op *ops, size_t n_ops, uint32_t T, uint32_t L, uint64_t *hist) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    if (compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err) != QIPB200_OK) return -1;
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  std::vector<PlanStep> steps;
  plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  for (int i = 0; i < 64; ++i) hist[i] = 0;
  const size_t gsz = prec == QIP_F32 ? sizeof(GlobalTerm<float>) : sizeof(GlobalTerm<double>);
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) {
      ++hist[54];
      continue;
    }
    const HostPass &p = steps[s].pass;
    ++hist[52];
    hist[55] += p.gterms.size() / gsz;
    const uint64_t tiles = 1ull << (n - p.hdr.T);
    if (hist[60] == 0 || tiles < hist[60]) hist[60] = tiles;
    if (p.jbits == 0) ++hist[62];
    if (p.jbits != 0 && p.jgroups.empty()) ++hist[63];
    std::vector<std::pair<uint64_t, uint64_t>> conds;
    for (size_t i = 0; i < p.ops.size(); ++i) {
      const MicroOp &mo = p.ops[i].h;
      if (mo.kind == MK_DENSE) ++hist[56];
      if (mo.kind == MK_DIAG) ++hist[57];
      if (mo.kind == MK_EXCH) ++hist[58];
      if (mo.kind != MK_SUPER) continue;
      const unsigned char *ep = p.ops[i].data.data();
      for (;;) {
        uint32_t op;
        memcpy(&op, ep, 4);
        if (elem_case(op) == EC_END) break;
        ++hist[elem_case(op)];
        if ((op & kElemHasCond) && elem_cond_slot(op) == kCondOverflow) ++hist[51];
        ep += elem_size_bytes(op);
      }
    }
    for (size_t g = 0; g < p.jgroups.size(); ++g)
      for (size_t e = 0; e < p.jgroups[g].elems.size(); ++e) {
        const JElem &d = p.jgroups[g].elems[e];
        ++hist[40 + d.kind];
        if (d.kind == JElem::PH && d.pm) ++hist[45];
        if (d.kind == JElem::PH && !d.tterms.empty()) ++hist[46];
        if (d.kind == JElem::PH && !d.terms.empty()) ++hist[47];
        if (d.gmask) ++hist[48];
        if (d.gmask && std::find(conds.begin(), conds.end(), std::make_pair(d.gmask, d.gval)) == conds.end())
          conds.push_back(std::make_pair(d.gmask, d.gval));
      }
    if (conds.size() > hist[59]) hist[59] = conds.size();
    JitProgram prog;
    std::string why;
    if (!jit_generate(p, (qip_prec)prec, &prog, &why)) {
      ++hist[53];
      if (p.jbits != 0 && !p.jgroups.empty()) ++hist[61];
      continue;
    }
    hist[49] += count_substr(prog.source, "const unsigned la");
    hist[50] += count_substr(prog.source, "const unsigned sa");
  }
  return 0;
}

// plan only (no amplitudes): pass / single-step counts for big circuits
extern "C" int emul_plan_stats(int prec, uint32_t n, const qip_op *ops, size_t n_ops, uint32_t T, uint32_t L,
                               int fuse_blocks, uint32_t max_k, uint64_t *stats) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err);
    if (st != QIPB200_OK) return st;
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  cfg.fuse_blocks = fuse_blocks != 0;
  if (max_k) cfg.compose_threshold = max_k;
  std::vector<PlanStep> steps;
  plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  uint64_t n_pass = 0, n_single = 0, n_micro = 0, n_gates_in_pass = 0, dense_k[4] = {0, 0, 0, 0}, diag_terms = 0, exch = 0;
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) {
      ++n_single;
      continue;
    }
    ++n_pass;
    n_micro += steps[s].pass.ops.size();
    n_gates_in_pass += steps[s].pass.n_gates;
    if (getenv("PLAN_TRACE")) {  // one line per pass: gates, then each micro-op as bits:elems
      fprintf(stderr, "pass %2llu: %3u gates |", (unsigned long long)n_pass, steps[s].pass.n_gates);
      for (size_t i = 0; i < steps[s].pass.ops.size(); ++i) {
        const MicroOp &mo = steps[s].pass.ops[i].h;
        fprintf(stderr, " {%u,%u,%u}:%u", mo.ins_pos[0], mo.ins_pos[1], mo.ins_pos[2], mo.nterms);
      }
      fprintf(stderr, "\n");
    }
    for (size_t i = 0; i < steps[s].pass.ops.size(); ++i) {
      const MicroOp &mo = steps[s].pass.ops[i].h;
      if (mo.kind == MK_DENSE) dense_k[mo.k]++;
      else if (mo.kind == MK_DIAG) diag_terms += mo.nterms;
      else if (mo.kind == MK_SUPER) {
        dense_k[0]++;
        exch += mo.nterms;
        const unsigned char *ep = steps[s].pass.ops[i].data.data();
        for (;;) {
          uint32_t op;
          memcpy(&op, ep, 4);
          if (elem_case(op) == EC_END) break;
          stats[16 + elem_case(op)]++;
          if (op & kElemHasCond) stats[15]++;
          ep += elem_size_bytes(op);
        }
      }
      else dense_k[1]++;
    }
  }
  stats[0] = n_pass; stats[1] = n_single; stats[2] = n_micro; stats[3] = n_gates_in_pass;
  stats[4] = dense_k[0]; /* super-ops */ stats[5] = exch; /* elementary ops */ stats[6] = dense_k[2] + dense_k[3]; stats[7] = diag_terms; stats[8] = dense_k[1];
  return 0;
}


// ---- generated (JIT) pass kernels, compiled for the HOST ------------------------------------------------
// Same planner, but every pass is turned into specialised source by jit_generate (rustqip_b200/csrc/jit_codegen.cpp),
// compiled with g++ -DQIP_JIT_HOST and run on the host copy of the state: the code generator (thread maps,
// addressing, renaming, zero/one folding, parameter block layout) is validated against the oracle without a GPU.
// stats: [0] passes run through generated code, [1] passes the generator declined (emulated instead),
//        [2] single-op steps, [3] CTA barriers, [4] warp syncs, [5] renamed (instruction-free) ops, [6] elementary ops
extern "C" int emul_schedule_jit(int prec, uint32_t n, const qip_op *ops, size_t n_ops, void *state, uint32_t T, uint32_t L,
                                 const char *workdir, uint64_t *stats, char *errbuf, size_t errlen) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err);
    if (st != QIPB200_OK) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
      return st;
    }
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  std::vector<PlanStep> steps;
  RotatePlan rplan;
  if (getenv("EMUL_ROTATE")) {  // the rotating planner's passes (end-of-pass swaps = renaming) through the generated kernels
    std::string err;
    int st = plan_rotating(ops, n_ops, (qip_prec)prec, n, cfg, &rplan, &err);
    if (st != QIPB200_OK) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
      return st;
    }
    steps = rplan.steps;
    flat = rplan.singles;  // single steps index the plan's own op list
  } else {
    plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  }
  const uint64_t N = 1ull << n;
  uint64_t st_[8] = {0};
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) {  // single op through the reference-semantics gather (via complex<double>)
      std::vector<cd> psi(N);
      if (prec == QIP_F32) {
        const float *f = (const float *)state;
        for (uint64_t i = 0; i < N; ++i) psi[i] = cd(f[2 * i], f[2 * i + 1]);
      } else {
        const double *f = (const double *)state;
        for (uint64_t i = 0; i < N; ++i) psi[i] = cd(f[2 * i], f[2 * i + 1]);
      }
      apply_single(flat[steps[s].op_index], n, psi);
      for (uint64_t i = 0; i < N; ++i) {
        if (prec == QIP_F32) {
          ((float *)state)[2 * i] = (float)psi[i].real();
          ((float *)state)[2 * i + 1] = (float)psi[i].imag();
        } else {
          ((double *)state)[2 * i] = psi[i].real();
          ((double *)state)[2 * i + 1] = psi[i].imag();
        }
      }
      ++st_[2];
      continue;
    }
    JitProgram prog;
    std::string why;
    if (!jit_generate(steps[s].pass, (qip_prec)prec, &prog, &why)) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "generator declined pass %zu: %s", s, why.c_str());
      ++st_[1];
      return -4;
    }
    char base[512];
    snprintf(base, sizeof(base), "%s/jitpass_%d_%zu", workdir, (int)getpid(), s);
    const std::string cu = std::string(base) + ".cpp", so = std::string(base) + ".so";
    FILE *f = fopen(cu.c_str(), "w");
    if (!f) return -5;
    fwrite(prog.source.data(), 1, prog.source.size(), f);
    fclose(f);
    const std::string cmd = "/usr/bin/g++ -x c++ -std=c++17 -O1 -ffp-contract=off -DQIP_JIT_HOST -fPIC -shared -o " + so + " " + cu + " 2> " +
                            std::string(base) + ".log";
    if (system(cmd.c_str()) != 0) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "g++ failed on the generated source of pass %zu (see %s.log)", s, base);
      return -6;
    }
    void *h = dlopen(so.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (!h) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "dlopen: %s", dlerror());
      return -7;
    }
    typedef void (*Fn)(void *, const void *, unsigned);
    Fn fn = (Fn)dlsym(h, "qip_host_pass");
    if (!fn) return -8;
    fn(state, prog.params.data(), n);
    dlclose(h);
    unlink(so.c_str());
    ++st_[0];
    st_[3] += prog.n_cta_barriers;
    st_[4] += prog.n_warp_syncs;
    st_[5] += prog.n_renamed;
    st_[6] += prog.n_elems;
  }
  if (stats) memcpy(stats, st_, sizeof(st_));
  return 0;
}

// Source + parameter block of every pass of a schedule (no execution): for offline inspection (nvcc / cuobjdump).
extern "C" int emul_dump_jit(int prec, uint32_t n, const qip_op *ops, size_t n_ops, const char *prefix) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    if (compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err) != QIPB200_OK) return -1;
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  std::vector<PlanStep> steps;
  plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  int k = 0;
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) continue;
    JitProgram prog;
    std::string why;
    char name[512];
    if (!jit_generate(steps[s].pass, (qip_prec)prec, &prog, &why, getenv("JIT_DUMP_PAIRED") != nullptr)) {
      fprintf(stderr, "pass %zu declined: %s\n", s, why.c_str());
      continue;
    }
    snprintf(name, sizeof(name), "%s_%03d.cu", prefix, k++);
    FILE *f = fopen(name, "w");
    if (!f) return -2;
    fwrite(prog.source.data(), 1, prog.source.size(), f);
    fclose(f);
    fprintf(stderr, "%s: %u super-ops, %u elems (%u renamed), %u CTA barriers, %u warp syncs, %u consts, %zu param bytes\n", name,
            prog.n_super, prog.n_elems, prog.n_renamed, prog.n_cta_barriers, prog.n_warp_syncs, prog.n_consts, prog.params.size());
  }
  return k;
}
