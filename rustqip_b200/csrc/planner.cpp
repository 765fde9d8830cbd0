// planner.cpp -- host-side fusion planner: turns a list of compiled local ops into
// fused shared-memory tile passes (tile.cuh) and single-op steps.  Pure C++.
//
// This is the "fusion scheduler" row of SURVEY.md section 8f (N4): what the reference's
// apply_ops (qip-iterators/src/matrix_ops.rs:158-219) aspired to.  The fused result
// is DEFINED as the sequential product of the single-op semantics.
//
// Reordering rule.  Every op acts on each of its index bits either DIAGONALLY (a
// control bit, or a bit of a diagonal gate) or NON-DIAGONALLY (a target of a dense
// block / X / Swap).  Two ops commute if on every shared bit both act diagonally.
// A pass takes ops in program order, skipping an op only when it does not fit; an
// op may overtake a skipped one only if the two commute by the rule above.
//
// Inside a pass, ops are grouped into SUPER-OPS: lists of elementary ops on <= 3
// tile-local bits that one thread executes on 8 register-resident amplitudes.  Groups
// on disjoint bit sets commute, so several stay open at once; an op whose bits span
// groups merges them (if <= 3 bits in total) or closes them.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "tile.cuh"

namespace qipb200 {

namespace {

inline int popc(uint64_t x) { return __builtin_popcountll(x); }
inline bool is_one(const cplx &c) { return c.real() == 1.0 && c.imag() == 0.0; }

struct OpInfo {
  uint64_t nd = 0;        // bits acted on non-diagonally
  uint64_t dg = 0;        // bits acted on diagonally
  uint64_t need_tile = 0; // bits that must be tile bits for the op to run in a pass
  bool tile_ok = false;
  double unfused_cost = 1.0;  // HBM sweeps of the per-gate kernel
  uint32_t est_bytes = 0;     // upper bound of the descriptor bytes in a pass
};

OpInfo analyse(const FlatOp &f) {
  OpInfo o;
  const int nctrl = popc(f.ctrl_mask);
  switch (f.cls) {
    case CLASS_DENSE:
      for (size_t i = 0; i < f.tgt_sorted.size(); ++i) o.nd |= 1ull << f.tgt_sorted[i];
      o.dg = f.ctrl_mask;
      o.need_tile = o.nd;
      o.tile_ok = f.tgt_sorted.size() <= 3 && f.tgt_sorted.size() + nctrl <= 6;
      o.unfused_cost = 1.0 / (1 << nctrl);
      o.est_bytes = f.tgt_sorted.size() == 1 ? 368 : (uint32_t)sizeof(MicroOp) + 2 * 112 + 1040;
      break;
    case CLASS_FLIP:
      o.nd = 1ull << f.tgt_sorted[0];
      o.dg = f.ctrl_mask;
      o.need_tile = o.nd;
      o.tile_ok = nctrl + 1 <= 6;
      o.unfused_cost = 1.0 / (1 << nctrl);
      o.est_bytes = 368;
      break;
    case CLASS_BITSWAP:
      for (size_t i = 0; i < f.swaps.size(); ++i) o.nd |= (1ull << f.swaps[i].first) | (1ull << f.swaps[i].second);
      o.dg = f.ctrl_mask;
      o.need_tile = o.nd;
      o.tile_ok = nctrl + 2 <= 6 && f.swaps.size() <= 3;
      o.unfused_cost = 0.5 * f.swaps.size() / (1 << nctrl);
      o.est_bytes = 640 * (uint32_t)f.swaps.size();
      break;
    case CLASS_DIAGONAL:
      o.dg = f.ctrl_mask;
      for (size_t i = 0; i < f.diag_bits.size(); ++i) o.dg |= 1ull << f.diag_bits[i];
      o.tile_ok = f.diag_bits.size() <= 3;  // expands to <= 8 masked-phase terms
      o.unfused_cost = 1.0 / (1 << nctrl);
      o.est_bytes = 368 * (1u << f.diag_bits.size());
      break;
    default:  // CLASS_GENERAL (CLASS_IDENTITY never reaches here)
      for (uint32_t j = 0; j < f.k; ++j) o.nd |= 1ull << f.idx_bits[j];
      o.tile_ok = false;
      break;
  }
  return o;
}

// ---- small dense linear algebra on the host ------------------------------------------
// Embed a matrix on `from` bits (ascending) into the sub-space of `to` bits (ascending, superset).
std::vector<cplx> embed(const std::vector<cplx> &m, const std::vector<uint32_t> &from,
                        const std::vector<uint32_t> &to) {
  const size_t kf = from.size(), kt = to.size();
  std::vector<int> pos(kf);
  for (size_t i = 0; i < kf; ++i) pos[i] = (int)(std::find(to.begin(), to.end(), from[i]) - to.begin());
  const size_t St = (size_t)1 << kt, Sf = (size_t)1 << kf;
  std::vector<cplx> out(St * St, cplx(0, 0));
  uint32_t from_mask = 0;
  for (size_t i = 0; i < kf; ++i) from_mask |= 1u << pos[i];
  for (size_t r = 0; r < St; ++r)
    for (size_t c = 0; c < St; ++c) {
      if ((r & ~(size_t)from_mask) != (c & ~(size_t)from_mask)) continue;  // identity on the other bits
      size_t rs = 0, cs = 0;
      for (size_t i = 0; i < kf; ++i) {
        rs |= ((r >> pos[i]) & 1) << i;
        cs |= ((c >> pos[i]) & 1) << i;
      }
      out[r * St + c] = m[rs * Sf + cs];
    }
  return out;
}

std::vector<cplx> matmul(const std::vector<cplx> &a, const std::vector<cplx> &b, size_t S) {
  std::vector<cplx> out(S * S, cplx(0, 0));
  for (size_t r = 0; r < S; ++r)
    for (size_t k = 0; k < S; ++k) {
      const cplx av = a[r * S + k];
      if (av.real() == 0.0 && av.imag() == 0.0) continue;
      for (size_t c = 0; c < S; ++c) out[r * S + c] += av * b[k * S + c];
    }
  return out;
}

// ---- host-side elementary op (tile-local bit numbers) ----------------------------------
struct HElem {
  int type = E_DENSE1;
  uint32_t lb_j = 0, lb_k = 0;   // target bit / swap pair (tile-local)
  uint32_t lctrl = 0;            // tile-local control mask
  uint32_t lmask = 0, lval = 0;  // PHASE condition (tile-local)
  uint64_t gmask = 0, gval = 0;  // CTA-uniform condition
  cplx m[4];                     // DENSE1 matrix / PHASE factor in m[0]
  struct CondPhase {
    uint64_t gmask, gval;
    cplx w;
  };
  std::vector<CondPhase> terms;   // PHASE: extra CTA-conditional factors on the same local mask (-> EC_PHASEN)
  std::vector<uint32_t> mbits;   // DENSE3: the local bits the matrix acts on (ascending, <= 3)
  std::vector<cplx> mk;          // DENSE3: 2^k x 2^k matrix on mbits
  uint32_t bits() const {
    uint32_t b = lctrl;
    switch (type) {
      case E_DENSE1:
      case E_X:
        b |= 1u << lb_j;
        break;
      case E_SWAP:
        b |= (1u << lb_j) | (1u << lb_k);
        break;
      case E_PHASE:
        b |= lmask;
        break;
      default:
        for (size_t i = 0; i < mbits.size(); ++i) b |= 1u << mbits[i];
    }
    return b;
  }
};

struct Group {
  uint32_t mask = 0;
  uint32_t pmask = 0;  // generated kernels only: bits outside `mask` that phases of this group are predicated on
  std::vector<HElem> elems;
};

// 8x8 matrix of an elementary op over the 3 bits P (ascending tile-local bits).
std::vector<cplx> elem_matrix(const HElem &e, const std::vector<uint32_t> &P) {
  auto sub_of = [&](uint32_t lb) { return (uint32_t)(std::find(P.begin(), P.end(), lb) - P.begin()); };
  uint32_t lc = 0;
  for (uint32_t b = 0; b < 32; ++b)
    if ((e.lctrl >> b) & 1) lc |= 1u << sub_of(b);
  std::vector<cplx> M(64, cplx(0, 0));
  for (uint32_t c = 0; c < 8; ++c) M[c * 8 + c] = cplx(1, 0);
  if (e.type == E_DENSE1 || e.type == E_X) {
    const uint32_t j = sub_of(e.lb_j);
    cplx mm[4] = {e.m[0], e.m[1], e.m[2], e.m[3]};
    if (e.type == E_X) {
      mm[0] = mm[3] = cplx(0, 0);
      mm[1] = mm[2] = cplx(1, 0);
    }
    for (uint32_t c = 0; c < 8; ++c) {
      if ((c >> j) & 1) continue;
      if ((c & lc) != lc) continue;
      const uint32_t i0 = c, i1 = c | (1u << j);
      M[i0 * 8 + i0] = mm[0];
      M[i0 * 8 + i1] = mm[1];
      M[i1 * 8 + i0] = mm[2];
      M[i1 * 8 + i1] = mm[3];
    }
  } else if (e.type == E_PHASE) {
    uint32_t lm = 0, lv = 0;
    for (uint32_t b = 0; b < 32; ++b)
      if ((e.lmask >> b) & 1) {
        lm |= 1u << sub_of(b);
        lv |= ((e.lval >> b) & 1u) << sub_of(b);
      }
    for (uint32_t c = 0; c < 8; ++c)
      if ((c & lm) == lv) M[c * 8 + c] = e.m[0];
  } else if (e.type == E_SWAP) {
    const uint32_t j = sub_of(e.lb_j), k = sub_of(e.lb_k);
    for (uint32_t c = 0; c < 8; ++c) {
      if ((c & lc) != lc) continue;
      const uint32_t bj = (c >> j) & 1, bk = (c >> k) & 1;
      if (bj == bk) continue;
      const uint32_t d = c ^ (1u << j) ^ (1u << k);
      M[c * 8 + c] = cplx(0, 0);
      M[c * 8 + d] = cplx(1, 0);
    }
  } else {  // DENSE3
    M = embed(e.mk, e.mbits, P);
  }
  return M;
}

template <typename R>
struct Emitter {
  HostPass *pass;
  uint32_t T;
  const PlanConfig *cfg;
  uint32_t gbits = 3;   // bits per group: 3 for the interpreter's records, cfg->jit_group_bits for the generated kernels
  bool jmode = false;   // emit JGroups (tile.cuh) instead of serialised records
  long jhad_group = -1; // jmode: where the last un-normalised Hadamard sits
  size_t jhad_elem = 0;
  bool jfail = false;   // jmode: the pass holds an op wider than a group (the interpreter's wide micro-ops serve it)
  std::vector<Group> open;
  std::vector<GlobalTerm<R>> gterms;
  // Un-normalised Hadamards: product of the scales not applied yet (a global scalar), and where the last
  // butterfly record sits so that it can be turned back into a scaled 2x2 if nothing else absorbs the product.
  double pending_scale = 1.0;
  long had_op = -1;
  size_t had_at = 0;
  uint32_t had_j = 0;

  // The same group for the generated kernels: any number of bits up to gbits, ops in sub-index coordinates.
  void emit_group_j(const Group &g) {
    std::vector<uint32_t> P;
    uint32_t mask = g.mask;
    // pad with the highest unused tile-local bits that do not take a bank-group bit's last provider away
    // (jit_codegen.cpp: bank bit k of a swizzled address needs tile bit k or k+3 outside the group)
    for (int pass_no = 0; pass_no < 2 && (uint32_t)popc(mask) < gbits; ++pass_no)
      for (int b = (int)T - 1; b >= 0 && (uint32_t)popc(mask) < gbits; --b) {
        if ((mask >> b) & 1) continue;
        if (pass_no == 0 && b < 7) {
          const int partner = b < 3 ? b + 3 : (b < 6 ? b - 3 : -1);
          if (partner < 0 || ((mask >> partner) & 1)) continue;  // would leave a bank bit without provider
        }
        mask |= 1u << b;
      }
    for (uint32_t b = 0; b < 32; ++b)
      if ((mask >> b) & 1) P.push_back(b);
    auto sub_of = [&](uint32_t lb) { return (uint32_t)(std::find(P.begin(), P.end(), lb) - P.begin()); };
    auto sub_mask = [&](uint32_t lmask) {
      uint32_t o = 0;
      for (uint32_t b = 0; b < 32; ++b)
        if ((lmask >> b) & 1) o |= 1u << sub_of(b);
      return o;
    };
    JGroup jg;
    jg.bits = P;
    for (size_t i = 0; i < g.elems.size(); ++i) {
      const HElem &e = g.elems[i];
      JElem d;
      d.gmask = e.gmask;
      d.gval = e.gval;
      const bool cond = e.gmask != 0;
      if (e.type == E_DENSE1 || e.type == E_X) {
        d.kind = e.type == E_X ? JElem::X : JElem::D1;
        d.j = sub_of(e.lb_j);
        d.lc = sub_mask(e.lctrl);
        for (int q = 0; q < 4; ++q) d.m[q] = e.m[q];
        if (e.type == E_X) {
          d.m[0] = d.m[3] = cplx(0, 0);
          d.m[1] = d.m[2] = cplx(1, 0);
        } else {
          bool real = true;
          for (int q = 0; q < 4; ++q) real &= e.m[q].imag() == 0.0;
          const bool everywhere = d.lc == 0 && !cond;
          const double hs = e.m[0].real();
          const bool is_h = real && everywhere && cfg->unnormalised_h && hs > 0.0 && e.m[1].real() == hs && e.m[2].real() == hs &&
                            e.m[3].real() == -hs;
          if (is_h) {  // s*[[1,1],[1,-1]]: butterfly now, the scale later (a global scalar commutes with everything)
            d.kind = JElem::HAD;
            pending_scale *= hs;
            jhad_group = (long)pass->jgroups.size();
            jhad_elem = jg.elems.size();
          } else if (everywhere && pending_scale != 1.0) {
            for (int q = 0; q < 4; ++q) d.m[q] *= pending_scale;
            pending_scale = 1.0;
            jhad_group = -1;
          }
        }
      } else if (e.type == E_PHASE) {
        d.kind = JElem::PH;
        d.lm = sub_mask(e.lmask & mask);
        d.lv = sub_mask(e.lval & mask);
        d.pm = e.lmask & ~mask;  // bits of the phase outside the group: a predicate on the thread's tile-local index
        d.pv = e.lval & ~mask;
        d.m[0] = e.m[0];
        for (size_t k = 0; k < e.terms.size(); ++k) {
          JCondPhase t = {e.terms[k].gmask, e.terms[k].gval, e.terms[k].w};
          d.terms.push_back(t);
        }
      } else {  // E_DENSE3: dense block on <= 3 of the group's bits
        d.kind = JElem::DK;
        for (size_t q = 0; q < e.mbits.size(); ++q) d.mb.push_back(sub_of(e.mbits[q]));
        d.mk = e.mk;
        if (!cond && pending_scale != 1.0) {
          for (size_t q = 0; q < d.mk.size(); ++q) d.mk[q] *= pending_scale;
          pending_scale = 1.0;
          jhad_group = -1;
        }
      }
      jg.elems.push_back(d);
    }
    // Runs of consecutive unconditional phases (all diagonal: any order) that act on the same amplitudes of the
    // group: one element with thread-conditional factors.
    {
      std::vector<JElem> out;
      for (size_t i = 0; i < jg.elems.size();) {
        size_t e = i;
        auto plain_phase = [](const JElem &x) { return x.kind == JElem::PH && x.gmask == 0; };
        while (e < jg.elems.size() && plain_phase(jg.elems[e])) ++e;
        if (e == i) {
          out.push_back(jg.elems[i++]);
          continue;
        }
        std::vector<char> used(e - i, 0);
        for (size_t a = i; a < e; ++a) {
          if (used[a - i]) continue;
          JElem head = jg.elems[a];
          used[a - i] = 1;
          std::vector<size_t> same;
          for (size_t b = a + 1; b < e; ++b)
            if (!used[b - i] && jg.elems[b].lm == head.lm && jg.elems[b].lv == head.lv) same.push_back(b);
          if (!same.empty() && (head.pm || !same.empty())) {
            // the unpredicated members multiply into the base factor, the predicated ones become thread terms
            cplx base(1, 0);
            std::vector<JElem::ThreadTerm> tt;
            std::vector<JCondPhase> ct;
            bool mixed = false;  // a member with CTA terms AND a thread predicate: its table factor is not unconditional
            auto take = [&](const JElem &x) {
              if (x.pm != 0 && !x.terms.empty()) mixed = true;
              if (x.pm == 0) {
                base *= x.m[0];
                ct.insert(ct.end(), x.terms.begin(), x.terms.end());
              } else {
                JElem::ThreadTerm t = {x.pm, x.pv, x.m[0]};
                tt.push_back(t);
              }
            };
            take(head);
            for (size_t q = 0; q < same.size(); ++q) {
              take(jg.elems[same[q]]);
              used[same[q] - i] = 1;
            }
            if (tt.size() <= 48 && ct.size() <= 48 && !mixed) {
              head.m[0] = base;
              head.pm = head.pv = 0;
              head.tterms = tt;
              head.terms = ct;
              out.push_back(head);
              continue;
            }
            for (size_t q = 0; q < same.size(); ++q) used[same[q] - i] = 0;  // too many: leave them as they are
          }
          out.push_back(jg.elems[a]);
        }
        i = e;
      }
      jg.elems.swap(out);
      if (jhad_group == (long)pass->jgroups.size())  // the positions moved: re-locate the group's last butterfly
        for (size_t q = 0; q < jg.elems.size(); ++q)
          if (jg.elems[q].kind == JElem::HAD) jhad_elem = q;
    }
    pass->jgroups.push_back(jg);
  }

  void emit_group(const Group &g) {
    if (jmode) {
      emit_group_j(g);
      return;
    }
    // pad the bit set to 3 with the highest unused tile-local bits (keeps the low bits for the lanes)
    std::vector<uint32_t> P;
    uint32_t mask = g.mask;
    for (int b = (int)T - 1; b >= 0 && popc(mask) < 3; --b)
      if (!((mask >> b) & 1)) mask |= 1u << b;
    for (uint32_t b = 0; b < 32; ++b)
      if ((mask >> b) & 1) P.push_back(b);
    auto sub_of = [&](uint32_t lb) { return (uint32_t)(std::find(P.begin(), P.end(), lb) - P.begin()); };

    std::vector<HElem> elems = g.elems;
    // many 2x2 gates and nothing conditional: one composed 8x8 is cheaper (32 vs 8 FMA-quads per gate)
    size_t n_dense = 0;
    bool conditional = false;
    for (size_t i = 0; i < elems.size(); ++i) {
      n_dense += elems[i].type == E_DENSE1 ? 1 : (elems[i].type == E_DENSE3 ? 4 : 0);  // host elems are never E_DENSE1R
      conditional |= elems[i].gmask != 0 || !elems[i].terms.empty();
    }
    if (!conditional && elems.size() > 1 && n_dense >= cfg->compose_threshold) {
      std::vector<cplx> acc(64, cplx(0, 0));
      for (uint32_t c = 0; c < 8; ++c) acc[c * 8 + c] = cplx(1, 0);
      for (size_t i = 0; i < elems.size(); ++i) acc = matmul(elem_matrix(elems[i], P), acc, 8);
      HElem d;
      d.type = E_DENSE3;
      d.mbits = P;
      d.mk = acc;
      elems.clear();
      elems.push_back(d);
    }

    {  // the per-CTA factor table has kMaxPhasen slots: beyond that, unfold into plain conditional phases
      std::vector<HElem> flat;
      uint32_t slots = pass->hdr.n_phasen;
      for (size_t i = 0; i < elems.size(); ++i) {
        if (elems[i].type != E_PHASE || elems[i].terms.empty() || slots < kMaxPhasen) {
          slots += (elems[i].type == E_PHASE && !elems[i].terms.empty()) ? 1u : 0u;
          flat.push_back(elems[i]);
          continue;
        }
        HElem base = elems[i];
        base.terms.clear();
        if (!is_one(base.m[0])) flat.push_back(base);
        for (size_t k = 0; k < elems[i].terms.size(); ++k) {
          HElem c = base;
          c.gmask = elems[i].terms[k].gmask;
          c.gval = elems[i].terms[k].gval;
          c.m[0] = elems[i].terms[k].w;
          flat.push_back(c);
        }
      }
      elems.swap(flat);
    }

    HostMicroOp mo;
    memset(&mo.h, 0, sizeof(mo.h));
    mo.h.kind = MK_SUPER;
    mo.h.k = 3;
    mo.h.ins_n = 3;
    for (uint32_t i = 0; i < 3; ++i) mo.h.ins_pos[i] = P[i];
    for (uint32_t u = 0; u < 8; ++u) {
      uint32_t off = 0;
      for (uint32_t i = 0; i < 3; ++i)
        if ((u >> i) & 1) off |= 1u << P[i];
      mo.h.off[u] = off;
      // swizzled byte offset (tile_kernel.cu: swz<R>): f64 t ^ ((t>>3)&7), 16 B; f32 t ^ (((t>>4)&7)<<1), 8 B
      mo.h.soff[u] = sizeof(R) == 8 ? (off ^ ((off >> 3) & 7u)) << 4 : (off ^ (((off >> 4) & 7u) << 1)) << 3;
    }
    mo.h.groups_log2 = T - 3;
    mo.h.nterms = (uint32_t)elems.size();
    for (size_t i = 0; i < elems.size(); ++i) {
      const HElem &e = elems[i];
      Elem<R> d;
      memset(&d, 0, sizeof(d));
      d.gmask = e.gmask;
      d.gval = e.gval;
      const bool cond = e.gmask != 0;
      uint32_t slot = 0;
      if (cond) {  // the CTA evaluates each distinct condition once (bit `slot` of its condition word)
        slot = kCondOverflow;
        for (size_t c = 0; c < pass->conds.size(); ++c)
          if (pass->conds[c].gmask == e.gmask && pass->conds[c].gval == e.gval) slot = (uint32_t)c;
        if (slot == kCondOverflow && pass->conds.size() < kCondOverflow) {
          CondTerm ct;
          ct.gmask = e.gmask;
          ct.gval = e.gval;
          slot = (uint32_t)pass->conds.size();
          pass->conds.push_back(ct);
        }
      }
      uint32_t lc = 0, lm = 0, lv = 0;
      for (uint32_t b = 0; b < 32; ++b) {
        if ((e.lctrl >> b) & 1) lc |= 1u << sub_of(b);
        if ((e.lmask >> b) & 1) {
          lm |= 1u << sub_of(b);
          lv |= ((e.lval >> b) & 1u) << sub_of(b);
        }
      }
      const uint32_t rec_bytes = (uint32_t)sizeof(d) + (e.type == E_DENSE3 ? (uint32_t)(128 * sizeof(R)) : 0u) +
                                 (uint32_t)(e.terms.size() * sizeof(PhaseTerm<R>));
      if (e.type == E_DENSE1 || e.type == E_X) {
        const uint32_t j = sub_of(e.lb_j);
        uint32_t pm = 0, p = 0;
        for (uint32_t c = 0; c < 8; ++c) {
          if ((c >> j) & 1) continue;
          if ((c & lc) == lc) pm |= 1u << p;
          ++p;
        }
        if (e.type == E_X) {
          d.op = elem_op(E_X, j, pm, cond, rec_bytes);
        } else {
        bool real = true;
        for (int q = 0; q < 4; ++q) real &= e.m[q].imag() == 0.0;
        d.op = elem_op(real ? E_DENSE1R : E_DENSE1, j, pm, cond, rec_bytes);
        cplx mm[4] = {e.m[0], e.m[1], e.m[2], e.m[3]};
        const bool everywhere = pm == 0xfu && !cond;  // acts on every amplitude of the state
        const double hs = mm[0].real();
        const bool is_h = real && everywhere && cfg->unnormalised_h && hs > 0.0 && mm[1].real() == hs && mm[2].real() == hs &&
                          mm[3].real() == -hs;
        if (is_h) {  // s*[[1,1],[1,-1]]: butterfly now, scale later
          d.op = (d.op & ~kElemCaseMask) | (EC_HAD + j);
          pending_scale *= hs;
          had_op = (long)pass->ops.size();
          had_at = mo.data.size();
          had_j = j;
        } else if (everywhere && pending_scale != 1.0) {
          for (int q = 0; q < 4; ++q) mm[q] *= pending_scale;
          pending_scale = 1.0;
          had_op = -1;
        }
        for (int q = 0; q < 4; ++q) {
          if (real) {
            d.m[q] = (R)mm[q].real();
          } else {
            d.m[2 * q] = (R)mm[q].real();
            d.m[2 * q + 1] = (R)mm[q].imag();
          }
        }
        }
      } else if (e.type == E_PHASE) {
        uint32_t am = 0;
        for (uint32_t c = 0; c < 8; ++c)
          if ((c & lm) == lv) am |= 1u << c;
        d.op = e.terms.empty() ? elem_op(E_PHASE, 0, am, cond, rec_bytes) : elem_op_phasen(am, rec_bytes);
        d.pad = e.terms.empty() ? 0u : pass->hdr.n_phasen++;
        d.m[0] = (R)e.m[0].real();
        d.m[1] = (R)e.m[0].imag();
      } else {  // E_DENSE3 (E_X / E_SWAP were lowered above)
        d.op = elem_op(E_DENSE3, 0, 0, cond, rec_bytes);
      }
      d.op |= slot << kElemCondShift;
      const size_t at = mo.data.size();
      mo.data.resize(at + sizeof(d));
      memcpy(mo.data.data() + at, &d, sizeof(d));
      for (size_t k = 0; k < e.terms.size(); ++k) {
        PhaseTerm<R> pt;
        memset(&pt, 0, sizeof(pt));
        pt.gmask = e.terms[k].gmask;
        pt.gval = e.terms[k].gval;
        pt.re = (R)e.terms[k].w.real();
        pt.im = (R)e.terms[k].w.imag();
        const size_t at3 = mo.data.size();
        mo.data.resize(at3 + sizeof(pt));
        memcpy(mo.data.data() + at3, &pt, sizeof(pt));
      }
      if (e.type == E_DENSE3) {
        std::vector<cplx> M = embed(e.mk, e.mbits, P);
        if (!cond && pending_scale != 1.0) {  // a dense block touches every amplitude: it takes the pending scale
          for (size_t q = 0; q < M.size(); ++q) M[q] *= pending_scale;
          pending_scale = 1.0;
          had_op = -1;
        }
        const size_t at2 = mo.data.size();
        mo.data.resize(at2 + 128 * sizeof(R));
        R *w = reinterpret_cast<R *>(mo.data.data() + at2);
        for (int q = 0; q < 64; ++q) {
          w[2 * q] = (R)M[q].real();
          w[2 * q + 1] = (R)M[q].imag();
        }
      }
    }
    {  // END sentinel: the interpreter loops until it reads case id 0
      Elem<R> endrec;
      memset(&endrec, 0, sizeof(endrec));
      const size_t at = mo.data.size();
      mo.data.resize(at + sizeof(endrec));
      memcpy(mo.data.data() + at, &endrec, sizeof(endrec));
    }
    mo.h.data_bytes = (uint32_t)mo.data.size();
    pass->ops.push_back(mo);
  }

  // End of the pass: a product of Hadamard scales nobody absorbed goes back into the last butterfly,
  // which becomes an ordinary real 2x2 again.
  void settle_scale() {
    if (pending_scale == 1.0) return;
    if (jmode) {
      JElem &d = pass->jgroups[(size_t)jhad_group].elems[jhad_elem];
      d.kind = JElem::D1;
      d.lc = 0;
      d.m[0] = d.m[1] = d.m[2] = cplx(pending_scale, 0);
      d.m[3] = cplx(-pending_scale, 0);
      pending_scale = 1.0;
      jhad_group = -1;
      return;
    }
    Elem<R> d;
    unsigned char *rec = pass->ops[(size_t)had_op].data.data() + had_at;
    memcpy(&d, rec, sizeof(d));
    d.op = (d.op & ~kElemCaseMask) | (EC_D1R_FULL + had_j);
    d.m[0] = d.m[1] = d.m[2] = (R)pending_scale;
    d.m[3] = (R)-pending_scale;
    memcpy(rec, &d, sizeof(d));
    pending_scale = 1.0;
    had_op = -1;
  }

  // Emit the open groups that touch `lmask` (or all of them).  Groups on disjoint bits commute,
  // so the ones leaving together are first packed into as few 3-bit super-ops as possible
  // (three 1-bit groups, or a 2-bit and a 1-bit group, share one shared-memory round trip).
  void flush_touching(uint32_t lmask, bool all, bool by_predicate = false) {
    std::vector<Group> out;
    for (size_t i = 0; i < open.size();) {
      if (all || ((by_predicate ? open[i].pmask : open[i].mask) & lmask)) {
        out.push_back(open[i]);
        open.erase(open.begin() + i);
      } else {
        ++i;
      }
    }
    if (cfg->fuse_blocks) {
      std::stable_sort(out.begin(), out.end(), [](const Group &a, const Group &b) { return popc(a.mask) > popc(b.mask); });
      std::vector<Group> packed;
      for (size_t i = 0; i < out.size(); ++i) {
        bool placed = false;
        for (size_t j = 0; j < packed.size() && !placed; ++j)
          if ((uint32_t)popc(packed[j].mask | out[i].mask) <= gbits) {
            packed[j].mask |= out[i].mask;
            packed[j].pmask |= out[i].pmask;
            packed[j].elems.insert(packed[j].elems.end(), out[i].elems.begin(), out[i].elems.end());
            placed = true;
          }
        if (!placed) packed.push_back(out[i]);
      }
      if (cfg->fill_on_flush && !all) {
        // A super-op that leaves with spare bits takes open groups that nothing forces out yet along for the
        // ride (disjoint bits commute; their later ops simply start a new group): their current ops cost no
        // shared-memory round trip of their own.
        for (size_t j = 0; j < packed.size(); ++j)
          for (size_t i = 0; i < open.size() && (uint32_t)popc(packed[j].mask) < gbits;) {
            if ((uint32_t)popc(packed[j].mask | open[i].mask) <= gbits) {
              packed[j].mask |= open[i].mask;
              packed[j].pmask |= open[i].pmask;
              packed[j].elems.insert(packed[j].elems.end(), open[i].elems.begin(), open[i].elems.end());
              open.erase(open.begin() + (long)i);
            } else {
              ++i;
            }
          }
      }
      out.swap(packed);
    }
    for (size_t i = 0; i < out.size(); ++i) emit_group(out[i]);
  }

  // Peephole: fold `e` into the last elementary op of a group when both act on the same
  // target bit under the same controls/condition (H.T.H -> one complex 2x2, T after a 2x2 ->
  // a scaled row, two phases on the same mask -> one phase).  Returns true when folded.
  static bool fold_into(HElem &b, const HElem &e, bool fold_cond, bool keep_real) {
    if (fold_cond && b.type == E_PHASE && e.type == E_PHASE && b.lmask == e.lmask && b.lval == e.lval &&
        (b.gmask != e.gmask || b.gval != e.gval || !b.terms.empty() || !e.terms.empty())) {
      // same amplitudes, different CTA-uniform conditions: keep one op with a list of conditional factors
      if (b.gmask) {
        HElem::CondPhase t = {b.gmask, b.gval, b.m[0]};
        b.terms.push_back(t);
        b.m[0] = cplx(1, 0);
        b.gmask = b.gval = 0;
      }
      if (e.gmask) {
        HElem::CondPhase t = {e.gmask, e.gval, e.m[0]};
        b.terms.push_back(t);
      } else {
        b.m[0] *= e.m[0];
      }
      b.terms.insert(b.terms.end(), e.terms.begin(), e.terms.end());
      return true;
    }
    if (b.gmask != e.gmask || b.gval != e.gval) return false;
    auto phase_target_ok = [](const HElem &ph, const HElem &d1) {
      // ph == diag(1, w) on d1's target bit under exactly d1's controls
      const uint32_t tb = 1u << d1.lb_j;
      return ph.lval == ph.lmask && (ph.lmask & tb) && (ph.lmask & ~tb) == d1.lctrl;
    };
    const bool b_mat = b.type == E_DENSE1 || b.type == E_X, e_mat = e.type == E_DENSE1 || e.type == E_X;
    if (b_mat && e_mat && !(b.type == E_X && e.type == E_X)) {
      if (b.lb_j != e.lb_j || b.lctrl != e.lctrl) return false;
      b.type = E_DENSE1;
      const cplx a0 = b.m[0], a1 = b.m[1], a2 = b.m[2], a3 = b.m[3];
      b.m[0] = e.m[0] * a0 + e.m[1] * a2;  // e.m * b.m
      b.m[1] = e.m[0] * a1 + e.m[1] * a3;
      b.m[2] = e.m[2] * a0 + e.m[3] * a2;
      b.m[3] = e.m[2] * a1 + e.m[3] * a3;
      return true;
    }
    // A real 2x2 costs half the FP64 work of a complex one, an (un-normalised) Hadamard a quarter, a phase on one
    // sub-bit a quarter: folding a non-real phase into a REAL matrix would make it complex and cost more than
    // the two ops apart.  (Complex matrices absorb phases for free.)
    auto is_real = [](const HElem &d1) {
      return d1.m[0].imag() == 0.0 && d1.m[1].imag() == 0.0 && d1.m[2].imag() == 0.0 && d1.m[3].imag() == 0.0;
    };
    if (b.type == E_DENSE1 && e.type == E_PHASE) {
      if (!e.terms.empty() || !phase_target_ok(e, b)) return false;
      if (keep_real && is_real(b) && e.m[0].imag() != 0.0) return false;
      b.m[2] *= e.m[0];  // diag(1,w) * M: scales the row of the |1> output
      b.m[3] *= e.m[0];
      return true;
    }
    if (b.type == E_PHASE && e.type == E_DENSE1) {
      if (!b.terms.empty() || !phase_target_ok(b, e)) return false;
      if (keep_real && is_real(e) && b.m[0].imag() != 0.0) return false;
      HElem d = e;
      d.m[1] *= b.m[0];  // M * diag(1,w): scales the column of the |1> input
      d.m[3] *= b.m[0];
      b = d;
      return true;
    }
    if (b.type == E_PHASE && e.type == E_PHASE) {
      if (b.lmask != e.lmask || b.lval != e.lval) return false;
      b.m[0] *= e.m[0];
      return true;
    }
    return false;
  }

  // Append an elementary op: merge the groups it touches when the union has <= 3 bits.
  void add(const HElem &e_in) {
    // Register-permuting ops are lowered to exact in-place arithmetic (0*x + 1*y == y for
    // finite amplitudes): X -> real 2x2 [0 1; 1 0]; SWAP(j,k) -> CX(j->k) CX(k->j) CX(j->k).
    if (e_in.type == E_SWAP) {
      for (int step = 0; step < 3; ++step) {
        HElem d = e_in;
        d.type = E_X;
        d.lb_j = (step == 1) ? e_in.lb_j : e_in.lb_k;
        d.lctrl = e_in.lctrl | (1u << ((step == 1) ? e_in.lb_k : e_in.lb_j));
        add(d);
      }
      return;
    }
    HElem e = e_in;
    if (e.type == E_X) {  // matrix kept for host-side composition / folding
      e.m[0] = e.m[3] = cplx(0, 0);
      e.m[1] = e.m[2] = cplx(1, 0);
      if (!cfg->x_as_moves) e.type = E_DENSE1;  // 0*x + 1*y == y exactly for finite amplitudes
    }
    const uint32_t bm = e.bits();
    if (!cfg->fuse_blocks) {
      Group g;
      g.mask = bm;
      g.elems.push_back(e);
      emit_group(g);
      return;
    }
    if (jmode) {
      // A group holding a phase predicated on bit b must run before anything that acts NON-diagonally on b
      // (everything diagonal on b commutes with it).
      const uint32_t ndb = nd_bits(e);
      bool any = false;
      for (size_t i = 0; i < open.size(); ++i) any |= (open[i].pmask & ndb) != 0;
      if (any) flush_touching(ndb, false, true);
    }
    uint32_t um = bm;
    std::vector<size_t> hit;
    for (size_t i = 0; i < open.size(); ++i)
      if (open[i].mask & bm) {
        hit.push_back(i);
        um |= open[i].mask;
      }
    if (jmode && e.type == E_PHASE && (uint32_t)popc(um) > gbits && !hit.empty()) {
      // A diagonal op needs none of its bits in registers: instead of closing every group it touches and
      // opening a new one, it joins the group that holds most of its bits; its other bits become per-thread
      // predicates there (JElem::pm).  The other groups on those bits leave first: they precede it in program order.
      size_t best = hit[0];
      for (size_t h = 1; h < hit.size(); ++h)
        if (popc(open[hit[h]].mask & bm) > popc(open[best].mask & bm)) best = hit[h];
      Group host = open[best];
      open.erase(open.begin() + (long)best);
      const uint32_t outside = bm & ~host.mask;
      flush_touching(outside, false);
      bool folded = false;
      if (cfg->peephole) {
        std::vector<HElem> &el = host.elems;
        for (size_t k = el.size(); k-- > 0;) {
          HElem &prev = el[k];
          const bool terms_ok = prev.type != E_PHASE || (prev.terms.size() < 48 && e.terms.size() < 48);
          if (terms_ok && fold_into(prev, e, cfg->fold_cond_phases, cfg->keep_real)) {
            folded = true;
            if (is_identity(prev)) el.erase(el.begin() + (long)k);
            break;
          }
          if (!cfg->lookback || !commute(prev, e)) break;
        }
      }
      if (!folded) host.elems.push_back(e);
      if ((uint32_t)popc(host.mask | bm) <= gbits)
        host.mask |= bm;  // the others are gone: the bits fit after all
      else
        host.pmask |= outside;
      host.pmask &= ~host.mask;
      if (!host.elems.empty()) open.push_back(host);
      return;
    }
    if ((uint32_t)popc(um) > gbits) {
      flush_touching(bm, false);
      Group g;
      g.mask = bm;
      g.elems.push_back(e);
      open.push_back(g);
      return;
    }
    Group merged;
    merged.mask = um;
    for (size_t h = 0; h < hit.size(); ++h) {  // disjoint groups commute: any order
      merged.elems.insert(merged.elems.end(), open[hit[h]].elems.begin(), open[hit[h]].elems.end());
      merged.pmask |= open[hit[h]].pmask;
    }
    merged.pmask &= ~merged.mask;
    for (size_t h = hit.size(); h-- > 0;) open.erase(open.begin() + hit[h]);
    bool folded = false;
    if (cfg->peephole) {
      // Fold `e` into an earlier op on the same target (see fold_into), looking back past the ops it
      // commutes with (disjoint bits, or diagonal on every shared bit): H(a) H(b) T(a) folds T into H(a)'s slot.
      std::vector<HElem> &el = merged.elems;
      for (size_t k = el.size(); k-- > 0;) {
        HElem &prev = el[k];
        const bool terms_ok = !(e.type == E_PHASE && prev.type == E_PHASE) || (prev.terms.size() < 48 && e.terms.size() < 48);
        if (terms_ok && fold_into(prev, e, cfg->fold_cond_phases, cfg->keep_real)) {
          folded = true;
          if (is_identity(prev)) el.erase(el.begin() + (long)k);  // H.H, X.X, T.T^-1 ...: nothing left to do
          break;
        }
        if (!cfg->lookback || !commute(prev, e)) break;
      }
    }
    if (!folded) merged.elems.push_back(e);
    if (!merged.elems.empty()) open.push_back(merged);
  }

  static uint32_t nd_bits(const HElem &h) {
    switch (h.type) {
      case E_DENSE1:
      case E_X:
        return 1u << h.lb_j;
      case E_SWAP:
        return (1u << h.lb_j) | (1u << h.lb_k);
      case E_PHASE:
        return 0;
      default:
        return h.bits();
    }
  }
  static bool commute(const HElem &a, const HElem &b) { return !(nd_bits(a) & b.bits()) && !(nd_bits(b) & a.bits()); }
  static bool is_identity(const HElem &h) {
    const double tol = 1e-15;
    if (h.type == E_PHASE) return h.terms.empty() && std::abs(h.m[0] - cplx(1, 0)) < tol;
    if (h.type != E_DENSE1) return false;
    return std::abs(h.m[0] - cplx(1, 0)) < tol && std::abs(h.m[3] - cplx(1, 0)) < tol && std::abs(h.m[1]) < tol &&
           std::abs(h.m[2]) < tol;
  }

  // ---- wide micro-ops for what does not fit 3 bits ----------------------------------
  void push_wide_dense(const FlatOp &f, const std::vector<uint32_t> &ltgt, uint32_t lctrl, uint64_t gmask) {
    HostMicroOp mo;
    memset(&mo.h, 0, sizeof(mo.h));
    std::vector<uint32_t> ins = ltgt;
    for (uint32_t b = 0; b < 32; ++b)
      if ((lctrl >> b) & 1) ins.push_back(b);
    std::sort(ins.begin(), ins.end());
    mo.h.ins_n = (uint32_t)ins.size();
    for (size_t i = 0; i < ins.size(); ++i) mo.h.ins_pos[i] = ins[i];
    mo.h.lor_mask = lctrl;
    mo.h.gmask = gmask;
    mo.h.groups_log2 = T - mo.h.ins_n;
    if (f.cls == CLASS_FLIP) {
      mo.h.kind = MK_EXCH;
      mo.h.off[0] = 0;
      mo.h.off[1] = 1u << ltgt[0];
    } else {
      mo.h.kind = MK_DENSE;
      mo.h.k = (uint32_t)ltgt.size();
      const uint32_t S = 1u << mo.h.k;
      for (uint32_t u = 0; u < S; ++u) {
        uint32_t off = 0;
        for (uint32_t i = 0; i < mo.h.k; ++i)
          if ((u >> i) & 1) off |= 1u << ltgt[i];
        mo.h.off[u] = off;
      }
      mo.data.resize((size_t)S * S * 2 * sizeof(R));
      R *d = reinterpret_cast<R *>(mo.data.data());
      for (uint32_t i = 0; i < S * S; ++i) {
        d[2 * i] = (R)f.m_sorted[i].real();
        d[2 * i + 1] = (R)f.m_sorted[i].imag();
      }
    }
    mo.h.data_bytes = (uint32_t)mo.data.size();
    pass->ops.push_back(mo);
  }

  void push_wide_exch(uint32_t a, uint32_t b, uint32_t lctrl, uint64_t gmask) {
    HostMicroOp mo;
    memset(&mo.h, 0, sizeof(mo.h));
    mo.h.kind = MK_EXCH;
    std::vector<uint32_t> ins = {a, b};
    for (uint32_t c = 0; c < 32; ++c)
      if ((lctrl >> c) & 1) ins.push_back(c);
    std::sort(ins.begin(), ins.end());
    mo.h.ins_n = (uint32_t)ins.size();
    for (size_t i = 0; i < ins.size(); ++i) mo.h.ins_pos[i] = ins[i];
    mo.h.lor_mask = lctrl;
    mo.h.gmask = gmask;
    mo.h.groups_log2 = T - mo.h.ins_n;
    mo.h.off[0] = 1u << a;
    mo.h.off[1] = 1u << b;
    pass->ops.push_back(mo);
  }

  void push_wide_diag(const std::vector<DiagTerm<R>> &terms) {
    for (size_t at = 0; at < terms.size(); at += kMaxDiagTerms) {
      const size_t n = std::min<size_t>(kMaxDiagTerms, terms.size() - at);
      HostMicroOp mo;
      memset(&mo.h, 0, sizeof(mo.h));
      mo.h.kind = MK_DIAG;
      mo.h.nterms = (uint32_t)n;
      mo.data.resize(n * sizeof(DiagTerm<R>));
      memcpy(mo.data.data(), terms.data() + at, mo.data.size());
      mo.h.data_bytes = (uint32_t)mo.data.size();
      pass->ops.push_back(mo);
    }
  }
};

// Translate the taken ops of one pass into micro-ops.
template <typename R>
void emit_pass(const std::vector<FlatOp> &ops, const std::vector<size_t> &taken, const PassHeader &hdr,
               const PlanConfig &cfg, HostPass *pass, bool jmode = false) {
  const uint32_t T = hdr.T, L = hdr.L;
  int local_of[64];  // physical bit -> tile-local bit (or -1)
  for (int b = 0; b < 64; ++b) local_of[b] = -1;
  for (uint32_t b = 0; b < L; ++b) local_of[b] = (int)b;
  for (uint32_t i = 0; i < hdr.m; ++i) local_of[hdr.hi_pos[i]] = (int)(L + i);

  Emitter<R> em;
  em.pass = pass;
  em.T = T;
  em.cfg = &cfg;
  em.jmode = jmode;
  em.gbits = jmode ? std::min<uint32_t>(cfg.jit_group_bits, T) : 3;

  for (size_t ti = 0; ti < taken.size(); ++ti) {
    const FlatOp &f = ops[taken[ti]];
    if (f.cls == CLASS_IDENTITY) continue;  // retired without emitting anything
    uint32_t lctrl = 0;
    uint64_t gmask = 0;
    for (uint32_t b = 0; b < 64; ++b)
      if ((f.ctrl_mask >> b) & 1) {
        if (local_of[b] >= 0)
          lctrl |= 1u << local_of[b];
        else
          gmask |= 1ull << b;
      }
    if (f.cls == CLASS_DIAGONAL) {
      const size_t nd = f.diag_bits.size();
      std::vector<DiagTerm<R>> wide;
      for (size_t u = 0; u < f.diag.size(); ++u) {
        if (is_one(f.diag[u])) continue;
        HElem e;
        e.type = E_PHASE;
        e.gmask = gmask;
        e.gval = gmask;
        e.lmask = lctrl;
        e.lval = lctrl;
        for (size_t i = 0; i < nd; ++i) {
          const uint32_t b = f.diag_bits[i];
          const uint64_t v = (u >> i) & 1;
          if (local_of[b] >= 0) {
            e.lmask |= 1u << local_of[b];
            e.lval |= (uint32_t)v << local_of[b];
          } else {
            e.gmask |= 1ull << b;
            e.gval |= v << b;
          }
        }
        e.m[0] = f.diag[u];
        if (e.lmask == 0 && em.gterms.size() < kMaxGlobalTerms) {
          // a scalar for this CTA: commutes with everything, applied once at store time
          GlobalTerm<R> g;
          g.gmask = e.gmask;
          g.gval = e.gval;
          g.re = (R)e.m[0].real();
          g.im = (R)e.m[0].imag();
          em.gterms.push_back(g);
        } else if ((uint32_t)popc(e.lmask) <= em.gbits) {
          em.add(e);
        } else if (jmode) {
          em.jfail = true;
        } else {
          DiagTerm<R> t;
          t.gmask = e.gmask;
          t.gval = e.gval;
          t.lmask = e.lmask;
          t.lval = e.lval;
          t.re = (R)e.m[0].real();
          t.im = (R)e.m[0].imag();
          wide.push_back(t);
        }
      }
      if (!wide.empty() && !jmode) {
        em.flush_touching(0, true);
        em.push_wide_diag(wide);
      }
      continue;
    }
    if (f.cls == CLASS_BITSWAP) {
      for (size_t i = 0; i < f.swaps.size(); ++i) {
        const uint32_t a = (uint32_t)local_of[f.swaps[i].first], b = (uint32_t)local_of[f.swaps[i].second];
        if ((uint32_t)popc(lctrl) + 2 <= em.gbits) {
          HElem e;
          e.type = E_SWAP;
          e.lb_j = a;
          e.lb_k = b;
          e.lctrl = lctrl;
          e.gmask = e.gval = gmask;
          em.add(e);
        } else if (jmode) {
          em.jfail = true;
        } else {
          em.flush_touching(0, true);
          em.push_wide_exch(std::min(a, b), std::max(a, b), lctrl, gmask);
        }
      }
      continue;
    }
    std::vector<uint32_t> ltgt;
    for (size_t i = 0; i < f.tgt_sorted.size(); ++i) ltgt.push_back((uint32_t)local_of[f.tgt_sorted[i]]);
    // local order equals physical order (low bits identity, high bits ascending), so m_sorted stays valid
    if ((size_t)popc(lctrl) + ltgt.size() > em.gbits || (ltgt.size() > 1 && (size_t)popc(lctrl) + ltgt.size() > 3)) {
      if (jmode) {
        em.jfail = true;
        continue;
      }
      em.flush_touching(0, true);
      em.push_wide_dense(f, ltgt, lctrl, gmask);
      continue;
    }
    HElem e;
    e.gmask = e.gval = gmask;
    e.lctrl = lctrl;
    if (f.cls == CLASS_FLIP) {
      e.type = E_X;
      e.lb_j = ltgt[0];
    } else if (ltgt.size() == 1) {
      e.type = E_DENSE1;
      e.lb_j = ltgt[0];
      for (int q = 0; q < 4; ++q) e.m[q] = f.m_sorted[q];
    } else {
      // dense 2- or 3-bit block: the controls (if any) are folded into the matrix
      e.type = E_DENSE3;
      e.lctrl = 0;
      std::vector<uint32_t> bits = ltgt;
      for (uint32_t b = 0; b < 32; ++b)
        if ((lctrl >> b) & 1) bits.push_back(b);
      std::sort(bits.begin(), bits.end());
      std::vector<cplx> full = embed(f.m_sorted, ltgt, bits);
      const size_t S = (size_t)1 << bits.size();
      uint32_t cm = 0;
      for (size_t i = 0; i < bits.size(); ++i)
        if ((lctrl >> bits[i]) & 1) cm |= 1u << i;
      if (cm)
        for (size_t r = 0; r < S; ++r)
          for (size_t c = 0; c < S; ++c)
            if ((r & cm) != cm || (c & cm) != cm) full[r * S + c] = (r == c) ? cplx(1, 0) : cplx(0, 0);
      e.mbits = bits;
      e.mk = full;
    }
    em.add(e);
  }
  em.flush_touching(0, true);
  em.settle_scale();
  if (jmode) {
    pass->jbits = em.jfail ? 0 : em.gbits;
    if (em.jfail) pass->jgroups.clear();
    return;  // global terms and conditions were produced by the record emission of the same pass
  }
  pass->gterms.resize(em.gterms.size() * sizeof(GlobalTerm<R>));
  if (!em.gterms.empty()) memcpy(pass->gterms.data(), em.gterms.data(), pass->gterms.size());
}

size_t pass_bytes(const HostPass &p) {
  size_t bytes = 0;
  for (size_t i = 0; i < p.ops.size(); ++i) bytes += sizeof(MicroOp) + ((p.ops[i].data.size() + 15) & ~(size_t)15);
  return bytes + ((p.gterms.size() + 15) & ~(size_t)15) + p.conds.size() * sizeof(CondTerm);
}

}  // namespace

PlanConfig default_plan_config(qip_prec prec, uint32_t n_local, bool sharded) {
  PlanConfig c;
  const char *j = getenv("QIPB200_JIT");
  const bool jit_off = j && (!strcmp(j, "off") || !strcmp(j, "0"));
  const bool generated = n_local >= 22 && !jit_off;  // passes run generated kernels (jit_runtime.cu: from 22 local qubits)
  c.T = prec == QIP_F32 ? 13 : 12;  // 64 KiB of amplitudes per tile
  c.L = prec == QIP_F32 ? 6 : 5;    // 512-byte contiguous runs in HBM
  // f64 states on generated kernels: 256-byte contiguous runs (L = 4), i.e. 8 instead of 7 freely chosen tile bits.  On one
  // H100 SXM (400 W power limit), N=30 f64 headline circuit, alternating runs: 21 passes, 285.9-287.2 ms against 25 passes,
  // 329.5-332.2 ms with L = 5 (pass 13.2 vs 12.9 ms).  Passes whose generated kernel is not ready (or every pass, when NVRTC
  // or the driver API is missing) run the interpreter kernel on the same L = 4 plan; its speed there is not measured.
  // Sharded states keep L = 5: the migration protocols have not been run at L = 4.
  if (prec == QIP_F64 && generated && !sharded) c.L = 4;
  // test / tuning knobs (tile geometry and grouping only; results are unaffected)
  if (const char *e = getenv("QIPB200_TILE_T")) c.T = std::min<uint32_t>((uint32_t)atoi(e), c.T);
  if (const char *e = getenv("QIPB200_TILE_L")) c.L = (uint32_t)atoi(e);
  if (const char *e = getenv("QIPB200_COMPOSE")) c.compose_threshold = (uint32_t)std::max(1, atoi(e));
  if (const char *e = getenv("QIPB200_TILE_G")) c.groups_per_thread = atoi(e) == 2 ? 2 : 1;
  // generated kernels: 2^4 (f64) / 2^5 (f32) amplitudes of a group in registers = 64 data registers per thread
  c.jit_group_bits = prec == QIP_F32 ? 5 : 4;
  if (const char *e = getenv("QIPB200_JIT_GROUP_BITS")) c.jit_group_bits = (uint32_t)std::min(6, std::max(3, atoi(e)));
  if (const char *e = getenv("QIPB200_NO_BLOCK_FUSION")) c.fuse_blocks = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_NO_PEEPHOLE")) c.peephole = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_SEED_SEARCH")) c.seed_search = atoi(e) != 0;
  if (const char *e = getenv("QIPB200_PLAN_LOOKAHEAD")) c.lookahead = (uint32_t)std::max(0, atoi(e));
  if (const char *e = getenv("QIPB200_NO_HAD")) c.unnormalised_h = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_KEEP_REAL")) c.keep_real = atoi(e) != 0;
  if (const char *e = getenv("QIPB200_NO_LOOKBACK")) c.lookback = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_NO_FILL")) c.fill_on_flush = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_X_MOVES")) c.x_as_moves = atoi(e) != 0;
  if (const char *e = getenv("QIPB200_NO_PHASEN")) c.fold_cond_phases = atoi(e) == 0;
  if (const char *e = getenv("QIPB200_NO_TMA")) c.use_tma = atoi(e) == 0;
  // States big enough for the generated kernels (jit_runtime.cu: from 22 local qubits): a pass costs one HBM sweep
  // almost regardless of what it folds in, so fewer passes win (tile-bit seed search: 25 instead of 29 for the N=30
  // circuit) and FP64 work is worth saving (phases kept out of real 2x2 gates).  On one H100 SXM (700 W), N=30 f64:
  // 25 passes, 300-304 ms with both options vs 29 passes, 347 ms without.  (The interpreter kernel is bound by its own
  // instruction stream and does not gain from either.)
  if (generated) {
    if (!getenv("QIPB200_SEED_SEARCH")) c.seed_search = true;
    if (!getenv("QIPB200_KEEP_REAL")) c.keep_real = true;
  }
  if (n_local < c.T) c.T = n_local;
  if (c.L > c.T) c.L = c.T;
  if (c.T - c.L > kTileMaxHigh) c.L = c.T - kTileMaxHigh;
  if (prec == QIP_F32 && c.L == 0 && c.T >= 1) c.L = 1;  // a 16-byte unit holds two f32 amplitudes
  return c;
}

// ---- tile-bit selection -----------------------------------------------------------------
// One greedy selection in program order, the tile's high bits pre-seeded with `seed`.
struct Pick {
  uint64_t S_high = 0;
  std::vector<size_t> taken, left;
  double unfused = 0.0;
  long single = -1;  // first op that may run alone right now: not blocked, commutes past EVERY earlier op
  size_t n_nd = 0;   // non-diagonal gates absorbed (diagonal ones ride along in any pass)
};

struct Selector {
  const std::vector<OpInfo> &info;
  const std::vector<char> *blocked;
  bool can_tile;
  uint64_t low_mask;
  uint32_t m;
  uint64_t budget;

  Pick select(const std::vector<size_t> &remaining, uint64_t seed) const {
    Pick pk;
    pk.S_high = seed;
    uint64_t pend_d = 0, pend_nd = 0, bytes = 0, seen_d = 0, seen_nd = 0;
    for (size_t r = 0; r < remaining.size(); ++r) {
      const size_t idx = remaining[r];
      const OpInfo &o = info[idx];
      const bool is_blocked = blocked && (*blocked)[idx];
      const bool conflict = (o.nd & (pend_d | pend_nd)) || (o.dg & pend_nd);
      if (pk.single < 0 && !is_blocked && !((o.nd & (seen_d | seen_nd)) || (o.dg & seen_nd))) pk.single = (long)r;
      seen_d |= o.dg;
      seen_nd |= o.nd;
      if (can_tile && !conflict && o.tile_ok && bytes + o.est_bytes <= budget) {
        const uint64_t need = o.need_tile & ~low_mask & ~pk.S_high;
        if ((uint32_t)popc(pk.S_high | need) <= m) {
          pk.S_high |= need;
          pk.taken.push_back(idx);
          pk.unfused += o.unfused_cost;
          pk.n_nd += o.nd ? 1 : 0;
          bytes += o.est_bytes;
          continue;
        }
      }
      pend_d |= o.dg;
      pend_nd |= o.nd;
      pk.left.push_back(idx);
    }
    return pk;
  }

  uint64_t candidate_bits(const Pick &pk) const {
    uint64_t cand = 0;
    for (size_t r = 0; r < pk.left.size() && r < 64; ++r) cand |= info[pk.left[r]].need_tile & ~low_mask;
    return cand & ~pk.S_high;
  }

  // The plain greedy fills the tile with the bits of the first gates it meets.  Try reserving slots for bits that
  // gates left behind need (forward selection, one bit at a time): keep whichever selection absorbs the most
  // non-diagonal gates.
  Pick seed_search(const std::vector<size_t> &remaining, Pick best, std::vector<Pick> *chain = nullptr) const {
    uint64_t seeds = 0;
    for (uint32_t round = 0; round < m && !best.left.empty(); ++round) {
      const uint64_t cand = candidate_bits(best);
      uint64_t best_bit = 0;
      for (uint32_t bit = 0; bit < 64; ++bit) {
        if (!((cand >> bit) & 1)) continue;
        Pick alt = select(remaining, seeds | (1ull << bit));
        if (alt.n_nd > best.n_nd) {
          if (chain) chain->push_back(best);
          best = std::move(alt);
          best_bit = 1ull << bit;
        }
      }
      if (!best_bit) break;
      seeds |= best_bit;
    }
    return best;
  }

  // Sweeps the plain greedy needs for `remaining`; what is left when it gets stuck behind blocked ops is charged at
  // the average rate of a pass.  (Rollouts cut off after a few passes or a window of ops were tried: the estimate of
  // the cut-off tail misleads the search -- 29..48 sweeps instead of 25 on the N=30 circuit.)
  double rollout(std::vector<size_t> remaining) const {
    double cost = 0.0;
    while (!remaining.empty()) {
      Pick pk = select(remaining, 0);
      if (pk.taken.empty() || pk.unfused <= 1.05) {
        if (pk.single < 0) {
          size_t nd = 0;
          for (size_t r = 0; r < remaining.size(); ++r) nd += info[remaining[r]].nd ? 1 : 0;
          return cost + nd / 24.0;
        }
        cost += std::min(1.0, info[remaining[(size_t)pk.single]].unfused_cost);
        remaining.erase(remaining.begin() + pk.single);
        continue;
      }
      cost += 1.0;
      remaining.swap(pk.left);
    }
    return cost;
  }

  // Look-ahead: a pass that absorbs the most gates NOW is not always the one that leaves the cheapest rest.  Score
  // candidate tile-bit sets by 1 + the sweeps a plain greedy needs for what they leave behind.
  Pick lookahead(const std::vector<size_t> &remaining, Pick incumbent, uint32_t width) const {
    std::vector<Pick> cands;
    cands.push_back(select(remaining, 0));
    (void)seed_search(remaining, cands[0], &cands);
    double best_cost = rollout(incumbent.left);
    std::vector<uint64_t> tried;
    tried.push_back(incumbent.S_high);
    // beam over seed sets: each round extends the best `width` seed sets by one more reserved bit
    struct Node {
      uint64_t seeds;
      double cost;
      size_t n_nd;
    };
    std::vector<Node> frontier(1, Node{0, 0.0, 0});
    Pick best = std::move(incumbent);
    for (size_t c = 0; c < cands.size(); ++c) {
      const double cost = rollout(cands[c].left);
      if (cost < best_cost - 1e-9 || (cost < best_cost + 1e-9 && cands[c].n_nd > best.n_nd)) {
        best_cost = cost;
        best = cands[c];
      }
    }
    for (uint32_t round = 0; round < m; ++round) {
      std::vector<Node> next;
      for (size_t f = 0; f < frontier.size(); ++f) {
        const Pick base = select(remaining, frontier[f].seeds);
        const uint64_t cand = candidate_bits(base);
        for (uint32_t bit = 0; bit < 64; ++bit) {
          if (!((cand >> bit) & 1)) continue;
          const uint64_t seeds = frontier[f].seeds | (1ull << bit);
          if ((uint32_t)popc(seeds) > m) continue;
          bool dup = false;
          for (size_t t = 0; t < next.size(); ++t) dup = dup || next[t].seeds == seeds;
          if (dup) continue;
          Pick alt = select(remaining, seeds);
          if (alt.taken.empty()) continue;
          const double cost = rollout(alt.left);
          next.push_back(Node{seeds, cost, alt.n_nd});
          if (cost < best_cost - 1e-9 || (cost < best_cost + 1e-9 && alt.n_nd > best.n_nd)) {
            best_cost = cost;
            best = std::move(alt);
          }
        }
      }
      if (next.empty()) break;
      std::sort(next.begin(), next.end(), [](const Node &a, const Node &b) { return a.cost != b.cost ? a.cost < b.cost : a.n_nd > b.n_nd; });
      if (next.size() > width) next.resize(width);
      frontier.swap(next);
    }
    return best;
  }
};

void op_dependency_masks(const FlatOp &f, DepMasks *out) {
  const OpInfo o = analyse(f);
  out->nd = o.nd;
  out->dg = o.dg;
}

void op_uniform_info(const FlatOp &f, DepMasks *out) {
  out->has_uniform = true;
  if (f.cls == CLASS_IDENTITY) {  // nothing to do on the virtual rank: rides along in any pass
    out->u_tile_ok = true;
    out->u_need_tile = 0;
    out->u_unfused_cost = 0.0;
    out->u_est_bytes = 0;
    return;
  }
  const OpInfo o = analyse(f);
  out->u_tile_ok = o.tile_ok;
  out->u_need_tile = o.need_tile;
  out->u_unfused_cost = o.unfused_cost;
  out->u_est_bytes = o.est_bytes;
}

void plan_passes(const std::vector<FlatOp> &ops, uint32_t n_local, qip_prec prec, const PlanConfig &cfg_in,
                 std::vector<PlanStep> *steps, const std::vector<char> *blocked, std::vector<size_t> *leftover,
                 const std::vector<DepMasks> *dep) {
  PlanConfig cfg = cfg_in;
  if (cfg.T > n_local) cfg.T = n_local;
  if (cfg.L > cfg.T) cfg.L = cfg.T;
  const uint32_t m = cfg.T - cfg.L;
  const uint64_t low_mask = (1ull << cfg.L) - 1ull;
  const bool can_tile = cfg.T >= 3;
  std::vector<OpInfo> info(ops.size());
  std::vector<size_t> remaining;
  const bool uniform = dep && !dep->empty() && (*dep)[0].has_uniform;
  for (size_t i = 0; i < ops.size(); ++i) {
    const bool is_blocked = blocked && (*blocked)[i];
    if (uniform) {  // nothing rank-specific may steer the selection
      const DepMasks &d = (*dep)[i];
      info[i] = OpInfo();
      info[i].nd = d.nd;
      info[i].dg = d.dg;
      info[i].need_tile = d.u_need_tile;
      info[i].tile_ok = d.u_tile_ok && !is_blocked;
      info[i].unfused_cost = d.u_unfused_cost;
      info[i].est_bytes = d.u_est_bytes;
      remaining.push_back(i);
      continue;
    }
    if (ops[i].cls == CLASS_IDENTITY && !is_blocked) {
      if (!dep) continue;  // a plain identity gate: nothing to do, nothing to order
      // identity ON THIS RANK under the current layout (e.g. a rank-held control is 0): it emits
      // nothing, but it may only be retired once everything it depends on has run -- if it stays
      // behind a blocked op it must be re-examined under the next layout.
      info[i] = OpInfo();
      info[i].nd = (*dep)[i].nd;
      info[i].dg = (*dep)[i].dg;
      info[i].tile_ok = true;
      info[i].unfused_cost = 0.0;
      remaining.push_back(i);
      continue;
    }
    info[i] = analyse(ops[i]);
    if (dep) {
      info[i].nd = (*dep)[i].nd;
      info[i].dg = (*dep)[i].dg;
    }
    if (is_blocked) info[i].tile_ok = false;
    remaining.push_back(i);
  }
  // est_bytes are upper bounds (every op opening its own super-op); real passes are several times
  // smaller after grouping and folding.  Try optimistic budgets first and fall back towards the
  // guaranteed one when the emitted pass does not fit the parameter space.
  const uint32_t byte_budget = kMaxPassBytes - 2048;
  static const uint32_t kBudgetScale[3] = {4, 2, 1};
  while (!remaining.empty()) {
    bool done = false, stuck = false;
    for (int attempt = uniform ? 2 : 0; attempt < 3 && !done; ++attempt) {  // uniform: the guaranteed budget only
      const uint64_t budget = (uint64_t)byte_budget * kBudgetScale[attempt];
      Selector sel{info, blocked, can_tile, low_mask, m, budget};
      Pick best = sel.select(remaining, 0);
      if (cfg.seed_search && can_tile) best = sel.seed_search(remaining, std::move(best));
      if (cfg.lookahead && can_tile && !best.left.empty()) best = sel.lookahead(remaining, std::move(best), cfg.lookahead);
      uint64_t S_high = best.S_high;
      std::vector<size_t> &taken = best.taken, &left = best.left;
      const double unfused = best.unfused;
      const long single = best.single;
      if (taken.empty() || unfused <= 1.05) {
        if (single < 0) {  // everything left is blocked or stuck behind a blocked op
          stuck = true;
          break;
        }
        // not worth a full sweep: run one op with its per-gate kernel
        PlanStep st;
        st.is_pass = false;
        st.op_index = remaining[(size_t)single];
        steps->push_back(st);
        remaining.erase(remaining.begin() + single);
        done = true;
        break;
      }
      PlanStep st;
      st.is_pass = true;
      PassHeader &h = st.pass.hdr;
      memset(&h, 0, sizeof(h));
      h.T = cfg.T;
      h.L = cfg.L;
      h.m = m;
      // pad the tile-bit set to exactly m bits with the highest unused bits
      for (int b = (int)n_local - 1; b >= (int)cfg.L && (uint32_t)popc(S_high) < m; --b)
        if (!((S_high >> b) & 1)) S_high |= 1ull << b;
      uint32_t c = 0;
      for (uint32_t b = 0; b < 64; ++b)
        if ((S_high >> b) & 1) h.hi_pos[c++] = b;
      for (uint32_t ch = 0; ch < (1u << m); ++ch) {
        uint64_t off = 0;
        for (uint32_t i = 0; i < m; ++i)
          if ((ch >> i) & 1) off |= 1ull << h.hi_pos[i];
        h.chunk_off[ch] = off;
      }
      if (prec == QIP_F32)
        emit_pass<float>(ops, taken, h, cfg, &st.pass);
      else
        emit_pass<double>(ops, taken, h, cfg, &st.pass);
      if (cfg.jit_group_bits >= 3) {  // the same gates once more, grouped for the generated kernels
        if (prec == QIP_F32)
          emit_pass<float>(ops, taken, h, cfg, &st.pass, true);
        else
          emit_pass<double>(ops, taken, h, cfg, &st.pass, true);
      }
      if (pass_bytes(st.pass) > kMaxPassBytes && attempt < 2) continue;  // too optimistic: retry with a smaller budget
      h.n_ops = (uint32_t)st.pass.ops.size();
      h.n_gterms = (uint32_t)(st.pass.gterms.size() / (prec == QIP_F32 ? sizeof(GlobalTerm<float>) : sizeof(GlobalTerm<double>)));
      st.pass.n_gates = (uint32_t)taken.size();
      steps->push_back(st);
      remaining.swap(left);
      done = true;
    }
    if (stuck) break;
  }
  if (leftover) *leftover = remaining;
}

// ---- planning with qubit rotation (tile.cuh: RotatePlan) -------------------------------------------------------
namespace {

// Greedy selection over LOGICAL qubits: a tile is any set S of <= T qubits with at most m of them from outside `prev`
// (the previous tile): the L low positions are filled from the previous tile by the swaps that end the previous pass.
struct RotSelector {
  const std::vector<OpInfo> &info;
  uint32_t T, m;
  uint64_t prev, budget;

  bool fits(uint64_t S) const { return (uint32_t)popc(S) <= T && (uint32_t)popc(S & ~prev) <= m; }

  Pick select(const std::vector<size_t> &remaining, uint64_t seed) const {
    Pick pk;
    pk.S_high = seed;  // here: the whole tile set
    uint64_t pend_d = 0, pend_nd = 0, bytes = 0, seen_d = 0, seen_nd = 0;
    for (size_t r = 0; r < remaining.size(); ++r) {
      const size_t idx = remaining[r];
      const OpInfo &o = info[idx];
      const bool conflict = (o.nd & (pend_d | pend_nd)) || (o.dg & pend_nd);
      if (pk.single < 0 && !((o.nd & (seen_d | seen_nd)) || (o.dg & seen_nd))) pk.single = (long)r;
      seen_d |= o.dg;
      seen_nd |= o.nd;
      if (!conflict && o.tile_ok && bytes + o.est_bytes <= budget && fits(pk.S_high | o.need_tile)) {
        pk.S_high |= o.need_tile;
        pk.taken.push_back(idx);
        pk.unfused += o.unfused_cost;
        pk.n_nd += o.nd ? 1 : 0;
        bytes += o.est_bytes;
        continue;
      }
      pend_d |= o.dg;
      pend_nd |= o.nd;
      pk.left.push_back(idx);
    }
    return pk;
  }

  Pick seed_search(const std::vector<size_t> &remaining, Pick best) const {
    uint64_t seeds = 0;
    for (uint32_t round = 0; round < T && !best.left.empty(); ++round) {
      uint64_t cand = 0;
      for (size_t r = 0; r < best.left.size() && r < 64; ++r) cand |= info[best.left[r]].need_tile;
      cand &= ~best.S_high;
      uint64_t best_bit = 0;
      for (uint32_t bit = 0; bit < 64; ++bit) {
        if (!((cand >> bit) & 1) || !fits(seeds | (1ull << bit))) continue;
        Pick alt = select(remaining, seeds | (1ull << bit));
        if (alt.n_nd > best.n_nd) {
          best = std::move(alt);
          best_bit = 1ull << bit;
        }
      }
      if (!best_bit) break;
      seeds |= best_bit;
    }
    return best;
  }
};

FlatOp make_bitswap(uint32_t p, uint32_t q, uint32_t n) {
  FlatOp f;
  f.base_kind = QIP_OP_SWAP;
  f.n = n;
  f.k = 2;
  f.kop = 2;
  f.nc = 0;
  f.idx_bits.push_back(p);
  f.idx_bits.push_back(q);
  f.cls = CLASS_BITSWAP;
  f.ctrl_mask = 0;
  f.swaps.push_back(std::make_pair(std::min(p, q), std::max(p, q)));
  return f;
}

// One pass over the physical tile bits low L + `S_high`, holding exactly `pops` (compiled under the current layout).
void build_forced_pass(const std::vector<FlatOp> &pops, uint64_t S_high, const PlanConfig &cfg, qip_prec prec, uint32_t n_gates,
                       PlanStep *st) {
  const uint32_t m = cfg.T - cfg.L;
  st->is_pass = true;
  PassHeader &h = st->pass.hdr;
  memset(&h, 0, sizeof(h));
  h.T = cfg.T;
  h.L = cfg.L;
  h.m = m;
  uint32_t c = 0;
  for (uint32_t b = 0; b < 64; ++b)
    if ((S_high >> b) & 1) h.hi_pos[c++] = b;
  for (uint32_t ch = 0; ch < (1u << m); ++ch) {
    uint64_t off = 0;
    for (uint32_t i = 0; i < m; ++i)
      if ((ch >> i) & 1) off |= 1ull << h.hi_pos[i];
    h.chunk_off[ch] = off;
  }
  std::vector<size_t> all(pops.size());
  for (size_t i = 0; i < pops.size(); ++i) all[i] = i;
  for (int jm = 0; jm < (cfg.jit_group_bits >= 3 ? 2 : 1); ++jm) {
    if (prec == QIP_F32)
      emit_pass<float>(pops, all, h, cfg, &st->pass, jm == 1);
    else
      emit_pass<double>(pops, all, h, cfg, &st->pass, jm == 1);
  }
  h.n_ops = (uint32_t)st->pass.ops.size();
  h.n_gterms = (uint32_t)(st->pass.gterms.size() / (prec == QIP_F32 ? sizeof(GlobalTerm<float>) : sizeof(GlobalTerm<double>)));
  st->pass.n_gates = n_gates;
}

}  // namespace

static int plan_rotating_scaled(const qip_op *ops, size_t n_ops, qip_prec prec, uint32_t n, const PlanConfig &cfg_in,
                                uint32_t budget_scale, RotatePlan *out, std::string *err, std::vector<uint32_t> *layout, bool restore);

// transpositions that bring `phys` home, packed into swap-only steps by the fixed-layout planner
static int append_restore(qip_prec prec, uint32_t n, const PlanConfig &cfg, std::vector<uint32_t> &phys, RotatePlan *out,
                          std::string *err) {
  std::vector<FlatOp> back;
  for (int b = (int)n - 1; b >= 0; --b) {
    if (phys[(size_t)b] == (uint32_t)b) continue;
    const uint32_t where = phys[(size_t)b];
    back.push_back(make_bitswap((uint32_t)b, where, n));
    for (uint32_t c = 0; c < n; ++c) {
      if (phys[c] == (uint32_t)b)
        phys[c] = where;
      else if (phys[c] == where)
        phys[c] = (uint32_t)b;
    }
  }
  if (back.empty()) return QIPB200_OK;
  std::vector<PlanStep> steps;
  std::vector<size_t> left;
  plan_passes(back, n, prec, cfg, &steps, nullptr, &left);
  if (!left.empty()) {
    if (err) *err = "internal: layout restore left ops behind";
    return QIPB200_ERR_UNSUPPORTED;
  }
  for (size_t i = 0; i < steps.size(); ++i) {
    if (!steps[i].is_pass) {
      out->singles.push_back(back[steps[i].op_index]);
      steps[i].op_index = out->singles.size() - 1;
    }
    out->steps.push_back(steps[i]);
    ++out->n_restore_steps;
  }
  return QIPB200_OK;
}

int plan_layout_restore(qip_prec prec, uint32_t n, const PlanConfig &cfg, uint32_t *layout, RotatePlan *out, std::string *err) {
  out->steps.clear();
  out->singles.clear();
  out->n_swaps = out->n_restore_steps = 0;
  std::vector<uint32_t> phys(layout, layout + n);
  int st = append_restore(prec, n, cfg, phys, out, err);
  if (st == QIPB200_OK)
    for (uint32_t b = 0; b < n; ++b) layout[b] = phys[b];
  return st;
}

int plan_rotating(const qip_op *ops, size_t n_ops, qip_prec prec, uint32_t n, const PlanConfig &cfg, RotatePlan *out,
                  std::string *err, uint32_t *layout, bool restore) {
  std::vector<uint32_t> start(n);
  for (uint32_t b = 0; b < n; ++b) start[b] = layout ? layout[b] : b;
  // the per-op byte estimates are upper bounds: optimistic budgets first, as plan_passes does
  static const uint32_t kScale[3] = {4, 2, 1};
  for (int attempt = 0; attempt < 3; ++attempt) {
    std::vector<uint32_t> phys = start;
    int st = plan_rotating_scaled(ops, n_ops, prec, n, cfg, kScale[attempt], out, err, &phys, restore);
    if (st != QIPB200_OK) return st;
    bool fits = true;
    for (size_t i = 0; i < out->steps.size(); ++i)
      if (out->steps[i].is_pass && pass_bytes(out->steps[i].pass) > kMaxPassBytes) fits = false;
    if (fits || attempt == 2) {
      if (layout)
        for (uint32_t b = 0; b < n; ++b) layout[b] = phys[b];
      return QIPB200_OK;
    }
  }
  return QIPB200_OK;
}

static int plan_rotating_scaled(const qip_op *ops, size_t n_ops, qip_prec prec, uint32_t n, const PlanConfig &cfg_in,
                                uint32_t budget_scale, RotatePlan *out, std::string *err, std::vector<uint32_t> *layout, bool restore) {
  out->steps.clear();
  out->singles.clear();
  out->n_swaps = out->n_restore_steps = 0;
  PlanConfig cfg = cfg_in;
  if (cfg.T > n) cfg.T = n;
  if (cfg.L > cfg.T) cfg.L = cfg.T;
  const uint32_t T = cfg.T, L = cfg.L, m = T - L;
  if (T < 3 || n > 62) {
    if (err) *err = "rotating plan: state too small / too large";
    return QIPB200_ERR_UNSUPPORTED;
  }
  // logical view: every op compiled under the identity layout
  std::vector<OpInfo> info(n_ops);
  std::vector<size_t> remaining;
  for (size_t i = 0; i < n_ops; ++i) {
    FlatOp f;
    int st = compile_op(&ops[i], prec, n, &f, err);
    if (st != QIPB200_OK) return st;
    if (f.cls == CLASS_IDENTITY) continue;
    info[i] = analyse(f);
    remaining.push_back(i);
  }
  std::vector<uint32_t> &phys = *layout;  // logical bit -> physical bit
  auto logical_at = [&](uint32_t p) {
    for (uint32_t b = 0; b < n; ++b)
      if (phys[b] == p) return b;
    return 0u;
  };
  auto compile_now = [&](size_t i, FlatOp *f) { return compile_op(&ops[i], prec, n, f, err, phys.data()); };
  const uint64_t byte_budget = (uint64_t)(kMaxPassBytes - 2048) * budget_scale;

  // the pass that is selected but not emitted yet (its end swaps depend on the NEXT selection)
  bool have_pending = false;
  uint64_t pend_tile = 0;           // logical qubits of the pending pass (exactly T)
  std::vector<size_t> pend_taken;
  uint64_t prev = 0;                // logical qubits the next tile may take its low positions from
  for (uint32_t p = 0; p < L; ++p) prev |= 1ull << logical_at(p);

  // emit the pending pass; `want_low` (logical, exactly L qubits of pend_tile) must sit in the low positions afterwards
  auto flush_pending = [&](uint64_t want_low, const std::vector<std::pair<uint32_t, uint32_t>> &extra_swaps) -> int {
    std::vector<FlatOp> pops(pend_taken.size());
    for (size_t i = 0; i < pend_taken.size(); ++i) {
      int st = compile_now(pend_taken[i], &pops[i]);
      if (st != QIPB200_OK) return st;
    }
    uint64_t S_high = 0;
    for (uint32_t b = 0; b < n; ++b)
      if (((pend_tile >> b) & 1) && phys[b] >= L) S_high |= 1ull << phys[b];
    if ((uint32_t)popc(S_high) != m) {
      if (err) *err = "internal: rotating plan lost track of the tile";
      return QIPB200_ERR_UNSUPPORTED;
    }
    // The pass may end with ANY permutation of its tile positions.  Target: the wanted qubits in the low positions (at
    // their own low position when they have one), every other tile qubit at its own position when that one is a high
    // position of this tile, the rest wherever is left (staying put when possible) -- the layout never drifts far from the
    // canonical one, which keeps the final restore short.
    auto do_swap = [&](uint32_t p, uint32_t q) {
      pops.push_back(make_bitswap(p, q, n));
      const uint32_t a = logical_at(p), b = logical_at(q);
      phys[a] = q;
      phys[b] = p;
      ++out->n_swaps;
    };
    {
      static const bool homing = !getenv("QIPB200_ROTATE_NO_HOMING");
      std::vector<uint32_t> pos;  // the tile's positions
      for (uint32_t p = 0; p < L; ++p) pos.push_back(p);
      for (uint32_t p = L; p < n; ++p)
        if ((S_high >> p) & 1) pos.push_back(p);
      std::vector<int> target(n, -1);       // target[position] = logical qubit
      std::vector<char> placed(n, 0);       // by logical qubit
      auto in_tile_pos = [&](uint32_t p) { return p < L || ((S_high >> p) & 1); };
      // 1. wanted-low qubits whose own position is low
      for (uint32_t b = 0; b < L; ++b)
        if ((want_low >> b) & 1) {
          target[b] = (int)b;
          placed[b] = 1;
        }
      // 2. the other wanted-low qubits: stay where they are if that is a free low position, else any free low position
      for (int round = 0; round < 2; ++round)
        for (uint32_t b = 0; b < n; ++b) {
          if (!((want_low >> b) & 1) || placed[b]) continue;
          if (round == 0) {
            if (phys[b] < L && target[phys[b]] < 0) {
              target[phys[b]] = (int)b;
              placed[b] = 1;
            }
            continue;
          }
          for (uint32_t p = 0; p < L; ++p)
            if (target[p] < 0) {
              target[p] = (int)b;
              placed[b] = 1;
              break;
            }
        }
      // 3. the remaining tile qubits: home if home is a high tile position, else stay put if still free, else anything
      std::vector<uint32_t> rest;
      for (size_t i = 0; i < pos.size(); ++i) {
        const uint32_t b = logical_at(pos[i]);
        if (!placed[b]) rest.push_back(b);
      }
      for (int round = 0; round < 3; ++round)
        for (size_t i = 0; i < rest.size(); ++i) {
          const uint32_t b = rest[i];
          if (placed[b]) continue;
          if (round == 0) {
            if (homing && b >= L && in_tile_pos(b) && target[b] < 0) {
              target[b] = (int)b;
              placed[b] = 1;
            }
          } else if (round == 1) {
            if (phys[b] >= L && target[phys[b]] < 0) {
              target[phys[b]] = (int)b;
              placed[b] = 1;
            }
          } else {
            for (size_t k = 0; k < pos.size(); ++k)
              if (pos[k] >= L && target[pos[k]] < 0) {
                target[pos[k]] = (int)b;
                placed[b] = 1;
                break;
              }
          }
        }
      // realise it: put the right qubit into every position in turn (a transposition each)
      for (size_t i = 0; i < pos.size(); ++i) {
        const uint32_t p = pos[i];
        if (target[p] < 0) {
          if (err) *err = "internal: rotating plan: tile position without a qubit";
          return QIPB200_ERR_UNSUPPORTED;
        }
        const uint32_t want = (uint32_t)target[p];
        if (logical_at(p) != want) do_swap(p, phys[want]);
      }
    }
    for (size_t i = 0; i < extra_swaps.size(); ++i) do_swap(extra_swaps[i].first, extra_swaps[i].second);
    PlanStep st;
    build_forced_pass(pops, S_high, cfg, prec, (uint32_t)pend_taken.size(), &st);
    out->steps.push_back(st);
    have_pending = false;
    return QIPB200_OK;
  };

  while (!remaining.empty()) {
    RotSelector sel{info, T, m, prev, byte_budget};
    Pick best = sel.select(remaining, 0);
    if (cfg.seed_search) best = sel.seed_search(remaining, std::move(best));
    if (best.taken.empty() || best.unfused <= 1.05) {
      // not worth a sweep: one op with its per-gate kernel, under the layout left by the pending pass
      if (best.single < 0) {
        if (err) *err = "internal: rotating plan made no progress";
        return QIPB200_ERR_UNSUPPORTED;
      }
      if (have_pending) {
        uint64_t keep = 0;  // nothing to prepare: the low positions stay as they are
        for (uint32_t p = 0; p < L; ++p) keep |= 1ull << logical_at(p);
        int st = flush_pending(keep, {});
        if (st != QIPB200_OK) return st;
      }
      FlatOp f;
      int st = compile_now(remaining[(size_t)best.single], &f);
      if (st != QIPB200_OK) return st;
      out->singles.push_back(f);
      PlanStep ps;
      ps.is_pass = false;
      ps.op_index = out->singles.size() - 1;
      out->steps.push_back(ps);
      remaining.erase(remaining.begin() + best.single);
      // no pass is pending any more: the next tile carries over only the qubits that now sit in the low positions
      // (not the whole tile of the flushed pass, whose high qubits no later swap brings down)
      prev = 0;
      for (uint32_t p = 0; p < L; ++p) prev |= 1ull << logical_at(p);
      continue;
    }
    // the tile of this pass: the selected qubits, padded to T (first from the previous tile: they cost nothing)
    uint64_t tile = best.S_high;
    for (int round = 0; round < 2 && (uint32_t)popc(tile) < T; ++round)
      for (int b = (int)n - 1; b >= 0 && (uint32_t)popc(tile) < T; --b) {
        const uint64_t bit = 1ull << b;
        if (tile & bit) continue;
        if (round == 0 ? ((prev & bit) != 0) : ((uint32_t)popc((tile | bit) & ~prev) <= m)) tile |= bit;
      }
    if ((uint32_t)popc(tile) != T || (uint32_t)popc(tile & ~prev) > m) {
      if (err) *err = "internal: rotating plan could not complete a tile";
      return QIPB200_ERR_UNSUPPORTED;
    }
    // its low positions: L qubits of tile & prev, preferring the ones that already sit low
    uint64_t want_low = 0;
    for (int round = 0; round < 2 && (uint32_t)popc(want_low) < L; ++round)
      for (uint32_t b = 0; b < n && (uint32_t)popc(want_low) < L; ++b) {
        const uint64_t bit = 1ull << b;
        if (!(tile & prev & bit) || (want_low & bit)) continue;
        if (round == 1 || phys[b] < L) want_low |= bit;
      }
    if ((uint32_t)popc(want_low) != L) {
      if (err) *err = "internal: rotating plan: fewer than L carried qubits";
      return QIPB200_ERR_UNSUPPORTED;
    }
    if (have_pending) {
      int st = flush_pending(want_low, {});
      if (st != QIPB200_OK) return st;
    }  // else: first pass -- prev is exactly the L qubits sitting low, so want_low == prev
    have_pending = true;
    pend_tile = tile;
    pend_taken = best.taken;
    prev = tile;
    remaining.swap(best.left);
  }
  if (have_pending) {
    // last pass: fold in every restoring transposition whose two positions are tile bits of this pass, in an order
    // that keeps the low positions filled from the tile; the rest is restored by swap-only passes below
    uint64_t keep = 0;
    for (uint32_t p = 0; p < L; ++p) keep |= 1ull << logical_at(p);
    uint64_t tile_phys = (1ull << L) - 1ull;
    for (uint32_t b = 0; b < n; ++b)
      if ((pend_tile >> b) & 1) tile_phys |= 1ull << phys[b];
    std::vector<std::pair<uint32_t, uint32_t>> extra;
    if (restore) {
      std::vector<uint32_t> sim = phys;  // simulate the transpositions b <-> home within the tile
      bool progress = true;
      while (progress) {
        progress = false;
        for (uint32_t b = 0; b < n; ++b) {
          const uint32_t where = sim[b];
          if (where == b || !((tile_phys >> where) & 1) || !((tile_phys >> b) & 1)) continue;
          extra.push_back(std::make_pair(b, where));  // physical positions b (home) and where
          for (uint32_t c = 0; c < n; ++c) {
            if (sim[c] == b)
              sim[c] = where;
            else if (c != b && sim[c] == where)
              sim[c] = b;
          }
          sim[b] = b;
          progress = true;
        }
      }
    }
    int st = flush_pending(keep, extra);
    if (st != QIPB200_OK) return st;
  }
  if (restore) return append_restore(prec, n, cfg_in, phys, out, err);
  return QIPB200_OK;
}

bool serialise_pass(const HostPass &p, PassParams *out) {
  const size_t bytes = pass_bytes(p);
  if (bytes > kMaxPassBytes) return false;
  out->h = p.hdr;
  unsigned char *w = out->recs;
  for (size_t i = 0; i < p.ops.size(); ++i) {
    MicroOp mh = p.ops[i].h;
    mh.data_bytes = (uint32_t)((p.ops[i].data.size() + 15) & ~(size_t)15);
    memcpy(w, &mh, sizeof(mh));
    w += sizeof(mh);
    if (!p.ops[i].data.empty()) memcpy(w, p.ops[i].data.data(), p.ops[i].data.size());
    w += mh.data_bytes;
  }
  out->h.gterm_off = (uint32_t)(w - out->recs);
  if (!p.gterms.empty()) memcpy(w, p.gterms.data(), p.gterms.size());
  w += (p.gterms.size() + 15) & ~(size_t)15;
  out->h.cond_off = (uint32_t)(w - out->recs);
  out->h.n_conds = (uint32_t)p.conds.size();
  if (!p.conds.empty()) memcpy(w, p.conds.data(), p.conds.size() * sizeof(CondTerm));
  out->h.blob_bytes = (uint32_t)bytes;
  return true;
}

}  // namespace qipb200
