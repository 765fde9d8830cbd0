// jit_codegen.cpp -- see jit_codegen.h.  Pure host C++.
//
// Reference semantics being specialised: one pass = the sequential product of the reference's per-entry
// sweeps (qip/src/builder.rs:423-514, qip-iterators/src/matrix_ops.rs:127-152) restricted to gates whose
// non-diagonal bits are tile bits; the arithmetic of every elementary op is issued in exactly the order of the
// interpreter kernel (tile_interp.cuh), with terms whose coefficient is exactly 0 dropped and coefficients of
// exactly +-1 turned into add/sub -- both exact for finite amplitudes, so the two kernels agree bit for bit
// (up to the sign of zero) and the interpreter's oracle parity carries over.
#include "jit_codegen.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <sstream>

namespace qipb200 {

namespace {

struct Cond {
  uint64_t gmask, gval;
};

struct PhTerm {
  uint64_t gmask, gval;
  double re, im;
};

// elementary op of a group, ready for emission (sub-index coordinates, K = bits of the group)
struct DElem {
  enum Kind { D1, X, PH, PHN, DK, HAD } kind = D1;
  bool real = false;
  uint32_t j = 0;          // D1 / X / HAD: target sub-bit
  uint32_t lc = 0;         // D1 / X: control sub-mask
  uint32_t lm = 0, lv = 0; // PH / PHN: acts on sub-indices c with (c & lm) == lv
  uint32_t pm = 0, pv = 0; // PH / PHN: in the threads whose tile-local group index t has (t & pm) == pv
  int cond = -1;           // index into the program's condition list
  double m[8] = {0};       // D1: real m00 m01 m10 m11 | complex (re,im) x 4; PH: w
  std::vector<uint32_t> mb;  // DK: sub-bits of the dense block (ascending)
  std::vector<double> mk;    // DK: 2^k x 2^k complex (re,im), row-major
  uint32_t slot = 0;       // PHN: factor-table slot
  struct TT {
    uint32_t pm, pv;
    double re, im;
  };
  std::vector<TT> tt;      // PH: thread-conditional factors (product formed in registers, applied once)
};

// value as it will be seen by a kernel of precision `f64` (constants are pooled after rounding)
inline double as_prec(bool f64, double v) { return f64 ? v : (double)(float)v; }

bool convert_group(const JGroup &jg, bool f64, std::vector<Cond> &conds, std::vector<DElem> *out,
                   std::vector<std::vector<PhTerm>> *phn_terms, std::vector<std::pair<double, double>> *phn_base,
                   std::string *why) {
  for (size_t i = 0; i < jg.elems.size(); ++i) {
    const JElem &e = jg.elems[i];
    DElem d;
    if (e.gmask) {
      int found = -1;
      for (size_t c = 0; c < conds.size(); ++c)
        if (conds[c].gmask == e.gmask && conds[c].gval == e.gval) found = (int)c;
      if (found < 0) {
        Cond c = {e.gmask, e.gval};
        found = (int)conds.size();
        conds.push_back(c);
      }
      d.cond = found;
    }
    switch (e.kind) {
      case JElem::D1:
      case JElem::X: {
        d.kind = e.kind == JElem::X ? DElem::X : DElem::D1;
        d.j = e.j;
        d.lc = e.lc;
        bool real = true;
        for (int q = 0; q < 4; ++q) real &= as_prec(f64, e.m[q].imag()) == 0.0;
        d.real = real;
        for (int q = 0; q < 4; ++q) {
          if (real) {
            d.m[q] = as_prec(f64, e.m[q].real());
          } else {
            d.m[2 * q] = as_prec(f64, e.m[q].real());
            d.m[2 * q + 1] = as_prec(f64, e.m[q].imag());
          }
        }
        break;
      }
      case JElem::HAD:
        d.kind = DElem::HAD, d.j = e.j;
        break;
      case JElem::PH:
        d.lm = e.lm, d.lv = e.lv;
        d.pm = e.pm, d.pv = e.pv;
        d.m[0] = as_prec(f64, e.m[0].real()), d.m[1] = as_prec(f64, e.m[0].imag());
        for (size_t k = 0; k < e.tterms.size(); ++k) {
          DElem::TT t = {e.tterms[k].pm, e.tterms[k].pv, as_prec(f64, e.tterms[k].w.real()), as_prec(f64, e.tterms[k].w.imag())};
          d.tt.push_back(t);
        }
        if (e.terms.empty()) {
          d.kind = DElem::PH;
        } else {

          if (e.gmask) return *why = "conditional phase run under a condition", false;
          d.kind = DElem::PHN;
          d.slot = (uint32_t)phn_terms->size();
          phn_base->push_back(std::make_pair(d.m[0], d.m[1]));
          std::vector<PhTerm> terms;
          for (size_t k = 0; k < e.terms.size(); ++k) {
            PhTerm t = {e.terms[k].gmask, e.terms[k].gval, as_prec(f64, e.terms[k].w.real()), as_prec(f64, e.terms[k].w.imag())};
            terms.push_back(t);
          }
          phn_terms->push_back(terms);
        }
        break;
      case JElem::DK: {
        d.kind = DElem::DK;
        d.mb = e.mb;
        if (e.mb.empty() || e.mb.size() > 3 || e.mk.size() != ((size_t)1 << (2 * e.mb.size()))) return *why = "malformed dense block", false;
        d.mk.resize(2 * e.mk.size());
        for (size_t q = 0; q < e.mk.size(); ++q) {
          d.mk[2 * q] = as_prec(f64, e.mk[q].real());
          d.mk[2 * q + 1] = as_prec(f64, e.mk[q].imag());
        }
        break;
      }
    }
    out->push_back(d);
  }
  return true;
}

// ---- source emission --------------------------------------------------------------------------
struct Gen {
  bool f64;
  std::ostringstream o;
  std::vector<double> pool;  // |value| of every pooled constant
  int nv = 0;
  uint32_t renamed = 0;

  std::string fresh() {
    char b[24];
    snprintf(b, sizeof(b), "v%d", nv++);
    return b;
  }
  // expression of constant v (never called with 0 / +-1 by the chain emitter)
  std::string K(double v) {
    const double a = std::fabs(v);
    size_t i = 0;
    for (; i < pool.size(); ++i)
      if (pool[i] == a) break;
    if (i == pool.size()) pool.push_back(a);
    char b[40];
    snprintf(b, sizeof(b), v < 0 ? "(-p.c[%zu])" : "p.c[%zu]", i);
    return b;
  }
  // acc = c0*v0; acc = fma(c1, v1, acc); ...   in this order, zero terms dropped, +-1 as add/sub
  std::string chain(const std::vector<std::pair<double, std::string>> &terms) {
    std::string acc;
    for (size_t i = 0; i < terms.size(); ++i) {
      const double c = terms[i].first;
      const std::string &v = terms[i].second;
      if (c == 0.0) continue;
      if (acc.empty()) {
        if (c == 1.0) acc = v;
        else if (c == -1.0) acc = "(-" + v + ")";
        else acc = "(" + K(c) + " * " + v + ")";
      } else {
        if (c == 1.0) acc = "(" + acc + " + " + v + ")";
        else if (c == -1.0) acc = "(" + acc + " - " + v + ")";
        else acc = "QFMA(" + K(c) + ", " + v + ", " + acc + ")";
      }
    }
    if (acc.empty()) acc = f64 ? "0.0" : "0.0f";
    return acc;
  }
};

uint32_t swz_units(bool f64, uint32_t t) { return f64 ? (t ^ ((t >> 3) & 7u)) : (t ^ (((t >> 4) & 7u) << 1)); }

}  // namespace

bool jit_generate(const HostPass &pass, qip_prec prec, JitProgram *out, std::string *why, bool paired,
                  const uint64_t *synth_index) {
  std::string dummy;
  if (!why) why = &dummy;
  const PassHeader &h = pass.hdr;
  const bool f64 = prec == QIP_F64;
  const uint32_t T = h.T, L = h.L, m = h.m;
  const uint32_t low3 = f64 ? 3 : 4;
  const uint32_t amp = f64 ? 16 : 8;
  const uint32_t K = pass.jbits;  // bits per group: 2^K amplitudes of a group live in one thread's registers
  if (K < 3 || K > 6 || pass.jgroups.empty()) return *why = "pass was not emitted as register groups (wide op, or generation off)", false;
  if (T < 11 || T > 14) return *why = "tile too small/large for the generated kernel", false;
  if (m < 3 || L < low3 || (1u << (L - low3)) > 256) return *why = "geometry has no TMA boxes", false;
  const uint32_t NA = 1u << K;
  // threads per CTA: every thread owns >= 1 group per super-op; 64 data registers (K = 4 f64 / K = 5 f32) leave
  // room for two 256-thread CTAs per SM, 32 for three
  static const uint32_t env_threads = []() {
    const char *e = getenv("QIPB200_JIT_CTA_THREADS");
    const int v = e ? atoi(e) : 0;
    return (uint32_t)(v == 128 || v == 256 ? v : 0);
  }();
  // 128 threads per CTA, three CTAs per SM.  On one H100 SXM (700 W) the N=30 f64 headline circuit took the same time
  // with 256 threads x 2 CTAs (299.1 / 303.0 ms vs 299.8 / 303.7 ms, alternating runs), so the default stays.
  uint32_t kThreads = env_threads ? env_threads : 128;
  while (kThreads > 32 && (1u << (T - K)) < kThreads) kThreads >>= 1;
  if ((1u << (T - K)) < kThreads) return *why = "tile holds fewer groups than a warp", false;
  const uint32_t kLaneBits = 5;
  uint32_t kWarpBits = 0;
  while ((32u << kWarpBits) < kThreads) ++kWarpBits;
  const uint32_t n_it_bits = T - K - kWarpBits - kLaneBits;
  const uint32_t NIT = 1u << n_it_bits;
  const uint32_t data_regs = NA * (f64 ? 4 : 2);
  const uint32_t ctas_per_sm = data_regs <= 32 ? 3 : (kThreads <= 128 ? 3 : 2);
  const char *RT = f64 ? "double" : "float";

  // ---- convert ----
  std::vector<Cond> conds;
  std::vector<std::vector<PhTerm>> phn_terms;
  std::vector<std::pair<double, double>> phn_base;
  std::vector<std::vector<DElem>> supers;
  std::vector<uint32_t> pmask;  // tile-local bit mask of each super-op
  std::vector<std::vector<uint32_t>> pbits;
  for (size_t i = 0; i < pass.jgroups.size(); ++i) {
    const JGroup &jg = pass.jgroups[i];
    if (jg.bits.size() != K) return *why = "malformed group bit list", false;
    std::vector<DElem> el;
    if (!convert_group(jg, f64, conds, &el, &phn_terms, &phn_base, why)) return false;
    supers.push_back(el);
    pbits.push_back(jg.bits);
    uint32_t pm = 0;
    for (uint32_t q = 0; q < K; ++q) {
      if (jg.bits[q] >= T || (q && jg.bits[q] <= jg.bits[q - 1])) return *why = "malformed group bit list", false;
      pm |= 1u << jg.bits[q];
    }
    pmask.push_back(pm);
  }
  if (conds.size() > 256) return *why = "more than 256 CTA-uniform conditions", false;
  const size_t S = supers.size();
  const size_t NC = conds.size(), NPH = phn_terms.size();
  size_t NPT = 0;
  for (size_t i = 0; i < NPH; ++i) NPT += phn_terms[i].size();
  if (NPH > 1024) return *why = "too many conditional phase runs", false;
  const size_t gsz = f64 ? sizeof(GlobalTerm<double>) : sizeof(GlobalTerm<float>);
  const size_t NG = pass.gterms.size() / gsz;

  // ---- thread maps: segments of super-ops that share their warp-id bits ----
  const uint32_t all_bits = (1u << T) - 1u;
  std::vector<uint32_t> wmask(S);
  std::vector<bool> cta_barrier_before(S, false);
  // Bank groups: with the 128-byte XOR swizzle the 16-byte bank group of tile-local index t is (t ^ t>>3) & 7 for
  // f64 (8-byte bank pair (t0, t1^t4, t2^t5, t3^t6) for f32).  A quarter warp (half warp for f32) is conflict free
  // iff its lane bits reach every bank-group bit: bank bit k needs tile bit k or k+3 among the lane bits (f32: bit 0
  // alone for k = 0).  A bank bit whose providers all sit in the sub-bits is lost anyway (inherent 2-way conflict);
  // the warp-id bits must not take the last provider away: a super-op already moves 2 x 64 KiB per tile through shared
  // memory, and every bank conflict adds to that.
  const uint32_t n_bank_bits = f64 ? 3 : 4;
  auto providers = [&](uint32_t k) -> uint32_t {  // tile bits that toggle bank bit k
    if (!f64 && k == 0) return 1u;
    return ((1u << k) | (1u << (k + 3))) & all_bits;
  };
  auto lost_bank_bits = [&](uint32_t taken) {  // bank bits no lane bit can reach once `taken` bits are gone
    uint32_t n = 0;
    for (uint32_t k = 0; k < n_bank_bits; ++k) n += (providers(k) & ~taken) == 0;
    return n;
  };
  auto extra_cost = [&](size_t s, size_t e, uint32_t w) {
    uint32_t c = 0;
    for (size_t k = s; k < e; ++k) c += lost_bank_bits(pmask[k] | w) - lost_bank_bits(pmask[k]);
    return c;
  };
  auto best_warp_bits = [&](size_t s, size_t e, uint32_t free_bits, uint32_t *cost) {
    // all kWarpBits-subsets of the free bits, highest bits first (ties go to the first hit)
    std::vector<uint32_t> fb;
    for (int b = (int)T - 1; b >= 0; --b)
      if ((free_bits >> b) & 1) fb.push_back((uint32_t)b);
    uint32_t best = 0, best_cost = ~0u;
    std::vector<uint32_t> idx(kWarpBits);
    for (uint32_t i = 0; i < kWarpBits; ++i) idx[i] = i;
    if (fb.size() < kWarpBits) {
      *cost = ~0u;
      return 0u;
    }
    for (;;) {
      uint32_t w = 0;
      for (uint32_t i = 0; i < kWarpBits; ++i) w |= 1u << fb[idx[i]];
      const uint32_t c = extra_cost(s, e, w);
      if (c < best_cost) best = w, best_cost = c;
      int q = (int)kWarpBits - 1;
      while (q >= 0 && idx[q] == fb.size() - kWarpBits + q) --q;
      if (q < 0) break;
      ++idx[q];
      for (uint32_t r = q + 1; r < kWarpBits; ++r) idx[r] = idx[r - 1] + 1;
    }
    *cost = best_cost;
    return best;
  };
  for (size_t s = 0; s < S;) {
    uint32_t free_bits = all_bits & ~pmask[s];
    uint32_t cost = 0;
    uint32_t w = best_warp_bits(s, s + 1, free_bits, &cost);
    size_t e = s + 1;
    // extend the segment while common free bits exist that cost no bank conflict: a CTA barrier is far cheaper than
    // a 2-way conflict on every access of a super-op
    while (e < S && (uint32_t)__builtin_popcount(free_bits & ~pmask[e]) >= kWarpBits) {
      uint32_t c2 = 0;
      const uint32_t w2 = best_warp_bits(s, e + 1, free_bits & ~pmask[e], &c2);
      if (c2 > cost) break;
      free_bits &= ~pmask[e++];
      w = w2;
      cost = c2;
    }
    for (size_t k = s; k < e; ++k) wmask[k] = w;
    cta_barrier_before[s] = s != 0;
    s = e;
  }

  Gen g;
  g.f64 = f64;
  std::ostringstream fn;  // the so_K functions
  uint32_t n_elems = 0;
  for (size_t s = 0; s < S; ++s) {
    // lane / iteration bits of this super-op
    uint32_t avail = all_bits & ~pmask[s] & ~wmask[s];
    std::vector<uint32_t> lane;  // tile bit of lane bit k
    for (uint32_t k = 0; k < n_bank_bits; ++k) {
      int pick = -1;
      if ((avail >> k) & 1) pick = (int)k;
      else if ((f64 || k >= 1) && k + 3 < T && ((avail >> (k + 3)) & 1)) pick = (int)(k + 3);
      if (pick >= 0) {
        lane.push_back((uint32_t)pick);
        avail &= ~(1u << pick);
      }
    }
    for (uint32_t b = 0; b < T && lane.size() < kLaneBits; ++b)
      if ((avail >> b) & 1) {
        lane.push_back(b);
        avail &= ~(1u << b);
      }
    std::vector<uint32_t> itb;
    for (uint32_t b = 0; b < T; ++b)
      if ((avail >> b) & 1) itb.push_back(b);
    if (lane.size() != kLaneBits || itb.size() != n_it_bits) return *why = "internal: thread map", false;
    const uint32_t n_tid_bits = kLaneBits + kWarpBits;
    std::vector<uint32_t> dst(n_tid_bits);  // tid bit -> tile bit
    for (uint32_t k = 0; k < kLaneBits; ++k) dst[k] = lane[k];
    {
      uint32_t k = 0;
      for (uint32_t b = 0; b < T; ++b)
        if ((wmask[s] >> b) & 1) dst[kLaneBits + k++] = b;
    }

    fn << "// super-op " << s << ": sub-bits {";
    for (uint32_t q = 0; q < K; ++q) fn << (q ? "," : "") << pbits[s][q];
    fn << "}, warp bits 0x" << std::hex << wmask[s] << std::dec << "\n";
    fn << "QIP_DEV void so_" << s << "(unsigned char* sm, const unsigned tid, const JP& p, const unsigned* condw, const "
       << RT << "* tbl, const " << RT << "* gt) {\n";
    fn << "  unsigned t = 0u;\n";
    for (uint32_t k = 0; k < n_tid_bits;) {
      uint32_t len = 1;
      while (k + len < n_tid_bits && dst[k + len] == dst[k] + len) ++len;
      fn << "  t |= ((tid >> " << k << ") & " << ((1u << len) - 1u) << "u) << " << dst[k] << ";\n";
      k += len;
    }
    bool needs_tt = false;
    for (size_t i = 0; i < supers[s].size(); ++i) needs_tt |= supers[s][i].pm != 0 || !supers[s][i].tt.empty();
    if (needs_tt) fn << "  const unsigned tt0 = t;\n";  // tile-local index of this thread's group (sub-bits zero)
    fn << (f64 ? "  t ^= (t >> 3) & 7u;\n  const unsigned a0 = t << 4;\n" : "  t ^= ((t >> 4) & 7u) << 1;\n  const unsigned a0 = t << 3;\n");
    // condition words this super-op tests
    {
      uint32_t words = 0;
      for (size_t i = 0; i < supers[s].size(); ++i)
        if (supers[s][i].cond >= 0) words |= 1u << (supers[s][i].cond >> 5);
      for (uint32_t w = 0; w < 8; ++w)
        if ((words >> w) & 1) fn << "  const unsigned cw" << w << " = condw[" << w << "];\n";
    }
    const bool last = s + 1 == S;
    if (last && NG) fn << "  const bool hasg = condw[8] != 0u;\n  const " << RT << " gr = gt[0], gi = gt[1];\n";
    // conditional-phase factors (one broadcast shared-memory read each) are loop invariants: read them once per
    // super-op, not once per group (the compiler cannot prove that the group's stores leave the table alone)
    std::vector<char> phn_hoisted(phn_terms.size(), 0);
    if (NIT > 1) {
      uint32_t budget = 12;
      for (size_t ei = 0; ei < supers[s].size() && budget; ++ei)
        if (supers[s][ei].kind == DElem::PHN && !phn_hoisted[supers[s][ei].slot]) {
          const uint32_t sl = supers[s][ei].slot;
          fn << "  const " << RT << " pw" << sl << "r = tbl[" << 2 * sl << "], pw" << sl << "i = tbl[" << 2 * sl + 1 << "];\n";
          phn_hoisted[sl] = 1;
          --budget;
        }
    }
    if (NIT > 1) fn << "#pragma unroll 1\n  for (unsigned it = 0; it < " << NIT << "u; ++it) {\n";
    else fn << "  {\n";
    {
      std::string a = "a0";
      for (uint32_t k = 0; k < n_it_bits; ++k) {
        char b[96];
        snprintf(b, sizeof(b), " ^ (((it >> %u) & 1u) * %uu)", k, swz_units(f64, 1u << itb[k]) * amp);
        a += b;
      }
      fn << "    const unsigned a = " << a << ";\n";
      if (needs_tt) {
        std::string tt = "tt0";
        for (uint32_t k = 0; k < n_it_bits; ++k) {
          char b[96];
          snprintf(b, sizeof(b), " | (((it >> %u) & 1u) << %u)", k, itb[k]);
          tt += b;
        }
        fn << "    const unsigned tt = " << tt << ";\n";
      }
    }
    // the 2^K addresses: XOR part (swizzle-modified bits) + additive part
    std::vector<uint32_t> soff(NA), xpart(NA), apart(NA), xs;
    for (uint32_t u = 0; u < NA; ++u) {
      uint32_t off = 0;
      for (uint32_t i = 0; i < K; ++i)
        if ((u >> i) & 1) off |= 1u << pbits[s][i];
      soff[u] = swz_units(f64, off) * amp;
      xpart[u] = soff[u] & 0x70u;
      apart[u] = soff[u] & ~0x70u;
      if (xpart[u] && std::find(xs.begin(), xs.end(), xpart[u]) == xs.end()) xs.push_back(xpart[u]);
    }
    for (size_t i = 0; i < xs.size(); ++i) fn << "    const unsigned ax" << xs[i] << " = a ^ " << xs[i] << "u;\n";
    auto addr = [&](uint32_t u) {
      std::ostringstream x;
      if (xpart[u]) x << "ax" << xpart[u];
      else x << "a";
      if (apart[u]) x << " + " << apart[u] << "u";
      return x.str();
    };
    // ---- conditional exchanges folded into the addresses ----
    // An X under a CTA-uniform condition (CNOT / Toffoli whose control lies outside the tile) cannot be a static
    // renaming; as arithmetic it costs four predicated moves per amplitude.  When it is the FIRST thing that
    // happens to its amplitudes it is a conditional choice of the LOAD address instead (one select per amplitude),
    // when it is the LAST thing, of the STORE address.
    const std::vector<DElem> &els = supers[s];
    auto is_xlike = [](const DElem &d) {
      return d.kind == DElem::X || (d.kind == DElem::D1 && d.real && d.m[0] == 0.0 && d.m[3] == 0.0 && d.m[1] == 1.0 && d.m[2] == 1.0);
    };
    auto pairs_list = [&](uint32_t j, uint32_t lc, std::vector<std::pair<uint32_t, uint32_t>> *pr) {
      for (uint32_t c = 0; c < NA; ++c) {
        if ((c >> j) & 1) continue;
        if ((c & lc) == lc) pr->push_back(std::make_pair(c, c | (1u << j)));
      }
    };
    auto amps_of = [&](const DElem &d) -> uint64_t {
      uint64_t a = 0;
      if (d.kind == DElem::DK) return NA == 64 ? ~0ull : ((1ull << NA) - 1ull);
      if (d.kind == DElem::PH || d.kind == DElem::PHN) {
        for (uint32_t c = 0; c < NA; ++c)
          if ((c & d.lm) == d.lv) a |= 1ull << c;
        return a;
      }
      std::vector<std::pair<uint32_t, uint32_t>> pr;
      pairs_list(d.j, d.kind == DElem::HAD ? 0u : d.lc, &pr);
      for (size_t k = 0; k < pr.size(); ++k) a |= (1ull << pr[k].first) | (1ull << pr[k].second);
      return a;
    };
    std::vector<char> folded(els.size(), 0);
    std::vector<int> lf_cond(NA, -1), sf_cond(NA, -1);
    std::vector<uint32_t> lf_other(NA), sf_other(NA);
    for (uint32_t u = 0; u < NA; ++u) lf_other[u] = sf_other[u] = u;
    {
      std::vector<uint32_t> slot_of(NA);
      uint64_t dirty = 0;
      for (uint32_t u = 0; u < NA; ++u) slot_of[u] = u;
      for (size_t ei = 0; ei < els.size(); ++ei) {
        const DElem &d = els[ei];
        const uint64_t am = amps_of(d);
        if (is_xlike(d)) {
          std::vector<std::pair<uint32_t, uint32_t>> pr;
          pairs_list(d.j, d.lc, &pr);
          if (d.cond < 0) {  // static renaming: follows the names, touches nothing
            for (size_t k = 0; k < pr.size(); ++k) std::swap(slot_of[pr[k].first], slot_of[pr[k].second]);
            continue;
          }
          if (!(am & dirty)) {
            for (size_t k = 0; k < pr.size(); ++k) {
              const uint32_t sx = slot_of[pr[k].first], sy = slot_of[pr[k].second];
              lf_cond[sx] = lf_cond[sy] = d.cond;
              lf_other[sx] = sy;
              lf_other[sy] = sx;
            }
            folded[ei] = 1;
          }
        }
        dirty |= am;
      }
      uint64_t later = 0;
      for (size_t ei = els.size(); ei-- > 0;) {
        if (folded[ei]) continue;
        const DElem &d = els[ei];
        const uint64_t am = amps_of(d);
        if (is_xlike(d) && d.cond >= 0 && !(am & later)) {
          std::vector<std::pair<uint32_t, uint32_t>> pr;
          pairs_list(d.j, d.lc, &pr);
          for (size_t k = 0; k < pr.size(); ++k) {
            sf_cond[pr[k].first] = sf_cond[pr[k].second] = d.cond;
            sf_other[pr[k].first] = pr[k].second;
            sf_other[pr[k].second] = pr[k].first;
          }
          folded[ei] = 1;
        }
        later |= am;
      }
    }
    auto cond_test = [](int c) {
      char b[64];
      snprintf(b, sizeof(b), "((cw%d >> %d) & 1u)", c >> 5, c & 31);
      return std::string(b);
    };
    auto sel_addr = [&](uint32_t u, int c, uint32_t other, const char *tag) {
      if (c < 0) return addr(u);
      const std::string nm = std::string(tag) + std::to_string(u);
      fn << "    const unsigned " << nm << " = " << cond_test(c) << " ? (" << addr(other) << ") : (" << addr(u) << ");\n";
      return nm;
    };
    std::vector<std::string> vr(NA), vi(NA);
    for (uint32_t u = 0; u < NA; ++u) {
      const std::string la = sel_addr(u, lf_cond[u], lf_other[u], "la");
      const std::string q = g.fresh();
      fn << "    const QV " << q << " = *reinterpret_cast<const QV*>(sm + " << la << ");\n";
      vr[u] = q + ".x";
      vi[u] = q + ".y";
    }
    // ---- elementary ops ----
    for (size_t ei = 0; ei < supers[s].size(); ++ei) {
      const DElem &d = supers[s][ei];
      ++n_elems;
      if (folded[ei]) {  // became a conditional load / store address
        ++g.renamed;
        continue;
      }
      const bool cond = d.cond >= 0 || d.pm != 0;
      std::string ctest = d.cond >= 0 ? cond_test(d.cond) : std::string();
      if (d.pm) {  // thread predicate of a phase whose bit lies outside the group
        char b[64];
        snprintf(b, sizeof(b), "((tt & %uu) == %uu)", d.pm, d.pv);
        ctest = ctest.empty() ? std::string(b) : "(" + ctest + " && " + b + ")";
      }
      // new values of the amplitudes this op changes: (u, new re expr, new im expr)
      struct Upd {
        uint32_t u;
        std::string re, im;
      };
      std::vector<Upd> upd;
      typedef std::vector<std::pair<double, std::string>> Terms;
      if (is_xlike(d)) {
        std::vector<std::pair<uint32_t, uint32_t>> pr;
        pairs_list(d.j, d.lc, &pr);
        if (!cond) {  // pure renaming: no instruction at all, exact for every bit pattern
          for (size_t k = 0; k < pr.size(); ++k) {
            std::swap(vr[pr[k].first], vr[pr[k].second]);
            std::swap(vi[pr[k].first], vi[pr[k].second]);
          }
          ++g.renamed;
          continue;
        }
        for (size_t k = 0; k < pr.size(); ++k) {
          Upd a = {pr[k].first, vr[pr[k].second], vi[pr[k].second]}, b = {pr[k].second, vr[pr[k].first], vi[pr[k].first]};
          upd.push_back(a);
          upd.push_back(b);
        }
      } else if (d.kind == DElem::HAD) {
        std::vector<std::pair<uint32_t, uint32_t>> pr;
        pairs_list(d.j, 0u, &pr);
        for (size_t k = 0; k < pr.size(); ++k) {
          const uint32_t x = pr[k].first, y = pr[k].second;
          Upd a = {x, "(" + vr[x] + " + " + vr[y] + ")", "(" + vi[x] + " + " + vi[y] + ")"};
          Upd b = {y, "(" + vr[x] + " - " + vr[y] + ")", "(" + vi[x] + " - " + vi[y] + ")"};
          upd.push_back(a);
          upd.push_back(b);
        }
      } else if (d.kind == DElem::D1) {
        std::vector<std::pair<uint32_t, uint32_t>> pr;
        pairs_list(d.j, d.lc, &pr);
        for (size_t k = 0; k < pr.size(); ++k) {
          const uint32_t x = pr[k].first, y = pr[k].second;
          const std::string &xr = vr[x], &xi = vi[x], &yr = vr[y], &yi = vi[y];
          Upd a, b;
          a.u = x;
          b.u = y;
          if (d.real) {  // tile_interp.cuh QIP_D1R: x' = fma(m00, x, m01*y); y' = fma(m10, x, m11*y)
            const double m00 = d.m[0], m01 = d.m[1], m10 = d.m[2], m11 = d.m[3];
            a.re = g.chain(Terms{{m01, yr}, {m00, xr}});
            a.im = g.chain(Terms{{m01, yi}, {m00, xi}});
            b.re = g.chain(Terms{{m11, yr}, {m10, xr}});
            b.im = g.chain(Terms{{m11, yi}, {m10, xi}});
          } else {  // QIP_D1C
            const double m00r = d.m[0], m00i = d.m[1], m01r = d.m[2], m01i = d.m[3], m10r = d.m[4], m10i = d.m[5],
                         m11r = d.m[6], m11i = d.m[7];
            a.re = g.chain(Terms{{m01r, yr}, {-m01i, yi}, {m00r, xr}, {-m00i, xi}});
            a.im = g.chain(Terms{{m01r, yi}, {m01i, yr}, {m00r, xi}, {m00i, xr}});
            b.re = g.chain(Terms{{m11r, yr}, {-m11i, yi}, {m10r, xr}, {-m10i, xi}});
            b.im = g.chain(Terms{{m11r, yi}, {m11i, yr}, {m10r, xi}, {m10i, xr}});
          }
          upd.push_back(a);
          upd.push_back(b);
        }
      } else if ((d.kind == DElem::PH || d.kind == DElem::PHN) && !d.tt.empty()) {
        // factor = base * product of the factors whose thread predicate holds: scalar work, then ONE application
        const std::string wr = g.fresh(), wi = g.fresh();
        auto lit = [&](double v) -> std::string {
          if (v == 0.0) return f64 ? "0.0" : "0.0f";
          if (v == 1.0) return f64 ? "1.0" : "1.0f";
          if (v == -1.0) return f64 ? "-1.0" : "-1.0f";
          return g.K(v);
        };
        if (d.kind == DElem::PHN)  // the CTA-conditional part of the product was formed once per CTA (factor table)
          fn << "    " << RT << " " << wr << " = tbl[" << 2 * d.slot << "], " << wi << " = tbl[" << 2 * d.slot + 1 << "];\n";
        else
          fn << "    " << RT << " " << wr << " = " << lit(d.m[0]) << ", " << wi << " = " << lit(d.m[1]) << ";\n";
        for (size_t k = 0; k < d.tt.size(); ++k) {
          const std::string nr2 = g.fresh(), ni2 = g.fresh();
          fn << "    if ((tt & " << d.tt[k].pm << "u) == " << d.tt[k].pv << "u) { const " << RT << " " << nr2 << " = "
             << g.chain(Terms{{-d.tt[k].im, wi}, {d.tt[k].re, wr}}) << ", " << ni2 << " = "
             << g.chain(Terms{{d.tt[k].im, wr}, {d.tt[k].re, wi}}) << "; " << wr << " = " << nr2 << "; " << wi << " = " << ni2 << "; }\n";
        }
        for (uint32_t c = 0; c < NA; ++c) {
          if ((c & d.lm) != d.lv) continue;
          Upd a = {c, "QFMA(" + wr + ", " + vr[c] + ", -(" + wi + " * " + vi[c] + "))",
                   "QFMA(" + wr + ", " + vi[c] + ", (" + wi + " * " + vr[c] + "))"};
          upd.push_back(a);
        }
      } else if (d.kind == DElem::PH) {  // QIP_PH: re' = fma(wr, re, -(wi*im)); im' = fma(wr, im, wi*re)
        for (uint32_t c = 0; c < NA; ++c) {
          if ((c & d.lm) != d.lv) continue;
          Upd a = {c, g.chain(Terms{{-d.m[1], vi[c]}, {d.m[0], vr[c]}}), g.chain(Terms{{d.m[1], vr[c]}, {d.m[0], vi[c]}})};
          upd.push_back(a);
        }
      } else if (d.kind == DElem::PHN) {  // factor formed once per CTA (table behind the tile)
        std::string wr, wi;
        if (phn_hoisted[d.slot]) {
          wr = "pw" + std::to_string(d.slot) + "r";
          wi = "pw" + std::to_string(d.slot) + "i";
        } else {
          wr = g.fresh(), wi = g.fresh();
          fn << "    const " << RT << " " << wr << " = tbl[" << 2 * d.slot << "], " << wi << " = tbl[" << 2 * d.slot + 1 << "];\n";
        }
        for (uint32_t c = 0; c < NA; ++c) {
          if ((c & d.lm) != d.lv) continue;
          Upd a = {c, "QFMA(" + wr + ", " + vr[c] + ", -(" + wi + " * " + vi[c] + "))",
                   "QFMA(" + wr + ", " + vi[c] + ", (" + wi + " * " + vr[c] + "))"};
          upd.push_back(a);
        }
      } else {  // DK: dense 2^k x 2^k on the sub-bits mb, for every setting of the group's other bits; rows in
                // order, re = fma(mr, xr, re); re = fma(-mi, xi, re); im likewise (tile_interp.cuh _QIP_D3_BODY)
        const uint32_t kb = (uint32_t)d.mb.size(), SB = 1u << kb;
        uint32_t mbm = 0;
        for (uint32_t q = 0; q < kb; ++q) mbm |= 1u << d.mb[q];
        for (uint32_t base = 0; base < NA; ++base) {
          if (base & mbm) continue;
          std::vector<uint32_t> idx(SB);
          for (uint32_t r = 0; r < SB; ++r) {
            uint32_t c = base;
            for (uint32_t q = 0; q < kb; ++q)
              if ((r >> q) & 1) c |= 1u << d.mb[q];
            idx[r] = c;
          }
          for (uint32_t u = 0; u < SB; ++u) {
            Terms tr, ti;
            for (uint32_t v = 0; v < SB; ++v) {
              const double mr = d.mk[2 * (u * SB + v)], mi = d.mk[2 * (u * SB + v) + 1];
              tr.push_back(std::make_pair(mr, vr[idx[v]]));
              tr.push_back(std::make_pair(-mi, vi[idx[v]]));
              ti.push_back(std::make_pair(mr, vi[idx[v]]));
              ti.push_back(std::make_pair(mi, vr[idx[v]]));
            }
            Upd a = {idx[u], g.chain(tr), g.chain(ti)};
            upd.push_back(a);
          }
        }
      }
      // materialise (all right-hand sides refer to the OLD names)
      std::vector<std::string> nr(upd.size()), ni(upd.size());
      for (size_t k = 0; k < upd.size(); ++k) {
        nr[k] = g.fresh();
        ni[k] = g.fresh();
      }
      if (!cond) {
        for (size_t k = 0; k < upd.size(); ++k)
          fn << "    const " << RT << " " << nr[k] << " = " << upd[k].re << ", " << ni[k] << " = " << upd[k].im << ";\n";
      } else {
        for (size_t k = 0; k < upd.size(); ++k)
          fn << "    " << RT << " " << nr[k] << " = " << vr[upd[k].u] << ", " << ni[k] << " = " << vi[upd[k].u] << ";\n";
        fn << "    if (" << ctest << ") {\n";
        for (size_t k = 0; k < upd.size(); ++k)
          fn << "      " << nr[k] << " = " << upd[k].re << "; " << ni[k] << " = " << upd[k].im << ";\n";
        fn << "    }\n";
      }
      for (size_t k = 0; k < upd.size(); ++k) {
        vr[upd[k].u] = nr[k];
        vi[upd[k].u] = ni[k];
      }
    }
    if (last && NG) {  // CTA-uniform phase product, folded into the last write of every amplitude
      std::vector<std::string> nr(NA), ni(NA);
      for (uint32_t u = 0; u < NA; ++u) {
        nr[u] = g.fresh();
        ni[u] = g.fresh();
        fn << "    " << RT << " " << nr[u] << " = " << vr[u] << ", " << ni[u] << " = " << vi[u] << ";\n";
      }
      fn << "    if (hasg) {\n";
      for (uint32_t u = 0; u < NA; ++u)
        fn << "      " << nr[u] << " = QFMA(gr, " << vr[u] << ", -(gi * " << vi[u] << ")); " << ni[u] << " = QFMA(gr, " << vi[u]
           << ", (gi * " << vr[u] << "));\n";
      fn << "    }\n";
      for (uint32_t u = 0; u < NA; ++u) {
        vr[u] = nr[u];
        vi[u] = ni[u];
      }
    }
    for (uint32_t u = 0; u < NA; ++u) {
      const std::string sa = sel_addr(u, sf_cond[u], sf_other[u], "sa");
      const std::string q = g.fresh();
      fn << "    { QV " << q << "; " << q << ".x = " << vr[u] << "; " << q << ".y = " << vi[u] << "; *reinterpret_cast<QV*>(sm + "
         << sa << ") = " << q << "; }\n";
    }
    fn << "  }\n}\n\n";
  }

  // ---- parameter block ----
  const uint32_t NBOX = 1u << (m - 3);
  const size_t NK = g.pool.size();
  std::ostringstream src;
  src << "// generated by rustqip_b200/csrc/jit_codegen.cpp -- one fused tile pass, specialised\n";
  src << "typedef unsigned long long u64;\n";
  src << "#define TILE_T " << T << "\n#define TILE_L " << L << "\n#define TILE_M " << m << "\n#define LOW3 " << low3 << "\n";
  src << "#define NBOX " << NBOX << "\n#define NC " << NC << "\n#define NPH " << NPH << "\n#define NPT " << NPT << "\n#define NG " << NG
      << "\n#define NK " << NK << "\n";
  src << "#define CTA_THREADS " << kThreads << "\n#define CTAS_PER_SM " << ctas_per_sm << "\n";
  src << "#define TILE_BYTES " << (amp << T) << "u\n#define BOX_BYTES " << (amp << (L + 3)) << "u\n";
  const uint32_t tbl_bytes = (uint32_t)(((NPH * 2 * (f64 ? 8 : 4)) + 15) & ~(size_t)15);
  const uint32_t off_tbl = amp << T, off_gt = off_tbl + tbl_bytes, off_condw = off_gt + 16, off_mbar = off_condw + 48;
  src << "#define OFF_TBL " << off_tbl << "u\n#define OFF_GT " << off_gt << "u\n#define OFF_CONDW " << off_condw << "u\n#define OFF_MBAR "
      << off_mbar << "u\n";
  src << "#define QIP_PAIRED " << (paired ? 1 : 0) << "\n";
  const bool synth = synth_index != nullptr;
  src << "#define QIP_SYNTH " << (synth ? 1 : 0) << "\n";
  src << "typedef " << RT << " R;\n";
  src << "struct JP {\n  u64 box_off[NBOX];\n";
  if (NC) src << "  u64 cm[NC], cv[NC];\n";
  if (NPT) src << "  u64 ptm[NPT], ptv[NPT];\n";
  if (NG) src << "  u64 gm[NG], gv[NG];\n";
  if (NK) src << "  R c[NK];\n";
  if (NPT) src << "  R ptw[2 * NPT];\n";
  if (NPH) src << "  R pw[2 * NPH];\n";
  if (NG) src << "  R gw[2 * NG];\n";
  src << "  unsigned hi_pos[8];\n";
  if (NPH) src << "  unsigned pt_begin[NPH + 1];\n";
  if (synth) src << "  unsigned init_lo, init_hi;\n";  // the basis index the tiles are built from
  // multi-GPU (paired send, below): tiles whose index bit `send_bit` equals `send_val` are stored to `tmap_out` (the
  // partner's shard) at the index with that bit flipped; send_bit >= 64: off
  src << "  unsigned send_bit, send_val;\n";
  // first tile of the launch in the tile counter (jit_runtime.cu writes 0: every launch covers the whole pass)
  src << "  unsigned tile_off_lo, tile_off_hi;\n";
  // tiles of this launch: a CTA walks the tile counter with stride gridDim.x (grid == tile count: one tile per CTA;
  // a grid of a few CTAs per SM: persistent CTAs, no CTA exit / launch / barrier init between tiles)
  src << "  unsigned tile_cnt_lo, tile_cnt_hi;\n";
  // > 0: ask the TMA unit to pull the tile `prefetch_dist` places ahead in the tile counter into L2 while this one is
  // processed (DRAM reads in flight are then no longer bounded by the shared memory of the resident CTAs)
  src << "  unsigned prefetch_dist, pad_;\n";
  // migration fused into this pass, in place ("paired send", multi-GPU): a tile of the half this rank gives away
  // (tile counter bit pair_cbit == send_val) is announced to the partner as soon as it sits in shared memory (partner's
  // flag word of the paired tile := pair_seq) and stored into the PARTNER's shard (tmap_out, index bit send_bit
  // flipped) once the partner has announced the tile it gives in return -- the slot being overwritten.  pair_my == 0: off
  src << "  unsigned pair_cbit, pair_seq, pair_my_lo, pair_my_hi, pair_peer_lo, pair_peer_hi, pair_err_lo, pair_err_hi;\n";
  src << "};\n";
  src << R"(#ifdef QIP_JIT_HOST
#include <cmath>
#include <cstring>
#define QIP_DEV static inline
#define QFMA(a, b, c) std::fma((a), (b), (c))
struct alignas(2 * sizeof(R)) QV { R x, y; };
struct alignas(16) QZ { unsigned x, y, z, w; };
#else
#define QIP_DEV __device__ __forceinline__
#define QFMA(a, b, c) fma((a), (b), (c))
)";
  src << (f64 ? "typedef double2 QV;\n" : "typedef float2 QV;\n");
  src << "typedef uint4 QZ;\n";
  src << "#endif\n\n";
  src << fn.str();

  // prelude: per-CTA condition word, conditional-phase factor table, CTA-uniform global factor
  const bool has_prelude = NC || NPH || NG;
  src << "QIP_DEV void prelude(unsigned char* sm, const unsigned tid, const JP& p, const u64 base) {\n";
  src << "  unsigned* condw = reinterpret_cast<unsigned*>(sm + OFF_CONDW);\n  (void)condw; (void)base; (void)tid;\n";
  if (NC) {
    src << "  for (unsigned cb = 0; cb < NC; cb += CTA_THREADS) {\n    const unsigned ci = cb + tid;\n    bool on = false;\n";
    src << "    if (ci < NC) on = (base & p.cm[ci]) == p.cv[ci];\n";
    src << "#ifdef QIP_JIT_HOST\n    if (on && ci < 256u) condw[ci >> 5] |= 1u << (ci & 31u);\n#else\n";
    src << "    const unsigned bits = __ballot_sync(0xffffffffu, on);\n    if ((tid & 31u) == 0u && ci < 256u) condw[ci >> 5] = bits;\n#endif\n  }\n";
  }
  if (NPH) {
    src << "  {\n    R* tbl = reinterpret_cast<R*>(sm + OFF_TBL);\n    for (unsigned e = tid; e < NPH; e += " << kThreads << "u) {\n";
    src << "      R wr = p.pw[2 * e], wi = p.pw[2 * e + 1];\n";
    src << "      for (unsigned k = p.pt_begin[e]; k < p.pt_begin[e + 1]; ++k) {\n";
    src << "        if ((base & p.ptm[k]) != p.ptv[k]) continue;\n";
    src << "        const R nr = wr * p.ptw[2 * k] - wi * p.ptw[2 * k + 1];\n";
    src << "        wi = wr * p.ptw[2 * k + 1] + wi * p.ptw[2 * k];\n        wr = nr;\n      }\n";
    src << "      tbl[2 * e] = wr;\n      tbl[2 * e + 1] = wi;\n    }\n  }\n";
  }
  if (NG) {
    src << "  if (tid == " << kThreads - 1 << "u) {\n    R gr = (R)1, gi = (R)0;\n    unsigned hasg = 0u;\n";
    src << "    for (unsigned k = 0; k < NG; ++k) {\n      if ((base & p.gm[k]) != p.gv[k]) continue;\n";
    src << "      const R nr = gr * p.gw[2 * k] - gi * p.gw[2 * k + 1];\n      gi = gr * p.gw[2 * k + 1] + gi * p.gw[2 * k];\n      gr = nr;\n      hasg = 1u;\n    }\n";
    src << "    R* gt = reinterpret_cast<R*>(sm + OFF_GT);\n    gt[0] = gr;\n    gt[1] = gi;\n    condw[8] = hasg;\n  }\n";
  }
  src << "}\n\n";

  // tile base index: the tile counter with zero bits inserted at the high tile bit positions
  src << "QIP_DEV u64 tile_base(const JP& p, u64 tile) {\n  u64 base = tile << TILE_L;\n";
  src << "  for (unsigned i = 0; i < TILE_M; ++i) {\n    const unsigned q = p.hi_pos[i];\n";
  src << "    base = ((base >> q) << (q + 1)) | (base & ((1ull << q) - 1ull));\n  }\n  return base;\n}\n\n";

  // synthesised pass: the tile of a basis state, written in the layout the TMA load would leave (128-byte swizzle)
  if (synth) {
    src << "QIP_DEV void synth_fill(unsigned char* sm, const unsigned tid, const JP& p, const u64 base) {\n";
    src << "  const u64 idx = ((u64)p.init_hi << 32) | (u64)p.init_lo;\n";
    src << "  u64 rest = idx & ~((1ull << TILE_L) - 1ull);\n  unsigned t = (unsigned)(idx & ((1ull << TILE_L) - 1ull));\n";
    src << "  for (unsigned i = 0; i < TILE_M; ++i) {\n    const u64 b = 1ull << p.hi_pos[i];\n";
    src << "    if (idx & b) t |= 1u << (TILE_L + i);\n    rest &= ~b;\n  }\n";
    src << (f64 ? "  t ^= (t >> 3) & 7u;\n" : "  t ^= ((t >> 4) & 7u) << 1;\n");
    src << "  const unsigned hit = rest == base ? t * (unsigned)sizeof(QV) : 0xffffffffu;  // byte offset of the one\n";
    src << "#pragma unroll 8\n  for (unsigned o = tid * 16u; o < TILE_BYTES; o += CTA_THREADS * 16u) {\n";
    src << "    QZ v;\n    v.x = v.y = v.z = v.w = 0u;\n";
    if (f64)
      src << "    if (o == hit) v.y = 0x3ff00000u;  // 1.0 + 0i\n";
    else
      src << "    if (o == (hit & ~15u)) {  // 1.0f + 0i\n      if (hit & 8u) v.z = 0x3f800000u;\n      else v.x = 0x3f800000u;\n    }\n";
    src << "    *reinterpret_cast<QZ*>(sm + o) = v;\n  }\n}\n\n";
  }

  // ---- host harness (validation without a GPU) ----
  src << "#ifdef QIP_JIT_HOST\n";
  src << "extern \"C\" void qip_host_pass(R* psi, const JP* pp, unsigned n_local) {\n  const JP& p = *pp;\n";
  src << "  static unsigned char sm[OFF_MBAR + 64];\n  const u64 tiles = 1ull << (n_local - TILE_T);\n";
  src << "  for (u64 tile = 0; tile < tiles; ++tile) {\n    const u64 base = tile_base(p, tile);\n";
  if (synth) {
    src << "    for (unsigned tid = 0; tid < " << kThreads << "u; ++tid) synth_fill(sm, tid, p, base);\n";
  } else {
    src << "    for (unsigned t = 0; t < (1u << TILE_T); ++t) {\n      u64 idx = base + (t & ((1u << TILE_L) - 1u));\n";
    src << "      for (unsigned i = 0; i < TILE_M; ++i) if ((t >> (TILE_L + i)) & 1u) idx |= 1ull << p.hi_pos[i];\n";
    src << (f64 ? "      const unsigned s = t ^ ((t >> 3) & 7u);\n" : "      const unsigned s = t ^ (((t >> 4) & 7u) << 1);\n");
    src << "      memcpy(sm + s * sizeof(QV), psi + 2 * idx, sizeof(QV));\n    }\n";
  }
  src << "    memset(sm + OFF_CONDW, 0, 48);\n";
  src << "    for (unsigned tid = 0; tid < " << kThreads << "u; ++tid) prelude(sm, tid, p, base);\n";
  for (size_t s = 0; s < S; ++s)
    src << "    for (unsigned tid = 0; tid < " << kThreads << "u; ++tid) so_" << s
        << "(sm, tid, p, reinterpret_cast<const unsigned*>(sm + OFF_CONDW), reinterpret_cast<const R*>(sm + OFF_TBL), "
           "reinterpret_cast<const R*>(sm + OFF_GT));\n";
  src << "    for (unsigned t = 0; t < (1u << TILE_T); ++t) {\n      u64 idx = base + (t & ((1u << TILE_L) - 1u));\n";
  src << "      for (unsigned i = 0; i < TILE_M; ++i) if ((t >> (TILE_L + i)) & 1u) idx |= 1ull << p.hi_pos[i];\n";
  src << (f64 ? "      const unsigned s = t ^ ((t >> 3) & 7u);\n" : "      const unsigned s = t ^ (((t >> 4) & 7u) << 1);\n");
  src << "      memcpy(psi + 2 * idx, sm + s * sizeof(QV), sizeof(QV));\n    }\n  }\n}\n";
  src << "#else\n";

  // ---- device kernel ----
  src << R"(struct alignas(64) CUtensorMap { u64 opaque[16]; };
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
  unsigned done;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void box_coords(const JP& p, u64 idx, int* c) {
  const unsigned h1 = p.hi_pos[0], h2 = p.hi_pos[1], h3 = p.hi_pos[2];
  c[0] = (int)((idx >> LOW3) & ((1ull << (h1 - LOW3)) - 1ull));
  c[1] = (int)((idx >> h1) & ((1ull << (h2 - h1)) - 1ull));
  c[2] = (int)((idx >> h2) & ((1ull << (h3 - h2)) - 1ull));
  c[3] = (int)(idx >> h3);
}
extern "C" __global__ void __launch_bounds__(CTA_THREADS, CTAS_PER_SM)
qip_pass(R* __restrict__ psi, const __grid_constant__ JP p, const __grid_constant__ CUtensorMap tmap,
         const __grid_constant__ CUtensorMap tmap_out) {
  extern __shared__ __align__(1024) unsigned char sm[];
  const unsigned tid = threadIdx.x;
  const unsigned smb = (unsigned)__cvta_generic_to_shared(sm);
  const unsigned mbar = smb + OFF_MBAR;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const u64 tile_off = ((u64)p.tile_off_hi << 32) | (u64)p.tile_off_lo, tile_cnt = ((u64)p.tile_cnt_hi << 32) | (u64)p.tile_cnt_lo;
  unsigned parity = 0u;
#if QIP_PAIRED
  const u64 pair_my = ((u64)p.pair_my_hi << 32) | (u64)p.pair_my_lo;
#endif
#pragma unroll 1
  for (u64 tile = blockIdx.x; tile < tile_cnt; tile += gridDim.x, parity ^= 1u) {
#if QIP_PAIRED
  // paired send: walk the tile counter with its bits 0 and pair_cbit exchanged, so that tiles this rank keeps and tiles it
  // gives away alternate (HBM and NVLink traffic overlap) and both ranks reach a pair of tiles at about the same time
  u64 tpos = tile;
  if (pair_my != 0ull && p.pair_cbit != 0u) {
    const u64 b0 = tpos & 1ull, bc = (tpos >> p.pair_cbit) & 1ull;
    tpos = (tpos & ~(1ull | (1ull << p.pair_cbit))) | bc | (b0 << p.pair_cbit);
  }
  const u64 tt = tpos + tile_off;
#else
  const u64 tt = tile + tile_off;
#endif
  const u64 base = tile_base(p, tt);
#if QIP_SYNTH
  if (tile != (u64)blockIdx.x) __syncthreads();  // the previous tile's stores have read the buffer (thread 0 waited)
  synth_fill(sm, tid, p, base);
#else
  if (tid == 0) {  // the tile buffer is free: this thread waited for the previous tile's stores to have read it
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(TILE_BYTES) : "memory");
#pragma unroll 1
    for (unsigned b = 0; b < NBOX; ++b) {
      int c[4];
      box_coords(p, base + p.box_off[b], c);
      asm volatile(
          "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
              smb + b * BOX_BYTES),
          "l"(&tmap), "r"(mbar), "r"(0), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3])
          : "memory");
    }
  }
  if (p.prefetch_dist && tid == 32u && tile + p.prefetch_dist < tile_cnt) {
    const u64 nbase = tile_base(p, tile + p.prefetch_dist + tile_off);
#pragma unroll 1
    for (unsigned b = 0; b < NBOX; ++b) {
      int c[4];
      box_coords(p, nbase + p.box_off[b], c);
      asm volatile("cp.async.bulk.prefetch.tensor.5d.L2.global [%0, {%1, %2, %3, %4, %5}];" ::"l"(&tmap), "r"(0), "r"(c[0]), "r"(c[1]),
                   "r"(c[2]), "r"(c[3])
                   : "memory");
    }
  }
#endif
)";
  src << "  prelude(sm, tid, p, base);\n";
  // (always needed with persistent CTAs: the previous tile's super-ops read what the prelude overwrites -- they are
  // all past the barrier before the stores -- and the prelude's results must be visible before the super-ops)
  // (a synthesised tile is written by all threads: it must be complete before the super-ops)
  if (has_prelude || synth) src << "  __syncthreads();\n";
  src << "  const unsigned* condw = reinterpret_cast<const unsigned*>(sm + OFF_CONDW);\n";
  src << "  const R* tbl = reinterpret_cast<const R*>(sm + OFF_TBL);\n  const R* gt = reinterpret_cast<const R*>(sm + OFF_GT);\n";
  if (!synth) src << "  mbar_wait(mbar, parity);\n";
  src << R"(#if QIP_PAIRED
  const bool pair_give = pair_my != 0ull && ((tt >> p.pair_cbit) & 1ull) == (u64)p.send_val;
  if (pair_give && tid == 0) {  // my copy of the tile is in shared memory: the partner may overwrite the slot
    const u64 peer_flags = ((u64)p.pair_peer_hi << 32) | (u64)p.pair_peer_lo;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_flags + 4ull * (tt ^ (1ull << p.pair_cbit))),
                 "r"(p.pair_seq)
                 : "memory");
  }
#endif
)";
  uint32_t n_bar = 0, n_ws = 0;
  for (size_t s = 0; s < S; ++s) {
    if (s) {
      if (cta_barrier_before[s]) {
        src << "  __syncthreads();\n";
        ++n_bar;
      } else {
        src << "  __syncwarp();\n";
        ++n_ws;
      }
    }
    src << "  so_" << s << "(sm, tid, p, condw, tbl, gt);\n";
  }
  src << R"(  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (tid == 0) {
#if QIP_PAIRED
    if (pair_give) {  // wait for the partner's copy of the tile this one replaces
      unsigned v;
      unsigned long long t0, t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      for (;;) {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(pair_my + 4ull * tt) : "memory");
        if ((int)(v - p.pair_seq) >= 0) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        volatile unsigned* errw = reinterpret_cast<volatile unsigned*>(((u64)p.pair_err_hi << 32) | (u64)p.pair_err_lo);
        if (t1 - t0 > 20000000000ull || *errw != 0u) {  // 20 s: the partner is gone (later tiles give up at once)
          *errw = 1u;
          break;
        }
      }
    }
#endif
#pragma unroll 1
    for (unsigned b = 0; b < NBOX; ++b) {
      int c[4];
      u64 idx = base + p.box_off[b];
      const CUtensorMap* tm = &tmap;
      if (p.send_bit < 64u && ((idx >> p.send_bit) & 1ull) == (u64)p.send_val) {
        tm = &tmap_out;
        idx ^= 1ull << p.send_bit;
      }
      box_coords(p, idx, c);
      asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(tm),
                   "r"(smb + b * BOX_BYTES), "r"(0), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3])
                   : "memory");
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    if (p.send_bit < 64u && ((base >> p.send_bit) & 1ull) == (u64)p.send_val)  // (bit send_bit is constant within a tile)
      asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores to the partner: wait until they are performed
    else
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
  }  // tile loop
  (void)psi;
}
#endif
)";

  // ---- the JP blob, in declaration order ----
  std::vector<unsigned char> blob;
  auto put = [&](const void *ptr, size_t n) {
    const unsigned char *b = static_cast<const unsigned char *>(ptr);
    blob.insert(blob.end(), b, b + n);
  };
  auto put_real = [&](double v) {
    if (f64) put(&v, 8);
    else {
      const float f = (float)v;
      put(&f, 4);
    }
  };
  for (uint32_t b = 0; b < NBOX; ++b) put(&h.chunk_off[b << 3], 8);
  for (size_t i = 0; i < NC; ++i) put(&conds[i].gmask, 8);
  for (size_t i = 0; i < NC; ++i) put(&conds[i].gval, 8);
  for (size_t i = 0; i < NPH; ++i)
    for (size_t k = 0; k < phn_terms[i].size(); ++k) put(&phn_terms[i][k].gmask, 8);
  for (size_t i = 0; i < NPH; ++i)
    for (size_t k = 0; k < phn_terms[i].size(); ++k) put(&phn_terms[i][k].gval, 8);
  std::vector<double> gre(NG), gim(NG);
  {
    std::vector<uint64_t> gm(NG), gv(NG);
    for (size_t i = 0; i < NG; ++i) {
      if (f64) {
        GlobalTerm<double> t;
        memcpy(&t, pass.gterms.data() + i * gsz, gsz);
        gm[i] = t.gmask, gv[i] = t.gval, gre[i] = t.re, gim[i] = t.im;
      } else {
        GlobalTerm<float> t;
        memcpy(&t, pass.gterms.data() + i * gsz, gsz);
        gm[i] = t.gmask, gv[i] = t.gval, gre[i] = t.re, gim[i] = t.im;
      }
    }
    for (size_t i = 0; i < NG; ++i) put(&gm[i], 8);
    for (size_t i = 0; i < NG; ++i) put(&gv[i], 8);
  }
  for (size_t i = 0; i < NK; ++i) put_real(g.pool[i]);
  for (size_t i = 0; i < NPH; ++i)
    for (size_t k = 0; k < phn_terms[i].size(); ++k) {
      put_real(phn_terms[i][k].re);
      put_real(phn_terms[i][k].im);
    }
  for (size_t i = 0; i < NPH; ++i) {
    put_real(phn_base[i].first);
    put_real(phn_base[i].second);
  }
  for (size_t i = 0; i < NG; ++i) {
    put_real(gre[i]);
    put_real(gim[i]);
  }
  for (uint32_t i = 0; i < 8; ++i) put(&h.hi_pos[i], 4);
  if (NPH) {
    uint32_t at = 0;
    for (size_t i = 0; i < NPH; ++i) {
      put(&at, 4);
      at += (uint32_t)phn_terms[i].size();
    }
    put(&at, 4);
  }
  if (synth) {
    const uint32_t w[2] = {(uint32_t)*synth_index, (uint32_t)(*synth_index >> 32)};
    put(w, 8);
  }
  out->send_offset = (uint32_t)blob.size();
  {
    const uint32_t off_bit = 64u, val = 0u;
    put(&off_bit, 4);
    put(&val, 4);
    put(&val, 4);  // tile_off_lo
    put(&val, 4);  // tile_off_hi
    put(&val, 4);  // tile_cnt_lo (set per launch)
    put(&val, 4);  // tile_cnt_hi
    put(&val, 4);  // prefetch_dist (set per launch)
    put(&val, 4);  // pad_
    for (int i = 0; i < 8; ++i) put(&val, 4);  // pair_* (set per launch)
  }
  while (blob.size() % 8) blob.push_back(0);  // sizeof(JP): the struct is 8-byte aligned

  out->source = src.str();
  out->params.swap(blob);
  out->synthesised = synth;
  out->smem_bytes = off_mbar + 64;
  out->threads = kThreads;
  out->tiles_log2_sub = T;
  out->n_super = (uint32_t)S;
  out->n_elems = n_elems;
  out->n_cta_barriers = n_bar;
  out->n_warp_syncs = n_ws;
  out->n_renamed = g.renamed;
  out->n_consts = (uint32_t)NK;
  return true;
}

}  // namespace qipb200
