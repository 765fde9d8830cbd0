// tile.cuh -- fused shared-memory tile pass: data structures shared by the host
// planner (planner.cpp) and the kernel (tile_kernel.cu).
//
// One PASS sweeps the state once: every CTA loads a TILE of 2^T amplitudes (the L
// lowest index bits, contiguous in HBM, plus m = T-L arbitrary higher "tile bits")
// into shared memory, applies a list of MICRO-OPS there, and writes the tile back.
// Any gate whose non-diagonal target bits are tile bits can run inside the pass;
// control bits and diagonal gates may sit on ANY bit (a non-tile bit is a CTA-uniform
// predicate).  Algorithmic HBM traffic of a pass = 2 * 2^n * sizeof(amplitude), the
// same as ONE gate of the reference's per-entry loop (qip/src/builder.rs:423-514).
//
// The work-horse micro-op is MK_SUPER: a set of 3 tile-local bits and a LIST of
// elementary ops on them.  A thread pulls the 8 amplitudes of one group into
// registers, runs the whole list there (2x2 gates, X, phases, bit swaps, optional
// CTA-uniform conditions for controls that live outside the tile) and writes the
// group back: one shared-memory round trip for many gates.  All descriptors travel
// as a __grid_constant__ kernel parameter, i.e. are read through the constant bank,
// not through the shared-memory pipe that carries the amplitudes.
#pragma once

#include <cstdint>
#include <vector>

#include "opcompile.h"

namespace qipb200 {

static const uint32_t kTileMaxHigh = 8;       // m <= 8 -> 256 chunk offsets
static const uint32_t kMaxPassBytes = 27 * 1024;  // micro-op records per pass (kernel parameter space)
static const uint32_t kMaxDiagTerms = 24;     // per MK_DIAG micro-op
static const uint32_t kMaxGlobalTerms = 32;   // CTA-uniform phase terms applied at store time
static const uint32_t kMaxPhasen = 256;       // EC_PHASEN ops per pass (4 KiB factor table in shared memory)

enum MicroKind { MK_DENSE = 0, MK_DIAG = 1, MK_EXCH = 2, MK_SUPER = 3 };
// Elementary-op kinds of a MK_SUPER group.  Real and complex 2x2 gates are separate kinds
// (a real matrix -- H, Ry, X-like -- needs half the FMAs).
// SWAP exists on the host side only: the planner lowers it to three controlled X.  X is a pair
// exchange done with register moves (bit-exact, no FP64 work).
enum ElemType { E_DENSE1 = 0, E_DENSE1R = 1, E_X = 2, E_PHASE = 3, E_SWAP = 4, E_DENSE3 = 5 };

// Elem::op layout (host-precomputed so the kernel's dispatch is one jump on the case id):
//   bits 0-5   interpreter case id: 0 END (sentinel after the last op of a super-op),
//              1-3 real 2x2 on sub-bit 0/1/2 with every pair active, 4-6 complex ditto,
//              7-9 real 2x2 masked (generic), 10-12 complex 2x2 masked, 13 PHASE (generic mask), 14 dense 8x8,
//              15-17 X (pair exchange by register moves) every pair active, 18-20 X masked,
//              21 PHASEN: one phase mask, base factor m[0..1] times the product of the CTA-uniform
//                 conditional factors listed after the record (slot of the per-CTA table in Elem::pad) -- a run of
//                 controlled phases whose controls lie outside the tile costs one application
//              22-24 PHASE on every amplitude with sub-bit j set (T, S, Rz ... : straight-line, no mask tests)
//              25-30 real 2x2 on sub-bit j under ONE control inside the group (CNOT, CRy): 25 + 2*j + w, w = 0/1:
//                 the control is the lower/higher of the two other sub-bits
//              31-33 real 2x2 on sub-bit j under BOTH other sub-bits (Toffoli)
//              34-36 PHASE on the amplitudes with two sub-bits set (CZ, controlled phase): (0,1), (0,2), (1,2)
//              37-39 UN-NORMALISED Hadamard butterfly on sub-bit j (x+y, x-y: half the FP64 work of a real 2x2);
//                 the planner folds the pending 1/sqrt(2)^k -- a global scalar, it commutes with everything --
//                 into a later full 2x2 of the same pass
//   bits 6-11  slot of the op's CTA-uniform condition in the pass's condition table (kCondOverflow: test
//              the record's own gmask/gval)
//   bits 12-19 active mask: 2x2 kinds: bit p <-> the p-th (ascending) sub-index with bit j
//              clear; PHASE: bit c <-> sub-index c
//   bits 20-30 record size in 16-byte units (the dense 8x8 matrix follows its record)
//   bit 31     the op has a CTA-uniform condition
static const uint32_t kElemHasCond = 1u << 31;
static const uint32_t kElemCaseMask = 0x3fu;
static const uint32_t kElemCondShift = 6;
static const uint32_t kCondOverflow = 63;  // slots 0..62 index the pass's condition table
enum ElemCase { EC_END = 0, EC_D1R_FULL = 1, EC_D1C_FULL = 4, EC_D1R_MASK = 7, EC_D1C_MASK = 10, EC_PHASE = 13, EC_DENSE3 = 14,
                EC_X_FULL = 15, EC_X_MASK = 18, EC_PHASEN = 21, EC_PHASE_J = 22, EC_D1R_C1 = 25, EC_D1R_C2 = 31,
                EC_PHASE_2 = 34, EC_HAD = 37, EC_N_CASES = 40 };
// pair mask of "the w-th other sub-bit is set" / "both other sub-bits set"; phase masks of the special cases
static const uint32_t kPairMaskC1[2] = {0xAu, 0xCu};
static const uint32_t kPairMaskC2 = 0x8u;
static const uint32_t kPhaseMaskJ[3] = {0xAAu, 0xCCu, 0xF0u};
static const uint32_t kPhaseMask2[3] = {0x88u, 0xA0u, 0xC0u};
inline uint32_t elem_op(uint32_t kind, uint32_t j, uint32_t mask, bool cond, uint32_t size_bytes) {
  uint32_t id;
  if (kind == E_DENSE1R) {
    if (mask == 0xfu) id = EC_D1R_FULL + j;
    else if (mask == kPairMaskC1[0]) id = EC_D1R_C1 + 2 * j;
    else if (mask == kPairMaskC1[1]) id = EC_D1R_C1 + 2 * j + 1;
    else if (mask == kPairMaskC2) id = EC_D1R_C2 + j;
    else id = EC_D1R_MASK + j;
  } else if (kind == E_DENSE1)
    id = (mask == 0xfu ? EC_D1C_FULL : EC_D1C_MASK) + j;
  else if (kind == E_X)
    id = (mask == 0xfu ? EC_X_FULL : EC_X_MASK) + j;
  else if (kind == E_PHASE) {
    id = EC_PHASE;
    for (uint32_t q = 0; q < 3; ++q) {
      if (mask == kPhaseMaskJ[q]) id = EC_PHASE_J + q;
      if (mask == kPhaseMask2[q]) id = EC_PHASE_2 + q;
    }
  } else
    id = EC_DENSE3;
  return id | (mask << 12) | ((size_bytes >> 4) << 20) | (cond ? kElemHasCond : 0u);
}
inline uint32_t elem_case(uint32_t op) { return op & kElemCaseMask; }
inline uint32_t elem_cond_slot(uint32_t op) { return (op >> kElemCondShift) & 63u; }
inline uint32_t elem_op_phasen(uint32_t mask, uint32_t size_bytes) { return EC_PHASEN | (mask << 12) | ((size_bytes >> 4) << 20); }
inline uint32_t elem_size_bytes(uint32_t op) { return ((op >> 20) & 0x7ffu) << 4; }

// Device-visible micro-op header (fixed 160 bytes), followed by its data:
//   MK_DENSE: 2^k x 2^k complex<R> (re,im interleaved), sub-index bit i <-> ins_pos order of targets
//   MK_DIAG : nterms x DiagTerm<R>
//   MK_SUPER: nterms elementary records (Elem<R>, dense 8x8 ones followed by 64 complex<R>) + END record
struct alignas(16) MicroOp {
  uint32_t kind;
  uint32_t k;            // dense: number of target bits (1..3); super: 3
  uint32_t ins_n;        // number of tile-local positions removed from the group counter
  uint32_t ins_pos[6];   // ascending tile-local positions (targets and local controls)
  uint32_t lor_mask;     // tile-local control bits (forced to 1)
  uint32_t off[8];       // dense/super: tile-local offset of sub-index u; exch: off[0] <-> off[1]
  uint32_t groups_log2;  // T - ins_n
  uint32_t nterms;       // diag terms / super elems
  uint32_t data_bytes;   // bytes of data following the header
  uint32_t pad0;
  uint64_t gmask;        // control bits outside the tile: tested against the tile's base index
  uint64_t pad1[3];
  uint32_t soff[8];      // super: SWIZZLED shared-memory BYTE offset of sub-index u (the XOR swizzle is GF(2)-linear,
                         // so address(t0 + off[u]) = tile + (swz_bytes(t0) ^ soff[u]))
};
static_assert(sizeof(MicroOp) == 160, "MicroOp must be 160 bytes");

template <typename R>
struct alignas(16) DiagTerm {  // multiply by (re,im) where (global & gmask)==gval and (local & lmask)==lval
  uint64_t gmask, gval;
  uint32_t lmask, lval;
  R re, im;
};

// Elementary op of a MK_SUPER group, in SUB-INDEX coordinates (bit i of the sub-index
// <-> ins_pos[i] of the enclosing micro-op).  E_DENSE3 records are followed by 64 complex<R>.
template <typename R>
struct alignas(16) Elem {
  uint32_t op;           // see elem_op()
  uint32_t pad;          // EC_PHASEN: slot of this op in the per-CTA factor table (terms follow the record)
  uint64_t gmask, gval;  // CTA-uniform condition on the tile's base index (read only if kElemHasCond)
  uint64_t pad2;
  R m[8];                // DENSE1: m00,m01,m10,m11 (re,im); DENSE1R: m00,m01,m10,m11 (re); PHASE: w (re,im)
};

template <typename R>
struct alignas(16) PhaseTerm {  // conditional factor of an EC_PHASEN record
  uint64_t gmask, gval;
  R re, im;
};

struct CondTerm {  // entry of a pass's condition table: (base & gmask) == gval, evaluated once per CTA
  uint64_t gmask, gval;
};

template <typename R>
struct GlobalTerm {  // multiply the whole tile by (re,im) where (base & gmask) == gval
  uint64_t gmask, gval;
  R re, im;
};

struct PassHeader {
  uint32_t T, L, m, n_ops;
  uint32_t hi_pos[kTileMaxHigh];           // the m high tile bit positions, ascending
  uint64_t chunk_off[1u << kTileMaxHigh];  // amplitude offset of chunk c (bits of c spread over hi_pos)
  uint32_t blob_bytes;                     // bytes of micro-op records
  uint32_t n_gterms;                       // GlobalTerm records at the very end of the blob
  uint32_t gterm_off;                      // byte offset of the GlobalTerm array inside the blob
  uint32_t n_phasen;                       // EC_PHASEN ops in this pass (slots of the per-CTA factor table)
  uint32_t use_tma;                        // set by the launcher: tile moved by TMA tensor copies
  uint32_t n_conds;                        // CondTerm records (<= kCondOverflow) at cond_off inside the blob
  uint32_t cond_off;
  uint32_t pad_[1];
};

// What the kernel receives by value (constant bank).  16-byte aligned so that the records
// (16-byte aligned relative to `recs`) keep their alignment in parameter space.
struct alignas(16) PassParams {
  PassHeader h;
  unsigned char recs[kMaxPassBytes];
};
static_assert(sizeof(PassParams) <= 32000, "kernel parameter space");
static_assert(sizeof(PassHeader) % 16 == 0, "records must start 16-byte aligned");

// ---- host side ---------------------------------------------------------------------
struct HostMicroOp {
  MicroOp h;
  std::vector<unsigned char> data;
};

// ---- the same pass for the GENERATED kernels (jit_codegen.cpp): groups of up to `jbits` tile-local bits ----
// The interpreter's records are tied to 3-bit groups (8 amplitudes, 8-bit masks); a generated kernel can keep
// 2^4 (f64) or 2^5 (f32) amplitudes of a group in registers, and every bit more per group means fewer shared-memory
// round trips per pass (2 x 64 KiB through shared memory per super-op and tile).  Elementary ops are given in SUB-INDEX coordinates: bit i of the sub-index <-> bits[i].
struct JCondPhase {
  uint64_t gmask, gval;
  cplx w;
};
struct JElem {
  enum Kind { D1 = 0, X = 1, PH = 2, DK = 3, HAD = 4 } kind = D1;
  uint32_t j = 0;                 // D1 / X / HAD: target sub-bit
  uint32_t lc = 0;                // D1 / X: control sub-mask (the op acts on pairs whose other bits contain lc)
  uint32_t lm = 0, lv = 0;        // PH: acts on sub-indices c with (c & lm) == lv
  uint32_t pm = 0, pv = 0;        // PH: ... in the groups whose TILE-LOCAL index t satisfies (t & pm) == pv: a diagonal op
                                  //     needs none of its bits in registers, a bit outside the group is a per-thread predicate
  uint64_t gmask = 0, gval = 0;   // CTA-uniform condition on the tile's base index (gmask == 0: none)
  cplx m[4];                      // D1: m00 m01 m10 m11; PH: factor in m[0]
  std::vector<JCondPhase> terms;  // PH: further factors, each under its own CTA-uniform condition
  // PH: further factors, each under its own THREAD predicate on the tile-local index ((t & pm) == pv): a run of phases
  // on the same amplitudes of the group that differ only in bits outside the group (QFT: the controlled phases of one
  // target) costs one scalar product per thread and ONE application (jit_codegen forms the product in registers)
  struct ThreadTerm {
    uint32_t pm, pv;
    cplx w;
  };
  std::vector<ThreadTerm> tterms;
  std::vector<uint32_t> mb;       // DK: the sub-bits the dense block acts on (ascending, <= 3)
  std::vector<cplx> mk;           // DK: 2^k x 2^k, row-major, bit i of the row index <-> mb[i]
};
struct JGroup {
  std::vector<uint32_t> bits;  // ascending tile-local bits, exactly jbits of them (padded)
  std::vector<JElem> elems;
};

struct HostPass {
  PassHeader hdr{};
  std::vector<JGroup> jgroups;  // generated-kernel view of the pass (empty: not produced)
  uint32_t jbits = 0;
  std::vector<HostMicroOp> ops;
  std::vector<unsigned char> gterms;  // GlobalTerm<R> records
  std::vector<CondTerm> conds;        // distinct CTA-uniform conditions of the pass's elementary ops
  uint32_t n_gates = 0;               // reference ops folded into this pass
};

// One step of a planned schedule: either a fused pass or a single op run by the
// per-gate kernels (index into the original op list).
struct PlanStep {
  bool is_pass = false;
  HostPass pass;
  size_t op_index = 0;
};

struct PlanConfig {
  uint32_t T = 12;        // tile bits
  uint32_t L = 5;         // contiguous low bits
  bool fuse_blocks = true;      // group ops into 3-bit register-resident super-ops
  bool peephole = true;         // fold consecutive ops on the same target bit into one 2x2
  bool fold_cond_phases = true; // fold phases that differ only in their CTA-uniform condition into one EC_PHASEN op
  bool use_tma = true;          // move tiles with TMA (cp.async.bulk.tensor, 128B-swizzle tensor map) when the geometry allows
  bool x_as_moves = false;      // X inside a tile as register moves (exact for non-finite amplitudes too) instead of the
                                // exact-for-finite 0/1 real 2x2; moves cost more issue slots, the FP64 pipe has slack
  bool fill_on_flush = true;    // a super-op leaving with spare bits takes small open groups along
  bool lookback = true;         // peephole: look back past commuting ops for a fold partner; drop ops that cancel
  bool keep_real = false;       // peephole: do not fold a non-real phase into a real 2x2 (less FP64 work, more elementary ops;
                                // on for the generated kernels, see plan_config in planner.cpp)
  bool unnormalised_h = true;   // Hadamards as add/sub butterflies, the scale folded into another gate of the pass
  bool seed_search = false;     // tile-bit choice: also try reserving slots for bits the greedy left out (fewer passes, but
                                // more elementary ops; on for the generated kernels, see plan_config in planner.cpp)
  uint32_t lookahead = 0;       // tile-bit choice: beam width of the look-ahead search (0 = off, env QIPB200_PLAN_LOOKAHEAD): candidate
                                // bit sets are scored by the sweeps a plain greedy needs for the gates they leave behind.  CPU
                                // measurements (tests/native emulator): N=30 d40 circuits 25/23/25 -> 24/22/22 sweeps, config 2
                                // 22 -> 20, at many times the planning time: worth it only for a circuit run many
                                // times, hence opt-in
  uint32_t jit_group_bits = 0;     // > 0: also emit the pass as groups of this many bits for the generated kernels
  int groups_per_thread = 1;       // register-resident groups per interpreter decode (1: 3 CTAs/SM, 2: 2 CTAs/SM)
  uint32_t compose_threshold = 8;  // >= this many 2x2 gates in one group: compose them into one 8x8
};

// Plan `ops` (already compiled against the current layout and restricted to local bits;
// ops[i].cls == CLASS_IDENTITY entries are dropped) for a local state of n_local bits.
// `blocked` (optional, same length as ops): ops that cannot run under the current layout (their
// non-diagonal targets are held by the rank index of a sharded state).  They are never emitted;
// they and everything that does not commute past them are returned in `leftover` (program order).
// `dep` (optional): per-op (non-diagonal, diagonal) bit masks to use for the commutation analysis
// instead of the ones derived from `ops` -- on a sharded state `ops` are restricted to the rank
// (rank-held controls dropped) but the ordering must respect the unrestricted bits.
struct DepMasks {
  uint64_t nd = 0, dg = 0;
  // Optional RANK-INDEPENDENT selection data (sharded states whose ranks must choose the same tile bits for every pass:
  // migrations fused into a pass pair up tiles across GPUs).  Filled by op_uniform_info from the op as restricted to a
  // virtual rank whose rank-held bits are all 1; when present, the planner selects with these instead of anything
  // derived from `ops` (which differ from rank to rank), and uses the guaranteed byte budget only (no size-driven retry).
  bool has_uniform = false, u_tile_ok = false;
  uint64_t u_need_tile = 0;
  double u_unfused_cost = 0.0;
  uint32_t u_est_bytes = 0;
};
void op_dependency_masks(const FlatOp &f, DepMasks *out);
void op_uniform_info(const FlatOp &restricted_to_virtual_rank, DepMasks *out);
void plan_passes(const std::vector<FlatOp> &ops, uint32_t n_local, qip_prec prec, const PlanConfig &cfg,
                 std::vector<PlanStep> *steps, const std::vector<char> *blocked = nullptr,
                 std::vector<size_t> *leftover = nullptr, const std::vector<DepMasks> *dep = nullptr);

// Planning with QUBIT ROTATION (single shard, opt-in: QIPB200_ROTATE=1; DESIGN.md section 8 item 0b).  The L lowest
// index bits are in every tile, so with a fixed layout the qubits living there are in EVERY pass although a pass leaves
// its qubits blocked on partners outside the tile -- those slots mostly idle.  Here a pass may END with a permutation of
// its own tile bits (Swap elements inside register groups: pure renaming in the generated kernels), so the low
// positions of the next tile can hold ANY L qubits of the previous tile: the selection runs over logical qubits with the
// only constraint that a pass brings in at most T - L qubits from outside the previous tile.  The logical -> physical
// map is tracked, every pass is emitted from its ops compiled under the layout of the moment, and the inverse permutation
// is folded into the last pass / appended as swap-only passes: the state ends in the canonical layout and the results
// are those of the plain schedule.  Headline circuit: 19 + restore instead of 25 sweeps (all 12 tile bits free: 16).
struct RotatePlan {
  std::vector<PlanStep> steps;   // PlanStep::op_index of a single step indexes `singles`
  std::vector<FlatOp> singles;
  uint32_t n_swaps = 0, n_restore_steps = 0;
};
// `layout` (n entries, logical bit -> physical bit, or NULL = canonical): the layout the state is in; on return the
// layout it is left in.  restore = true: the plan ends in the canonical layout (inverse permutation folded into the last
// pass + swap-only passes); false: the state keeps the layout of the last pass (the API restores it lazily, like the
// migrated qubits of a sharded state: before a download, never between schedules).
int plan_rotating(const qip_op *ops, size_t n_ops, qip_prec prec, uint32_t n, const PlanConfig &cfg, RotatePlan *out,
                  std::string *err, uint32_t *layout = nullptr, bool restore = true);
// Swap-only steps that bring `layout` back to the canonical one (layout is updated to the identity).
int plan_layout_restore(qip_prec prec, uint32_t n, const PlanConfig &cfg, uint32_t *layout, RotatePlan *out, std::string *err);

// Serialise a pass: header + micro-op records + global terms.  Returns false if the
// records do not fit kMaxPassBytes (the planner bounds passes so that they do).
bool serialise_pass(const HostPass &p, PassParams *out);

// Tile geometry defaults per precision; `sharded`: the state is split over several GPUs.
PlanConfig default_plan_config(qip_prec prec, uint32_t n_local, bool sharded = false);

}  // namespace qipb200
