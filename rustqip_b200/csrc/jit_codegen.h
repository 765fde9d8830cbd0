// jit_codegen.h -- per-pass specialised tile kernels: source generator (pure host C++, no CUDA).
//
// The generic tile kernel (tile_kernel.cu) INTERPRETS a pass: per elementary op it loads a descriptor word,
// walks a compare chain and loads the gate constants.  Here the planner's pass is turned into straight-line CUDA C++ instead:
// one kernel per pass STRUCTURE (which sub-bits, which op shapes, which constants are exactly 0 / +-1), with the
// numeric gate constants, the tile geometry and the CTA-uniform conditions passed as kernel parameters (constant
// bank operands of the FP64 instructions).  No dispatch, no descriptor loads; X / CNOT / SWAP inside a group
// become register renaming (zero instructions, bit-exact); thread->amplitude maps are chosen per super-op so that
// consecutive super-ops whose bits leave three common tile bits free need a __syncwarp, not a CTA barrier.
//
// The generated source also compiles for the HOST (-DQIP_JIT_HOST): tests/test_jit_cpu.py runs it through g++
// against the oracle, so the generator is validated without a GPU.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "tile.cuh"

namespace qipb200 {

struct JitProgram {
  std::string source;                 // CUDA C++ (entry point `qip_pass`), also host-compilable
  std::vector<unsigned char> params;  // the JP parameter block the source declares
  uint32_t smem_bytes = 0;            // dynamic shared memory of one CTA
  uint32_t threads = 256;
  uint32_t tiles_log2_sub = 0;        // grid = 1 << (n_local - T)
  uint32_t send_offset = 0;           // byte offset of JP::send_bit / send_val in `params` (patched per launch)
  bool synthesised = false;           // the pass builds its tiles from a basis index instead of loading them
  // statistics
  uint32_t n_super = 0, n_elems = 0, n_cta_barriers = 0, n_warp_syncs = 0, n_renamed = 0, n_consts = 0;
};

// Returns false (and says why) when the pass holds something the generator does not cover (wide micro-ops,
// geometry without TMA boxes, > 256 CTA-uniform conditions ...): the caller then runs the interpreter kernel.
// `paired`: the kernel can also play the per-tile handshake of a migration fused into the pass (multi-GPU, JP::pair_*).
// `synth_index`: the pass is the first one on a state that is still the basis state |*synth_index> (unsharded): every
// CTA fills its shared-memory tile with zeros and, in the tile that holds the index, a one, instead of loading the tile.
bool jit_generate(const HostPass &pass, qip_prec prec, JitProgram *out, std::string *why, bool paired = false,
                  const uint64_t *synth_index = nullptr);

}  // namespace qipb200
