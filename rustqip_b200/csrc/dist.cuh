// dist.cuh -- launch interface of the NVLink pair-exchange kernels (see dist.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/qipb200.h"

namespace qipb200 {

static const int kMaxWorld = 16;
static const int kFlagErrorSlot = 32;   // flags[kFlagErrorSlot] != 0 => a barrier timed out
static const int kFlagWords = 64;
// The flag page is followed, in the same (peer-mapped) allocation, by one reduction slot of kCommDoubles doubles:
// small cross-rank sums (measurement histograms, norms, sampling prefixes) are exchanged through it.
static const int kCommDoubles = 1 << 16;
static const size_t kCommOffsetBytes = 256;
// ... and by one 32-bit flag per tile of a fused pass (up to 2^22 tiles): the per-tile handshake of a migration that is
// fused into a tile pass (paired send: "my copy of this tile is in shared memory, you may overwrite it").
static const size_t kPairFlagOffsetBytes = kCommOffsetBytes + (size_t)kCommDoubles * sizeof(double);
static const uint32_t kPairFlagLog2 = 22;
static const size_t kFlagAllocBytes = kPairFlagOffsetBytes + (sizeof(uint32_t) << kPairFlagLog2);

// Trade the half-shard selected by local bit `l` with the partner's (see dist.cu).
// rb = this rank's value of the rank bit being migrated; s_bit = pair-ownership bit.
cudaError_t launch_pair_exchange(qip_prec prec, void *mine, void *peer, uint32_t n_local, uint32_t l,
                                 uint32_t s_bit, int rb, cudaStream_t s, uint64_t *launches);

// The protocol of a migration fused into a tile pass (jit_codegen.cpp: pair_*), played by a stand-alone kernel for a
// rank whose last pass could not do it itself: every tile of the half this rank gives away is read, announced to the
// partner ("loaded": partner's flag word of the paired tile := seq), and written into the partner's shard at the index
// with bit l flipped once the partner has announced its own tile.  Tile geometry = the pass header's.
struct PairedSendArgs {
  void *mine, *peer;
  uint32_t *my_flags, *peer_flags, *error_word;
  uint32_t seq, n_local, T, L, m, l, cbit, give;
  uint32_t hi_pos[8];
};
cudaError_t launch_paired_send(qip_prec prec, const PairedSendArgs &a, cudaStream_t s, uint64_t *launches);

// All-rank barrier through peer-mapped flag pages; stream-ordered.
cudaError_t launch_flag_barrier(uint32_t *const *peer_flags, uint32_t *my_flags, int rank, int world,
                                uint32_t epoch, uint32_t *error_word, cudaStream_t s, uint64_t *launches);

// out[i] = sum over ranks t (ascending: the same order, hence the same bits, on every rank) of comm_t[i], where
// comm_t is rank t's reduction slot read over NVLink.  The caller brackets it with flag barriers.
cudaError_t launch_comm_sum(const double *const *peer_comm, int world, double *out, uint32_t count, cudaStream_t s,
                            uint64_t *launches);

}  // namespace qipb200
