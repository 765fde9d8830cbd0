// schedule.h -- the gate schedule executor (the fold of builder.rs:423-514).
#pragma once

#include <cstddef>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "opcompile.h"
#include "state.h"
#include "tile.cuh"

namespace qipb200 {

// api.cu
int apply_flat_local(qipb200_state *s, const FlatOp &f);
int restrict_to_rank(const qipb200_state *s, const FlatOp &f_in, FlatOp *out, bool *skip);
int restrict_to_rank_as(const qipb200_state *s, int rank, const FlatOp &f_in, FlatOp *out, bool *skip);
int launch_local_op(qipb200_state *s, const FlatOp &f);
int report_error(qipb200_state *s, int status, const std::string &msg);
int report_cuda_error(qipb200_state *s, cudaError_t e, const char *what);
int compile_and_localize(qipb200_state *s, const qip_op *op, FlatOp *f, const uint64_t *next_use);
bool peek_first_exchange(const qipb200_state *s, const qip_op *op, const uint64_t *next_use, uint32_t *R, uint32_t *l);
// migration fused into the epoch's last tile pass, in place (paired send): who the partner is / what is left to do after
// the pass (or its stand-in kernel) ran: the closing barrier and the bit-map update
void paired_partner(const qipb200_state *s, uint32_t R, int *partner, int *give);
int paired_send_standin(qipb200_state *s, uint32_t R, uint32_t l, uint32_t cbit, uint32_t seq, const PassHeader &hdr);
int finish_paired_exchange(qipb200_state *s, uint32_t R, uint32_t l);
// write the basis state qipb200_state_set_basis left pending (no-op when there is none)
int materialise_init(qipb200_state *s);

// qubit rotation (opt-in, QIPB200_ROTATE=1, unsharded states; planner.cpp: plan_rotating): is it on / run swap-only steps
// that bring the state's layout back to the canonical one (api.cu: restore_layout)
bool rotate_enabled();
int restore_layout_planned(qipb200_state *s);

// schedule.cu: state <- ops[n-1] ... ops[0] state
int run_schedule(qipb200_state *s, const qip_op *ops, size_t n_ops, uint32_t flags);

}  // namespace qipb200
