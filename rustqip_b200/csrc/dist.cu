// dist.cu -- multi-GPU pair exchange over NVLink peer memory.
//
// The 2^n state is sharded by its top log2(world) PHYSICAL index bits, one process
// per GPU.  A gate that acts non-diagonally on a rank bit R is made local by
// swapping R with a local bit l ("qubit migration"): rank r and its partner
// r ^ (1 << (R - n_local)) trade the half-shards selected by bit l.  The kernel
// below does the trade IN PLACE with direct loads/stores on the partner's
// CUDA-IPC-mapped buffer (P2P over NVLink / NVSwitch): every (mine[i], peer[j])
// pair is owned by exactly one of the two ranks (split by a second local bit s),
// which reads both sides and writes both sides -- no staging buffer, no
// read-old/write-new hazard.  Per rank and direction 2^(n_local-1) amplitudes cross
// the link (half pulled by me, half pushed by the partner).
//
// The paired send (QIPB200_PAIRED_SEND=1) does the trade inside the epoch's last
// tile pass instead (jit_codegen.cpp: QIP_PAIRED); k_paired_send below plays the
// same per-tile protocol for a rank whose pass could not.
//
// Cross-GPU ordering is a flag barrier in peer-visible memory (system-scope
// release/acquire), launched on the same stream before and after the trade.
#include "dist.cuh"

namespace qipb200 {

static const int kThreads = 256;

struct ExArgs {
  uint32_t pos_lo, pos_hi;  // the two removed bit positions (l and s), ascending
  uint64_t fixed;           // bits to OR in: (!rb << l) | (rb << s)
  uint64_t flip;            // 1 << l
  uint64_t n_items;
};

// U independent pairs per thread: U remote 16-byte loads in flight per lane (NVLink round trips are ~2 us; the
// link needs a few MB outstanding per direction).  Items of one thread are a CTA-stride apart, so every
// warp-instruction still covers contiguous runs.
template <typename V, int U>
__global__ void __launch_bounds__(kThreads)
    k_pair_exchange(V *__restrict__ mine, V *__restrict__ peer, const ExArgs a) {
  for (uint64_t blk = blockIdx.x; blk * (uint64_t)(kThreads * U) < a.n_items; blk += gridDim.x) {  // grid-stride over CTA chunks
  const uint64_t w0 = blk * (kThreads * U) + threadIdx.x;
  uint64_t ii[U], jj[U];
  V x[U], y[U];
  bool on[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const uint64_t w = w0 + (uint64_t)u * kThreads;
    on[u] = w < a.n_items;
    uint64_t idx = on[u] ? w : 0;
    idx = ((idx >> a.pos_lo) << (a.pos_lo + 1)) | (idx & ((1ull << a.pos_lo) - 1ull));
    idx = ((idx >> a.pos_hi) << (a.pos_hi + 1)) | (idx & ((1ull << a.pos_hi) - 1ull));
    ii[u] = idx | a.fixed;
    jj[u] = ii[u] ^ a.flip;
  }
#pragma unroll
  for (int u = 0; u < U; ++u)
    if (on[u]) y[u] = peer[jj[u]];  // NVLink loads, all issued before the first use
#pragma unroll
  for (int u = 0; u < U; ++u)
    if (on[u]) x[u] = mine[ii[u]];
#pragma unroll
  for (int u = 0; u < U; ++u)
    if (on[u]) {
      mine[ii[u]] = y[u];
      peer[jj[u]] = x[u];  // NVLink store (posted)
    }
  }
}

cudaError_t launch_pair_exchange(qip_prec prec, void *mine, void *peer, uint32_t n_local, uint32_t l,
                                 uint32_t s_bit, int rb, cudaStream_t s, uint64_t *launches) {
  if (n_local < 2 || l == s_bit || l >= n_local || s_bit >= n_local) return cudaErrorInvalidValue;
  ExArgs a;
  a.pos_lo = l < s_bit ? l : s_bit;
  a.pos_hi = l < s_bit ? s_bit : l;
  a.fixed = ((uint64_t)(rb ? 0 : 1) << l) | ((uint64_t)(rb ? 1 : 0) << s_bit);
  a.flip = 1ull << l;
  a.n_items = 1ull << (n_local - 2);
  const unsigned grid = (unsigned)((a.n_items + (uint64_t)kThreads * 4 - 1) / ((uint64_t)kThreads * 4));
  if (prec == QIP_F32)
    k_pair_exchange<float2, 4><<<grid, kThreads, 0, s>>>((float2 *)mine, (float2 *)peer, a);
  else
    k_pair_exchange<double2, 4><<<grid, kThreads, 0, s>>>((double2 *)mine, (double2 *)peer, a);
  ++*launches;
  return cudaGetLastError();
}

// ---- flag barrier -----------------------------------------------------------------
struct BarrierArgs {
  uint32_t *peer_flags[kMaxWorld];  // peer_flags[t] = rank t's flag page (mapped), slot [rank] is ours
  uint32_t *my_flags;
  int rank, world;
  uint32_t epoch;
  uint32_t *error_word;  // set to 1 on timeout (pinned host or device memory)
};

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__global__ void k_flag_barrier(const BarrierArgs a) {
  const int t = threadIdx.x;
  if (t >= a.world) return;
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.peer_flags[t] + a.rank), "r"(a.epoch) : "memory");
  const uint64_t t0 = globaltimer_ns();
  uint32_t v;
  for (;;) {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.my_flags + t) : "memory");
    if ((int32_t)(v - a.epoch) >= 0) break;
    if (globaltimer_ns() - t0 > 20ull * 1000ull * 1000ull * 1000ull) {  // 20 s: a peer is gone
      *a.error_word = 1u;
      break;
    }
  }
  __threadfence_system();
}

cudaError_t launch_flag_barrier(uint32_t *const *peer_flags, uint32_t *my_flags, int rank, int world,
                                uint32_t epoch, uint32_t *error_word, cudaStream_t s, uint64_t *launches) {
  if (world > kMaxWorld) return cudaErrorInvalidValue;
  BarrierArgs a;
  for (int t = 0; t < world; ++t) a.peer_flags[t] = peer_flags[t];
  a.my_flags = my_flags;
  a.rank = rank;
  a.world = world;
  a.epoch = epoch;
  a.error_word = error_word;
  k_flag_barrier<<<1, 32, 0, s>>>(a);
  ++*launches;
  return cudaGetLastError();
}

// ---- stand-in for the fused (paired) migration ------------------------------------------------------------------
// One CTA per tile of the give-half; 2^T amplitudes through the registers of 256 threads.
template <typename V, int PER>
__global__ void __launch_bounds__(256) k_paired_send(const PairedSendArgs a) {
  const V *mine = static_cast<const V *>(a.mine);
  V *peer = static_cast<V *>(a.peer);
  // tile counter of this CTA: the j-th tile of the give-half IN THE ORDER THE FUSED PASS WALKS THEM (launch position
  // 2 j + give with bits 0 and cbit exchanged, jit_codegen.cpp) -- both sides of a pair must come up in the same order, or
  // the two bounded sets of resident CTAs can wait for each other
  uint64_t t = 2ull * blockIdx.x + a.give;
  if (a.cbit != 0u) {
    const uint64_t b0 = t & 1ull, bc = (t >> a.cbit) & 1ull;
    t = (t & ~(1ull | (1ull << a.cbit))) | bc | (b0 << a.cbit);
  }
  uint64_t base = t << a.L;
  for (uint32_t i = 0; i < a.m; ++i) {
    const uint32_t q = a.hi_pos[i];
    base = ((base >> q) << (q + 1)) | (base & ((1ull << q) - 1ull));
  }
  V x[PER];  // PER = 2^T / 256 amplitudes per thread
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const uint32_t e = threadIdx.x + (uint32_t)j * 256u;
    uint64_t idx = base + (e & ((1u << a.L) - 1u));
    for (uint32_t i = 0; i < a.m; ++i)
      if ((e >> (a.L + i)) & 1u) idx |= 1ull << a.hi_pos[i];
    x[j] = mine[idx];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.peer_flags + (t ^ (1ull << a.cbit))), "r"(a.seq) : "memory");
    const uint64_t t0 = globaltimer_ns();
    uint32_t v;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.my_flags + t) : "memory");
      if ((int32_t)(v - a.seq) >= 0) break;
      if (globaltimer_ns() - t0 > 20ull * 1000ull * 1000ull * 1000ull || *(volatile uint32_t *)a.error_word != 0u) {
        *a.error_word = 1u;  // the partner is gone; later tiles give up at once
        break;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const uint32_t e = threadIdx.x + (uint32_t)j * 256u;
    uint64_t idx = base + (e & ((1u << a.L) - 1u));
    for (uint32_t i = 0; i < a.m; ++i)
      if ((e >> (a.L + i)) & 1u) idx |= 1ull << a.hi_pos[i];
    peer[idx ^ (1ull << a.l)] = x[j];
  }
}

cudaError_t launch_paired_send(qip_prec prec, const PairedSendArgs &a, cudaStream_t s, uint64_t *launches) {
  if (a.T != (prec == QIP_F32 ? 13u : 12u) || a.n_local <= a.T || a.m > 8) return cudaErrorInvalidValue;  // full-size tiles only
  const unsigned grid = 1u << (a.n_local - a.T - 1);
  if (prec == QIP_F32)
    k_paired_send<float2, 32><<<grid, 256, 0, s>>>(a);
  else
    k_paired_send<double2, 16><<<grid, 256, 0, s>>>(a);
  ++*launches;
  return cudaGetLastError();
}

// ---- small all-reduce through the peers' reduction slots ----------------------------------
struct CommSumArgs {
  const double *comm[kMaxWorld];
  int world;
  uint32_t count;
};

__global__ void __launch_bounds__(256) k_comm_sum(double *__restrict__ out, const CommSumArgs a) {
  const uint32_t i = blockIdx.x * 256u + threadIdx.x;
  if (i >= a.count) return;
  double acc = 0.0;
  for (int t = 0; t < a.world; ++t) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(a.comm[t] + i) : "memory");
    acc += v;
  }
  out[i] = acc;
}

cudaError_t launch_comm_sum(const double *const *peer_comm, int world, double *out, uint32_t count, cudaStream_t s,
                            uint64_t *launches) {
  if (world > kMaxWorld || count > (uint32_t)kCommDoubles) return cudaErrorInvalidValue;
  CommSumArgs a;
  for (int t = 0; t < world; ++t) a.comm[t] = peer_comm[t];
  a.world = world;
  a.count = count;
  k_comm_sum<<<(count + 255u) / 256u, 256, 0, s>>>(out, a);
  ++*launches;
  return cudaGetLastError();
}

}  // namespace qipb200
