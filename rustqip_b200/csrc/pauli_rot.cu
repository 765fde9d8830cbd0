// pauli_rot.cu -- psi <- exp(-i theta_t/2 P_t) psi for many Pauli strings P_t per read-write sweep of the state
// (qipb200_state_apply_pauli_rotations).
//
// Write P = i^nY X^x Z^z (x: index-bit mask of the X/Y letters, z: of the Z/Y letters).  Then
//   (P psi)_j = i^nY (-1)^popc((j ^ x) & z) psi_{j ^ x},
//   exp(-i theta/2 P) psi = c psi + s w,   c = cos(theta/2), s = sin(theta/2),   w_j = -i (P psi)_j,
// so a rotation mixes only the pairs (j, j ^ x), and w is psi_{j ^ x} times a power of i and a sign: a component swap
// and negations, exact.  Per component the update is RN(RN(c psi_j) + RN(s w_j)) in the state's precision (explicit
// __dmul_rn / __dadd_rn or __fmul_rn / __fadd_rn, no FMA contraction), from the values before the term.  c and s are
// rounded once from double on the host.  Amplitudes stay in the state's precision between terms, so the result does
// not depend on how terms are grouped into sweeps, on the tile geometry or on the layout.
//
// Sweep = tile geometry + x_out (planner: pauli_rot.h).  A tile (sweep.cuh) is the kSweepL lowest index bits plus up to
// kRotM chosen high bits (2^11 amplitudes, runs of 16 contiguous amplitudes).  Each term's X/Y mask splits as
// x = x_in ^ x_out with x_in on tile bits and x_out either 0 or the one out-of-tile mask the sweep shares.  With
// x_out == 0 a CTA stages one tile (double-buffered: the next tile loads with cp.async while the current one is
// rotated); otherwise it stages the pair (B, B ^ x_out), visited from the side whose lowest x_out bit is clear.  Every
// amplitude belongs to exactly one CTA visit per sweep, so the tiles are written back in place.  The CTA applies the
// sweep's terms in order on the staged tile(s) and writes them back once.  Z/Y bits outside the tile give a CTA-uniform
// sign, popc(base & z_out).
//
// Ownership: for a term with x_in != 0 on one tile a thread updates the pairs (e, e ^ x_in) it enumerates, for a term
// that reaches the partner tile the pairs (A[e], B[e ^ x_in]) for its own e, for a diagonal term (x == 0) its own
// elements e; a barrier separates two terms only when their ownership differs (the host marks them).  A run of diagonal
// terms keeps the thread's elements in registers.  The first kRotSmemTerms descriptors of a sweep are staged in shared
// memory, later ones are read from global memory, so a run of any length fits one sweep if its geometry does.
// Shared memory: two tiles plus the staged descriptors, at most 74 KiB per CTA (two CTAs per SM).
#include "pauli_rot.h"
#include "pauli_rot_dev.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

#include "../../include/qipb200.h"

namespace qipb200 {

namespace {

const uint32_t kRotM = 7;   // chosen high bits of a tile
const uint32_t kRotTile = 1u << (kSweepL + kRotM);
const int kRotThreads = 256;
const int kRotPer = kRotTile / kRotThreads;  // tile amplitudes per thread
const uint32_t kRotSmemTerms = 256;          // descriptors staged in shared memory; later ones are read from global

// One one-tile term with x_in != 0 on tile X (base b): the thread's pairs (e, e ^ x_in), e with bit h clear.
template <typename R, typename V>
__device__ __forceinline__ void rot_in_tile(V *X, uint64_t b, const RotTermDev &T, uint32_t tsize, int t) {
  const uint32_t ph = T.flags & kRotPhase, h = T.aux;
  const R c = (R)T.c, s = flip_sign((R)T.s, (ph >> 1) ^ (uint32_t)parity(b & T.z_out));
  const bool swap = ph & 1;
#pragma unroll
  for (int k = 0; k < kRotPer / 2; ++k) {
    const uint32_t p = t + kRotThreads * k;
    if (2 * p >= tsize) continue;
    const uint32_t e = ((p >> h) << (h + 1)) | (p & ((1u << h) - 1)), f = e ^ T.x_in;
    const V u = X[e], w = X[f];
    X[e] = rot1<R, V>(u, w, c, flip_sign(s, __popc(f & T.z_in) & 1), swap);
    X[f] = rot1<R, V>(w, u, c, flip_sign(s, __popc(e & T.z_in) & 1), swap);
  }
}

template <typename R, bool PAIR>
__global__ void __launch_bounds__(kRotThreads, 2)
    k_pauli_rot(R *__restrict__ psi, const __grid_constant__ RotArgs a, const RotTermDev *__restrict__ terms) {
  typedef typename SweepV<R>::type V;
  extern __shared__ __align__(16) unsigned char smem[];
  V *tiles = reinterpret_cast<V *>(smem);  // [2][kRotTile]: two buffers of one tile, or the tiles A and B of a pair
  RotTermDev *sT = reinterpret_cast<RotTermDev *>(smem + 2 * kRotTile * sizeof(V));
  const int t = threadIdx.x;
  const uint32_t n_smem = min(a.n_terms, kRotSmemTerms);
  for (uint32_t i = t; i < n_smem; i += kRotThreads) sT[i] = terms[i];  // ordered by the first barrier of the loop
  const uint32_t tsize = 1u << a.geo.tb;
  uint64_t off[kRotPer];
#pragma unroll
  for (int k = 0; k < kRotPer; ++k) off[k] = tile_offset(a.geo, t + kRotThreads * k);
  auto issue = [&](uint64_t v, V *dst) {
    const uint64_t b = visit_base(a.geo, v);
#pragma unroll
    for (int k = 0; k < kRotPer; ++k) {
      const uint32_t e = t + kRotThreads * k;
      if (e >= tsize) continue;
      cp_async<sizeof(V)>(dst + e, psi + 2 * (b | off[k]));
      if (PAIR) cp_async<sizeof(V)>(dst + kRotTile + e, psi + 2 * ((b ^ a.geo.x_out) | off[k]));
    }
  };
  uint64_t v = blockIdx.x;
  if (!PAIR) {
    if (v < a.geo.n_visits) issue(v, tiles);
    cp_async_commit();
  }
  int cur = 0;
  for (; v < a.geo.n_visits; v += gridDim.x) {
    if (PAIR) {
      issue(v, tiles);
      cp_async_commit();
      cp_async_wait<0>();
    } else {  // the next tile into the other buffer, then wait for the current one only
      const uint64_t nv = v + gridDim.x;
      if (nv < a.geo.n_visits) issue(nv, tiles + (cur ^ 1) * kRotTile);
      cp_async_commit();
      cp_async_wait<1>();
    }
    __syncthreads();
    V *A = tiles + (PAIR ? 0 : cur) * kRotTile;
    V *Bt = A + kRotTile;  // PAIR only
    const uint64_t bA = visit_base(a.geo, v), bB = bA ^ a.geo.x_out;
    for (uint32_t i = 0; i < a.n_terms;) {
      const RotTermDev T = i < kRotSmemTerms ? sT[i] : terms[i];
      if (T.flags & kRotBarrier) __syncthreads();
      if (T.flags & kRotDiag) {  // a run of diagonal terms on the thread's own elements, in registers, tile by tile
        const uint32_t end = i + T.aux;
#pragma unroll 1
        for (int side = 0; side < (PAIR ? 2 : 1); ++side) {
          V *X = side ? Bt : A;
          const uint64_t b = side ? bB : bA;
          V r[kRotPer];
#pragma unroll
          for (int k = 0; k < kRotPer; ++k) {
            const uint32_t e = t + kRotThreads * k;
            r[k].x = r[k].y = (R)0;  // elements past a small tile are rotated too but never stored
            if (e < tsize) r[k] = X[e];
          }
          for (uint32_t j = i; j < end; ++j) {
            const RotTermDev D = j < kRotSmemTerms ? sT[j] : terms[j];
            const uint32_t ph = D.flags & kRotPhase;
            const R c = (R)D.c, s = flip_sign((R)D.s, ph >> 1);
            // sign of element k (e = t + 256 k): parity(t & z_in) ^ parity(k & z_in >> 8) ^ parity(base & z_out)
            const uint32_t zk = D.z_in >> 8;
            const uint32_t par8 = ((zk & 1) ? 0xAAu : 0u) ^ ((zk & 2) ? 0xCCu : 0u) ^ ((zk & 4) ? 0xF0u : 0u);
            const uint32_t f = par8 ^ (((__popc((uint32_t)t & D.z_in) & 1) ^ (uint32_t)parity(b & D.z_out)) ? 0xFFu : 0u);
            if (ph & 1) {
#pragma unroll
              for (int k = 0; k < kRotPer; ++k) r[k] = rot1<R, V>(r[k], r[k], c, flip_sign(s, (f >> k) & 1), true);
            } else {
#pragma unroll
              for (int k = 0; k < kRotPer; ++k) r[k] = rot1<R, V>(r[k], r[k], c, flip_sign(s, (f >> k) & 1), false);
            }
          }
#pragma unroll
          for (int k = 0; k < kRotPer; ++k) {
            const uint32_t e = t + kRotThreads * k;
            if (e < tsize) X[e] = r[k];
          }
        }
        i = end;
        continue;
      }
      if (PAIR && (T.flags & kRotPair)) {  // (A[e], B[e ^ x_in]) for the thread's own e
        const uint32_t ph = T.flags & kRotPhase;
        const R c = (R)T.c, s = flip_sign((R)T.s, ph >> 1);
        const bool swap = ph & 1;
        const uint32_t nA = parity(bA & T.z_out), nB = parity(bB & T.z_out);
#pragma unroll
        for (int k = 0; k < kRotPer; ++k) {
          const uint32_t e = t + kRotThreads * k;
          if (e >= tsize) continue;
          const uint32_t f = e ^ T.x_in;
          const V u = A[e], w = Bt[f];
          A[e] = rot1<R, V>(u, w, c, flip_sign(s, nB ^ (__popc(f & T.z_in) & 1)), swap);
          Bt[f] = rot1<R, V>(w, u, c, flip_sign(s, nA ^ (__popc(e & T.z_in) & 1)), swap);
        }
      } else {
        rot_in_tile<R, V>(A, bA, T, tsize, t);
        if (PAIR) rot_in_tile<R, V>(Bt, bB, T, tsize, t);
      }
      ++i;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kRotPer; ++k) {
      const uint32_t e = t + kRotThreads * k;
      if (e >= tsize) continue;
      *reinterpret_cast<V *>(psi + 2 * (bA | off[k])) = A[e];
      if (PAIR) *reinterpret_cast<V *>(psi + 2 * (bB | off[k])) = Bt[e];
    }
    __syncthreads();  // the stores have read this buffer before the next cp.async writes it
    if (!PAIR) cur ^= 1;
  }
  cp_async_wait<0>();
}

template <typename R, bool PAIR>
cudaError_t launch_rot(void *psi, const RotArgs &a, const RotTermDev *terms, int grid, cudaStream_t s) {
  typedef typename SweepV<R>::type V;
  static_assert(kRotThreads == 256 && kRotPer == 8, "the diagonal path's sign table assumes e = t + 256 k, k < 8");
  static_assert(2 * kRotTile * sizeof(double2) + kRotSmemTerms * sizeof(RotTermDev) <= 113 * 1024,
                "two CTAs per SM: at most 113 KiB of shared memory each");
  const size_t smem = 2 * kRotTile * sizeof(V) + std::min(a.n_terms, kRotSmemTerms) * sizeof(RotTermDev);
  const size_t smem_max = 2 * kRotTile * sizeof(V) + kRotSmemTerms * sizeof(RotTermDev);
  cudaError_t e = cudaFuncSetAttribute(k_pauli_rot<R, PAIR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
  if (e != cudaSuccess) return e;
  k_pauli_rot<R, PAIR><<<grid, kRotThreads, smem, s>>>((R *)psi, a, terms);
  return cudaGetLastError();
}

}  // namespace

// ---- host: the sweep planner (policy in pauli_rot.h) and the descriptor tables --------------------------------------

bool rot_sweep_join(RotSweep *S, uint64_t x, uint64_t low, uint32_t m) {
  const uint64_t r = x & ~(low | S->hi);
  if (r == 0 || r == S->x_out) return true;
  if (!(r & S->x_out) && (uint32_t)(__builtin_popcountll(S->hi) + __builtin_popcountll(r)) <= m) {
    S->hi |= r;
    return true;
  }
  if (S->x_out == 0) {
    S->x_out = r;
    return true;
  }
  return false;
}

void plan_rot_sweeps(uint32_t n, uint32_t m_max, const std::vector<PauliTerm> &terms, std::vector<RotSweep> *out) {
  const uint32_t L = std::min(kSweepL, n), m = std::min(m_max, n - L);
  const uint64_t low = (1ull << L) - 1;
  std::vector<RotSweep> &sw = *out;
  sw.clear();
  if (terms.empty()) return;
  sw.push_back(RotSweep());
  for (uint32_t t = 0; t < (uint32_t)terms.size(); ++t) {
    if (rot_sweep_join(&sw.back(), terms[t].x, low, m)) continue;
    sw.back().end = t;
    sw.push_back(RotSweep());
    sw.back().first = t;
    rot_sweep_join(&sw.back(), terms[t].x, low, m);  // always joins an empty sweep
  }
  sw.back().end = (uint32_t)terms.size();
  for (RotSweep &S : sw) sweep_fill(&S.hi, &S.x_out, n, L, m);
}

bool build_rot_tables(qip_prec prec, uint32_t n, const std::vector<PauliTerm> &terms, const double *angles,
                      bool negate_s, const std::vector<RotSweep> &sw, std::vector<RotArgs> *args_out,
                      std::vector<RotTermDev> *ht_out) {
  const uint32_t L = std::min(kSweepL, n);
  const uint64_t low = (1ull << L) - 1;
  std::vector<RotArgs> &args = *args_out;
  std::vector<RotTermDev> &ht = *ht_out;
  args.assign(sw.size(), RotArgs());
  ht.assign(terms.size(), RotTermDev());
  for (size_t k = 0; k < sw.size(); ++k) {
    const RotSweep &S = sw[k];
    RotArgs &a = args[k];
    memset(&a, 0, sizeof(a));
    a.geo = sweep_tiles(n, L, S.hi, S.x_out);
    const uint64_t tile = low | S.hi;
    a.n_terms = S.end - S.first;
    uint64_t prev_key = ~0ull;  // ownership of the previous term: (x_in, pair), diagonal terms (0, 0)
    for (uint32_t t = S.first; t < S.end; ++t) {
      const PauliTerm &P = terms[t];
      RotTermDev &d = ht[t];
      memset(&d, 0, sizeof(d));
      const uint64_t xo = P.x & ~tile;
      if (xo != 0 && xo != S.x_out) return false;  // the planner's invariant
      d.z_out = P.z & ~tile;
      d.x_in = tile_local(a.geo, P.x & tile);
      d.z_in = tile_local(a.geo, P.z & tile);
      double c = cos(angles[t] / 2), sn = sin(angles[t] / 2);
      if (prec == QIP_F32) {
        c = (double)(float)c;
        sn = (double)(float)sn;
      }
      d.c = c;
      d.s = negate_s ? -sn : sn;
      d.flags = (P.n_y + 3) & kRotPhase;  // w = -i * i^nY * sign * psi_partner
      if (P.x == 0) {
        d.flags |= kRotDiag;
      } else if (xo) {
        d.flags |= kRotPair;
      } else {
        d.aux = (uint32_t)__builtin_ctz(d.x_in);
      }
      const uint64_t key = ((uint64_t)d.x_in << 1) | (xo ? 1u : 0u);
      if (t > S.first && key != prev_key) d.flags |= kRotBarrier;
      prev_key = key;
    }
    // diagonal runs: the first term of each carries the run's length
    for (uint32_t t = S.first; t < S.end;) {
      if (!(ht[t].flags & kRotDiag)) {
        ++t;
        continue;
      }
      uint32_t e = t;
      while (e < S.end && (ht[e].flags & kRotDiag)) ++e;
      ht[t].aux = e - t;
      t = e;
    }
  }
  return true;
}

uint32_t pauli_rotation_sweep_count(uint32_t n, const std::vector<PauliTerm> &terms) {
  std::vector<RotSweep> sw;
  plan_rot_sweeps(n, kRotM, terms, &sw);
  return (uint32_t)sw.size();
}

cudaError_t run_pauli_rotations(qip_prec prec, void *psi, uint32_t n, const std::vector<PauliTerm> &terms,
                                const double *angles, int grid, cudaStream_t s, uint64_t *launches) {
  if (terms.empty()) return cudaSuccess;
  std::vector<RotSweep> sw;
  plan_rot_sweeps(n, kRotM, terms, &sw);
  std::vector<RotArgs> args;
  std::vector<RotTermDev> ht;
  if (!build_rot_tables(prec, n, terms, angles, false, sw, &args, &ht)) return cudaErrorInvalidValue;
  RotTermDev *d = nullptr;
  cudaError_t e = cudaMallocAsync((void **)&d, ht.size() * sizeof(RotTermDev), s);
  if (e != cudaSuccess) return e;
  // pageable source: the copy is staged before cudaMemcpyAsync returns, so ht may go when this function does
  e = cudaMemcpyAsync(d, ht.data(), ht.size() * sizeof(RotTermDev), cudaMemcpyHostToDevice, s);
  for (size_t k = 0; k < sw.size() && e == cudaSuccess; ++k) {
    const int g = (int)std::min<uint64_t>(args[k].geo.n_visits, (uint64_t)std::max(grid, 1));
    const RotTermDev *td = d + sw[k].first;
    if (prec == QIP_F32)
      e = args[k].geo.x_out ? launch_rot<float, true>(psi, args[k], td, g, s)
                            : launch_rot<float, false>(psi, args[k], td, g, s);
    else
      e = args[k].geo.x_out ? launch_rot<double, true>(psi, args[k], td, g, s)
                            : launch_rot<double, false>(psi, args[k], td, g, s);
    ++*launches;
  }
  const cudaError_t ef = cudaFreeAsync(d, s);
  return e != cudaSuccess ? e : ef;
}

}  // namespace qipb200
