// density.cu -- exact noisy simulation on density matrices (qipb200_density_*): the doubling of a circuit with Kraus
// channels into one schedule on vec(rho), and the readout kernels.
//
// Layout.  A density matrix of n qubits is a state of 2n qubits.  Row qubit q is state qubit q and column qubit q is
// state qubit n + q, so in the qip_op convention (qubit q at index bit N - 1 - q) rho_rc sits at index r 2^n + c: the
// row index is the high half, each row is contiguous, and the downloaded vector reshaped to 2^n x 2^n is rho.
//
// Doubling.  rho -> U rho U^dagger is U on row qubits and conj(U) on column qubits: a gate op is emitted as itself,
// then as its conjugate (every index + n, MAT and sparse values conjugated, Swap and Control structure unchanged).
// A channel {K_i} on [q_1..q_k] is one MAT op on [q_1..q_k, q_1 + n..q_k + n] with S = sum_i kron(K_i, conj K_i): the
// row-major vec of K rho K^dagger.  S is formed in double, terms added in ascending i starting from the first, each
// part rounded once to the state's precision.  The result runs through qipb200_state_apply_schedule as it is, so the
// planner's fused tile passes and generated kernels carry over.
//
// Readouts honour the state's logical -> physical bit map (a QIPB200_ROTATE schedule leaves it permuted): index bits
// are moved with per-byte tables (a key's byte b selects tables[b][byte], the ORed masks are the physical index),
// staged in shared memory.  Every reduction has a fixed grid and order and no atomics, so results are deterministic
// (the spectrum's eigen-solve is cuSOLVER's and is not promised to repeat bit for bit).
//   - k_density_sums: entries of rho summed over index sets, one thread group per output entry (measure_probs and
//     the trace read only the diagonal; reduced reads the 2^(n + k) entries of the kept block pairs a <= a').
//   - k_density_expect: Re Tr(rho P) = Re i^nY sum_r (-1)^popc(r & z) rho_{r, r ^ x}, 2^n entries per term, a grid of
//     term x CTA blocks per launch.
//   - k_density_fidelity: <psi|rho|psi> = sum_rc conj(psi_r) rho_rc psi_c in one read sweep of rho, psi from L2.
//   - k_density_from_state: rho = |psi><psi| in one write sweep.
//   - k_density_widen: rho widened to double into the eigen-solver's matrix (qipb200_density_spectrum).
#include "density.h"

#include <algorithm>
#include <complex>
#include <cstring>
#include <type_traits>

#include "opcompile.h"
#include "kraus.h"

namespace qipb200 {

namespace {

const int kDenThreads = 256;
const int kDenGrid = 1056;       // fixed reduction grid: 8 CTAs per SM of a 132-SM H100
const int kDenExpectBlocks = 64; // CTAs per term at most
const uint32_t kDenTermBatch = 4096;

template <typename R>
using VecOf = typename std::conditional<std::is_same<R, float>::value, float2, double2>::type;

// Byte tables of a key -> physical index map: masks[j] is what key bit j sets.
std::vector<uint64_t> byte_tables(const std::vector<uint64_t> &masks, uint32_t *nbytes) {
  *nbytes = (uint32_t)((masks.size() + 7) / 8);
  std::vector<uint64_t> t((size_t)*nbytes * 256, 0);
  for (uint32_t b = 0; b < *nbytes; ++b)
    for (uint32_t v = 0; v < 256; ++v) {
      uint64_t m = 0;
      for (uint32_t j = 0; j < 8 && 8 * b + j < masks.size(); ++j)
        if ((v >> j) & 1) m |= masks[8 * b + j];
      t[(size_t)b * 256 + v] = m;
    }
  return t;
}

// The tables of the logical -> physical map (pol[l] is the physical bit of logical bit l), or of its inverse.
std::vector<uint64_t> layout_tables(const std::vector<uint32_t> &pol, bool inverse, uint32_t *nbytes) {
  std::vector<uint64_t> masks(pol.size());
  for (size_t l = 0; l < pol.size(); ++l) {
    if (inverse)
      masks[pol[l]] = 1ull << l;
    else
      masks[l] = 1ull << pol[l];
  }
  return byte_tables(masks, nbytes);
}

bool is_identity(const std::vector<uint32_t> &pol) {
  for (size_t l = 0; l < pol.size(); ++l)
    if (pol[l] != l) return false;
  return true;
}

__device__ __forceinline__ void load_tables(uint64_t *sh, const uint64_t *tab, uint32_t nbytes) {
  for (uint32_t i = threadIdx.x; i < nbytes * 256; i += blockDim.x) sh[i] = tab[i];
  __syncthreads();
}

__device__ __forceinline__ uint64_t scatter(const uint64_t *sh, uint32_t nbytes, uint64_t key) {
  uint64_t p = 0;
  for (uint32_t b = 0; b < nbytes; ++b) p |= sh[(b << 8) | ((key >> (8 * b)) & 255)];
  return p;
}

// The CTA's sum of v: a fixed tree over the threads.
__device__ __forceinline__ double2 block_sum(double2 v) {
  __shared__ double2 red[kDenThreads];
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
  for (int s = kDenThreads / 2; s > 0; s >>= 1) {
    if (t < s) {
      red[t].x += red[t + s].x;
      red[t].y += red[t + s].y;
    }
    __syncthreads();
  }
  return red[0];
}

template <typename R>
__global__ void __launch_bounds__(kDenThreads) k_density_from_state(VecOf<R> *__restrict__ rho,
                                                                    const VecOf<R> *__restrict__ psi, uint32_t n,
                                                                    uint64_t total) {
  const uint64_t mask = (1ull << n) - 1, stride = (uint64_t)gridDim.x * kDenThreads;
  for (uint64_t i = (uint64_t)blockIdx.x * kDenThreads + threadIdx.x; i < total; i += stride) {
    const VecOf<R> a = __ldg(psi + (i >> n)), b = __ldg(psi + (i & mask));
    VecOf<R> o;
    o.x = a.x * b.x + a.y * b.y;
    o.y = a.y * b.x - a.x * b.y;
    rho[i] = o;
  }
}

// Per CTA: sum over its indices i (grid-stride, ascending) of conj(psi_r) (rho_i psi_c) in double.
template <typename R, bool IDENT>
__global__ void __launch_bounds__(kDenThreads) k_density_fidelity(const VecOf<R> *__restrict__ rho,
                                                                  const VecOf<R> *__restrict__ psi, uint32_t n,
                                                                  uint64_t total, const uint64_t *__restrict__ tab,
                                                                  uint32_t nbytes, double2 *__restrict__ partials) {
  extern __shared__ uint64_t sh[];
  if (!IDENT) load_tables(sh, tab, nbytes);
  const uint64_t mask = (1ull << n) - 1, stride = (uint64_t)gridDim.x * kDenThreads;
  double ar = 0.0, ai = 0.0;
#pragma unroll 4
  for (uint64_t i = (uint64_t)blockIdx.x * kDenThreads + threadIdx.x; i < total; i += stride) {
    const uint64_t l = IDENT ? i : scatter(sh, nbytes, i);
    const VecOf<R> v = rho[i], pc = __ldg(psi + (l & mask)), pr = __ldg(psi + (l >> n));
    const double tr = (double)v.x * pc.x - (double)v.y * pc.y, ti = (double)v.x * pc.y + (double)v.y * pc.x;
    ar += (double)pr.x * tr + (double)pr.y * ti;
    ai += (double)pr.x * ti - (double)pr.y * tr;
  }
  const double2 s = block_sum(make_double2(ar, ai));
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// out[g] = sum of partials[g * per .. (g + 1) * per) in order, one thread per g.
__global__ void k_density_finish(const double2 *__restrict__ partials, uint32_t groups, uint32_t per,
                                 double2 *__restrict__ out) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  double2 s = partials[(size_t)g * per];
  for (uint32_t j = 1; j < per; ++j) {
    s.x += partials[(size_t)g * per + j].x;
    s.y += partials[(size_t)g * per + j].y;
  }
  out[g] = s;
}

struct DenTerm {
  uint64_t x, z;
};

// Per (term, CTA): sum over r of (-1)^popc(r & z) rho_{r, r ^ x}; the phase i^nY is applied on the host.
template <typename R>
__global__ void __launch_bounds__(kDenThreads) k_density_expect(const VecOf<R> *__restrict__ rho, uint32_t n,
                                                                const DenTerm *__restrict__ terms,
                                                                const uint64_t *__restrict__ tab, uint32_t nbytes,
                                                                double2 *__restrict__ partials) {
  extern __shared__ uint64_t sh[];
  load_tables(sh, tab, nbytes);
  const DenTerm P = terms[blockIdx.y];
  const uint64_t side = 1ull << n, stride = (uint64_t)gridDim.x * kDenThreads;
  double sr = 0.0, si = 0.0;
  for (uint64_t r = (uint64_t)blockIdx.x * kDenThreads + threadIdx.x; r < side; r += stride) {
    const VecOf<R> v = rho[scatter(sh, nbytes, (r << n) | (r ^ P.x))];
    if (__popcll(r & P.z) & 1) {
      sr -= v.x;
      si -= v.y;
    } else {
      sr += v.x;
      si += v.y;
    }
  }
  const double2 s = block_sum(make_double2(sr, si));
  if (threadIdx.x == 0) partials[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
}

// One group of T = 2^tlog threads per output entry e: lanes stride over b, then a fixed tree over the group.
template <typename R>
__global__ void __launch_bounds__(kDenThreads) k_density_sums(const VecOf<R> *__restrict__ rho,
                                                              const uint64_t *__restrict__ tab, uint32_t nbytes,
                                                              uint32_t nb, uint32_t ke, uint32_t kc, uint32_t tlog,
                                                              double2 *__restrict__ out) {
  extern __shared__ uint64_t sh[];
  __shared__ double2 red[kDenThreads];
  load_tables(sh, tab, nbytes);
  const uint32_t t = threadIdx.x, T = 1u << tlog, lane = t & (T - 1);
  const uint64_t e = (uint64_t)blockIdx.x * (kDenThreads >> tlog) + (t >> tlog);
  bool live = e < (1ull << ke);
  if (live && kc) {
    const uint32_t ka = ke - kc;
    live = (e & ((1ull << ka) - 1)) <= (e >> ka);
  }
  double sr = 0.0, si = 0.0;
  if (live)
    for (uint64_t b = lane; b < (1ull << nb); b += T) {
      const VecOf<R> v = rho[scatter(sh, nbytes, b | (e << nb))];
      sr += v.x;
      si += v.y;
    }
  red[t] = make_double2(sr, si);
  __syncthreads();
  for (uint32_t s = T >> 1; s > 0; s >>= 1) {
    if (lane < s) {
      red[t].x += red[t + s].x;
      red[t].y += red[t + s].y;
    }
    __syncthreads();
  }
  if (live && lane == 0) out[e] = red[t];
}

template <typename R, bool IDENT>
__global__ void __launch_bounds__(kDenThreads) k_density_widen(const VecOf<R> *__restrict__ rho, uint64_t total,
                                                               const uint64_t *__restrict__ tab, uint32_t nbytes,
                                                               double2 *__restrict__ G) {
  extern __shared__ uint64_t sh[];
  if (!IDENT) load_tables(sh, tab, nbytes);
  const uint64_t stride = (uint64_t)gridDim.x * kDenThreads;
  for (uint64_t i = (uint64_t)blockIdx.x * kDenThreads + threadIdx.x; i < total; i += stride) {
    const VecOf<R> v = rho[i];
    G[IDENT ? i : scatter(sh, nbytes, i)] = make_double2((double)v.x, (double)v.y);
  }
}

// Stream-ordered device scratch, freed on the stream when the scope ends.
struct Scratch {
  cudaStream_t s;
  void *p = nullptr;
  explicit Scratch(cudaStream_t st) : s(st) {}
  cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, s); }
  ~Scratch() {
    if (p) cudaFreeAsync(p, s);
  }
};

#define DEN_TRY(call)                          \
  do {                                         \
    const cudaError_t e__ = (call);            \
    if (e__ != cudaSuccess) return e__;        \
  } while (0)

size_t tables_bytes(uint32_t nbytes) { return (size_t)nbytes * 256 * sizeof(uint64_t); }

// Tables first in the scratch, then `extra` bytes (16-byte aligned).
cudaError_t stage_tables(Scratch *sc, const std::vector<uint64_t> &tab, size_t extra) {
  const size_t tb = (tab.size() * sizeof(uint64_t) + 15) & ~(size_t)15;
  DEN_TRY(sc->alloc(tb + extra + 16));
  if (!tab.empty())
    DEN_TRY(cudaMemcpyAsync(sc->p, tab.data(), tab.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, sc->s));
  return cudaSuccess;
}

double2 *after_tables(const Scratch &sc, const std::vector<uint64_t> &tab) {
  const size_t tb = (tab.size() * sizeof(uint64_t) + 15) & ~(size_t)15;
  return reinterpret_cast<double2 *>((char *)sc.p + tb);
}

template <typename R>
cudaError_t fidelity_prec(const void *rho, const void *psi, uint32_t n, const std::vector<uint32_t> &pol,
                          double *out2, cudaStream_t s, uint64_t *launches) {
  const bool ident = is_identity(pol);
  uint32_t nbytes = 0;
  const std::vector<uint64_t> tab = ident ? std::vector<uint64_t>() : layout_tables(pol, true, &nbytes);
  Scratch sc(s);
  DEN_TRY(stage_tables(&sc, tab, (kDenGrid + 1) * sizeof(double2)));
  double2 *parts = after_tables(sc, tab);
  const uint64_t total = 1ull << (2 * n);
  const VecOf<R> *r = (const VecOf<R> *)rho, *p = (const VecOf<R> *)psi;
  if (ident)
    k_density_fidelity<R, true><<<kDenGrid, kDenThreads, 0, s>>>(r, p, n, total, nullptr, 0, parts);
  else
    k_density_fidelity<R, false><<<kDenGrid, kDenThreads, tables_bytes(nbytes), s>>>(
        r, p, n, total, (const uint64_t *)sc.p, nbytes, parts);
  DEN_TRY(cudaGetLastError());
  k_density_finish<<<1, 32, 0, s>>>(parts, 1, kDenGrid, parts + kDenGrid);
  DEN_TRY(cudaGetLastError());
  *launches += 2;
  DEN_TRY(cudaMemcpyAsync(out2, parts + kDenGrid, sizeof(double2), cudaMemcpyDeviceToHost, s));
  return cudaStreamSynchronize(s);
}

template <typename R>
cudaError_t expect_prec(const void *rho, uint32_t n, const std::vector<uint32_t> &pol,
                        const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches) {
  uint32_t nbytes = 0;
  const std::vector<uint64_t> tab = layout_tables(pol, false, &nbytes);
  const uint64_t side = 1ull << n;
  const uint32_t B = (uint32_t)std::max<uint64_t>(
      1, std::min<uint64_t>(kDenExpectBlocks, side / (kDenThreads * 16)));
  const uint32_t batch = (uint32_t)std::min<size_t>(terms.size(), kDenTermBatch);
  Scratch sc(s);
  DEN_TRY(stage_tables(&sc, tab, (size_t)batch * (sizeof(DenTerm) + (B + 1) * sizeof(double2))));
  double2 *parts = after_tables(sc, tab), *sums = parts + (size_t)batch * B;
  DenTerm *dterms = reinterpret_cast<DenTerm *>(sums + batch);
  std::vector<DenTerm> ht(batch);
  std::vector<double2> hs(batch);
  for (size_t t0 = 0; t0 < terms.size(); t0 += batch) {
    const uint32_t nt = (uint32_t)std::min<size_t>(batch, terms.size() - t0);
    for (uint32_t t = 0; t < nt; ++t) ht[t] = DenTerm{terms[t0 + t].x, terms[t0 + t].z};
    DEN_TRY(cudaMemcpyAsync(dterms, ht.data(), nt * sizeof(DenTerm), cudaMemcpyHostToDevice, s));
    k_density_expect<R><<<dim3(B, nt), kDenThreads, tables_bytes(nbytes), s>>>(
        (const VecOf<R> *)rho, n, dterms, (const uint64_t *)sc.p, nbytes, parts);
    DEN_TRY(cudaGetLastError());
    k_density_finish<<<(nt + 127) / 128, 128, 0, s>>>(parts, nt, B, sums);
    DEN_TRY(cudaGetLastError());
    *launches += 2;
    DEN_TRY(cudaMemcpyAsync(hs.data(), sums, nt * sizeof(double2), cudaMemcpyDeviceToHost, s));
    DEN_TRY(cudaStreamSynchronize(s));  // ht and hs are reused by the next batch
    for (uint32_t t = 0; t < nt; ++t) {
      const double2 v = hs[t];
      switch (terms[t0 + t].n_y & 3) {  // Re(i^nY v)
        case 0: out[t0 + t] = v.x; break;
        case 1: out[t0 + t] = -v.y; break;
        case 2: out[t0 + t] = -v.x; break;
        default: out[t0 + t] = v.y; break;
      }
    }
  }
  return cudaSuccess;
}

template <typename R>
cudaError_t sums_prec(const void *rho, const std::vector<uint64_t> &key_masks, uint32_t nb, uint32_t ke, uint32_t kc,
                      double *out, cudaStream_t s, uint64_t *launches) {
  uint32_t nbytes = 0;
  const std::vector<uint64_t> tab = byte_tables(key_masks, &nbytes);
  const uint64_t E = 1ull << ke;
  const uint32_t tlog = std::min<uint32_t>(nb, 8);  // 256 threads per entry at most
  const uint64_t per_cta = kDenThreads >> tlog;
  Scratch sc(s);
  DEN_TRY(stage_tables(&sc, tab, E * sizeof(double2)));
  double2 *res = after_tables(sc, tab);
  DEN_TRY(cudaMemsetAsync(res, 0, E * sizeof(double2), s));
  k_density_sums<R><<<(unsigned)((E + per_cta - 1) / per_cta), kDenThreads, tables_bytes(nbytes), s>>>(
      (const VecOf<R> *)rho, (const uint64_t *)sc.p, nbytes, nb, ke, kc, tlog, res);
  DEN_TRY(cudaGetLastError());
  *launches += 1;
  DEN_TRY(cudaMemcpyAsync(out, res, E * sizeof(double2), cudaMemcpyDeviceToHost, s));
  return cudaStreamSynchronize(s);
}

template <typename R>
cudaError_t widen_prec(const void *rho, uint32_t n, const std::vector<uint32_t> &pol, double2 *G, cudaStream_t s,
                       uint64_t *launches) {
  const bool ident = is_identity(pol);
  uint32_t nbytes = 0;
  const std::vector<uint64_t> tab = ident ? std::vector<uint64_t>() : layout_tables(pol, true, &nbytes);
  Scratch sc(s);
  DEN_TRY(stage_tables(&sc, tab, 0));
  const uint64_t total = 1ull << (2 * n);
  const unsigned grid = (unsigned)std::min<uint64_t>((total + kDenThreads - 1) / kDenThreads, 132 * 16);
  if (ident)
    k_density_widen<R, true><<<grid, kDenThreads, 0, s>>>((const VecOf<R> *)rho, total, nullptr, 0, G);
  else
    k_density_widen<R, false><<<grid, kDenThreads, tables_bytes(nbytes), s>>>(
        (const VecOf<R> *)rho, total, (const uint64_t *)sc.p, nbytes, G);
  DEN_TRY(cudaGetLastError());
  *launches += 1;
  return cudaSuccess;
}

// The conjugate of a gate op on the column qubits: indices + n, values conjugated, structure unchanged.
qip_op conjugate_op(const qip_op &op, uint32_t n, size_t amp, DensitySchedule *d) {
  qip_op o = op;
  d->u64s.emplace_back(op.indices, op.indices + op.n_indices);
  for (uint64_t &q : d->u64s.back()) q += n;
  o.indices = d->u64s.back().data();
  auto conj_values = [&](const void *src, size_t count) {
    d->blobs.emplace_back((const unsigned char *)src, (const unsigned char *)src + count * amp);
    unsigned char *b = d->blobs.back().data();
    for (size_t i = 0; i < count; ++i) {
      if (amp == 8) {
        float *v = reinterpret_cast<float *>(b + i * amp) + 1;
        *v = -*v;
      } else {
        double *v = reinterpret_cast<double *>(b + i * amp) + 1;
        *v = -*v;
      }
    }
    return (const void *)b;
  };
  switch (op.kind) {
    case QIP_OP_MATRIX:
      o.dense = conj_values(op.dense, (size_t)op.n_entries);
      break;
    case QIP_OP_SPARSE:
      o.sp_val = conj_values(op.sp_val, (size_t)op.sp_rowptr[op.n_entries]);
      break;
    case QIP_OP_CONTROL:
      d->nested.push_back(conjugate_op(*op.inner, n, amp, d));
      o.inner = &d->nested.back();
      break;
    default:
      break;
  }
  return o;
}

// The superoperator of channel c as one MAT op on [q.., q + n..].
qip_op superop(const KrausSet &ks, size_t c, uint32_t n, qip_prec prec, DensitySchedule *d) {
  const uint32_t k = ks.arity(c), D = 1u << k, DD = D * D;
  std::vector<double> S(2 * (size_t)DD * DD);
  for (uint32_t i = ks.first[c]; i < ks.first[c + 1]; ++i) {
    const double *K = ks.mat[i];
    const bool first = i == ks.first[c];
    for (uint32_t r1 = 0; r1 < D; ++r1)
      for (uint32_t r2 = 0; r2 < D; ++r2)
        for (uint32_t c1 = 0; c1 < D; ++c1)
          for (uint32_t c2 = 0; c2 < D; ++c2) {
            const double a = K[2 * (r1 * D + c1)], b = K[2 * (r1 * D + c1) + 1];
            const double x = K[2 * (r2 * D + c2)], y = K[2 * (r2 * D + c2) + 1];
            const double re = a * x + b * y, im = b * x - a * y;  // K[r1][c1] conj(K[r2][c2])
            double *e = &S[2 * ((size_t)(r1 * D + r2) * DD + (c1 * D + c2))];
            e[0] = first ? re : e[0] + re;
            e[1] = first ? im : e[1] + im;
          }
  }
  const size_t amp = prec == QIP_F32 ? 8 : 16;
  d->blobs.emplace_back(S.size() / 2 * amp);
  unsigned char *b = d->blobs.back().data();
  for (size_t i = 0; i < S.size(); ++i) {
    if (prec == QIP_F32)
      reinterpret_cast<float *>(b)[i] = (float)S[i];
    else
      reinterpret_cast<double *>(b)[i] = S[i];
  }
  d->u64s.emplace_back();
  std::vector<uint64_t> &idx = d->u64s.back();
  for (uint32_t j = 0; j < k; ++j) idx.push_back(ks.qubits[ks.qfirst[c] + j]);
  for (uint32_t j = 0; j < k; ++j) idx.push_back(ks.qubits[ks.qfirst[c] + j] + n);
  qip_op o;
  memset(&o, 0, sizeof(o));
  o.kind = QIP_OP_MATRIX;
  o.n_indices = 2 * k;
  o.n_entries = (uint64_t)DD * DD;
  o.indices = idx.data();
  o.dense = b;
  return o;
}

}  // namespace

int build_density_schedule(const std::string &who, qip_prec prec, uint32_t n, const qip_op *ops, size_t n_ops,
                           size_t n_channels, const uint64_t *channel_pos, const uint32_t *arity,
                           const uint64_t *qubits, const uint32_t *n_kraus, const double *kraus, DensitySchedule *out,
                           std::string *err) {
  if (prec != QIP_F32 && prec != QIP_F64) {
    *err = who + ": bad precision";
    return QIPB200_ERR_INVALID_ARG;
  }
  if (n == 0 || n > 20) {
    *err = who + ": a density matrix has 1..20 qubits (its state 2..40), got " + std::to_string(n);
    return QIPB200_ERR_INVALID_ARG;
  }
  if ((n_ops && !ops) || (n_channels && !channel_pos)) {
    *err = who + ": NULL ops or channel_pos";
    return QIPB200_ERR_INVALID_ARG;
  }
  for (size_t i = 0; i < n_ops; ++i) {
    std::string e;
    const int st = validate_op(&ops[i], prec, n, &e);
    if (st != QIPB200_OK) {
      *err = who + ": op " + std::to_string(i) + ": " + e;
      return st;
    }
  }
  for (size_t c = 0; c < n_channels; ++c)
    if (channel_pos[c] > n_ops || (c && channel_pos[c] < channel_pos[c - 1])) {
      *err = who + ": channel_pos[" + std::to_string(c) + "] = " + std::to_string(channel_pos[c]) +
             " (positions must be non-decreasing and at most n_ops = " + std::to_string(n_ops) + ")";
      return QIPB200_ERR_INVALID_ARG;
    }
  KrausSet ks;
  const int st = parse_kraus_channels(who, n, n_channels, arity, qubits, n_kraus, kraus, &ks, err, true);
  if (st != QIPB200_OK) return st;
  DensitySchedule &d = *out;
  d = DensitySchedule();
  const size_t amp = prec == QIP_F32 ? 8 : 16;
  size_t c = 0;
  for (size_t i = 0; i <= n_ops; ++i) {
    for (; c < n_channels && channel_pos[c] == i; ++c) d.ops.push_back(superop(ks, c, n, prec, &d));
    if (i == n_ops) break;
    d.ops.push_back(ops[i]);
    d.ops.push_back(conjugate_op(ops[i], n, amp, &d));
  }
  return QIPB200_OK;
}

cudaError_t run_density_from_state(qip_prec prec, void *rho, const void *psi, uint32_t n, cudaStream_t s,
                                   uint64_t *launches) {
  const uint64_t total = 1ull << (2 * n);
  const unsigned grid = (unsigned)std::min<uint64_t>((total + kDenThreads - 1) / kDenThreads, 132 * 16);
  if (prec == QIP_F32)
    k_density_from_state<float><<<grid, kDenThreads, 0, s>>>((float2 *)rho, (const float2 *)psi, n, total);
  else
    k_density_from_state<double><<<grid, kDenThreads, 0, s>>>((double2 *)rho, (const double2 *)psi, n, total);
  *launches += 1;
  return cudaGetLastError();
}

cudaError_t run_density_sums(qip_prec prec, const void *rho, const std::vector<uint64_t> &key_masks, uint32_t nb,
                             uint32_t ke, uint32_t kc, double *out, cudaStream_t s, uint64_t *launches) {
  return prec == QIP_F32 ? sums_prec<float>(rho, key_masks, nb, ke, kc, out, s, launches)
                         : sums_prec<double>(rho, key_masks, nb, ke, kc, out, s, launches);
}

cudaError_t run_density_expect(qip_prec prec, const void *rho, uint32_t n, const std::vector<uint32_t> &pol,
                               const std::vector<PauliTerm> &terms, double *out, cudaStream_t s, uint64_t *launches) {
  return prec == QIP_F32 ? expect_prec<float>(rho, n, pol, terms, out, s, launches)
                         : expect_prec<double>(rho, n, pol, terms, out, s, launches);
}

cudaError_t run_density_fidelity(qip_prec prec, const void *rho, const void *psi, uint32_t n,
                                 const std::vector<uint32_t> &pol, double *out2, cudaStream_t s, uint64_t *launches) {
  return prec == QIP_F32 ? fidelity_prec<float>(rho, psi, n, pol, out2, s, launches)
                         : fidelity_prec<double>(rho, psi, n, pol, out2, s, launches);
}

cudaError_t run_density_widen(qip_prec prec, const void *rho, uint32_t n, const std::vector<uint32_t> &pol, double2 *G,
                              cudaStream_t s, uint64_t *launches) {
  return prec == QIP_F32 ? widen_prec<float>(rho, n, pol, G, s, launches)
                         : widen_prec<double>(rho, n, pol, G, s, launches);
}

}  // namespace qipb200
