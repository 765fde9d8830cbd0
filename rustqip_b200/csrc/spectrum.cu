// spectrum.cu -- see spectrum.h.
//
// cuSOLVER is loaded at run time (dlopen), as jit_runtime.cu loads NVRTC: the library itself links only a static
// cudart and libdl, loads without cuSOLVER, and every other entry point works without it.  cuSOLVER brings its own
// CUDA runtime, so nothing here relies on implicit ordering between the two: the caller's kernels are synchronised
// before the solver starts, the solver's stream is set to the context's stream (and read back), and that stream is
// synchronised before the eigenvalues are read.
#include "spectrum.h"

#include <cusolverDn.h>
#include <dlfcn.h>

#include <algorithm>
#include <mutex>

#include "../../include/qipb200.h"

namespace qipb200 {

namespace {

struct Cusolver {
  void *h = nullptr;
  decltype(&cusolverDnCreate) create = nullptr;
  decltype(&cusolverDnDestroy) destroy = nullptr;
  decltype(&cusolverDnSetStream) set_stream = nullptr;
  decltype(&cusolverDnGetStream) get_stream = nullptr;
  decltype(&cusolverDnZheevd_bufferSize) zheevd_size = nullptr;
  decltype(&cusolverDnZheevd) zheevd = nullptr;
  std::string why;
  bool ok = false;
};

Cusolver &cusolver() {
  static Cusolver c;
  static std::once_flag once;
  std::call_once(once, [&]() {
    const char *names[] = {"libcusolver.so.11", "/usr/local/cuda/lib64/libcusolver.so.11"};
    std::string reasons;
    for (const char *nm : names) {
      if ((c.h = dlopen(nm, RTLD_NOW | RTLD_LOCAL))) break;
      const char *e = dlerror();
      reasons += std::string(reasons.empty() ? "" : "; ") + (e ? e : nm);
    }
    if (!c.h) {
      c.why = "libcusolver not found: " + reasons;
      return;
    }
#define QIP_SYM(field, name)                       \
  *(void **)(&c.field) = dlsym(c.h, name);         \
  if (!c.field) {                                  \
    c.why = std::string("libcusolver lacks ") + name; \
    return;                                        \
  }
    QIP_SYM(create, "cusolverDnCreate")
    QIP_SYM(destroy, "cusolverDnDestroy")
    QIP_SYM(set_stream, "cusolverDnSetStream")
    QIP_SYM(get_stream, "cusolverDnGetStream")
    QIP_SYM(zheevd_size, "cusolverDnZheevd_bufferSize")
    QIP_SYM(zheevd, "cusolverDnZheevd")
#undef QIP_SYM
    c.ok = true;
  });
  return c;
}

int solver_fail(cusolverStatus_t st, const char *what, std::string *err) {
  *err = std::string(what) + " failed (cusolverStatus_t " + std::to_string((int)st) + ")";
  return st == CUSOLVER_STATUS_ALLOC_FAILED ? QIPB200_ERR_OOM : QIPB200_ERR_CUDA;
}

int cuda_status(cudaError_t e, const char *what, std::string *err) {
  *err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  cudaGetLastError();
  return e == cudaErrorMemoryAllocation ? QIPB200_ERR_OOM : QIPB200_ERR_CUDA;
}

}  // namespace

bool eig_solver_available(std::string *why) {
  Cusolver &c = cusolver();
  if (!c.ok && why) *why = c.why;
  return c.ok;
}

void eig_work_free(EigWork *w, cudaStream_t s) {
  if (w->G) cudaFreeAsync(w->G, s);
  if (w->work) cudaFreeAsync(w->work, s);
  *w = EigWork();
}

int eig_work_alloc(void **handle, uint32_t K, EigWork *w, cudaStream_t s, std::string *err) {
  Cusolver &c = cusolver();
  if (!c.ok) {
    *err = c.why;
    return QIPB200_ERR_UNSUPPORTED;
  }
  if (!*handle) {
    cusolverDnHandle_t h = nullptr;
    const cusolverStatus_t st = c.create(&h);
    if (st != CUSOLVER_STATUS_SUCCESS) return solver_fail(st, "cusolverDnCreate", err);
    *handle = h;
  }
  // Stream-ordered pool allocations on the context's stream (no device-wide synchronisation per call): G, then
  // the eigenvalues and the info word; the workspace, once its size is known, in a second allocation.
  w->K = K;
  const size_t g_bytes = (size_t)K * K * sizeof(double2), w_off = (g_bytes + 255) & ~(size_t)255;
  const size_t i_off = w_off + (((size_t)K * sizeof(double) + 255) & ~(size_t)255);
  cudaError_t e = cudaMallocAsync((void **)&w->G, i_off + sizeof(int), s);
  if (e != cudaSuccess) {
    w->G = nullptr;
    return cuda_status(e, "cudaMallocAsync(entanglement_spectrum matrix)", err);
  }
  w->W = (double *)((char *)w->G + w_off);
  w->info = (int *)((char *)w->G + i_off);
  const cusolverStatus_t st =
      c.zheevd_size((cusolverDnHandle_t)*handle, CUSOLVER_EIG_MODE_NOVECTOR, CUBLAS_FILL_MODE_UPPER, (int)K,
                    (const cuDoubleComplex *)w->G, (int)K, w->W, &w->lwork);
  if (st != CUSOLVER_STATUS_SUCCESS) {
    eig_work_free(w, s);
    return solver_fail(st, "cusolverDnZheevd_bufferSize", err);
  }
  e = cudaMallocAsync((void **)&w->work, (size_t)std::max(w->lwork, 1) * sizeof(double2), s);
  if (e != cudaSuccess) {
    w->work = nullptr;
    eig_work_free(w, s);
    return cuda_status(e, "cudaMallocAsync(eigen-solver workspace)", err);
  }
  return QIPB200_OK;
}

int eig_solve(void *handle, EigWork *w, cudaStream_t s, double *eigs_asc, std::string *err) {
  Cusolver &c = cusolver();
  cusolverDnHandle_t h = (cusolverDnHandle_t)handle;
  cudaError_t e = cudaStreamSynchronize(s);  // everything this library queued for G has finished
  if (e != cudaSuccess) return cuda_status(e, "cudaStreamSynchronize(before the eigen-solve)", err);
  cusolverStatus_t st = c.set_stream(h, s);
  if (st != CUSOLVER_STATUS_SUCCESS) return solver_fail(st, "cusolverDnSetStream", err);
  cudaStream_t got = nullptr;
  st = c.get_stream(h, &got);
  if (st != CUSOLVER_STATUS_SUCCESS || got != s) {
    *err = "cusolverDnSetStream did not take the context's stream";
    return QIPB200_ERR_CUDA;
  }
  // Row-major G read column-major is G^T = conj(G): the same eigenvalues.
  st = c.zheevd(h, CUSOLVER_EIG_MODE_NOVECTOR, CUBLAS_FILL_MODE_UPPER, (int)w->K, (cuDoubleComplex *)w->G, (int)w->K,
                w->W, (cuDoubleComplex *)w->work, w->lwork, w->info);
  if (st != CUSOLVER_STATUS_SUCCESS) {
    cudaStreamSynchronize(s);
    return solver_fail(st, "cusolverDnZheevd", err);
  }
  e = cudaStreamSynchronize(s);  // the solver's work on the stream has finished
  int info = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&info, w->info, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(eigs_asc, w->W, (size_t)w->K * sizeof(double), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return cuda_status(e, "eigen-solve", err);
  if (info != 0) {
    *err = "cusolverDnZheevd: info = " + std::to_string(info) + (info > 0 ? " (no convergence)" : " (bad argument)");
    return QIPB200_ERR_CUDA;
  }
  return QIPB200_OK;
}

void eig_handle_destroy(void *handle) {
  if (handle && cusolver().ok) cusolver().destroy((cusolverDnHandle_t)handle);
}

}  // namespace qipb200
