// spectrum.h -- eigenvalues of a Hermitian matrix on the device for qipb200_state_entanglement_spectrum (spectrum.cu).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>

namespace qipb200 {

// Largest side of qipb200_state_entanglement_spectrum: G is 4^13 double2 = 1 GiB (2^14 would be 4 GiB).
const uint32_t kSpectrumMaxSide = 13;

// Whether cuSOLVER could be loaded into this process (dlopen once, on the first call); *why gets the loader's reason
// when not.  Host-only: needs no device.
bool eig_solver_available(std::string *why);

// The device buffers of one eigen-solve of a K x K Hermitian matrix, allocated before the state is touched so that a
// refusal for memory leaves it as it was.
struct EigWork {
  double2 *G = nullptr;    // K x K, row-major; the solve overwrites it (one allocation with W and info)
  double *W = nullptr;     // K eigenvalues, ascending up to rounding
  double2 *work = nullptr;
  int *info = nullptr;
  int lwork = 0;
  uint32_t K = 0;
};

// Create the context's solver handle if *handle is null (on the current device), then allocate w for K x K from the
// stream-ordered pool of stream s.  Returns a QIPB200_* status and the reason in *err; QIPB200_ERR_OOM when a buffer
// cannot be allocated.
int eig_work_alloc(void **handle, uint32_t K, EigWork *w, cudaStream_t s, std::string *err);
void eig_work_free(EigWork *w, cudaStream_t s);

// Eigenvalues of the Hermitian matrix in w->G (cusolverDnZheevd, values only) into the host array eigs_asc (K doubles,
// ascending).  The solver runs on stream s; the stream is synchronised before and after.
int eig_solve(void *handle, EigWork *w, cudaStream_t s, double *eigs_asc, std::string *err);

// Destroy a handle eig_work_alloc created (qipb200_shutdown).
void eig_handle_destroy(void *handle);

}  // namespace qipb200
