// indicator.cuh -- what the indicator builders share: shapes on a regular grid (indicator.cu) and
// shapes on shapes (overlay.cu).  The CSR handle, the keep rule and the host side of a call:
// device buffers, CUB scratch and the handle's lifetime.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

// Rows n_shapes, columns ny * nx; filled on the host from the device results and read with
// atl_indicator_nnz / _export.
struct AtlIndicator {
  int32_t n_shapes = 0, ny = 0, nx = 0;
  std::vector<int64_t> indptr;
  std::vector<int32_t> indices;
  std::vector<double> data;
};

namespace atl {

constexpr double kKeep = 1e-10;  // fractions at or below this are not stored

template <class T>
struct DevBuf {
  T* p = nullptr;
  ~DevBuf() { cudaFree(p); }
  cudaError_t alloc(size_t n) { return cudaMalloc((void**)&p, std::max<size_t>(n, 1) * sizeof(T)); }
};

// CUB scratch that grows as needed
struct Temp {
  DevBuf<char> buf;
  size_t bytes = 0;
  cudaError_t need(size_t b) {
    if (b <= bytes) return cudaSuccess;
    cudaFree(buf.p);
    buf.p = nullptr;
    bytes = 0;
    cudaError_t e = buf.alloc(b);
    if (e == cudaSuccess) bytes = b;
    return e;
  }
  // A two-phase CUB call cub(temp, bytes): the size query (temp = NULL), the scratch grown to fit,
  // then the call itself.
  template <class Cub>
  cudaError_t run(Cub&& cub) {
    size_t b = 0;
    cudaError_t e = cub(nullptr, b);
    if (e == cudaSuccess) e = need(b);
    return e == cudaSuccess ? cub(buf.p, b) : e;
  }
  // run(cub) for an exclusive scan whose input ends with a 0, then the scan's total, *last (its
  // last output), copied to the host.
  template <class Cub, class T>
  cudaError_t run(Cub&& cub, const T* last, T& total) {
    const cudaError_t e = run(cub);
    return e == cudaSuccess ? cudaMemcpy(&total, last, sizeof(T), cudaMemcpyDeviceToHost) : e;
  }
};

// The end of a call that filled R on the device with result rc: waits for the device, then hands R
// out through *out, or deletes it when anything failed.  `what` names the call in a CUDA error.
inline int hand_out(AtlIndicator* R, int rc, const char* what, AtlIndicator** out) {
  if (rc == ATL_OK) {
    const cudaError_t ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) rc = cuda_fail(ce, what);
  }
  if (rc != ATL_OK) {
    delete R;
    return rc;
  }
  *out = R;
  return ATL_OK;
}

}  // namespace atl
