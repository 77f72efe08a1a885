// indicator.cuh -- the CSR handle and keep rule shared by the indicator kernels: shapes on a
// regular grid (indicator.cu) and shapes on shapes (overlay.cu).
#pragma once
#include <stdint.h>

#include <vector>

namespace atl {

constexpr double kKeep = 1e-10;  // fractions at or below this are not stored

}  // namespace atl

// Rows n_shapes, columns ny * nx; filled on the host from the device results and read with
// atl_indicator_nnz / _export.
struct AtlIndicator {
  int32_t n_shapes = 0, ny = 0, nx = 0;
  std::vector<int64_t> indptr;
  std::vector<int32_t> indices;
  std::vector<double> data;
};
