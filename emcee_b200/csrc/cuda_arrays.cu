// The one kernel of the device-memory transfers (eb_set_state_from): the NaN check of an initial log_prob that
// never reaches the host.  Everything else those entry points do is copies on the copy engines (capi.cu).
#include <algorithm>

#include "engine.cuh"

namespace eb {
namespace {

// status |= flag when any of x[n] is NaN (ensemble.py:357-358 `np.any(np.isnan(log_prob))`): one vote per warp
__global__ void __launch_bounds__(256) flag_nan_kernel(const double* __restrict__ x, size_t n, int flag, int* status) {
  bool nan = false;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x)
    nan |= isnan(x[k]);
  if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(status, flag);
}

}  // namespace

cudaError_t launch_flag_nan(const double* x, size_t n, int flag, int* status, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, 1024);
  flag_nan_kernel<<<grid, 256, 0, st>>>(x, n, flag, status);
  return cudaGetLastError();
}

}  // namespace eb
