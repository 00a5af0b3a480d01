// Gather of a user red-blue move (eb_move_set_proposal): the rows a user get_proposal receives, s then c
// (red_blue.py:85-87 `s = coords[inds == split]`, `c = [coords[inds == j] for j != split]`), in one launch per
// half-step.  The split table `order` already lists the walkers grouped by set, ascending inside a set, so output row
// r reads walker
//   order[a_start + r]            r <  a_count             (the active set)
//   order[r - a_count]            a_count <= r < a_count + a_start   (the sets before it)
//   order[r]                      r >= a_count + a_start   (the sets after it)
// and the host gets s and c back to back with one contiguous copy.
#include "engine.cuh"

namespace eb {

namespace {

constexpr int GATHER_WARPS = 8;

// one warp per output row; V = double2 when rows are a whole number of 16-byte vectors (even D: cudaMalloc bases
// are 256-byte aligned, so every row is 16-byte aligned), else double
template <class V>
__global__ void __launch_bounds__(GATHER_WARPS * 32) split_gather_kernel(const V* __restrict__ coords,
                                                                         const int32_t* __restrict__ order, int64_t N,
                                                                         int a_start, int a_count, int64_t vpr,
                                                                         V* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * GATHER_WARPS + threadIdx.y;
  if (r >= N) return;
  const int64_t k = r < a_count ? a_start + r : (r < (int64_t)a_count + a_start ? r - a_count : r);
  const int64_t w = order[k];
  const V* src = coords + w * vpr;
  V* dst = out + r * vpr;
  for (int64_t v = threadIdx.x; v < vpr; v += 32) dst[v] = src[v];
}

}  // namespace

cudaError_t launch_split_gather(const double* coords, const int32_t* order, int64_t N, int D, int a_start, int a_count,
                                double* out, cudaStream_t st) {
  if (N <= 0) return cudaSuccess;
  const dim3 block(32, GATHER_WARPS);
  const unsigned grid = (unsigned)((N + GATHER_WARPS - 1) / GATHER_WARPS);
  if (D % 2 == 0)
    split_gather_kernel<double2><<<grid, block, 0, st>>>(reinterpret_cast<const double2*>(coords), order, N, a_start,
                                                         a_count, D / 2, reinterpret_cast<double2*>(out));
  else
    split_gather_kernel<double><<<grid, block, 0, st>>>(coords, order, N, a_start, a_count, D, out);
  return cudaGetLastError();
}

}  // namespace eb
