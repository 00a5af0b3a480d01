// The two kernels around a captured log-probability graph (eb_model_set_graphs): `stage` copies a split's rows into
// the graph's static input, `result` reads its static output into the engine's lp buffer.  The graph is launched
// between them on the engine's stream, so a half-step of a graph model needs no host synchronisation.
//
// Errors stay on the device.  Once the status word holds any error, `stage` copies nothing (the graph never sees a
// non-finite row from the caller or a move, ensemble.py:476-479; it runs on what x last held, which may be its own
// writes, and its output is discarded) and `result` writes NaN into every lp entry, so the accept kernel that follows
// rejects every row and the state, the accept counters and the log-probabilities freeze at the offending half-step.
// The first error is recorded once, as flags | split << 8 | step << 16 (graph_err_word), for the host to report.
#include <algorithm>

#include "engine.cuh"

namespace eb {
namespace {

__device__ __forceinline__ void record_first(unsigned long long* err, unsigned long long tag, int flags) {
  atomicCAS(err, 0ull, tag | (unsigned long long)(flags & 0xff));
}

// x[r] = src[min(r, rows - 1)] for r < m: the last real row pads the rows of a short chunk
__global__ void __launch_bounds__(256) graph_stage_kernel(const double* __restrict__ src, int64_t rows, int64_t m, int D,
                                                          double* __restrict__ x, int64_t x_stride,
                                                          const int* __restrict__ status, unsigned long long* err,
                                                          unsigned long long tag) {
  const int f = *status;
  if (f != 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) record_first(err, tag, f);
    return;
  }
  const size_t n = (size_t)m * (size_t)D;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
    const int64_t r = (int64_t)(k / (size_t)D);
    const int e = (int)(k - (size_t)r * D);
    const int64_t s = r < rows ? r : rows - 1;
    x[r * x_stride + e] = src[(size_t)s * D + e];
  }
}

// out[i] = lp[i * lp_stride] for i < rows; a NaN raises FLAG_NAN_LOGPROB at this half-step (ensemble.py:550-551).
// One block: whether any entry is NaN decides what every entry becomes.
__global__ void __launch_bounds__(GRAPH_RESULT_THREADS) graph_result_kernel(const double* __restrict__ lp,
                                                                            int64_t lp_stride, int64_t rows,
                                                                            double* __restrict__ out, int* status,
                                                                            unsigned long long* err,
                                                                            unsigned long long tag) {
  bool nan = false;
  for (int64_t i = threadIdx.x; i < rows; i += blockDim.x) {
    const double v = lp[i * lp_stride];
    nan |= isnan(v);
    out[i] = v;
  }
  const bool any_nan = __syncthreads_or(nan) != 0;
  const int f = *status;  // the errors of earlier launches; this block's own flag is raised below
  __syncthreads();
  if (any_nan && threadIdx.x == 0) {
    atomicOr(status, FLAG_NAN_LOGPROB);
    record_first(err, tag, f | FLAG_NAN_LOGPROB);
  }
  if (any_nan || f != 0)
    for (int64_t i = threadIdx.x; i < rows; i += blockDim.x) out[i] = __longlong_as_double(0x7ff8000000000000ll);
}

}  // namespace

cudaError_t launch_graph_stage(const double* src, int64_t rows, int64_t m, int D, double* x, int64_t x_stride_bytes,
                               const int* status, unsigned long long* err, unsigned long long tag, cudaStream_t st) {
  const size_t n = (size_t)m * (size_t)D;
  const unsigned grid = (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, 4096));
  graph_stage_kernel<<<grid, 256, 0, st>>>(src, rows, m, D, x, x_stride_bytes / (int64_t)sizeof(double), status, err,
                                           tag);
  return cudaGetLastError();
}

cudaError_t launch_graph_result(const double* lp, int64_t lp_stride_bytes, int64_t rows, double* out, int* status,
                                unsigned long long* err, unsigned long long tag, cudaStream_t st) {
  graph_result_kernel<<<1, GRAPH_RESULT_THREADS, 0, st>>>(lp, lp_stride_bytes / (int64_t)sizeof(double), rows, out,
                                                          status, err, tag);
  return cudaGetLastError();
}

}  // namespace eb
