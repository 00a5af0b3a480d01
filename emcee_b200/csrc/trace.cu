// Running trace of the live state (eb_trace_config / eb_trace_read / eb_trace_best): one row of ensemble statistics
// per recorded step, for runs that store no chain.  Two launches per recorded step, both behind the step on the
// engine's stream: trace_partial_kernel reads the [N, D] state once and leaves one partial sum per chunk of rows,
// trace_finish_kernel folds the chunks, writes the row and keeps the best sample.  The order of every floating-point
// addition is the one trace_sum.h lays down, so a row does not depend on the launch.
#include <algorithm>

#include "engine.cuh"
#include "trace_sum.h"

namespace eb {
namespace {

constexpr int TRACE_LANES = 16;                // threads across a column tile, two columns each
constexpr int TRACE_TILE = 2 * TRACE_LANES;    // columns per block
constexpr int TRACE_THREADS = TRACE_LANES * TRACE_CHUNK_LEAVES;
constexpr int TRACE_LOAD = 8;                  // rows whose loads are in flight together in one thread
constexpr int FINISH_COLS = 32, FINISH_LANES = 32;

// Block (chunk, tile): thread (lane, leaf) sums the TRACE_LEAF_ROWS rows of its leaf for columns j, j + 1 about
// walker 0's row; the leaves meet in shared memory in leaf order.  VEC (D even): every row starts 16 bytes aligned
// and the two columns are one double2 load; an odd D leaves odd rows 8 bytes off, so it loads scalars.  The blocks of
// tile 0 also reduce the chunk's log-probabilities and accept mask.  partial[chunk] = [S1 D | S2 D | TraceLp].
template <bool VEC>
__global__ void __launch_bounds__(TRACE_THREADS, 4)
    trace_partial_kernel(const double* __restrict__ x, const double* __restrict__ logp,
                         const uint8_t* __restrict__ acc, uint32_t N, int D, double* __restrict__ partial) {
  __shared__ double sm[TRACE_CHUNK_LEAVES][TRACE_LANES][4];
  __shared__ TraceLp slp[TRACE_CHUNK_LEAVES];
  const int lane = threadIdx.x % TRACE_LANES, leaf = threadIdx.x / TRACE_LANES;
  const uint32_t chunk = blockIdx.x;
  const int j = blockIdx.y * TRACE_TILE + 2 * lane;
  const uint32_t c0 = chunk * (uint32_t)TRACE_CHUNK_ROWS;
  const uint32_t r0 = c0 + leaf * TRACE_LEAF_ROWS;
  const uint32_t r1 = min(N, r0 + (uint32_t)TRACE_LEAF_ROWS);
  const bool has0 = j < D, has1 = j + 1 < D;
  double a1 = 0.0, a2 = 0.0, b1 = 0.0, b2 = 0.0;
  if (has0 && r0 < N) {
    const double sh0 = x[j], sh1 = has1 ? x[j + 1] : 0.0;
    const double* p = x + (size_t)r0 * D + j;
    if (VEC) {
      uint32_t r = r0;
      for (; r + TRACE_LOAD <= r1; r += TRACE_LOAD, p += (size_t)TRACE_LOAD * D) {
        double2 v[TRACE_LOAD];
#pragma unroll
        for (int k = 0; k < TRACE_LOAD; ++k) v[k] = *reinterpret_cast<const double2*>(p + (size_t)k * D);
#pragma unroll
        for (int k = 0; k < TRACE_LOAD; ++k) {
          trace_term(v[k].x, sh0, a1, a2);
          trace_term(v[k].y, sh1, b1, b2);
        }
      }
      for (; r < r1; ++r, p += D) {
        const double2 v = *reinterpret_cast<const double2*>(p);
        trace_term(v.x, sh0, a1, a2);
        trace_term(v.y, sh1, b1, b2);
      }
    } else {
#pragma unroll 4
      for (uint32_t r = r0; r < r1; ++r, p += D) {
        trace_term(p[0], sh0, a1, a2);
        if (has1) trace_term(p[1], sh1, b1, b2);
      }
    }
  }
  sm[leaf][lane][0] = a1;
  sm[leaf][lane][1] = b1;
  sm[leaf][lane][2] = a2;
  sm[leaf][lane][3] = b2;
  if (blockIdx.y == 0 && lane == 0 && r0 < N) {
    TraceLp t = trace_lp_first(logp[r0], r0, acc[r0]);
    for (uint32_t r = r0 + 1; r < r1; ++r) trace_lp_term(t, logp[r], r, acc[r]);
    slp[leaf] = t;
  }
  __syncthreads();
  const int nleaves = (int)((min(N, c0 + (uint32_t)TRACE_CHUNK_ROWS) - c0 + TRACE_LEAF_ROWS - 1) / TRACE_LEAF_ROWS);
  double* out = partial + (size_t)chunk * (2 * D + TRACE_EXTRA);
  if (threadIdx.x < 4 * TRACE_LANES) {
    const int l = threadIdx.x / 4, k = threadIdx.x % 4;
    const int col = blockIdx.y * TRACE_TILE + 2 * l + (k & 1);
    if (col < D) {
      double v = sm[0][l][k];
      for (int f = 1; f < nleaves; ++f) v = trace_add(v, sm[f][l][k]);
      out[(k < 2 ? 0 : D) + col] = v;
    }
  } else if (threadIdx.x == 4 * TRACE_LANES && blockIdx.y == 0) {
    TraceLp t = slp[0];
    for (int f = 1; f < nleaves; ++f) trace_lp_join(t, slp[f]);
    *reinterpret_cast<TraceLp*>(out + 2 * D) = t;
  }
}

// Folds the n chunk sums in place with trace_sum.h's tree and writes the row.  Blocks 0 .. gridDim.x - 2 own
// FINISH_COLS columns each (S1 and S2 of a column in one thread); the last block folds the log-probability side,
// and replaces the best sample when this step's maximum is larger than every earlier one.
__global__ void __launch_bounds__(FINISH_COLS * FINISH_LANES)
    trace_finish_kernel(const double* __restrict__ x, uint32_t N, int D, double* __restrict__ partial, uint32_t n,
                        double* __restrict__ row, unsigned long long step, TraceBest* __restrict__ best,
                        double* __restrict__ best_coords) {
  const size_t W = 2 * (size_t)D + TRACE_EXTRA;
  const int tx = threadIdx.x % FINISH_COLS, ty = threadIdx.x / FINISH_COLS;
  if (blockIdx.x + 1 < gridDim.x) {
    const int j = blockIdx.x * FINISH_COLS + tx;
    for (uint32_t s = (uint32_t)trace_tree_start(n); s >= 1; s >>= 1) {
      if (j < D)
        for (uint32_t i = ty; i < s && i + s < n; i += FINISH_LANES) {
          double* a = partial + i * W + j;
          const double* b = partial + (i + s) * W + j;
          a[0] = trace_add(a[0], b[0]);
          a[D] = trace_add(a[D], b[D]);
        }
      __syncthreads();
    }
    if (ty == 0 && j < D) {
      row[j] = trace_mean(x[j], partial[j], N);
      row[D + j] = trace_var(partial[j], partial[D + j], N);
    }
    return;
  }
  __shared__ unsigned long long take;  // walker + 1 when the best sample is replaced
  for (uint32_t s = (uint32_t)trace_tree_start(n); s >= 1; s >>= 1) {
    for (uint32_t i = threadIdx.x; i < s && i + s < n; i += blockDim.x)
      trace_lp_join(*reinterpret_cast<TraceLp*>(partial + i * W + 2 * D),
                    *reinterpret_cast<const TraceLp*>(partial + (i + s) * W + 2 * D));
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const TraceLp t = *reinterpret_cast<const TraceLp*>(partial + 2 * D);
    row[2 * D] = __ddiv_rn(t.sum, (double)N);
    row[2 * D + 1] = t.max;
    row[2 * D + 2] = t.accepted;
    row[2 * D + 3] = t.walker;
    take = 0;
    if (!best->have || t.max > best->log_prob) {  // a tie keeps the earlier step
      best->have = 1;
      best->log_prob = t.max;
      best->step = step;
      best->walker = (unsigned long long)t.walker;
      take = best->walker + 1;
    }
  }
  __syncthreads();
  if (take)
    for (int j = threadIdx.x; j < D; j += blockDim.x) best_coords[j] = x[(size_t)(take - 1) * D + j];
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

size_t live_trace_fixed_bytes(uint32_t N, int D) {
  const size_t W = 2 * (size_t)D + TRACE_EXTRA;
  return align256(trace_nchunks(N) * W * sizeof(double)) + align256(sizeof(TraceBest)) +
         align256((size_t)D * sizeof(double));
}

cudaError_t live_trace_setup(LiveTrace* t, void* mem, uint32_t N, int D, const double* coords, const double* logp,
                             const uint8_t* accepted, cudaStream_t st) {
  const size_t W = 2 * (size_t)D + TRACE_EXTRA;
  char* p = static_cast<char*>(mem);
  *t = LiveTrace{};
  t->N = N;
  t->D = D;
  t->coords = coords;
  t->logp = logp;
  t->accepted = accepted;
  t->mem = mem;
  t->partial = reinterpret_cast<double*>(p);
  p += align256(trace_nchunks(N) * W * sizeof(double));
  t->best = reinterpret_cast<TraceBest*>(p);
  p += align256(sizeof(TraceBest));
  t->best_coords = reinterpret_cast<double*>(p);
  cudaError_t e = cudaMemsetAsync(t->best, 0, sizeof(TraceBest), st);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(st);
}

cudaError_t live_trace_launch(const LiveTrace& t, double* row, uint64_t step, cudaStream_t st, uint64_t& launches) {
  const uint32_t n = (uint32_t)trace_nchunks(t.N);
  const dim3 grid(n, (unsigned)((t.D + TRACE_TILE - 1) / TRACE_TILE));
  if (t.D % 2 == 0)
    trace_partial_kernel<true><<<grid, TRACE_THREADS, 0, st>>>(t.coords, t.logp, t.accepted, t.N, t.D, t.partial);
  else
    trace_partial_kernel<false><<<grid, TRACE_THREADS, 0, st>>>(t.coords, t.logp, t.accepted, t.N, t.D, t.partial);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const unsigned fin = (unsigned)((t.D + FINISH_COLS - 1) / FINISH_COLS) + 1;
  trace_finish_kernel<<<fin, FINISH_COLS * FINISH_LANES, 0, st>>>(t.coords, t.N, t.D, t.partial, n, row,
                                                                   (unsigned long long)step, t.best, t.best_coords);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  launches += 2;
  return cudaSuccess;
}

cudaError_t live_trace_best(const LiveTrace& t, TraceBest* best, double* coords, cudaStream_t st) {
  cudaError_t e = cudaMemcpyAsync(best, t.best, sizeof(TraceBest), cudaMemcpyDeviceToHost, st);
  if (e != cudaSuccess) return e;
  if (coords) {
    e = cudaMemcpyAsync(coords, t.best_coords, (size_t)t.D * sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return e;
  }
  return cudaStreamSynchronize(st);
}

}  // namespace eb
