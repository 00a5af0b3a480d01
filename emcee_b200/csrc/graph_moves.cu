// The two kernels around a captured proposal graph (eb_move_set_proposal_graphs): `stage` gathers a split's rows
// into the graph's static inputs s and c and fills its draws, `result` reads its static outputs q and factors into
// the engine.  The graph is launched between them on the engine's stream, so a half-step of a captured proposal
// needs no host synchronisation.
//
// Errors stay on the device, as around a log-probability graph (graph_fn.cu).  Once the status word holds any
// error, `stage` writes nothing and records the error, and `result` sets every factor to NaN, so the accept that
// follows rejects every row and the state freezes at the offending half-step.  A non-finite q raised by `result`
// itself is recorded by the launch's last block, which alone knows the verdict of every row.
#include <algorithm>

#include "draws.cuh"
#include "engine.cuh"

namespace eb {
namespace {

constexpr int GM_THREADS = 256;
constexpr int GM_WARPS = GM_THREADS / 32;

__device__ __forceinline__ void record_first_error(unsigned long long* err, unsigned long long tag, int flags) {
  atomicCAS(err, 0ull, tag | (unsigned long long)(flags & 0xff));
}

__device__ __forceinline__ bool finite2(double2 v) { return isfinite(v.x) && isfinite(v.y); }
__device__ __forceinline__ bool finite2(double v) { return isfinite(v); }
__device__ __forceinline__ bool has_inf(double2 v) { return isinf(v.x) || isinf(v.y); }
__device__ __forceinline__ bool has_inf(double v) { return isinf(v); }
__device__ __forceinline__ bool has_nan(double2 v) { return isnan(v.x) || isnan(v.y); }
__device__ __forceinline__ bool has_nan(double v) { return isnan(v); }

// blocks [0, gather_blocks): one warp per row r < N of s | c, split_gather_kernel's row mapping; the blocks after
// them: one thread per (row i < a_count, draw pair k).  V = double2 when every row of coords, s and c is a whole
// number of 16-byte aligned vectors.  Strides are in V.
template <class V>
__global__ void __launch_bounds__(GM_THREADS) graph_move_stage_kernel(
    const V* __restrict__ coords, const int32_t* __restrict__ order, int64_t N, int a_start, int a_count, int64_t vpr,
    V* __restrict__ s, int64_t s_stride, V* __restrict__ c, int64_t c_stride, unsigned gather_blocks,
    double* __restrict__ draws, int64_t d_stride, int normal, int64_t ndraws, uint64_t seed, uint64_t step,
    uint32_t split, const int* __restrict__ status, unsigned long long* err, unsigned long long tag) {
  const int f = *status;
  if (f != 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) record_first_error(err, tag, f);
    return;
  }
  if (blockIdx.x < gather_blocks) {
    const int64_t r = (int64_t)blockIdx.x * GM_WARPS + threadIdx.x / 32;
    if (r >= N) return;
    int64_t w = r;
    if (order) {
      const int64_t k = r < a_count ? a_start + r : (r < (int64_t)a_count + a_start ? r - a_count : r);
      w = order[k];
    }
    const V* src = coords + w * vpr;
    V* dst = r < a_count ? s + r * s_stride : c + (r - a_count) * c_stride;
    for (int64_t v = threadIdx.x % 32; v < vpr; v += 32) dst[v] = src[v];
    return;
  }
  const int64_t npair = (ndraws + 1) / 2;
  const int64_t t = (int64_t)(blockIdx.x - gather_blocks) * GM_THREADS + threadIdx.x;
  if (t >= (int64_t)a_count * npair) return;
  const int64_t i = t / npair;
  const int64_t k = t - i * npair;
  const u32x4 wd = draw_words(seed, step, sub_split(split, (uint32_t)k), TAG_GRAPH, (uint32_t)i);
  double d0, d1;
  graph_draw_pair(wd, normal, d0, d1);
  double* row = draws + i * d_stride;
  row[2 * k] = d0;
  if (2 * k + 1 < ndraws) row[2 * k + 1] = d1;
}

// one warp per row i < ns: qbuf[i] = q[i], f[i] = factors[i]; then the last block to finish applies the verdict
template <class V>
__global__ void __launch_bounds__(GM_THREADS) graph_move_result_kernel(
    const V* __restrict__ q, int64_t q_stride, int64_t vpr, const double* __restrict__ fsrc, int64_t f_stride,
    int64_t ns, V* __restrict__ qbuf, double* f, int* status, unsigned* ticket, unsigned long long* err,
    unsigned long long tag) {
  const int64_t r = (int64_t)blockIdx.x * GM_WARPS + threadIdx.x / 32;
  bool inf = false, nan = false;
  if (r < ns) {
    const V* src = q + r * q_stride;
    V* dst = qbuf + r * vpr;
    for (int64_t v = threadIdx.x % 32; v < vpr; v += 32) {
      const V x = src[v];
      dst[v] = x;
      if (!finite2(x)) {
        inf |= has_inf(x);
        nan |= has_nan(x);
      }
    }
    if (threadIdx.x % 32 == 0) f[r] = fsrc[r * f_stride];
  }
  const int flags = (__syncthreads_or(inf) ? FLAG_INF_PARAM : 0) | (__syncthreads_or(nan) ? FLAG_NAN_PARAM : 0);
  __shared__ bool last;
  __threadfence();  // this block's factors before its ticket: the last block may overwrite them
  __syncthreads();
  if (threadIdx.x == 0) {
    if (flags) atomicOr(status, flags);
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  const int fs = *(volatile int*)status;
  __syncthreads();
  if (threadIdx.x == 0) {
    *ticket = 0;
    if (fs != 0) record_first_error(err, tag, fs);
  }
  if (fs != 0)
    for (int64_t i = threadIdx.x; i < ns; i += blockDim.x) f[i] = __longlong_as_double(0x7ff8000000000000ll);
}

bool aligned16(const void* p, int64_t stride_doubles) {
  return ((uintptr_t)p % 16 == 0) && (stride_doubles % 2 == 0);
}

}  // namespace

cudaError_t launch_graph_move_stage(const double* coords, const int32_t* order, int64_t N, int D, int a_start,
                                    int a_count, const GraphMoveBufs& b, int normal, int64_t ndraws, uint64_t seed,
                                    uint64_t step, uint32_t split, const int* status, unsigned long long* err,
                                    unsigned long long tag, cudaStream_t st) {
  const unsigned gather_blocks = (unsigned)((N + GM_WARPS - 1) / GM_WARPS);
  const int64_t pairs = (int64_t)a_count * ((ndraws + 1) / 2);
  const unsigned grid = gather_blocks + (unsigned)((pairs + GM_THREADS - 1) / GM_THREADS);
  const int64_t nc = N - a_count;
  // cudaMalloc bases are 256-byte aligned: an even D makes every coords row 16-byte aligned
  const bool vec = D % 2 == 0 && aligned16(b.s, b.s_stride) && (nc == 0 || aligned16(b.c, b.c_stride));
  if (vec)
    graph_move_stage_kernel<double2><<<grid, GM_THREADS, 0, st>>>(
        reinterpret_cast<const double2*>(coords), order, N, a_start, a_count, D / 2, reinterpret_cast<double2*>(b.s),
        b.s_stride / 2, reinterpret_cast<double2*>(b.c), b.c_stride / 2, gather_blocks, b.draws, b.draws_stride, normal,
        ndraws, seed, step, split, status, err, tag);
  else
    graph_move_stage_kernel<double><<<grid, GM_THREADS, 0, st>>>(coords, order, N, a_start, a_count, D, b.s,
                                                                 b.s_stride, b.c, b.c_stride, gather_blocks, b.draws,
                                                                 b.draws_stride, normal, ndraws, seed, step, split,
                                                                 status, err, tag);
  return cudaGetLastError();
}

cudaError_t launch_graph_move_result(const GraphMoveBufs& b, int64_t ns, int D, double* qbuf, double* f, int* status,
                                     unsigned* ticket, unsigned long long* err, unsigned long long tag,
                                     cudaStream_t st) {
  const unsigned grid = (unsigned)std::max<int64_t>(1, (ns + GM_WARPS - 1) / GM_WARPS);
  if (D % 2 == 0 && aligned16(b.q, b.q_stride))
    graph_move_result_kernel<double2><<<grid, GM_THREADS, 0, st>>>(
        reinterpret_cast<const double2*>(b.q), b.q_stride / 2, D / 2, b.f, b.f_stride, ns,
        reinterpret_cast<double2*>(qbuf), f, status, ticket, err, tag);
  else
    graph_move_result_kernel<double><<<grid, GM_THREADS, 0, st>>>(b.q, b.q_stride, D, b.f, b.f_stride, ns, qbuf, f,
                                                                  status, ticket, err, tag);
  return cudaGetLastError();
}

}  // namespace eb
