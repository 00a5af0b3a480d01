// Running reservoir (eb_reservoir_config / eb_reservoir_read): a uniform sample without replacement of K of the
// (step, walker) rows a run records, kept in device memory however long the run is.  reservoir_plan.h states what is
// kept and when the buffer is compacted; this file holds the kernels.
//
//   record    res_filter_kernel, one thread per walker: the row's tag-10 key, the filter, a warp-aggregated append,
//             and the warp copies each surviving row with 16-byte loads (8-byte for odd ndim).  A row that fails
//             reads nothing of the state.
//   compact   res_begin_kernel, RES_PASSES x res_hist_kernel (shared-memory histogram of one digit; the last block
//             to finish picks the digit, so the decisions stay on the device), res_mark_kernel (holes below K, keepers
//             from K on, the boundary group), res_group_kernel (orders a boundary group of more than the wanted
//             number of entries by (step, walker, buffer index)), res_move_kernel (keepers into the holes, count = K).
//   read      keys, steps and walkers to the host, sorted there; the rows follow in that order.
#include <algorithm>
#include <numeric>
#include <vector>

#include "engine.cuh"
#include "philox.cuh"
#include "reservoir_plan.h"

namespace eb {

struct ResCtl {
  unsigned long long count;   // live entries
  unsigned long long tau;     // the K-th key, once full
  unsigned long long prefix;  // the select: digits chosen so far (ResSelect)
  unsigned long long rank;
  unsigned long long group_size;  // entries with the K-th key (set by the last pass)
  unsigned int full;
  unsigned int active;  // this compaction has more than K entries to cut
  unsigned int ticket;  // blocks of the running pass that are done
  unsigned int nhole, nmove, ngroup;
  unsigned int hist[RES_BINS];
};

namespace {

constexpr int RES_THREADS = 256;
constexpr int RES_WARPS = RES_THREADS / 32;

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// slot of each lane with `pred` set in a run of appends to *ctr: one atomic per warp; every lane of the warp calls it
template <class T>
__device__ __forceinline__ T warp_append(bool pred, T* ctr) {
  const unsigned mask = __ballot_sync(0xffffffffu, pred);
  const int lane = threadIdx.x & 31, leader = mask ? __ffs(mask) - 1 : 0;
  T base = 0;
  if (mask && lane == leader) base = atomicAdd(ctr, (T)__popc(mask));
  base = __shfl_sync(0xffffffffu, base, leader);
  return base + (T)__popc(mask & lanemask_lt());
}

// the warp copies row `src` of x to row `dst` of y, D doubles each
template <bool VEC>
__device__ __forceinline__ void warp_copy_row(const double* __restrict__ x, size_t src, double* __restrict__ y,
                                              size_t dst, int D, int lane) {
  if (VEC) {
    const double2* s = reinterpret_cast<const double2*>(x + src * D);
    double2* d = reinterpret_cast<double2*>(y + dst * D);
    for (int j = lane; j < D / 2; j += 32) d[j] = s[j];
  } else {
    const double* s = x + src * D;
    double* d = y + dst * D;
    for (int j = lane; j < D; j += 32) d[j] = s[j];
  }
}

template <bool VEC>
__global__ void __launch_bounds__(RES_THREADS) res_filter_kernel(LiveReservoir r, unsigned long long seed,
                                                                 unsigned long long step) {
  const uint32_t w = blockIdx.x * RES_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool in = w < r.N;
  const unsigned long long key = in ? reservoir_key(seed, step, w) : 0ull;
  const bool pass = in && res_passes(r.ctl->full != 0, r.ctl->tau, key);
  unsigned mask = __ballot_sync(0xffffffffu, pass);
  if (!mask) return;
  const unsigned long long slot = warp_append(pass, &r.ctl->count);
  if (pass) {
    r.key[slot] = key;
    r.step[slot] = step;
    r.walker[slot] = w;
    r.lp[slot] = r.logp[w];
  }
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const uint32_t ws = __shfl_sync(0xffffffffu, w, src);
    const unsigned long long s = __shfl_sync(0xffffffffu, slot, src);
    warp_copy_row<VEC>(r.coords, ws, r.x, s, r.D, lane);
  }
}

__global__ void res_begin_kernel(ResCtl* ctl, unsigned long long K) {
  ctl->hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    ctl->active = ctl->count > K ? 1u : 0u;
    const ResSelect s = res_select_start(K);
    ctl->prefix = s.prefix;
    ctl->rank = s.rank;
    ctl->ticket = 0;
    ctl->nhole = ctl->nmove = ctl->ngroup = 0;
  }
}

// pass `pass` of the select: counts digit `pass` of the live keys that match the prefix; the last block picks the
// digit, moves the prefix and the rank on, and clears the histogram for the next pass
__global__ void __launch_bounds__(RES_THREADS) res_hist_kernel(const unsigned long long* __restrict__ key,
                                                               ResCtl* ctl, int pass) {
  if (!ctl->active) return;
  __shared__ unsigned sh[RES_BINS];
  __shared__ unsigned long long scan[RES_BINS];
  __shared__ bool last;
  const unsigned long long count = ctl->count, prefix = ctl->prefix;
  sh[threadIdx.x] = 0;
  __syncthreads();
  for (unsigned long long i = blockIdx.x * RES_THREADS + threadIdx.x; i < count; i += (size_t)gridDim.x * RES_THREADS) {
    const unsigned long long k = key[i];
    if (res_in_prefix(k, prefix, pass)) atomicAdd(&sh[res_digit(k, pass)], 1u);
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&ctl->hist[threadIdx.x], sh[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&ctl->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  const unsigned long long here = *(volatile unsigned*)&ctl->hist[threadIdx.x];
  scan[threadIdx.x] = here;  // inclusive scan over the bins
  __syncthreads();
  for (int o = 1; o < RES_BINS; o <<= 1) {
    const unsigned long long v = threadIdx.x >= o ? scan[threadIdx.x - o] : 0ull;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  const unsigned long long below = scan[threadIdx.x] - here;
  const unsigned long long rank = ctl->rank;
  __syncthreads();
  if (res_digit_holds(below, here, rank)) {
    ResSelect s{prefix, rank};
    res_take_digit(s, pass, threadIdx.x, below);
    ctl->prefix = s.prefix;
    ctl->rank = s.rank;
    ctl->group_size = here;
  }
  ctl->hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) ctl->ticket = 0;
}

// entry i is kept when its key is below the K-th key T, or is T and the whole group of T is kept; an entry of a group
// that has to be cut is listed for res_group_kernel.  Holes are dropped entries below K, movers kept entries from K on.
__global__ void __launch_bounds__(RES_THREADS) res_mark_kernel(LiveReservoir r) {
  ResCtl* ctl = r.ctl;
  if (!ctl->active) return;
  const unsigned long long count = ctl->count, T = ctl->prefix, need = ctl->rank + 1, g = ctl->group_size;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ctl->tau = T;
    ctl->full = 1;
  }
  const int warp = (blockIdx.x * RES_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const unsigned long long nwarps = (unsigned long long)gridDim.x * RES_WARPS;
  for (unsigned long long i0 = (unsigned long long)warp * 32; i0 < count; i0 += nwarps * 32) {
    const unsigned long long i = i0 + lane;
    const bool in = i < count;
    const unsigned long long k = in ? r.key[i] : 0ull;
    const bool grouped = in && k == T && g != need;
    const bool kept = in && (k < T || (k == T && g == need));
    const bool hole = in && !grouped && i < r.K && !kept;
    const bool mover = in && !grouped && i >= r.K && kept;
    const unsigned gs = warp_append(grouped, &ctl->ngroup);
    if (grouped) r.group[gs] = (uint32_t)i;
    const unsigned hs = warp_append(hole, &ctl->nhole);
    if (hole) r.holes[hs] = (uint32_t)i;
    const unsigned ms = warp_append(mover, &ctl->nmove);
    if (mover) r.movers[ms] = (uint32_t)i;
  }
}

// a boundary group larger than the entries it may keep: the first `need` by (step, walker, buffer index) stay
// (quadratic in the group, which has one entry unless two keys collide)
__global__ void __launch_bounds__(RES_THREADS) res_group_kernel(LiveReservoir r) {
  ResCtl* ctl = r.ctl;
  if (!ctl->active) return;
  const unsigned n = ctl->ngroup;
  const unsigned long long need = ctl->rank + 1;
  for (unsigned j = threadIdx.x; j < n; j += RES_THREADS) {
    const uint32_t e = r.group[j];
    unsigned long long before = 0;
    for (unsigned o = 0; o < n; ++o) {
      const uint32_t f = r.group[o];
      before += res_entry_before(r.step[f], r.walker[f], f, r.step[e], r.walker[e], e) ? 1 : 0;
    }
    const bool kept = before < need;
    if (e < r.K && !kept) r.holes[atomicAdd(&ctl->nhole, 1u)] = e;
    if (e >= r.K && kept) r.movers[atomicAdd(&ctl->nmove, 1u)] = e;
  }
}

template <bool VEC>
__global__ void __launch_bounds__(RES_THREADS) res_move_kernel(LiveReservoir r) {
  ResCtl* ctl = r.ctl;
  if (!ctl->active) return;
  const unsigned n = min(ctl->nmove, ctl->nhole);  // equal: exactly K entries are kept
  if (blockIdx.x == 0 && threadIdx.x == 0) ctl->count = r.K;
  const int lane = threadIdx.x & 31;
  for (unsigned j = (blockIdx.x * RES_THREADS + threadIdx.x) >> 5; j < n; j += gridDim.x * RES_WARPS) {
    const uint32_t src = r.movers[j], dst = r.holes[j];
    if (lane == 0) {
      r.key[dst] = r.key[src];
      r.step[dst] = r.step[src];
      r.walker[dst] = r.walker[src];
      r.lp[dst] = r.lp[src];
    }
    warp_copy_row<VEC>(r.x, src, r.x, dst, r.D, lane);
  }
}

// out row j = entry order[j]
template <bool VEC>
__global__ void __launch_bounds__(RES_THREADS) res_gather_kernel(LiveReservoir r, unsigned n, double* __restrict__ x,
                                                                 double* __restrict__ lp) {
  const int lane = threadIdx.x & 31;
  for (unsigned j = (blockIdx.x * RES_THREADS + threadIdx.x) >> 5; j < n; j += gridDim.x * RES_WARPS) {
    const uint32_t e = r.group[j];
    if (lp && lane == 0) lp[j] = r.lp[e];
    if (x) warp_copy_row<VEC>(r.x, e, x, j, r.D, lane);
  }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

unsigned grid_for(uint64_t items, uint64_t per_block, int sm_count) {
  const uint64_t g = (items + per_block - 1) / per_block;
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(g, 4 * (uint64_t)std::max(sm_count, 1)));
}

}  // namespace

size_t live_reservoir_bytes(uint64_t K, uint32_t N, int D) {
  const size_t cap = (size_t)res_cap(K, N);
  return align256(cap * (size_t)D * sizeof(double)) + align256(cap * sizeof(double)) +
         2 * align256(cap * sizeof(unsigned long long)) + 2 * align256(cap * sizeof(uint32_t)) +
         2 * align256((size_t)K * sizeof(uint32_t)) + align256(sizeof(ResCtl));
}

cudaError_t live_reservoir_setup(LiveReservoir* r, void* mem, uint64_t K, uint32_t N, int D, const double* coords,
                                 const double* logp, int sm_count, cudaStream_t st) {
  const size_t cap = (size_t)res_cap(K, N);
  char* p = static_cast<char*>(mem);
  auto take = [&p](size_t bytes) {
    char* q = p;
    p += align256(bytes);
    return q;
  };
  *r = LiveReservoir{};
  r->N = N;
  r->D = D;
  r->K = K;
  r->cap = cap;
  r->sm_count = sm_count;
  r->coords = coords;
  r->logp = logp;
  r->x = reinterpret_cast<double*>(take(cap * (size_t)D * sizeof(double)));
  r->lp = reinterpret_cast<double*>(take(cap * sizeof(double)));
  r->key = reinterpret_cast<unsigned long long*>(take(cap * sizeof(unsigned long long)));
  r->step = reinterpret_cast<unsigned long long*>(take(cap * sizeof(unsigned long long)));
  r->walker = reinterpret_cast<uint32_t*>(take(cap * sizeof(uint32_t)));
  r->group = reinterpret_cast<uint32_t*>(take(cap * sizeof(uint32_t)));
  r->holes = reinterpret_cast<uint32_t*>(take((size_t)K * sizeof(uint32_t)));
  r->movers = reinterpret_cast<uint32_t*>(take((size_t)K * sizeof(uint32_t)));
  r->ctl = reinterpret_cast<ResCtl*>(take(sizeof(ResCtl)));
  cudaError_t e = cudaMemsetAsync(r->ctl, 0, sizeof(ResCtl), st);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(st);
}

cudaError_t live_reservoir_record(const LiveReservoir& r, uint64_t seed, uint64_t step, cudaStream_t st,
                                  uint64_t& launches) {
  const unsigned grid = (r.N + RES_THREADS - 1) / RES_THREADS;
  if (r.D % 2 == 0)
    res_filter_kernel<true><<<grid, RES_THREADS, 0, st>>>(r, seed, step);
  else
    res_filter_kernel<false><<<grid, RES_THREADS, 0, st>>>(r, seed, step);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  launches += 1;
  return cudaSuccess;
}

cudaError_t live_reservoir_compact(const LiveReservoir& r, uint64_t bound, cudaStream_t st, uint64_t& launches) {
  res_begin_kernel<<<1, RES_BINS, 0, st>>>(r.ctl, r.K);
  const unsigned g = grid_for(bound, 4 * RES_THREADS, r.sm_count);
  for (int pass = 0; pass < RES_PASSES; ++pass) res_hist_kernel<<<g, RES_THREADS, 0, st>>>(r.key, r.ctl, pass);
  res_mark_kernel<<<g, RES_THREADS, 0, st>>>(r);
  res_group_kernel<<<1, RES_THREADS, 0, st>>>(r);
  // at most min(K, bound - K) entries move, one warp each
  const uint64_t moves = bound > r.K ? std::min<uint64_t>(r.K, bound - r.K) : 1;
  const unsigned gm = grid_for(moves, RES_WARPS, r.sm_count);
  if (r.D % 2 == 0)
    res_move_kernel<true><<<gm, RES_THREADS, 0, st>>>(r);
  else
    res_move_kernel<false><<<gm, RES_THREADS, 0, st>>>(r);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  launches += 4 + RES_PASSES;
  return cudaSuccess;
}

cudaError_t live_reservoir_read(const LiveReservoir& r, uint64_t kept, double* coords, double* lp, uint64_t* step,
                                int64_t* walker, bool device_out, cudaStream_t st) {
  if (kept == 0) return cudaSuccess;
  const size_t n = (size_t)kept, D = (size_t)r.D;
  std::vector<unsigned long long> k(n), s(n);
  std::vector<uint32_t> w(n);
  cudaError_t e = cudaMemcpyAsync(k.data(), r.key, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(s.data(), r.step, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(w.data(), r.walker, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return e;
  std::vector<uint32_t> order(n);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    return k[a] != k[b] ? k[a] < k[b] : res_row_before(s[a], w[a], s[b], w[b]);
  });
  for (size_t j = 0; j < n; ++j) {
    if (step) step[j] = s[order[j]];
    if (walker) walker[j] = (int64_t)w[order[j]];
  }
  if (!coords && !lp) return cudaSuccess;
  if (device_out) {
    e = cudaMemcpyAsync(r.group, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    const unsigned g = grid_for(n, RES_WARPS, r.sm_count);
    if (D % 2 == 0 && ((uintptr_t)coords & 15) == 0)  // 16-byte stores into a caller's buffer that allows them
      res_gather_kernel<true><<<g, RES_THREADS, 0, st>>>(r, (unsigned)n, coords, lp);
    else
      res_gather_kernel<false><<<g, RES_THREADS, 0, st>>>(r, (unsigned)n, coords, lp);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(st);
  }
  std::vector<double> x(coords ? n * D : 0), l(lp ? n : 0);
  if (coords) e = cudaMemcpyAsync(x.data(), r.x, n * D * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && lp) e = cudaMemcpyAsync(l.data(), r.lp, n * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return e;
  for (size_t j = 0; j < n; ++j) {
    if (coords) std::copy(x.begin() + order[j] * D, x.begin() + (order[j] + 1) * D, coords + j * D);
    if (lp) lp[j] = l[order[j]];
  }
  return cudaSuccess;
}

}  // namespace eb
