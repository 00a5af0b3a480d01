// Running autocorrelation function of the live state (eb_running_acf_config / eb_running_acf_read): per (walker,
// parameter) series, the lag sums S(tau) for tau <= max_lag, kept in device memory of a fixed size however long the
// run is, for runs that store no chain.  Every recorded step only writes the shifted state into a ring
// (racf_record_kernel); every RACF_B recorded steps racf_fold_kernel adds the block's lag products into the
// double-double sums, reading and writing each S(tau) once.  A read folds the pending values of the unfinished block
// into copies, combines, normalises and averages over the walkers (racf_read_kernel, racf_finish_kernel); only rho
// crosses PCIe.  Every floating-point operation is the one running_acf.h lays down, in its order.
#include <algorithm>

#include "engine.cuh"
#include "running_acf.h"

namespace eb {
namespace {

// racf_fold_kernel tiling: FOLD_TS series per block (one per lane of a warp), FOLD_LY warps across the lags, each
// thread FOLD_TR lags of one series; a lag tile is FOLD_TL = FOLD_LY * FOLD_TR lags.  The products of a chunk of
// FOLD_KC block values meet the FOLD_KC + FOLD_TR - 1 history values they need in registers (a Hankel tile).
constexpr int FOLD_TS = 32, FOLD_LY = 4, FOLD_TR = 8, FOLD_KC = 8;
constexpr int FOLD_TL = FOLD_LY * FOLD_TR;
constexpr int FOLD_THREADS = FOLD_TS * FOLD_LY;
constexpr int FOLD_WIN = RACF_B + FOLD_TL - 1;
constexpr int READ_BATCH = 16;  // lags whose per-walker ratios meet in shared memory together
constexpr int FINISH_THREADS = 256;

__global__ void racf_record_kernel(const double* __restrict__ x, uint64_t ND, uint64_t n, uint64_t ring_rows,
                                   uint64_t max_lag, double* __restrict__ x0, double* __restrict__ ring,
                                   double* __restrict__ head) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= ND) return;
  const double v = x[s];
  double y = 0.0;
  if (n == 0) x0[s] = v;
  else y = __dsub_rn(v, x0[s]);
  ring[(n % ring_rows) * ND + s] = y;
  if (n < max_lag) head[n * ND + s] = y;
}

// Block b of every series: S(tau) += sum_k y_{bB+k} y_{bB+k-tau} for tau <= max_lag, and each y_{bB+k} added into
// the double-double Y.  Values below index 0, or older than the ring keeps, are staged as 0; so are the rows only lags
// past max_lag read, and the warps whose lags all lie past max_lag skip their products (the last tile of a max_lag
// that is not a multiple of FOLD_TL).  Ring slots are found from one 64-bit remainder per block.
__global__ void __launch_bounds__(FOLD_THREADS)
    racf_fold_kernel(const double* __restrict__ ring, uint64_t ring_rows, uint64_t ND, uint64_t b, uint64_t max_lag,
                     double* __restrict__ s_hi, double* __restrict__ s_lo, double* __restrict__ y_hi,
                     double* __restrict__ y_lo) {
  __shared__ double v[RACF_B][FOLD_TS];
  __shared__ double win[FOLD_WIN][FOLD_TS];
  const int tx = threadIdx.x % FOLD_TS, ly = threadIdx.x / FOLD_TS;
  const uint64_t s = (uint64_t)blockIdx.x * FOLD_TS + tx;
  const bool live = s < ND;
  const int64_t bB = (int64_t)(b * RACF_B);
  const int64_t R = (int64_t)ring_rows, slot0 = (int64_t)((uint64_t)bB % ring_rows);
  // the ring row of recorded index t, for bB - max_lag <= t < bB + RACF_B (|t - bB| < R)
  const auto row = [&](int64_t t) {
    int64_t k = slot0 + (t - bB);
    k = k < 0 ? k + R : (k >= R ? k - R : k);
    return ring + (uint64_t)k * ND + s;
  };
  for (int r = ly; r < RACF_B; r += FOLD_LY) v[r][tx] = live ? *row(bB + r) : 0.0;
  __syncthreads();
  if (ly == 0 && live) {
    RacfDd y{y_hi[s], y_lo[s]};
    for (int k = 0; k < RACF_B; ++k) y = racf_dd_add_d(y, v[k][tx]);
    y_hi[s] = y.hi;
    y_lo[s] = y.lo;
  }
  const int64_t oldest = bB - (int64_t)max_lag;
  for (uint64_t tau0 = 0; tau0 <= max_lag; tau0 += FOLD_TL) {
    __syncthreads();  // the previous tile's reads of win are done
    const int64_t t0 = bB - (int64_t)tau0 - (FOLD_TL - 1);
    // rows below r_lo are read only for lags past max_lag
    const uint64_t tau_hi = min(tau0 + (FOLD_TL - 1), max_lag);
    const int r_lo = (int)(tau0 + (FOLD_TL - 1) - tau_hi);
    for (int r = ly; r < FOLD_WIN; r += FOLD_LY) {
      const int64_t t = t0 + r;
      win[r][tx] = (live && r >= r_lo && t >= 0 && t >= oldest) ? *row(t) : 0.0;
    }
    __syncthreads();
    if (tau0 + (uint64_t)(ly * FOLD_TR) > max_lag) continue;  // warp-uniform: every lag of this warp is past max_lag
    double acc[FOLD_TR];
#pragma unroll
    for (int j = 0; j < FOLD_TR; ++j) acc[j] = 0.0;
    // lag tau0 + ly FOLD_TR + j, block value k: history row k - ly FOLD_TR - j + FOLD_TL - 1 of win
    const int base = FOLD_TL - FOLD_TR - ly * FOLD_TR;
#pragma unroll 1
    for (int k0 = 0; k0 < RACF_B; k0 += FOLD_KC) {
      double vv[FOLD_KC], yy[FOLD_KC + FOLD_TR - 1];
#pragma unroll
      for (int i = 0; i < FOLD_KC; ++i) vv[i] = v[k0 + i][tx];
#pragma unroll
      for (int i = 0; i < FOLD_KC + FOLD_TR - 1; ++i) yy[i] = win[base + k0 + i][tx];
#pragma unroll
      for (int kk = 0; kk < FOLD_KC; ++kk)
#pragma unroll
        for (int j = 0; j < FOLD_TR; ++j) acc[j] = racf_fma(vv[kk], yy[kk - j + FOLD_TR - 1], acc[j]);
    }
    if (live) {
#pragma unroll
      for (int j = 0; j < FOLD_TR; ++j) {
        const uint64_t tau = tau0 + (uint64_t)(ly * FOLD_TR + j);
        if (tau <= max_lag) {
          const size_t at = tau * ND + s;
          const RacfDd r = racf_dd_add_d(RacfDd{s_hi[at], s_lo[at]}, acc[j]);
          s_hi[at] = r.hi;
          s_lo[at] = r.lo;
        }
      }
    }
  }
}

// Block (walker chunk, parameters d = blockIdx.y + k gridDim.y), one thread per walker: r_w(tau) for tau < L, summed
// over the chunk's walkers in walker order into partial[chunk, tau, d].  The folded sums are read, never written.
// Not on the step path (a read runs when the user asks for rho): neighbouring threads load at a stride of D doubles,
// and a read in the middle of a block re-runs the pending chain of m terms from global memory for every lag, O(L m)
// loads per series.  That costs milliseconds per read (DESIGN §5.7), which the simple layout is worth.
__global__ void __launch_bounds__(RACF_WCHUNK)
    racf_read_kernel(const double* __restrict__ ring, uint64_t ring_rows, const double* __restrict__ head,
                     const double* __restrict__ s_hi, const double* __restrict__ s_lo,
                     const double* __restrict__ y_hi, const double* __restrict__ y_lo, uint32_t N, int D, uint64_t n,
                     uint64_t L, double* __restrict__ partial) {
  __shared__ double sh[READ_BATCH][RACF_WCHUNK];
  const uint64_t ND = (uint64_t)N * D;
  const uint32_t chunk = blockIdx.x;
  for (int d = blockIdx.y; d < D; d += gridDim.y) {
    const uint32_t w = chunk * RACF_WCHUNK + threadIdx.x;
    const bool live = w < N;
    const uint32_t cnt = min((uint32_t)RACF_WCHUNK, N - chunk * RACF_WCHUNK);
    const uint64_t s = (uint64_t)w * D + d;
    const uint64_t base = n / RACF_B * RACF_B, m = n % RACF_B;
    const auto yat = [&](int64_t t) { return t < 0 ? 0.0 : ring[((uint64_t)t % ring_rows) * ND + s]; };
    RacfDd Y{0.0, 0.0}, hd{0.0, 0.0}, tl{0.0, 0.0};
    double c0 = 0.0;
    if (live) {
      Y = RacfDd{y_hi[s], y_lo[s]};
      for (uint64_t k = 0; k < m; ++k) Y = racf_dd_add_d(Y, yat((int64_t)(base + k)));
    }
    for (uint64_t tau0 = 0; tau0 < L; tau0 += READ_BATCH) {
      for (int j = 0; j < READ_BATCH; ++j) {
        const uint64_t tau = tau0 + j;
        if (!live || tau >= L) break;
        if (tau > 0) {
          hd = racf_dd_add_d(hd, head[(tau - 1) * ND + s]);
          tl = racf_dd_add_d(tl, yat((int64_t)(n - tau)));
        }
        RacfDd S{s_hi[tau * ND + s], s_lo[tau * ND + s]};
        if (m > 0) {
          double p = 0.0;
          for (uint64_t k = 0; k < m; ++k)
            p = racf_fma(yat((int64_t)(base + k)), yat((int64_t)(base + k) - (int64_t)tau), p);
          S = racf_dd_add_d(S, p);
        }
        const double c = racf_cov(S, Y, hd, tl, n, tau);
        if (tau == 0) c0 = c;
        sh[j][threadIdx.x] = racf_div(c, c0);
      }
      __syncthreads();
      if (threadIdx.x < READ_BATCH && tau0 + threadIdx.x < L) {
        const int j = threadIdx.x;
        double a = sh[j][0];
        for (uint32_t i = 1; i < cnt; ++i) a = racf_add(a, sh[j][i]);
        partial[((uint64_t)chunk * L + tau0 + j) * D + d] = a;
      }
      __syncthreads();
    }
  }
}

__global__ void racf_finish_kernel(const double* __restrict__ partial, uint64_t nchunks, uint64_t L, int D, uint32_t N,
                                   double* __restrict__ rho) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;  // tau * D + d
  if (i >= L * D) return;
  double a = partial[i];
  for (uint64_t c = 1; c < nchunks; ++c) a = racf_add(a, partial[c * L * D + i]);
  rho[i] = racf_div(a, (double)N);
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// doubles of each buffer, in layout order
struct RacfLayout {
  size_t sizes[10];
};
RacfLayout racf_layout(uint32_t N, int D, uint64_t max_lag) {
  const size_t ND = (size_t)N * D, L = max_lag + 1;
  return RacfLayout{{ND, racf_ring(max_lag) * ND, max_lag * ND, L * ND, L * ND, ND, ND,
                     racf_nchunks(N) * L * (size_t)D, L * (size_t)D, 0}};
}

}  // namespace

size_t live_racf_bytes(uint32_t N, int D, uint64_t max_lag) {
  const size_t ND = (size_t)N * D;
  // 4 max_lag + RACF_B + 5 rows of ND doubles, plus the walker-chunk partials and rho: refuse what a size_t cannot hold
  const uint64_t rows_cap = SIZE_MAX / 16 / (ND + 1);
  if (max_lag > rows_cap / 8) return SIZE_MAX;
  const RacfLayout l = racf_layout(N, D, max_lag);
  size_t total = 0;
  for (size_t k : l.sizes) total += align256(k * sizeof(double));
  return total;
}

cudaError_t live_racf_setup(LiveRacf* r, void* mem, uint32_t N, int D, uint64_t max_lag, const double* coords,
                            cudaStream_t st) {
  const RacfLayout l = racf_layout(N, D, max_lag);
  double* ptr[9];
  char* p = static_cast<char*>(mem);
  for (int k = 0; k < 9; ++k) {
    ptr[k] = reinterpret_cast<double*>(p);
    p += align256(l.sizes[k] * sizeof(double));
  }
  *r = LiveRacf{};
  r->N = N;
  r->D = D;
  r->max_lag = max_lag;
  r->coords = coords;
  r->x0 = ptr[0];
  r->ring = ptr[1];
  r->head = ptr[2];
  r->s_hi = ptr[3];
  r->s_lo = ptr[4];
  r->y_hi = ptr[5];
  r->y_lo = ptr[6];
  r->partial = ptr[7];
  r->rho = ptr[8];
  // S and Y start at zero; x0, the ring and head are written before they are read
  cudaError_t e = cudaMemsetAsync(r->s_hi, 0, (size_t)(reinterpret_cast<char*>(ptr[7]) - reinterpret_cast<char*>(ptr[3])),
                                  st);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(st);
}

cudaError_t live_racf_record(const LiveRacf& r, uint64_t n, cudaStream_t st, uint64_t& launches) {
  const uint64_t ND = (uint64_t)r.N * r.D;
  const unsigned threads = 256;
  racf_record_kernel<<<(unsigned)((ND + threads - 1) / threads), threads, 0, st>>>(
      r.coords, ND, n, racf_ring(r.max_lag), r.max_lag, r.x0, r.ring, r.head);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  ++launches;
  if ((n + 1) % RACF_B == 0) {
    racf_fold_kernel<<<(unsigned)((ND + FOLD_TS - 1) / FOLD_TS), FOLD_THREADS, 0, st>>>(
        r.ring, racf_ring(r.max_lag), ND, n / RACF_B, r.max_lag, r.s_hi, r.s_lo, r.y_hi, r.y_lo);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++launches;
  }
  return cudaSuccess;
}

cudaError_t live_racf_read(const LiveRacf& r, uint64_t n, double* rho, cudaStream_t st) {
  const uint64_t L = racf_rows(n, r.max_lag);
  if (L == 0) return cudaSuccess;
  const uint64_t nchunks = racf_nchunks(r.N);
  racf_read_kernel<<<dim3((unsigned)nchunks, (unsigned)std::min(r.D, 65535)), RACF_WCHUNK, 0, st>>>(
      r.ring, racf_ring(r.max_lag), r.head, r.s_hi, r.s_lo, r.y_hi, r.y_lo, r.N, r.D, n, L, r.partial);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const uint64_t LD = L * (uint64_t)r.D;
  racf_finish_kernel<<<(unsigned)((LD + FINISH_THREADS - 1) / FINISH_THREADS), FINISH_THREADS, 0, st>>>(
      r.partial, nchunks, L, r.D, r.N, r.rho);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(rho, r.rho, (size_t)LD * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(st);
}

}  // namespace eb
