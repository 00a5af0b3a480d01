// Chain analysis on the device: running moments of the ensemble (mean / covariance of a
// store=False run), the Gram matrix behind the initial-state independence check, and the
// walker-averaged autocorrelation function of a stored chain.
//
// Reference semantics (file:line relative to the reference):
//   chain mean / covariance of a run ........ what a caller computes from get_chain(flat=True)
//                                              (backends/backend.py:42-58); here accumulated on the
//                                              device so that store=False runs (ensemble.py:287-291)
//                                              need no D2H of the state
//   walkers_independent ...................... ensemble.py:653-663
//   autocorr.function_1d / integrated_time ... autocorr.py:21-46, 49-123
#include <math.h>

#include <algorithm>

#include "engine.cuh"

namespace eb {

namespace {

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// ===========================================================================
// column statistics: mean of each column (fixed summation order) + non-finite flags
// ===========================================================================
// grid = ceil(D / 32) blocks of (32, 8) threads; thread (x, y) sums rows y, y+8, ... of column 32 b + x
__global__ void __launch_bounds__(256) colmean_kernel(const double* __restrict__ X, int64_t nrows, int D,
                                                      double* __restrict__ mean, int* status) {
  __shared__ double part[8][33];
  const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
  const int d = blockIdx.x * 32 + x;
  double acc = 0.0;
  bool any_inf = false, any_nan = false;
  if (d < D)
    for (int64_t r = y; r < nrows; r += 8) {
      const double v = X[(size_t)r * D + d];
      acc += v;
      any_inf |= isinf(v);
      any_nan |= isnan(v);
    }
  part[y][x] = acc;
  if (status) {
    if (any_inf) atomicOr(status, FLAG_INF_PARAM);
    if (any_nan) atomicOr(status, FLAG_NAN_PARAM);
  }
  __syncthreads();
  if (y == 0 && d < D) {
    double s = 0.0;
    for (int k = 0; k < 8; ++k) s += part[k][x];
    mean[d] = s / (double)nrows;
  }
}

// ===========================================================================
// second moments on the FP64 tensor pipe: S2 += (X - shift)^T (X - shift), S1 += sum(X - shift)
// ===========================================================================
// The D x D result is tiled into 8 x 8 blocks; only blocks (i <= j) are computed.  A CTA stages
// CH rows in shared memory; warp w owns block pairs base + w, base + w + 8, ... (MAXB of them,
// accumulators in registers) and walks the staged rows 4 at a time: one DMMA m8n8k4 per block per
// 4 rows with A[g][t] = x[row t][8 i + g], B[t][g] = x[row t][8 j + g].  blockIdx.y selects the
// group of 8 * MAXB block pairs (large D needs several passes over the rows).
constexpr int MOM_WARPS = 8;
constexpr int MOM_MAXB = 18;  // 8 * 18 = 144 >= 136 pairs of D = 128: one pass

__global__ void __launch_bounds__(32 * MOM_WARPS)
    moments_partial_kernel(const double* __restrict__ X, int64_t nrows, int D, const double* __restrict__ shift,
                           double* __restrict__ partial, int CH, int RS, const int32_t* __restrict__ rowidx,
                           int skip_start, int skip_count) {
  extern __shared__ double xs[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int nblk = (D + 7) >> 3, Dp = 8 * nblk;
  const int npairs = nblk * (nblk + 1) / 2;
  const int base = blockIdx.y * MOM_WARPS * MOM_MAXB;
  int bi[MOM_MAXB], bj[MOM_MAXB];
  double c0[MOM_MAXB], c1[MOM_MAXB];
#pragma unroll
  for (int m = 0; m < MOM_MAXB; ++m) {
    const int p = base + warp + MOM_WARPS * m;
    c0[m] = c1[m] = 0.0;
    bi[m] = -1;
    bj[m] = 0;
    if (p < npairs) {  // row-major walk of the upper triangle: row i holds nblk - i pairs
      int i = 0, rem = p;
      while (rem >= nblk - i) {
        rem -= nblk - i;
        ++i;
      }
      bi[m] = i;
      bj[m] = i + rem;
    }
  }
  double s1[4] = {0.0, 0.0, 0.0, 0.0};  // column sums of dims tid, tid + 256, ... (pass 0 only; Dp <= 1024)
  const int64_t nchunks = (nrows + CH - 1) / CH;
  for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
    for (int idx = tid; idx < CH * Dp; idx += 32 * MOM_WARPS) {
      const int r = idx / Dp, d = idx - r * Dp;
      const int64_t row = chunk * CH + r;
      double v = 0.0;
      if (row < nrows && d < D) {
        // optional indirection: row r of the set is walker rowidx[r < skip_start ? r : r + skip_count]
        // (the complement of a split in the order of red_blue.py:85-87)
        const int64_t src = rowidx ? (int64_t)rowidx[row < skip_start ? row : row + skip_count] : row;
        v = X[(size_t)src * D + d] - shift[d];
      }
      xs[r * RS + d] = v;
    }
    __syncthreads();
    if (blockIdx.y == 0) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int d = tid + 32 * MOM_WARPS * q;
        if (d < Dp)
          for (int r = 0; r < CH; ++r) s1[q] += xs[r * RS + d];
      }
    }
    for (int k4 = 0; k4 < CH / 4; ++k4) {
      const double* rowp = xs + (4 * k4 + t) * RS + g;
#pragma unroll
      for (int m = 0; m < MOM_MAXB; ++m) {
        if (bi[m] >= 0) {  // warp-uniform
          const double av = rowp[8 * bi[m]];
          const double bv = rowp[8 * bj[m]];
          dmma884(c0[m], c1[m], av, bv);
        }
      }
    }
    __syncthreads();
  }
  double* out = partial + (size_t)blockIdx.x * ((size_t)Dp + (size_t)Dp * Dp);
  if (blockIdx.y == 0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int d = tid + 32 * MOM_WARPS * q;
      if (d < Dp) out[d] = s1[q];
    }
  }
#pragma unroll
  for (int m = 0; m < MOM_MAXB; ++m) {
    if (bi[m] >= 0) {
      double* o = out + Dp + (size_t)(8 * bi[m] + g) * Dp + 8 * bj[m] + 2 * t;
      o[0] = c0[m];
      o[1] = c1[m];
    }
  }
}

// acc[D + D*D] += sum over the CTA partials, in CTA order (deterministic); mirrors the lower triangle
__global__ void moments_reduce_kernel(const double* __restrict__ partial, int nparts, int D, double* __restrict__ acc) {
  const int nblk = (D + 7) >> 3, Dp = 8 * nblk;
  const size_t stride = (size_t)Dp + (size_t)Dp * Dp;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)D + (size_t)D * D) return;
  size_t src;
  if (e < (size_t)D) {
    src = e;
  } else {
    const size_t f = e - D;
    int r = (int)(f / D), c = (int)(f - (size_t)r * D);
    if ((r >> 3) > (c >> 3)) {
      const int tmp = r;
      r = c;
      c = tmp;
    }
    src = (size_t)Dp + (size_t)r * Dp + c;
  }
  double s = 0.0;
  for (int p = 0; p < nparts; ++p) s += partial[(size_t)p * stride + src];
  acc[e] += s;
}

// ===========================================================================
// walker-averaged normalised autocorrelation function of a stored chain (autocorr.py:21-46, 101-107)
// ===========================================================================
// Per series (walker, parameter): x - mean, zero-padded to M = 2 * next_pow_two(n_t); forward FFT,
// |F|^2, inverse FFT, acf / acf[0].  The transform is an in-place radix-2 pair that needs no
// bit-reversal pass: decimation-in-frequency forward (natural in, bit-reversed out), the pointwise
// power spectrum (order-agnostic), decimation-in-time inverse (bit-reversed in, natural out).
// Butterflies of span h < ACF_BLOCK / 2 stay inside aligned blocks of ACF_BLOCK points and run in
// shared memory (one CTA per block: all small-span forward stages, the power spectrum and all
// small-span inverse stages in one pass); larger spans are one global-memory pass each.  Every grid is 1-D
// (acf_grid.h): a slab may hold millions of series, and grid y stops at 65 535.

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// tw[k] = exp(-2 pi i k / M), k < M / 2
__global__ void acf_twiddle_kernel(double2* __restrict__ tw, int M) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= M / 2) return;
  double sn, cs;
  sincospi(-2.0 * (double)k / (double)M, &sn, &cs);
  tw[k] = make_double2(cs, sn);
}

// xin[n_t][S] (series contiguous) -> mean[S]; one thread per series, fixed order over t
__global__ void acf_mean_kernel(const double* __restrict__ xin, int n_t, int S, double* __restrict__ mean) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  double acc = 0.0;
  for (int t = 0; t < n_t; ++t) acc += xin[(size_t)t * S + s];
  mean[s] = acc / (double)n_t;
}

// z[s][t] = (xin[t][s] - mean[s], 0) for t < n_t, 0 beyond: 32 x 32 tiles through shared memory, CTA
// k = series tile * tiles_t + t tile
__global__ void __launch_bounds__(256) acf_load_kernel(const double* __restrict__ xin, const double* __restrict__ mean,
                                                       int n_t, int S, int M, unsigned tiles_t,
                                                       double2* __restrict__ z) {
  __shared__ double tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const unsigned st = blockIdx.x / tiles_t;
  const int t0 = (int)(blockIdx.x - st * tiles_t) * 32, s0 = (int)st * 32;
  for (int y = ty; y < 32; y += 8) {
    const int t = t0 + y, s = s0 + tx;
    tile[y][tx] = (t < n_t && s < S) ? xin[(size_t)t * S + s] - mean[s] : 0.0;
  }
  __syncthreads();
  for (int y = ty; y < 32; y += 8) {
    const int s = s0 + y, t = t0 + tx;
    if (s < S && t < M) z[(size_t)s * M + t] = make_double2(tile[tx][y], 0.0);
  }
}

// one butterfly stage of span h over every series (global memory): forward = DIF, inverse = DIT
__global__ void fft_global_stage_kernel(double2* __restrict__ z, const double2* __restrict__ tw, int S, int M, int h,
                                        int inverse) {
  const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t half = (size_t)M / 2;
  if (id >= (size_t)S * half) return;
  const size_t s = id / half;
  const int b = (int)(id - s * half);
  const int j = b & (h - 1);
  const int i = ((b - j) << 1) + j;
  double2* x = z + s * M;
  double2 w = tw[(size_t)j * (M / (2 * h))];
  const double2 u = x[i], v = x[i + h];
  if (!inverse) {
    x[i] = make_double2(u.x + v.x, u.y + v.y);
    x[i + h] = cmul(make_double2(u.x - v.x, u.y - v.y), w);
  } else {
    w.y = -w.y;
    const double2 vw = cmul(v, w);
    x[i] = make_double2(u.x + vw.x, u.y + vw.y);
    x[i + h] = make_double2(u.x - vw.x, u.y - vw.y);
  }
}

// the stages of span < B of one aligned block of B points, in shared memory: CTA k holds z[k B, (k + 1) B), block
// k mod (M / B) of series k / (M / B)
__global__ void __launch_bounds__(512) fft_local_kernel(double2* __restrict__ z, const double2* __restrict__ tw, int M,
                                                        int B) {
  extern __shared__ double2 sz[];
  double2* base = z + (size_t)blockIdx.x * B;
  for (int i = threadIdx.x; i < B; i += blockDim.x) sz[i] = base[i];
  for (int h = B / 2; h >= 1; h >>= 1) {  // forward, decimation in frequency
    __syncthreads();
    const int tstep = M / (2 * h);
    for (int b = threadIdx.x; b < B / 2; b += blockDim.x) {
      const int j = b & (h - 1);
      const int i = ((b - j) << 1) + j;
      const double2 u = sz[i], v = sz[i + h];
      sz[i] = make_double2(u.x + v.x, u.y + v.y);
      sz[i + h] = cmul(make_double2(u.x - v.x, u.y - v.y), tw[(size_t)j * tstep]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) {  // power spectrum (autocorr.py:43-44)
    const double2 v = sz[i];
    sz[i] = make_double2(v.x * v.x + v.y * v.y, 0.0);
  }
  for (int h = 1; h <= B / 2; h <<= 1) {  // inverse, decimation in time
    __syncthreads();
    const int tstep = M / (2 * h);
    for (int b = threadIdx.x; b < B / 2; b += blockDim.x) {
      const int j = b & (h - 1);
      const int i = ((b - j) << 1) + j;
      double2 w = tw[(size_t)j * tstep];
      w.y = -w.y;
      const double2 u = sz[i], vw = cmul(sz[i + h], w);
      sz[i] = make_double2(u.x + vw.x, u.y + vw.y);
      sz[i + h] = make_double2(u.x - vw.x, u.y - vw.y);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) base[i] = sz[i];
}

// f[k][d][lag] += sum over the slab's walkers of segment k (ascending) of acf[(w, d)][lag] / acf[(w, d)][0]
// (autocorr.py:45,105).  The slab holds walkers [w0, w0 + wb) of a chain of segments of seg_w walkers; CTA
// c = (j * nd + d) * lag_tiles + lag tile serves the slab's j-th segment, k = w0 / seg_w + j.
__global__ void acf_accumulate_kernel(const double2* __restrict__ z, int wb, int nd, int n_t, int M,
                                      unsigned lag_tiles, int64_t seg_w, int64_t w0, double* __restrict__ f) {
  const unsigned sd = blockIdx.x / lag_tiles;
  const int d = (int)(sd % (unsigned)nd);
  const int64_t k = w0 / seg_w + (int64_t)(sd / (unsigned)nd);
  const int lag = (int)(blockIdx.x - sd * lag_tiles) * blockDim.x + threadIdx.x;
  if (lag >= n_t) return;
  const int lo = (int)(max(k * seg_w, w0) - w0), hi = (int)(min((k + 1) * seg_w, w0 + (int64_t)wb) - w0);
  double acc = 0.0;
  for (int w = lo; w < hi; ++w) {
    const double2* x = z + (size_t)(w * nd + d) * M;
    acc += x[lag].x / x[0].x;
  }
  f[((size_t)k * nd + d) * n_t + lag] += acc;
}

__global__ void acf_scale_kernel(double* __restrict__ f, size_t n, double scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) f[i] *= scale;
}

// ===========================================================================
// segmented moments of a stored slice: nseg ensembles of N walkers stacked in every stored step
// ===========================================================================
// The batch regime: many segments of a few dozen walkers in a few dimensions, where one 8 x 8 DMMA block per
// (step, segment) would be mostly padding and launches.  One thread per (segment k, i, j) of the D x D sums, a
// chunk of stored steps per grid row y; every sum runs in (step, walker) order, so the result does not depend on
// the schedule.  Element (k, w, d) of stored step s is slots[s][(k * N + w) * D + d].

// shift[k][d] = the mean over walkers (ascending) of stored step 0's segment k
__global__ void moments_seg_shift_kernel(const double* const* __restrict__ slots, int64_t nseg, int64_t N, int D,
                                         double* __restrict__ shift) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nseg * D) return;
  const int64_t k = e / D;
  const int d = (int)(e - k * D);
  const double* x = slots[0] + (size_t)k * N * D + d;
  double acc = 0.0;
  for (int64_t w = 0; w < N; ++w) acc += x[(size_t)w * D];
  shift[e] = acc / (double)N;
}

// partial[y][k][D + D*D]: [sum(x - shift) | (x - shift)^T (x - shift)] of segment k over stored steps
// [y * cs, min(count, (y + 1) * cs)); thread (k, i, j) forms S2[i][j], and S1[i] when j == i
__global__ void __launch_bounds__(256)
    moments_seg_partial_kernel(const double* const* __restrict__ slots, uint64_t count, uint64_t cs, int64_t nseg,
                               int64_t N, int D, const double* __restrict__ shift, double* __restrict__ partial) {
  const int64_t DD = (int64_t)D * D;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nseg * DD) return;
  const int64_t k = e / DD;
  const int i = (int)((e - k * DD) / D), j = (int)(e - k * DD - (int64_t)i * D);
  const double si = shift[k * D + i], sj = shift[k * D + j];
  const uint64_t s0 = (uint64_t)blockIdx.y * cs, s1 = min(count, s0 + cs);
  double a1 = 0.0, a2 = 0.0;
  for (uint64_t s = s0; s < s1; ++s) {
    const double* x = slots[s] + (size_t)k * N * D;
    for (int64_t w = 0; w < N; ++w) {
      const double xi = x[(size_t)w * D + i] - si, xj = x[(size_t)w * D + j] - sj;
      a1 += xi;
      a2 = fma(xi, xj, a2);
    }
  }
  double* out = partial + ((size_t)blockIdx.y * nseg + k) * (size_t)(D + DD);
  if (i == j) out[i] = a1;
  out[D + (int64_t)i * D + j] = a2;
}

// acc[k][D + D*D] = sum over the chunks (ascending) of partial[y][k][...]
__global__ void moments_seg_reduce_kernel(const double* __restrict__ partial, uint64_t nchunks, size_t n,
                                          double* __restrict__ acc) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  double s = 0.0;
  for (uint64_t y = 0; y < nchunks; ++y) s += partial[y * n + e];
  acc[e] = s;
}

}  // namespace

// ---- host-side launchers -----------------------------------------------------------------
cudaError_t launch_colmean(const double* X, int64_t nrows, int D, double* mean, int* status, cudaStream_t st) {
  if (nrows <= 0 || D <= 0) return cudaSuccess;
  colmean_kernel<<<(D + 31) / 32, 256, 0, st>>>(X, nrows, D, mean, status);
  return cudaGetLastError();
}

int moments_grid(int D, int sm_count) {
  const int nblk = (D + 7) / 8, Dp = 8 * nblk;
  const size_t per = ((size_t)Dp + (size_t)Dp * Dp) * sizeof(double);
  size_t g = ((size_t)64 << 20) / per;  // <= 64 MiB of partials
  if (g < 1) g = 1;
  if (g > (size_t)sm_count) g = (size_t)sm_count;
  return (int)g;
}

size_t moments_partial_bytes(int D, int sm_count) {
  const int nblk = (D + 7) / 8, Dp = 8 * nblk;
  return (size_t)moments_grid(D, sm_count) * ((size_t)Dp + (size_t)Dp * Dp) * sizeof(double);
}

// acc[D + D*D] += [sum(x - shift), (x - shift)^T (x - shift)] over the rows of X
cudaError_t launch_moments(const double* X, int64_t nrows, int D, const double* shift, double* partial, double* acc,
                           int sm_count, cudaStream_t st, const int32_t* rowidx, int skip_start, int skip_count) {
  if (D > 1024) return cudaErrorNotSupported;
  if (nrows <= 0) return cudaSuccess;
  const int nblk = (D + 7) / 8, Dp = 8 * nblk;
  int RS = Dp;
  while (RS % 32 != 8) RS += 8;  // 4 staged rows x 8 dims of one fragment hit 32 distinct 8-byte banks
  int CH = (int)((96 * 1024) / ((size_t)RS * sizeof(double))) & ~3;
  if (CH > 64) CH = 64;
  if (CH < 4) CH = 4;
  const size_t smem = (size_t)CH * RS * sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(moments_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int grid = moments_grid(D, sm_count);
  const int64_t nchunks = (nrows + CH - 1) / CH;
  if (grid > nchunks) grid = (int)nchunks;
  const int npairs = nblk * (nblk + 1) / 2;
  const int passes = (npairs + MOM_WARPS * MOM_MAXB - 1) / (MOM_WARPS * MOM_MAXB);
  moments_partial_kernel<<<dim3(grid, passes), 32 * MOM_WARPS, smem, st>>>(X, nrows, D, shift, partial, CH, RS, rowidx,
                                                                           skip_start, skip_count);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const size_t n = (size_t)D + (size_t)D * D;
  moments_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, grid, D, acc);
  return cudaGetLastError();
}


// ---- autocorrelation -------------------------------------------------------------------------
cudaError_t launch_acf_twiddles(double2* tw, int M, cudaStream_t st) {
  acf_twiddle_kernel<<<(M / 2 + 255) / 256, 256, 0, st>>>(tw, M);
  return cudaGetLastError();
}

// One slab, walkers [w0, w0 + wb) of a chain of segments of seg_w walkers: xin[n_t][S = wb * nd] (device) ->
// f[k][nd][n_t] += sum over the slab's walkers of segment k of the normalised autocorrelation functions.
// z: S * M complex scratch, mean: S doubles.
cudaError_t launch_acf_slab(const double* xin, int n_t, int wb, int nd, int M, const double2* tw, double2* z,
                            double* mean, double* f, int64_t seg_w, int64_t w0, cudaStream_t st) {
  const int S = wb * nd;
  const int64_t nks = (w0 + wb - 1) / seg_w - w0 / seg_w + 1;
  const AcfGrid g = acf_grid(n_t, wb, nd, M, (uint64_t)nks);
  const int B = g.B;
  acf_mean_kernel<<<(unsigned)g.mean_blocks, 128, 0, st>>>(xin, n_t, S, mean);
  acf_load_kernel<<<(unsigned)g.load_blocks, 256, 0, st>>>(xin, mean, n_t, S, M, (unsigned)g.load_tiles_t, z);
  for (int h = M / 2; h >= B; h >>= 1)
    fft_global_stage_kernel<<<(unsigned)g.global_blocks, 256, 0, st>>>(z, tw, S, M, h, 0);
  const size_t smem = (size_t)B * sizeof(double2);
  cudaError_t e = cudaFuncSetAttribute(fft_local_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  fft_local_kernel<<<(unsigned)g.local_blocks, g.local_threads, smem, st>>>(z, tw, M, B);
  for (int h = B; h <= M / 2; h <<= 1)
    fft_global_stage_kernel<<<(unsigned)g.global_blocks, 256, 0, st>>>(z, tw, S, M, h, 1);
  acf_accumulate_kernel<<<(unsigned)g.accumulate_blocks, 256, 0, st>>>(z, wb, nd, n_t, M, (unsigned)g.lag_tiles, seg_w,
                                                                      w0, f);
  return cudaGetLastError();
}

// chunks of stored steps the segmented moments split a slice into: about 2^19 threads in all, at most one chunk per
// stored step, at most 65 535 (grid y) and at most 256 MiB of partial sums.  A pure function of the shape, so repeated calls are bit-identical.
uint64_t moments_seg_chunks(uint64_t count, int64_t nseg, int D) {
  const uint64_t per = (uint64_t)nseg * ((uint64_t)D + (uint64_t)D * D);
  uint64_t c = (((uint64_t)1 << 19) + per - 1) / per;
  c = std::min<uint64_t>(std::min<uint64_t>(c, 65535), ((uint64_t)1 << 25) / per);
  return std::max<uint64_t>(1, std::min<uint64_t>(c, count));
}

// shift[nseg][D], partial[nchunks][nseg][D + D*D] and acc[nseg][D + D*D] of a slice of `count` stored steps (slots:
// device table of count pointers)
cudaError_t launch_moments_segments(const double* const* slots, uint64_t count, int64_t nseg, int64_t N, int D,
                                    uint64_t nchunks, double* shift, double* partial, double* acc, cudaStream_t st) {
  const int64_t ne = nseg * D;
  moments_seg_shift_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, st>>>(slots, nseg, N, D, shift);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const uint64_t cs = (count + nchunks - 1) / nchunks;
  const uint64_t ny = (count + cs - 1) / cs;
  const int64_t nt = nseg * D * D;
  moments_seg_partial_kernel<<<dim3((unsigned)((nt + 255) / 256), (unsigned)ny), 256, 0, st>>>(slots, count, cs, nseg,
                                                                                             N, D, shift, partial);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const size_t n = (size_t)nseg * ((size_t)D + (size_t)D * D);
  moments_seg_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(partial, ny, n, acc);
  return cudaGetLastError();
}

cudaError_t launch_acf_scale(double* f, size_t n, double scale, cudaStream_t st) {
  acf_scale_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(f, n, scale);
  return cudaGetLastError();
}

}  // namespace eb
