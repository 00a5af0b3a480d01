// KDEMove (moves/kde.py): kernel-density proposals of the complement and their Hastings factors.
//
// Reference semantics (scipy.stats.gaussian_kde with uniform weights, as kde.py:39-43 calls it):
//   c = concatenate(complement sets); kde = gaussian_kde(c.T, bw_method)
//   q_i = c[j_i] + bw L z_i           (kde.resample: choice(nc, p=uniform) and multivariate_normal(0, bw^2 cov))
//   factor_i = logpdf(s_i) - logpdf(q_i) = LSE_c(-|y_s - y_c|^2 / 2) - LSE_c(-|y_q - y_c|^2 / 2)
// with y = (bw L)^-1 (x - mean_c), L the lower Cholesky factor of np.cov(c) (the kernel normaliser and the uniform
// log-weights cancel in the difference; centring on the complement mean changes no difference y_p - y_c).
//
// Per split the engine runs (step.cu, launch_step_kde): the complement moment sums and cov_chol_kernel that the
// whole-complement WalkMove uses, then
//   kde_factor_kernel   one CTA: refuses a singular factor (FLAG_KDE_SINGULAR), (bw L)^-1 and mean_c
//   kde_prepare_kernel  one lane group per row: the proposals q (qbuf), whitened s | q rows and complement rows
//   kde_lse_kernel      64 points x 64 centres per tile pass; |y_p - y_c|^2 from direct differences on the FP64
//                       CUDA cores, an online (max, sum) log-sum-exp per point; the centre tiles may be split over
//                       gridDim.y CTAs, whose partial (max, sum) pairs kde_merge_kernel folds into the factors
// and the accept of precomputed rows with a Hastings factor buffer (half_step_generic_kernel<EB_MOVE_USER>).
//
// Draws (DESIGN.md §2, draws.cuh): the kernel centre j_i from block (index = i, TAG_PROP_A), z_i = the TAG_NORMAL
// normals of row i (as WalkMove).
#include <math.h>

#include "draws.cuh"
#include "engine.cuh"

namespace eb {

namespace {

constexpr int KT = 64;          // points and centres per tile
constexpr int KD = 32;          // dimensions per staged chunk
constexpr int KPAD = KT + 1;    // smem row pitch of a transposed chunk: [KD][KT + 1]
constexpr int LSE_THREADS = 256;  // 16 point lanes x 16 centre lanes, each 4 points x 4 centres

// L (cov_chol_kernel) -> minv = (bw L)^-1 (lower, row-major), mean = shift + S1 / nc.  A zero pivot (at or below
// chol_psd's 1e-12 max-diag threshold, or past the rank bound nc - 1) sets FLAG_KDE_SINGULAR and writes nothing.
__global__ void __launch_bounds__(1024) kde_factor_kernel(const double* __restrict__ L, const double* __restrict__ acc,
                                                          const double* __restrict__ shift, double nc, int D, double bw,
                                                          double* __restrict__ minv, double* __restrict__ mean,
                                                          int* status) {
  __shared__ int s_bad;
  const int tid = threadIdx.x, nt = blockDim.x;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int j = tid; j < D; j += nt)
    if (!(L[(size_t)j * D + j] > 0.0)) s_bad = 1;
  __syncthreads();
  if (s_bad) {
    if (tid == 0) atomicOr(status, FLAG_KDE_SINGULAR);
    return;
  }
  for (int d = tid; d < D; d += nt) mean[d] = shift[d] + acc[d] / nc;
  // column j of the inverse by forward substitution, one thread per column
  for (int j = tid; j < D; j += nt) {
    for (int i = 0; i < j; ++i) minv[(size_t)i * D + j] = 0.0;
    minv[(size_t)j * D + j] = 1.0 / (bw * L[(size_t)j * D + j]);
    for (int i = j + 1; i < D; ++i) {
      double v = 0.0;
      for (int k = j; k < i; ++k) v = fma(bw * L[(size_t)i * D + k], minv[(size_t)k * D + j], v);
      minv[(size_t)i * D + j] = -v / (bw * L[(size_t)i * D + i]);
    }
  }
}

// y[e] = sum_{k <= e} minv[e, k] (x[k] - mean[k]) for the row x staged in v (group lanes g, G)
__device__ __forceinline__ void whiten_row(const double* v, const double* __restrict__ minv, int D, int g, int G,
                                           double* __restrict__ y) {
  for (int e = g; e < D; e += G) {
    const double* Mr = minv + (size_t)e * D;
    double acc = 0.0;
    for (int k = 0; k <= e; ++k) acc = fma(__ldg(Mr + k), v[k], acc);
    y[e] = acc;
  }
}

// rows [0, ns): the active walkers -> yp[r]; [ns, 2 ns): proposal i = r - ns -> qbuf[i], yp[r], jw[i] (walker id of
// its kernel centre); [2 ns, 2 ns + nc): complement rank k -> yc[k]
__global__ void __launch_bounds__(256) kde_prepare_kernel(const HalfStepArgs a, const double* __restrict__ L,
                                                          const double* __restrict__ minv,
                                                          const double* __restrict__ mean, double bw,
                                                          double* __restrict__ qbuf, double* __restrict__ yp,
                                                          double* __restrict__ yc, int64_t* __restrict__ jw,
                                                          const int G) {
  extern __shared__ double smem[];
  const int D = a.D;
  const int groups = blockDim.x / G;
  const int gid = threadIdx.x / G, g = threadIdx.x % G;
  const int lane = threadIdx.x & 31;
  const unsigned mask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
  const int64_t ns = a.a_count, nc = a.N - a.a_count;
  const int64_t r = (int64_t)blockIdx.x * groups + gid;
  if (r >= 2 * ns + nc) return;
  double* v = smem + (size_t)gid * 2 * D;  // the centred row
  double* z = v + D;                       // normals, then L z
  double* y;
  if (r < ns || r >= 2 * ns) {
    const int64_t k = r - 2 * ns;
    const int64_t w = r < ns ? a.order[a.a_start + r] : a.order[complement_slot(k, a.a_start, a.a_count)];
    const double* x = a.coords + (size_t)w * D;
    for (int e = g; e < D; e += G) v[e] = x[e] - mean[e];
    y = r < ns ? yp + (size_t)r * D : yc + (size_t)k * D;
  } else {
    const int64_t i = r - ns;
    const int64_t k = kde_centre_rank(prop_a(a.seed, a.step, (uint32_t)a.split, (uint32_t)i), nc);
    const int64_t cw = a.order[complement_slot(k, a.a_start, a.a_count)];
    for (int kk = g; 2 * kk < D; kk += G) {
      double n0, n1;
      normal_pair(a.seed, a.step, (uint32_t)a.split, (uint32_t)kk, (uint32_t)i, n0, n1);
      z[2 * kk] = n0;
      if (2 * kk + 1 < D) z[2 * kk + 1] = n1;
    }
    __syncwarp(mask);
    const double* c_row = a.coords + (size_t)cw * D;
    double* q = qbuf + (size_t)i * D;
    for (int e = g; e < D; e += G) {
      double acc = 0.0;
      const double* Lr = L + (size_t)e * D;
      for (int kk = 0; kk <= e; ++kk) acc = fma(__ldg(Lr + kk), z[kk], acc);
      const double qe = __dadd_rn(c_row[e], __dmul_rn(bw, acc));  // means + norm
      q[e] = qe;
      v[e] = qe - mean[e];
    }
    if (g == 0) jw[i] = cw;
    y = yp + (size_t)r * D;
  }
  __syncwarp(mask);
  whiten_row(v, minv, D, g, G, y);
}

// rows [row0, row0 + KT) x dims [d0, d0 + dk) of src[nrows, D] -> dst[k * KPAD + r]; zero outside
__device__ __forceinline__ void stage_chunk(double* dst, const double* __restrict__ src, int64_t row0, int64_t nrows,
                                            int d0, int dk, int D) {
  for (int e = threadIdx.x; e < KT * KD; e += LSE_THREADS) {
    const int r = e / KD, k = e - r * KD;
    double v = 0.0;
    if (k < dk && row0 + r < nrows) v = src[(size_t)(row0 + r) * D + d0 + k];
    dst[k * KPAD + r] = v;
  }
}

// fold (mo, so) into (m, s): the pair (max, sum of exp(t - max))
__device__ __forceinline__ void lse_fold(double& m, double& s, double mo, double so) {
  const double M = fmax(m, mo);
  if (M == -INFINITY) return;
  s = s * exp(m - M) + so * exp(mo - M);
  m = M;
}

// gridDim.x: point tiles of KT; gridDim.y: chunks of `tpc` centre tiles.  part_m / part_s [gridDim.y, P].
__global__ void __launch_bounds__(LSE_THREADS) kde_lse_kernel(const double* __restrict__ yp, int64_t P,
                                                              const double* __restrict__ yc, int64_t nc, int D,
                                                              int tpc, double* __restrict__ part_m,
                                                              double* __restrict__ part_s) {
  __shared__ double sp[KD * KPAD];
  __shared__ double sc[KD * KPAD];
  const int tc = threadIdx.x & 15, tp = threadIdx.x >> 4;
  const int64_t p0 = (int64_t)blockIdx.x * KT;
  const int64_t ctiles = (nc + KT - 1) / KT;
  const int64_t ct_lo = (int64_t)blockIdx.y * tpc;
  const int64_t ct_hi = ct_lo + tpc < ctiles ? ct_lo + tpc : ctiles;
  const bool one_chunk = D <= KD;
  double m[4], s[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    m[r] = -INFINITY;
    s[r] = 0.0;
  }
  if (one_chunk) stage_chunk(sp, yp, p0, P, 0, D, D);
  for (int64_t ct = ct_lo; ct < ct_hi; ++ct) {
    const int64_t c0 = ct * KT;
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int d0 = 0; d0 < D; d0 += KD) {
      const int dk = D - d0 < KD ? D - d0 : KD;
      __syncthreads();  // the previous chunk's readers are done
      if (!one_chunk) stage_chunk(sp, yp, p0, P, d0, dk, D);
      stage_chunk(sc, yc, c0, nc, d0, dk, D);
      __syncthreads();
#pragma unroll 4
      for (int k = 0; k < dk; ++k) {
        double pv[4], cv[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) pv[r] = sp[k * KPAD + tp + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) cv[c] = sc[k * KPAD + tc + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const double d = pv[r] - cv[c];  // a direct difference: no |a|^2 + |b|^2 - 2 a.b cancellation
            acc[r][c] = fma(d, d, acc[r][c]);
          }
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      double t[4], tmax = -INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        t[c] = c0 + tc + 16 * c < nc ? -0.5 * acc[r][c] : -INFINITY;
        tmax = fmax(tmax, t[c]);
      }
      if (tmax > m[r]) {
        s[r] *= exp(m[r] - tmax);
        m[r] = tmax;
      }
      if (m[r] > -INFINITY)
#pragma unroll
        for (int c = 0; c < 4; ++c) s[r] += exp(t[c] - m[r]);
    }
  }
  // the 16 centre lanes of a point hold disjoint centre sets: fold them
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      const double mo = __shfl_xor_sync(0xffffffffu, m[r], off, 16);
      const double so = __shfl_xor_sync(0xffffffffu, s[r], off, 16);
      lse_fold(m[r], s[r], mo, so);
    }
    const int64_t p = p0 + tp + 16 * r;
    if (tc == 0 && p < P) {
      part_m[(size_t)blockIdx.y * P + p] = m[r];
      part_s[(size_t)blockIdx.y * P + p] = s[r];
    }
  }
}

__device__ __forceinline__ double lse_merge(const double* __restrict__ part_m, const double* __restrict__ part_s,
                                            int64_t P, int nchunks, int64_t p) {
  double m = -INFINITY, s = 0.0;
  for (int y = 0; y < nchunks; ++y) lse_fold(m, s, part_m[(size_t)y * P + p], part_s[(size_t)y * P + p]);
  return m + log(s);
}

// f[i] = logpdf(s_i) - logpdf(q_i) (kde.py:42): points i and ns + i
__global__ void kde_merge_kernel(const double* __restrict__ part_m, const double* __restrict__ part_s, int64_t ns,
                                 int nchunks, double* __restrict__ f) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ns) return;
  const int64_t P = 2 * ns;
  f[i] = lse_merge(part_m, part_s, P, nchunks, i) - lse_merge(part_m, part_s, P, nchunks, ns + i);
}

}  // namespace

// ---- launchers -----------------------------------------------------------------------------------
KdePlan kde_plan(int64_t ns, int64_t nc, int sm_count) {
  KdePlan p;
  const int64_t P = 2 * ns;
  p.ptiles = (P + KT - 1) / KT;
  const int64_t ctiles = (nc + KT - 1) / KT;
  // enough CTAs for four per SM: a small ensemble splits its centre tiles over gridDim.y
  int64_t want = (4 * (int64_t)sm_count + p.ptiles - 1) / p.ptiles;
  if (want < 1) want = 1;
  if (want > ctiles) want = ctiles;
  p.tpc = (int)((ctiles + want - 1) / want);
  p.nchunks = (int)((ctiles + p.tpc - 1) / p.tpc);
  return p;
}

size_t kde_partial_doubles(int64_t N, int sm_count) {
  // nchunks * P <= (4 sm / ptiles + 1) * ptiles * KT, for pairs (m, s); P <= N + 1
  return 2 * (size_t)((4 * (int64_t)sm_count + (N + 1 + KT - 1) / KT + 1) * KT);
}

cudaError_t launch_kde_factor(const double* L, const double* acc, const double* shift, double nc, int D, double bw,
                              double* minv, double* mean, int* status, cudaStream_t st) {
  int threads = 32;
  while (threads < D && threads < 1024) threads <<= 1;
  kde_factor_kernel<<<1, threads, 0, st>>>(L, acc, shift, nc, D, bw, minv, mean, status);
  return cudaGetLastError();
}

cudaError_t launch_kde_prepare(const HalfStepArgs& a, const double* L, const double* minv, const double* mean,
                               double bw, double* qbuf, double* yp, double* yc, int64_t* jw, cudaStream_t st) {
  const int64_t rows = 2 * (int64_t)a.a_count + (a.N - a.a_count);
  const int G = lanes_per_walker(a.D);
  int threads = 256;
  size_t smem = (size_t)(threads / G) * 2 * a.D * sizeof(double);
  while (smem > 200 * 1024 && threads > G) {
    threads >>= 1;
    smem = (size_t)(threads / G) * 2 * a.D * sizeof(double);
  }
  if (smem > 200 * 1024) return cudaErrorInvalidConfiguration;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kde_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int groups = threads / G;
  kde_prepare_kernel<<<(unsigned)((rows + groups - 1) / groups), threads, smem, st>>>(a, L, minv, mean, bw, qbuf, yp,
                                                                                       yc, jw, G);
  return cudaGetLastError();
}

cudaError_t launch_kde_factors(const double* yp, const double* yc, int64_t ns, int64_t nc, int D, const KdePlan& p,
                               double* part, double* f, cudaStream_t st) {
  if (ns <= 0) return cudaSuccess;
  const int64_t P = 2 * ns;
  double* part_m = part;
  double* part_s = part + (size_t)p.nchunks * P;
  kde_lse_kernel<<<dim3((unsigned)p.ptiles, (unsigned)p.nchunks), LSE_THREADS, 0, st>>>(yp, P, yc, nc, D, p.tpc,
                                                                                         part_m, part_s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  kde_merge_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, st>>>(part_m, part_s, ns, p.nchunks, f);
  return cudaGetLastError();
}

}  // namespace eb
