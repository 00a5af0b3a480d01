// Proposal generators of the moves whose proposal is not a per-walker row formula: WalkMove and
// GaussianMove (MHMove).  Each writes the proposals q[count, D] to a scratch buffer; the fused
// log-prob + accept + update then runs in half_step_generic_kernel<MOVE_PRECOMPUTED, MODEL>.
//
// Reference semantics (file:line relative to the reference):
//   WalkMove.get_proposal ............ moves/walk.py:27-37
//   GaussianMove proposals ........... moves/gaussian.py:72-119   (called from MHMove.propose, mh.py:51)
// Draw specification (DESIGN.md, oracle/philox.py): standard normals 2k, 2k+1 of row i are the cosine / sine
// Box-Muller branches of block (index = i, sub-index = k, TAG_NORMAL); the helper subset of active rank i is
// the first s images of a Feistel permutation keyed by blocks (index = i, sub-index 0..1, TAG_SUBSET);
// multivariate_normal(mean, cov) := mean + L z with L the thresholded lower Cholesky factor of cov.
#include <math.h>

#include "draws.cuh"
#include "engine.cuh"
#include "rowops.cuh"

namespace eb {

namespace {

// ===========================================================================
// thresholded Cholesky of a covariance held as moment sums (oracle/philox.py chol_psd)
// ===========================================================================
// acc = [S1[D] | S2[D*D]] about `shift` over n rows  ->  cov = (S2 - S1 S1^T / n) / (n - 1) (np.cov,
// walk.py:35) -> L (row-major lower factor, upper part zero).  One CTA; column j needs columns < j.
__global__ void __launch_bounds__(1024) cov_chol_kernel(const double* __restrict__ acc, double n, int D,
                                                        double* __restrict__ cov, double* __restrict__ L) {
  __shared__ double s_piv, s_tol;
  __shared__ int s_left;  // pivots still allowed: rank(cov of n rows) <= n - 1
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int e = tid; e < D * D; e += nt) {
    const int r = e / D, c = e - r * D;
    cov[e] = (acc[D + e] - acc[r] * acc[c] / n) / (n - 1.0);
    L[e] = 0.0;
  }
  __syncthreads();
  if (tid == 0) {
    double m = 0.0;
    for (int j = 0; j < D; ++j) m = fmax(m, cov[(size_t)j * D + j]);
    s_tol = 1e-12 * m;
    s_left = n - 1.0 < (double)D ? (int)(n - 1.0) : D;
  }
  __syncthreads();
  for (int j = 0; j < D; ++j) {
    if (tid == 0) {
      double d = cov[(size_t)j * D + j];
      for (int k = 0; k < j; ++k) d -= L[(size_t)j * D + k] * L[(size_t)j * D + k];
      s_piv = (s_left > 0 && d > s_tol) ? sqrt(d) : 0.0;
      if (s_piv > 0.0) s_left -= 1;
      L[(size_t)j * D + j] = s_piv;
    }
    __syncthreads();
    const double piv = s_piv;
    if (piv > 0.0)
      for (int i = j + 1 + tid; i < D; i += nt) {
        double v = cov[(size_t)i * D + j];
        for (int k = 0; k < j; ++k) v -= L[(size_t)i * D + k] * L[(size_t)j * D + k];
        L[(size_t)i * D + j] = v / piv;
      }
    __syncthreads();
  }
}

// ===========================================================================
// WalkMove, s = None: one covariance per split (the whole complement), q_i = s_i + L z_i
// ===========================================================================
__global__ void __launch_bounds__(256) walk_shared_propose_kernel(const HalfStepArgs a, const double* __restrict__ L,
                                                                  double* __restrict__ qbuf, const int G) {
  extern __shared__ double smem[];
  const int D = a.D;
  const int groups = blockDim.x / G;
  const int gid = threadIdx.x / G, g = threadIdx.x % G;
  const int lane = threadIdx.x & 31;
  const unsigned mask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
  const int64_t i = (int64_t)blockIdx.x * groups + gid;
  if (i >= a.a_count) return;
  double* z = smem + (size_t)gid * D;
  const int64_t w = a.order[a.a_start + i];
  const double* s_row = a.coords + (size_t)w * D;
  for (int k = g; 2 * k < D; k += G) {
    double n0, n1;
    normal_pair(a.seed, a.step, (uint32_t)a.split, (uint32_t)k, (uint32_t)i, n0, n1);
    z[2 * k] = n0;
    if (2 * k + 1 < D) z[2 * k + 1] = n1;
  }
  __syncwarp(mask);
  for (int e = g; e < D; e += G) {
    double acc = 0.0;
    const double* Lr = L + (size_t)e * D;
    for (int k = 0; k <= e; ++k) acc = fma(__ldg(Lr + k), z[k], acc);
    qbuf[(size_t)i * D + e] = __dadd_rn(s_row[e], acc);  // walk.py:36
  }
}

// ===========================================================================
// WalkMove, s helpers per walker: one CTA per active walker (D <= 64, s <= 4096)
// ===========================================================================
constexpr int WALK_MAX_D = 64;
constexpr int WALK_MAX_S = 4096;

__global__ void __launch_bounds__(128) walk_subset_propose_kernel(const HalfStepArgs a, const int s0,
                                                                  double* __restrict__ qbuf) {
  extern __shared__ double smem[];
  const int D = a.D, tid = threadIdx.x, nt = blockDim.x;
  double* mean = smem;               // [D]
  double* z = mean + D;              // [D]
  double* cov = z + D;               // [D * D]
  double* L = cov + (size_t)D * D;   // [D * D]
  int32_t* ids = reinterpret_cast<int32_t*>(L + (size_t)D * D);  // [s0] helper walker ids
  __shared__ double s_piv, s_tol;
  __shared__ int s_left;  // pivots still allowed: rank(cov of s0 rows) <= s0 - 1
  const int64_t i = blockIdx.x;
  const int64_t Nc = a.N - a.a_count;
  // walk.py:34  inds = random.choice(Nc, s, replace=False): first s images of the keyed permutation
  FeistelKeys fk;
#pragma unroll
  for (int b = 0; b < FEISTEL_ROUNDS / 4; ++b) {
    const u32x4 kw = draw_words(a.seed, a.step, sub_split((uint32_t)a.split, (uint32_t)b), TAG_SUBSET, (uint32_t)i);
    fk.k[4 * b + 0] = kw.x;
    fk.k[4 * b + 1] = kw.y;
    fk.k[4 * b + 2] = kw.z;
    fk.k[4 * b + 3] = kw.w;
  }
  const int h = feistel_half_bits((uint64_t)Nc);
  for (int j = tid; j < s0; j += nt) {
    const int64_t r = (int64_t)split_permute((uint64_t)j, (uint64_t)Nc, h, fk);
    ids[j] = a.order[complement_slot(r, a.a_start, a.a_count)];
  }
  for (int k = tid; 2 * k < D; k += nt) {
    double n0, n1;
    normal_pair(a.seed, a.step, (uint32_t)a.split, (uint32_t)k, (uint32_t)i, n0, n1);
    z[2 * k] = n0;
    if (2 * k + 1 < D) z[2 * k + 1] = n1;
  }
  __syncthreads();
  // walk.py:35  cov = np.cov(c[inds], rowvar=0): X -= mean; X^T X / (s - 1)
  for (int d = tid; d < D; d += nt) {
    double acc = 0.0;
    for (int j = 0; j < s0; ++j) acc += a.coords[(size_t)ids[j] * D + d];
    mean[d] = acc / (double)s0;
  }
  __syncthreads();
  for (int e = tid; e < D * D; e += nt) {
    const int r = e / D, c = e - r * D;
    if (c < r) continue;
    double acc = 0.0;
    for (int j = 0; j < s0; ++j) {
      const double* x = a.coords + (size_t)ids[j] * D;
      acc = fma(x[r] - mean[r], x[c] - mean[c], acc);
    }
    acc /= (double)(s0 - 1);
    cov[r * D + c] = acc;
    cov[c * D + r] = acc;
    L[r * D + c] = 0.0;
    L[c * D + r] = 0.0;
  }
  __syncthreads();
  if (tid == 0) {
    double m = 0.0;
    for (int j = 0; j < D; ++j) m = fmax(m, cov[j * D + j]);
    s_tol = 1e-12 * m;
    s_left = s0 - 1 < D ? s0 - 1 : D;
  }
  __syncthreads();
  for (int j = 0; j < D; ++j) {
    if (tid == 0) {
      double d = cov[j * D + j];
      for (int k = 0; k < j; ++k) d -= L[j * D + k] * L[j * D + k];
      s_piv = (s_left > 0 && d > s_tol) ? sqrt(d) : 0.0;
      if (s_piv > 0.0) s_left -= 1;
      L[j * D + j] = s_piv;
    }
    __syncthreads();
    const double piv = s_piv;
    if (piv > 0.0)
      for (int r = j + 1 + tid; r < D; r += nt) {
        double v = cov[r * D + j];
        for (int k = 0; k < j; ++k) v -= L[r * D + k] * L[j * D + k];
        L[r * D + j] = v / piv;
      }
    __syncthreads();
  }
  const int64_t w = a.order[a.a_start + i];
  for (int e = tid; e < D; e += nt) {
    double acc = 0.0;
    for (int k = 0; k <= e; ++k) acc = fma(L[e * D + k], z[k], acc);
    qbuf[(size_t)i * D + e] = __dadd_rn(a.coords[(size_t)w * D + e], acc);  // walk.py:36
  }
}

// ===========================================================================
// GaussianMove (gaussian.py:72-119): q = x0 + f * scale * randn (scalar / vector scale), or
// q = x0 + f * (L z) with ONE z for the whole ensemble (full covariance, :116-118); modes
// "vector" (all dims), "random" (one drawn dim per walker), "sequential" (dim = index for everyone)
// ===========================================================================
// v[d] = f * (L z)[d], one CTA
__global__ void gaussian_shift_kernel(const double* __restrict__ L, int D, double f, uint64_t seed, uint64_t step,
                                      double* __restrict__ v) {
  extern __shared__ double z[];
  for (int k = threadIdx.x; 2 * k < D; k += blockDim.x) {
    double n0, n1;
    normal_pair(seed, step, 0u, (uint32_t)k, 0u, n0, n1);
    z[2 * k] = n0;
    if (2 * k + 1 < D) z[2 * k + 1] = n1;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < D; e += blockDim.x) {
    double acc = 0.0;
    for (int k = 0; k <= e; ++k) acc = fma(L[(size_t)e * D + k], z[k], acc);
    v[e] = f * (0.0 + acc);  // gaussian.py:116  np.zeros(D) + L z
  }
}

// one thread per (walker, dim pair).  form: 0 scalar scale[0], 1 per-dim scale[d], 2 shared shift v[d]
__global__ void gaussian_propose_kernel(const double* __restrict__ x0, int64_t row0, int64_t nrows, int D, int form,
                                        const double* __restrict__ scale, double f, int mode, int seq_dim,
                                        uint64_t seed, uint64_t step, double* __restrict__ qbuf) {
  const int npair = (D + 1) / 2;
  const size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (size_t)nrows * npair) return;
  const int64_t r = (int64_t)(id / npair);
  const int k = (int)(id - (size_t)r * npair);
  const int64_t w = row0 + r;
  int dim = -1;  // "vector": every dimension moves
  if (mode == 1) {
    dim = gaussian_random_dim(prop_b(seed, step, 0, (uint32_t)w), D);
  } else if (mode == 2) {
    dim = seq_dim;  // gaussian.py:102
  }
  double n0 = 0.0, n1 = 0.0;
  if (form != 2) normal_pair(seed, step, 0u, (uint32_t)k, (uint32_t)w, n0, n1);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int d = 2 * k + half;
    if (d >= D) break;
    const double x = x0[(size_t)w * D + d];
    double v;
    if (form == 2)
      v = __dadd_rn(x, scale[d]);  // scale = the shared shift f * (L z)
    else  // gaussian.py:97  x0 + factor * scale * randn  (left to right)
      v = __dadd_rn(x, __dmul_rn(__dmul_rn(f, form == 0 ? scale[0] : scale[d]), half ? n1 : n0));
    qbuf[(size_t)r * D + d] = (dim < 0 || dim == d) ? v : x;  // gaussian.py:105-107
  }
}

}  // namespace

// ---- launchers -----------------------------------------------------------------------------------
cudaError_t launch_cov_chol(const double* acc, double n, int D, double* cov, double* L, cudaStream_t st) {
  cov_chol_kernel<<<1, D >= 512 ? 1024 : 256, 0, st>>>(acc, n, D, cov, L);
  return cudaGetLastError();
}

cudaError_t launch_walk_shared_propose(const HalfStepArgs& a, const double* L, double* qbuf, cudaStream_t st) {
  if (a.a_count <= 0) return cudaSuccess;
  const int G = lanes_per_walker(a.D);
  int threads = 256;
  size_t smem = (size_t)(threads / G) * a.D * sizeof(double);
  while (smem > 200 * 1024 && threads > G) {
    threads >>= 1;
    smem = (size_t)(threads / G) * a.D * sizeof(double);
  }
  if (smem > 200 * 1024) return cudaErrorInvalidConfiguration;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(walk_shared_propose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int groups = threads / G;
  walk_shared_propose_kernel<<<(unsigned)((a.a_count + groups - 1) / groups), threads, smem, st>>>(a, L, qbuf, G);
  return cudaGetLastError();
}

bool walk_subset_supported(int D, int s0) { return D <= WALK_MAX_D && s0 <= WALK_MAX_S && s0 >= 2; }

cudaError_t launch_walk_subset_propose(const HalfStepArgs& a, int s0, double* qbuf, cudaStream_t st) {
  if (a.a_count <= 0) return cudaSuccess;
  // (+8: the compiler reads helper ids in pairs, so an odd count touches one id past the end)
  const size_t smem = ((size_t)2 * a.D + (size_t)2 * a.D * a.D) * sizeof(double) + (size_t)s0 * sizeof(int32_t) + 8;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(walk_subset_propose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  walk_subset_propose_kernel<<<(unsigned)a.a_count, 128, smem, st>>>(a, s0, qbuf);
  return cudaGetLastError();
}

cudaError_t launch_gaussian_shift(const double* L, int D, double f, uint64_t seed, uint64_t step, double* v,
                                  cudaStream_t st) {
  gaussian_shift_kernel<<<1, 256, (size_t)(D + 1) * sizeof(double), st>>>(L, D, f, seed, step, v);
  return cudaGetLastError();
}

cudaError_t launch_gaussian_propose(const double* x0, int64_t row0, int64_t nrows, int D, int form, const double* scale,
                                    double f, int mode, int seq_dim, uint64_t seed, uint64_t step, double* qbuf,
                                    cudaStream_t st) {
  if (nrows <= 0) return cudaSuccess;
  const size_t n = (size_t)nrows * ((D + 1) / 2);
  gaussian_propose_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x0, row0, nrows, D, form, scale, f, mode, seq_dim,
                                                                      seed, step, qbuf);
  return cudaGetLastError();
}

}  // namespace eb
