// Per-row device helpers shared by the fused half-step kernels: group reductions, the
// registered log-probability models on a row staged in shared memory, status flags, and
// the (possibly peer-mapped) address of a walker's row.
#pragma once
#include <math.h>

#include "engine.cuh"

namespace eb {

// ===========================================================================
// model log-probabilities on a row staged in shared memory
// ===========================================================================
// G lanes (a power of two <= 32, aligned inside the warp) cooperate on one row
// x[0..D).  Every lane returns the reduced value.  The summation order depends
// only on (D, G) so results are independent of nwalkers and of the GPU count.
__device__ __forceinline__ double group_sum(double v, int G, unsigned mask) {
  for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
  return v;
}

template <int MODEL>
__device__ __forceinline__ double model_logprob(const double* __restrict__ x, double* __restrict__ xc,
                                                int D, int g, int G, unsigned mask, const ModelDev& m) {
  double acc = 0.0;
  if (MODEL == EB_MODEL_GAUSS_ISO) {
    for (int e = g; e < D; e += G) acc = fma(x[e], x[e], acc);
    return -0.5 * group_sum(acc, G, mask);
  } else if (MODEL == EB_MODEL_RING) {
    for (int e = g; e < D; e += G) acc = fma(x[e], x[e], acc);
    const double r = sqrt(group_sum(acc, G, mask));
    const double d = r - m.s0;
    return -(d * d) / (2.0 * m.s1 * m.s1);
  } else if (MODEL == EB_MODEL_ROSENBROCK) {
    for (int e = g; e < D - 1; e += G) {
      const double x0 = x[e], x1 = x[e + 1];
      const double t = x1 - x0 * x0;
      const double u = m.s0 - x0;
      acc += m.s1 * (t * t) + u * u;
    }
    return -group_sum(acc, G, mask);
  } else {  // EB_MODEL_GAUSS_DENSE, CUDA-core fallback for any D
    const double* __restrict__ mu = m.params;
    const double* __restrict__ A = m.params + D;
    for (int e = g; e < D; e += G) xc[e] = x[e] - mu[e];
    __syncwarp(mask);
    for (int j = g; j < D; j += G) {
      double y = 0.0;
      for (int k = 0; k < D; ++k) y = fma(__ldg(A + (size_t)k * D + j), xc[k], y);
      acc = fma(y, xc[j], acc);
    }
    return -0.5 * group_sum(acc, G, mask);
  }
}

// the prior's support (m.lo != nullptr): true on every lane of the group when lo[e] <= x[e] <= hi[e] for all e of
// the staged row (a NaN coordinate is outside); callers then select -inf for a row outside the box
__device__ __forceinline__ bool row_in_box(const double* __restrict__ x, int D, int g, int G, unsigned mask,
                                           const ModelDev& m) {
  bool in = true;
  for (int e = g; e < D; e += G) in &= (__ldg(m.lo + e) <= x[e]) & (x[e] <= __ldg(m.hi + e));
  return __all_sync(mask, in);
}

__device__ __forceinline__ void flag_nonfinite(double v, int* status) {
  if (isinf(v)) atomicOr(status, FLAG_INF_PARAM);
  if (isnan(v)) atomicOr(status, FLAG_NAN_PARAM);
}

// row pointer of walker w: local state, or the owner's buffer over NVLink
__device__ __forceinline__ const double* row_ptr(const HalfStepArgs& a, int64_t w) {
  if (a.peer_coords != nullptr) return a.peer_coords[w / a.rows_per_rank] + (size_t)w * a.D;
  return a.coords + (size_t)w * a.D;
}

}  // namespace eb
