// The summation order of the running trace (trace.cu, eb_trace_config / eb_trace_read): how the N rows of one step's
// ensemble are cut up and in which order the partial sums meet.  Everything here is a function of N alone -- not of
// the grid, the SM count or ndim -- so a row of the trace is the same bytes whatever launched it, and
// tests/helpers/trace_sum_host.cpp, which includes this file without CUDA, reproduces it with `==`.
//
//   leaf    TRACE_LEAF_ROWS consecutive rows, summed one after the other in row order (trace_term / trace_lp_term);
//           the last leaf may be short.
//   chunk   TRACE_CHUNK_LEAVES consecutive leaves, their sums added one after the other in leaf order, starting
//           from leaf 0's sum; the last chunk may hold fewer leaves.
//   tree    the n = trace_nchunks(N) chunk sums p[0 .. n - 1], folded in place:
//             for (s = trace_tree_start(n); s >= 1; s /= 2)  for every i < s with i + s < n:  p[i] += p[i + s]
//           (the additions of one level do not depend on each other); p[0] is the total.
//
// Per column j the sums are taken about the shift x[0][j], walker 0's coordinate: d = x[r][j] - shift,
// S1 += d, S2 = fma(d, d, S2).  Then mean = shift + S1 / N and var = (S2 - S1 (S1 / N)) / (N - 1), the product
// folded with one fma and a rounding-negative result set to 0 (trace_mean, trace_var).  A constant column has d == 0
// in every row and so var == 0 exactly; N == 1 gives 0 / 0 = NaN, numpy's ddof=1 answer.  The log-probabilities are
// summed raw (no shift: walker 0 may sit at -inf) through the same leaves, chunks and tree, together with their
// maximum, its lowest walker and the number of set bytes of the accept mask (TraceLp, trace_lp_join).
//
// Rounding: a total passes through at most TRACE_LEAF_ROWS - 1 + TRACE_CHUNK_LEAVES - 1 + ceil(log2 n) additions,
// so |S1 - sum d| <= trace_depth(N) u sum|d| to first order (u = 2^-53), and likewise S2 with one more rounding for
// the fma.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define EB_TRACE_HD __host__ __device__ __forceinline__
#else
#define EB_TRACE_HD inline
#endif

namespace eb {

constexpr int TRACE_LEAF_ROWS = 16;
constexpr int TRACE_CHUNK_LEAVES = 16;
constexpr int TRACE_CHUNK_ROWS = TRACE_LEAF_ROWS * TRACE_CHUNK_LEAVES;
constexpr int TRACE_EXTRA = 4;  // a trace row is [mean D | var D | log_prob_mean, log_prob_max, accepted, argmax]

EB_TRACE_HD uint64_t trace_nchunks(uint64_t N) { return (N + TRACE_CHUNK_ROWS - 1) / TRACE_CHUNK_ROWS; }

// the first stride of the tree over n >= 1 chunk sums: half the smallest power of two >= n (0 when n == 1)
EB_TRACE_HD uint64_t trace_tree_start(uint64_t n) {
  uint64_t p = 1;
  while (p < n) p <<= 1;
  return p >> 1;
}

// additions on the longest path from one term to the total
EB_TRACE_HD int trace_depth(uint64_t N) {
  int levels = 0;
  for (uint64_t s = trace_tree_start(trace_nchunks(N)); s >= 1; s >>= 1) ++levels;
  return TRACE_LEAF_ROWS - 1 + TRACE_CHUNK_LEAVES - 1 + levels;
}

EB_TRACE_HD double trace_fma(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}
EB_TRACE_HD double trace_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// one row's term of one column, about `shift`
EB_TRACE_HD void trace_term(double x, double shift, double& s1, double& s2) {
#ifdef __CUDA_ARCH__
  const double d = __dsub_rn(x, shift);
#else
  const double d = x - shift;
#endif
  s1 = trace_add(s1, d);
  s2 = trace_fma(d, d, s2);
}

EB_TRACE_HD double trace_mean(double shift, double s1, uint64_t N) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(shift, __ddiv_rn(s1, (double)N));
#else
  return shift + s1 / (double)N;
#endif
}

EB_TRACE_HD double trace_var(double s1, double s2, uint64_t N) {
#ifdef __CUDA_ARCH__
  const double t = __ddiv_rn(s1, (double)N);
  const double v = __ddiv_rn(__fma_rn(-s1, t, s2), (double)(N - 1));
#else
  const double t = s1 / (double)N;
  const double v = fma(-s1, t, s2) / (double)(N - 1);
#endif
  return v < 0.0 ? 0.0 : v;  // NaN (N == 1) passes through
}

// the log-probability side of a leaf, a chunk or the whole ensemble
struct TraceLp {
  double sum;     // of log_prob
  double max;     // largest log_prob ...
  double walker;  // ... and the lowest walker holding it (exact in a double)
  double accepted;  // set bytes of the accept mask (exact in a double)
};

EB_TRACE_HD TraceLp trace_lp_first(double lp, uint64_t walker, unsigned accepted) {
  return TraceLp{lp, lp, (double)walker, accepted ? 1.0 : 0.0};
}

// the next row of a leaf (walker ascending): a later walker replaces the maximum only when strictly larger
EB_TRACE_HD void trace_lp_term(TraceLp& a, double lp, uint64_t walker, unsigned accepted) {
  a.sum = trace_add(a.sum, lp);
  if (lp > a.max) {
    a.max = lp;
    a.walker = (double)walker;
  }
  a.accepted += accepted ? 1.0 : 0.0;
}

// a += b, for leaves into a chunk and for the tree; the tree joins chunks out of walker order, so a tie is settled
// by the walker number
EB_TRACE_HD void trace_lp_join(TraceLp& a, const TraceLp& b) {
  a.sum = trace_add(a.sum, b.sum);
  if (b.max > a.max || (b.max == a.max && b.walker < a.walker)) {
    a.max = b.max;
    a.walker = b.walker;
  }
  a.accepted += b.accepted;
}

}  // namespace eb
