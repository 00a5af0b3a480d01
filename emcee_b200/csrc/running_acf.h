// The arithmetic of the running autocorrelation function (running_acf.cu, eb_running_acf_config / eb_running_acf_read):
// the block fold of the lag sums, the final combination and the walker reduction, in the order the device runs them.
// Everything here is a function of the recorded states alone -- not of the grid, the tiling or how the steps were cut
// into calls -- so tests/helpers/running_acf_host.cpp, which includes this file without CUDA, reproduces the device's
// rho with `==`.
//
// Series.  Every (walker w, parameter d) is one series s = w D + d of recorded values x_0, x_1, .. x_{n-1}, kept
// shifted by its first value: y_t = x_t - x_0 (one rounding; y_0 = 0), and y_t = 0 for t < 0.
//
// Blocks.  Recorded index t belongs to block t / RACF_B.  Once a block is complete its lag products are folded:
//   p(tau) = fma chain over k = 0 .. RACF_B - 1, ascending, from 0.0:  p = fma(y_{bB+k}, y_{bB+k-tau}, p)
//   S(tau) = racf_dd_add_d(S(tau), p(tau))   for tau = 0 .. max_lag    (S double-double, starting at 0)
//   Y = racf_dd_add_d(Y, y_{bB+k})   for k = 0 .. RACF_B - 1, ascending    (Y double-double, starting at 0)
// A read with m = n mod RACF_B > 0 pending values folds the first m terms of the next block's chains the same way into
// copies of S and Y, so later reads see the same S and Y.
//
// Combination.  With head_tau = sum_{t < tau} y_t (added ascending into a double-double) and tail_tau =
// sum_{t >= n - tau} y_t (added descending), ybar = Y / n:
//   c(tau) = S(tau) - ybar ((Y - head_tau) + (Y - tail_tau)) + (n - tau) ybar^2        (all double-double, racf_cov)
// then r_w(tau) = hi(c(tau)) / hi(c(0)) in double (0 / 0 = NaN for a constant series, numpy's answer).
//
// Walker reduction.  rho(tau, d) = (sum over walker chunks of RACF_WCHUNK walkers, each summed ascending from its first
// walker; the chunk sums added ascending from chunk 0's) / N.
//
// Rounding (DESIGN §5.7 derives it; tests/running_acf_ref.py evaluates it): a block partial is an fma chain of
// RACF_B terms, |p^ - p| <= gamma_B sum |y_t y_{t-tau}|, so the lag sum is within gamma_B A(tau) + O((n / B + max_lag)
// u^2) of the exact lag sum of y, A(tau) = sum |y_t y_{t-tau}|.  Every value enters Y through its own double-double
// addition (accurate to 2 u^2 of the running sum), never through a plain-double partial sum, so Y is within
// 3 n u^2 sum |y| of the exact sum and its error is second order in c(tau) as well.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define EB_RACF_HD __host__ __device__ __forceinline__
#else
#define EB_RACF_HD inline
#endif

namespace eb {

constexpr int RACF_B = 64;        // recorded steps per block of the lag-sum fold
constexpr int RACF_WCHUNK = 64;   // walkers per chunk of the walker reduction

struct RacfDd {
  double hi, lo;
};

EB_RACF_HD double racf_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
EB_RACF_HD double racf_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
EB_RACF_HD double racf_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
EB_RACF_HD double racf_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
EB_RACF_HD double racf_fma(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}

// s + e == a + b exactly (Knuth)
EB_RACF_HD RacfDd racf_two_sum(double a, double b) {
  const double s = racf_add(a, b);
  const double bb = racf_sub(s, a);
  const double e = racf_add(racf_sub(a, racf_sub(s, bb)), racf_sub(b, bb));
  return RacfDd{s, e};
}
// s + e == a + b exactly when |a| >= |b| or a == 0
EB_RACF_HD RacfDd racf_fast_two_sum(double a, double b) {
  const double s = racf_add(a, b);
  return RacfDd{s, racf_sub(b, racf_sub(s, a))};
}

EB_RACF_HD RacfDd racf_dd_add_d(RacfDd a, double b) {
  const RacfDd s = racf_two_sum(a.hi, b);
  return racf_fast_two_sum(s.hi, racf_add(s.lo, a.lo));
}
EB_RACF_HD RacfDd racf_dd_add(RacfDd a, RacfDd b) {
  RacfDd s = racf_two_sum(a.hi, b.hi);
  const RacfDd t = racf_two_sum(a.lo, b.lo);
  s = racf_fast_two_sum(s.hi, racf_add(s.lo, t.hi));
  return racf_fast_two_sum(s.hi, racf_add(s.lo, t.lo));
}
EB_RACF_HD RacfDd racf_dd_neg(RacfDd a) { return RacfDd{-a.hi, -a.lo}; }
EB_RACF_HD RacfDd racf_dd_sub(RacfDd a, RacfDd b) { return racf_dd_add(a, racf_dd_neg(b)); }
EB_RACF_HD RacfDd racf_dd_mul(RacfDd a, RacfDd b) {
  const double p = racf_mul(a.hi, b.hi);
  double e = racf_fma(a.hi, b.hi, -p);
  e = racf_fma(a.hi, b.lo, e);
  e = racf_fma(a.lo, b.hi, e);
  return racf_fast_two_sum(p, e);
}
EB_RACF_HD RacfDd racf_dd_mul_d(RacfDd a, double b) {
  const double p = racf_mul(a.hi, b);
  const double e = racf_fma(a.lo, b, racf_fma(a.hi, b, -p));
  return racf_fast_two_sum(p, e);
}
EB_RACF_HD RacfDd racf_dd_div_d(RacfDd a, double b) {
  const double q1 = racf_div(a.hi, b);
  const double p = racf_mul(q1, b);
  const double pe = racf_fma(q1, b, -p);
  const double r = racf_add(racf_sub(a.hi, p), racf_sub(a.lo, pe));
  return racf_fast_two_sum(q1, racf_div(r, b));
}

// the unnormalised autocovariance c(tau) of n recorded values (the combination above); s, y, head, tail at this tau
EB_RACF_HD double racf_cov(RacfDd s, RacfDd y, RacfDd head, RacfDd tail, uint64_t n, uint64_t tau) {
  const RacfDd ybar = racf_dd_div_d(y, (double)n);
  const RacfDd t = racf_dd_add(racf_dd_sub(y, head), racf_dd_sub(y, tail));
  RacfDd c = racf_dd_sub(s, racf_dd_mul(ybar, t));
  c = racf_dd_add(c, racf_dd_mul_d(racf_dd_mul(ybar, ybar), (double)(n - tau)));
  return c.hi;
}

EB_RACF_HD uint64_t racf_nchunks(uint64_t N) { return (N + RACF_WCHUNK - 1) / RACF_WCHUNK; }

// slots of the ring: the last max_lag + RACF_B recorded values of every series
EB_RACF_HD uint64_t racf_ring(uint64_t max_lag) { return max_lag + RACF_B; }

// rows of rho a read returns after n recorded steps
EB_RACF_HD uint64_t racf_rows(uint64_t n, uint64_t max_lag) { return n < max_lag + 1 ? n : max_lag + 1; }

}  // namespace eb
