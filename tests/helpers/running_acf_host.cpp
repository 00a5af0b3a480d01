// Host-side restatement of emcee_b200/csrc/running_acf.cu, built with g++ by tests/test_running_acf_host.py and
// tests/test_gpu_running_acf.py: the ring, the first values, the double-double sums and their block fold, and a read,
// laid out and ordered as the kernels do it, with the arithmetic of running_acf.h.
#include <stdint.h>

#include <vector>

#include "../../emcee_b200/csrc/running_acf.h"

namespace {

using namespace eb;

struct Sums {
  uint64_t S, max_lag, R, n = 0;
  std::vector<double> x0, ring, head, s_hi, s_lo, y_hi, y_lo;
  Sums(uint64_t series, uint64_t lags)
      : S(series), max_lag(lags), R(racf_ring(lags)), x0(series), ring(R * series), head(lags * series),
        s_hi((lags + 1) * series), s_lo((lags + 1) * series), y_hi(series), y_lo(series) {}
  double yat(int64_t t, uint64_t s) const { return t < 0 ? 0.0 : ring[((uint64_t)t % R) * S + s]; }

  void record(const double* x) {
    for (uint64_t s = 0; s < S; ++s) {
      double y = 0.0;
      if (n == 0) x0[s] = x[s];
      else y = x[s] - x0[s];
      ring[(n % R) * S + s] = y;
      if (n < max_lag) head[n * S + s] = y;
    }
    if ((n + 1) % RACF_B == 0) fold(n / RACF_B);
    ++n;
  }

  void fold(uint64_t b) {
    const int64_t bB = (int64_t)(b * RACF_B), oldest = bB - (int64_t)max_lag;
    for (uint64_t s = 0; s < S; ++s) {
      RacfDd y{y_hi[s], y_lo[s]};
      for (int k = 0; k < RACF_B; ++k) y = racf_dd_add_d(y, yat(bB + k, s));
      y_hi[s] = y.hi;
      y_lo[s] = y.lo;
      for (uint64_t tau = 0; tau <= max_lag; ++tau) {
        double p = 0.0;
        for (int k = 0; k < RACF_B; ++k) {
          const int64_t t = bB + k - (int64_t)tau;
          p = racf_fma(yat(bB + k, s), (t >= 0 && t >= oldest) ? yat(t, s) : 0.0, p);
        }
        const RacfDd r = racf_dd_add_d(RacfDd{s_hi[tau * S + s], s_lo[tau * S + s]}, p);
        s_hi[tau * S + s] = r.hi;
        s_lo[tau * S + s] = r.lo;
      }
    }
  }

  // rho[L, D] of walkers N (S = N D)
  void read(uint64_t N, int D, double* rho) const {
    const uint64_t L = racf_rows(n, max_lag), base = n / RACF_B * RACF_B, m = n % RACF_B;
    std::vector<double> r(L * S);
    for (uint64_t s = 0; s < S; ++s) {
      RacfDd Y{y_hi[s], y_lo[s]}, hd{0.0, 0.0}, tl{0.0, 0.0};
      for (uint64_t k = 0; k < m; ++k) Y = racf_dd_add_d(Y, yat((int64_t)(base + k), s));
      double c0 = 0.0;
      for (uint64_t tau = 0; tau < L; ++tau) {
        if (tau > 0) {
          hd = racf_dd_add_d(hd, head[(tau - 1) * S + s]);
          tl = racf_dd_add_d(tl, yat((int64_t)(n - tau), s));
        }
        RacfDd Sd{s_hi[tau * S + s], s_lo[tau * S + s]};
        if (m > 0) {
          double p = 0.0;
          for (uint64_t k = 0; k < m; ++k)
            p = racf_fma(yat((int64_t)(base + k), s), yat((int64_t)(base + k) - (int64_t)tau, s), p);
          Sd = racf_dd_add_d(Sd, p);
        }
        const double c = racf_cov(Sd, Y, hd, tl, n, tau);
        if (tau == 0) c0 = c;
        r[tau * S + s] = racf_div(c, c0);
      }
    }
    const uint64_t nch = racf_nchunks(N);
    for (uint64_t tau = 0; tau < L; ++tau)
      for (int d = 0; d < D; ++d) {
        double total = 0.0;
        for (uint64_t ch = 0; ch < nch; ++ch) {
          const uint64_t w0 = ch * RACF_WCHUNK, w1 = w0 + RACF_WCHUNK < N ? w0 + RACF_WCHUNK : N;
          double a = r[tau * S + w0 * D + d];
          for (uint64_t w = w0 + 1; w < w1; ++w) a = racf_add(a, r[tau * S + w * D + d]);
          total = ch == 0 ? a : racf_add(total, a);
        }
        rho[tau * D + d] = racf_div(total, (double)N);
      }
  }
};

}  // namespace

extern "C" {

// x[n, N, D]: record every state; after each index listed in `reads` (ascending) a read whose result is dropped.
// rho[min(n, max_lag + 1), D] of the final read.
void probe_running_acf(const double* x, uint64_t n, uint64_t N, int D, uint64_t max_lag, const uint64_t* reads,
                       uint64_t nreads, double* rho) {
  Sums sums(N * D, max_lag);
  std::vector<double> scratch((max_lag + 1) * D);
  uint64_t next = 0;
  for (uint64_t t = 0; t < n; ++t) {
    sums.record(x + t * N * D);
    while (next < nreads && reads[next] == t) {
      sums.read(N, D, scratch.data());
      ++next;
    }
  }
  sums.read(N, D, rho);
}

// elementwise fma, to check the numpy statement's emulation
void probe_fma(const double* a, const double* b, const double* c, uint64_t n, double* out) {
  for (uint64_t i = 0; i < n; ++i) out[i] = racf_fma(a[i], b[i], c[i]);
}
}
