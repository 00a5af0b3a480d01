// Host-side restatement of emcee_b200/csrc/trace_sum.h, built with g++ by tests/test_trace_host.py and
// tests/test_gpu_trace.py: one row of the running trace computed on the CPU with the header's leaves, chunks and
// tree, its terms and its closing formulas -- what trace_partial_kernel and trace_finish_kernel compute in parallel.
#include <vector>

#include "../../emcee_b200/csrc/trace_sum.h"

namespace {

// p[0 .. n - 1] folded in place in the header's tree order; Join(a, b) is a += b
template <class T, class Join>
void tree(std::vector<T>& p, Join join) {
  const uint64_t n = p.size();
  for (uint64_t s = eb::trace_tree_start(n); s >= 1; s >>= 1)
    for (uint64_t i = 0; i < s && i + s < n; ++i) join(p[i], p[i + s]);
}

}  // namespace

extern "C" {

int probe_trace_depth(uint64_t N) { return eb::trace_depth(N); }

// x[N, D] row-major -> mean[D], var[D]
void probe_trace_columns(const double* x, uint64_t N, int D, double* mean, double* var) {
  using namespace eb;
  const uint64_t n = trace_nchunks(N);
  std::vector<double> p1(n), p2(n);
  for (int j = 0; j < D; ++j) {
    const double shift = x[j];
    for (uint64_t c = 0; c < n; ++c) {
      double c1 = 0.0, c2 = 0.0;
      const uint64_t c0 = c * TRACE_CHUNK_ROWS;
      for (int leaf = 0; leaf < TRACE_CHUNK_LEAVES; ++leaf) {
        const uint64_t r0 = c0 + (uint64_t)leaf * TRACE_LEAF_ROWS;
        if (r0 >= N) break;
        const uint64_t r1 = r0 + TRACE_LEAF_ROWS < N ? r0 + TRACE_LEAF_ROWS : N;
        double s1 = 0.0, s2 = 0.0;
        for (uint64_t r = r0; r < r1; ++r) trace_term(x[r * D + j], shift, s1, s2);
        if (leaf == 0) {
          c1 = s1;
          c2 = s2;
        } else {
          c1 = trace_add(c1, s1);
          c2 = trace_add(c2, s2);
        }
      }
      p1[c] = c1;
      p2[c] = c2;
    }
    tree(p1, [](double& a, double b) { a = trace_add(a, b); });
    tree(p2, [](double& a, double b) { a = trace_add(a, b); });
    mean[j] = trace_mean(shift, p1[0], N);
    var[j] = trace_var(p1[0], p2[0], N);
  }
}

// lp[N], acc[N] (bytes) -> out = {log_prob_mean, log_prob_max, accepted, argmax walker}
void probe_trace_log_prob(const double* lp, const uint8_t* acc, uint64_t N, double* out) {
  using namespace eb;
  const uint64_t n = trace_nchunks(N);
  std::vector<TraceLp> p(n);
  for (uint64_t c = 0; c < n; ++c) {
    const uint64_t c0 = c * TRACE_CHUNK_ROWS;
    for (int leaf = 0; leaf < TRACE_CHUNK_LEAVES; ++leaf) {
      const uint64_t r0 = c0 + (uint64_t)leaf * TRACE_LEAF_ROWS;
      if (r0 >= N) break;
      const uint64_t r1 = r0 + TRACE_LEAF_ROWS < N ? r0 + TRACE_LEAF_ROWS : N;
      TraceLp t = trace_lp_first(lp[r0], r0, acc[r0]);
      for (uint64_t r = r0 + 1; r < r1; ++r) trace_lp_term(t, lp[r], r, acc[r]);
      if (leaf == 0) p[c] = t;
      else trace_lp_join(p[c], t);
    }
  }
  tree(p, [](TraceLp& a, const TraceLp& b) { trace_lp_join(a, b); });
  out[0] = p[0].sum / (double)N;
  out[1] = p[0].max;
  out[2] = p[0].accepted;
  out[3] = p[0].walker;
}
}
