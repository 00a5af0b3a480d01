// Host-side probe of the segmented selection of eb_chain_select_segments, built by
// tests/test_batch_device_backend_host.py with g++.  It runs the CPU selection of select_host.cpp (the plan of
// select_keys.h, its CTA column blocks, group lookup and sorts) over the nseg * D columns the device reads.
#include "select_host.cpp"

extern "C" {
// x[count, nseg, N, D] (each stored step holds nseg segments of N rows), read as select_pass_kernel reads it: column
// c = k * D + d at offset k * N * D + w * D + d of a step.  out[nseg, nranks, D], has_nan[nseg, D]; returns the
// passes, or -1 as probe_select does.
int probe_select_segments(const double* x, uint64_t count, uint64_t nseg, uint64_t N, int D, const uint64_t* ranks,
                          size_t nranks, uint64_t cand_budget, double* out, uint8_t* has_nan) {
  const uint64_t C = nseg * (uint64_t)D, rows = count * N;
  std::vector<double> v(rows * C);
  for (uint64_t s = 0; s < count; ++s)
    for (uint64_t w = 0; w < N; ++w)
      for (uint64_t c = 0; c < C; ++c) {
        const uint64_t k = c / (uint64_t)D, d = c % (uint64_t)D;
        v[(s * N + w) * C + c] = x[s * nseg * N * D + k * N * D + w * D + d];
      }
  std::vector<double> o(nranks * C);
  const int passes = probe_select(v.data(), rows, (int)C, ranks, nranks, cand_budget, o.data(), has_nan);
  for (uint64_t c = 0; c < C; ++c)
    for (size_t r = 0; r < nranks; ++r) out[((c / D) * nranks + r) * D + c % D] = o[r * C + c];
  return passes;
}
}
