// Host-side probe of the ring origin of emcee_b200/csrc/chain_map.h (the slot map of a running window's ring), built by
// tests/test_window_host.py with g++.
#include "../../emcee_b200/csrc/chain_map.h"

extern "C" {
// runs of the slice read from ring origin `origin` as rows (seg, off, k0, n) in out[4 * max_runs]; returns the number
// of runs, or -1 when the slice is refused
long long probe_ring_runs(const uint64_t* start, size_t nseg, uint64_t origin, uint64_t first, uint64_t stride,
                          uint64_t count, uint64_t* out, size_t max_runs) {
  size_t r = 0;
  const bool ok = eb::for_each_chain_run(start, nseg, origin, first, stride, count,
                                         [&](size_t s, uint64_t off, uint64_t k0, uint64_t n) {
                                           if (r < max_runs) {
                                             out[4 * r + 0] = s;
                                             out[4 * r + 1] = off;
                                             out[4 * r + 2] = k0;
                                             out[4 * r + 3] = n;
                                           }
                                           ++r;
                                         });
  return ok ? (long long)r : -1;
}

// the same slice through the map without an origin (what every chain that is not a ring reads)
long long probe_plain_runs(const uint64_t* start, size_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                           uint64_t* out, size_t max_runs) {
  size_t r = 0;
  const bool ok = eb::for_each_chain_run(start, nseg, first, stride, count,
                                         [&](size_t s, uint64_t off, uint64_t k0, uint64_t n) {
                                           if (r < max_runs) {
                                             out[4 * r + 0] = s;
                                             out[4 * r + 1] = off;
                                             out[4 * r + 2] = k0;
                                             out[4 * r + 3] = n;
                                           }
                                           ++r;
                                         });
  return ok ? (long long)r : -1;
}
}
