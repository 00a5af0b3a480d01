// Host-side probe of emcee_b200/csrc/acf_grid.h (the slab size of acf_slabs and the grids of launch_acf_slab),
// built by tests/test_autocorr_exact_host.py with g++.
#include "../../emcee_b200/csrc/acf_grid.h"

extern "C" {
// out[12] = M, walkers per slab, scratch bytes per series, then the AcfGrid of a full slab: B, local_threads,
// local_blocks, mean_blocks, load_tiles_t, load_blocks, global_blocks, lag_tiles, accumulate_blocks
void probe_acf_grid(uint64_t n_t, uint64_t nw, uint64_t nd, uint64_t* out) {
  const int M = eb::acf_fft_length(n_t);
  const uint64_t wb = eb::acf_slab_walkers(n_t, nw, nd);
  const eb::AcfGrid g = eb::acf_grid(n_t, wb, nd, M);
  const uint64_t v[12] = {(uint64_t)M,       wb,          eb::acf_bytes_per_series(n_t),
                          (uint64_t)g.B,     (uint64_t)g.local_threads, g.local_blocks,
                          g.mean_blocks,     g.load_tiles_t, g.load_blocks,
                          g.global_blocks,   g.lag_tiles,    g.accumulate_blocks};
  for (int i = 0; i < 12; ++i) out[i] = v[i];
}
}
