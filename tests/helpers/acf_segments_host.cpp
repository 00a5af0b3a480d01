// Host-side probe of the segment slab planning in emcee_b200/csrc/acf_grid.h (acf_segment_slab_walkers,
// acf_slab_next and the accumulate grid of acf_slabs / launch_acf_slab), built by
// tests/test_batch_device_backend_host.py with g++.
#include "../../emcee_b200/csrc/acf_grid.h"

extern "C" {
// the slabs acf_slabs runs over nseg segments of nw / nseg walkers: w0[i], wn[i] and the accumulate grid's CTAs of
// each, at most cap of them; returns the number of slabs
uint64_t probe_acf_segment_slabs(uint64_t n_t, uint64_t nw, uint64_t nd, uint64_t nseg, uint64_t* w0, uint64_t* wn,
                                 uint64_t* blocks, uint64_t cap) {
  const int M = eb::acf_fft_length(n_t);
  const uint64_t seg_w = nw / nseg, wb = eb::acf_segment_slab_walkers(n_t, nw, nd, nseg);
  uint64_t i = 0;
  for (uint64_t w = 0, n = 0; w < nw; w += n, ++i) {
    n = eb::acf_slab_next(w, nw, seg_w, wb);
    if (i < cap) {
      w0[i] = w;
      wn[i] = n;
      blocks[i] = eb::acf_grid(n_t, n, nd, M, (w + n - 1) / seg_w - w / seg_w + 1).accumulate_blocks;
    }
  }
  return i;
}
}
