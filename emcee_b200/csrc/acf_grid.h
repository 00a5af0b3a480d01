// Launch geometry of the autocorrelation kernels (analysis.cu, launch_acf_slab) and the walker slabs that feed
// them (capi.cu, acf_slabs).  Host code only, without CUDA, so that tests/helpers/acf_grid_host.cpp can build it
// for the CPU tests.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace eb {

constexpr int ACF_BLOCK = 8192;                      // fft_local_kernel's block: 128 KB of double2 in shared memory
constexpr size_t ACF_SLAB_BYTES = (size_t)1 << 30;  // device scratch a walker slab is sized to

// M = 2 * next_pow_two(n_t): the zero-padded FFT length (autocorr.py:12-17)
inline int acf_fft_length(size_t n_t) {
  size_t n = 1;
  while (n < n_t) n <<= 1;
  return (int)(2 * n);
}

// bytes of device scratch per series of the slab: complex work array + its row of the chain slab
inline size_t acf_bytes_per_series(size_t n_t) { return (size_t)acf_fft_length(n_t) * 2 * sizeof(double) + n_t * sizeof(double); }

// walkers per slab: ~ACF_SLAB_BYTES of scratch, at least one walker, at most nw
inline size_t acf_slab_walkers(size_t n_t, size_t nw, size_t nd) {
  const size_t wb = ACF_SLAB_BYTES / (acf_bytes_per_series(n_t) * nd);
  return wb < 1 ? 1 : (wb > nw ? nw : wb);
}

// Walkers per slab of a chain of nseg segments (ensembles) of seg_w = nw / nseg walkers each: whole segments, as many
// as ~ACF_SLAB_BYTES of scratch holds, when one segment fits; otherwise the slab acf_slab_walkers gives one segment
// alone, so that a segment is split exactly as the chain of that ensemble alone would be.  nseg = 1: acf_slab_walkers.
inline size_t acf_segment_slab_walkers(size_t n_t, size_t nw, size_t nd, size_t nseg) {
  const size_t seg_w = nw / nseg;
  const size_t one = acf_slab_walkers(n_t, seg_w, nd);
  if (one < seg_w) return one;
  return acf_slab_walkers(n_t, nw, nd) / seg_w * seg_w;
}

// Walkers of the slab starting at walker w0 (slabs of wb walkers from acf_segment_slab_walkers): a slab of whole
// segments stops at the chain's end, a slab inside one segment at that segment's end.
inline size_t acf_slab_next(size_t w0, size_t nw, size_t seg_w, size_t wb) {
  const size_t end = wb >= seg_w ? nw : (w0 / seg_w + 1) * seg_w;
  return wb < end - w0 ? wb : end - w0;
}

// Grids of the kernels launch_acf_slab runs over a slab of S = wb * nd series of n_t samples.  Every grid is 1-D,
// on x (limit 2^31 - 1), so the series and parameter counts are bounded by memory, not by grid y's 65 535.
struct AcfGrid {
  int B;                        // fft_local_kernel: one CTA per aligned block of B = min(M, ACF_BLOCK) points ...
  int local_threads;            //   ... with 512 threads from B = 1024 on, 128 below
  uint64_t local_blocks;        //   ... S * M / B CTAs: CTA k holds points [k B, (k + 1) B) of the slab's z
  uint64_t mean_blocks;         // acf_mean_kernel: 128 series per CTA
  uint64_t load_tiles_t;        // acf_load_kernel: 32 x 32 (t, series) tiles, ceil(M / 32) along t ...
  uint64_t load_blocks;         //   ... times ceil(S / 32) along the series: CTA k = series tile * load_tiles_t + t tile
  uint64_t global_blocks;       // fft_global_stage_kernel: S * M / 2 butterflies, 256 per CTA
  uint64_t lag_tiles;           // acf_accumulate_kernel: ceil(n_t / 256) tiles of 256 lags ...
  uint64_t accumulate_blocks;   //   ... times nd times the segments the slab holds: CTA k = (segment * nd + parameter)
                                //   * lag_tiles + lag tile
};

// nks: the segments the slab's walkers belong to (1 for a single ensemble)
inline AcfGrid acf_grid(uint64_t n_t, uint64_t wb, uint64_t nd, int M, uint64_t nks = 1) {
  const uint64_t S = wb * nd, m = (uint64_t)M;
  AcfGrid g;
  g.B = M < ACF_BLOCK ? M : ACF_BLOCK;
  g.local_threads = g.B >= 1024 ? 512 : 128;
  g.local_blocks = S * (m / (uint64_t)g.B);
  g.mean_blocks = (S + 127) / 128;
  g.load_tiles_t = (m + 31) / 32;
  g.load_blocks = g.load_tiles_t * ((S + 31) / 32);
  g.global_blocks = (S * (m / 2) + 255) / 256;
  g.lag_tiles = (n_t + 255) / 256;
  g.accumulate_blocks = g.lag_tiles * nd * nks;
  return g;
}

}  // namespace eb
