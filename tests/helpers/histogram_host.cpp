// Host-side probe of emcee_b200/csrc/hist_bins.h, built by tests/test_chain_histogram_host.py with g++: the two bin
// rules one value at a time, and the whole pair histogram of eb_chain_histogram2d run on the CPU with the same tiles
// (hist2_block, hist2_tiles), the same per-value bins and the same output pair index as hist2_kernel.
#include <vector>

#include "../../emcee_b200/csrc/hist_bins.h"

extern "C" {

// out[i] = the bin of x[i] under np.histogram's uniform rule, HIST_DROP or HIST_BAD
void probe_uniform(const double* x, size_t n, double first, double last, double span, int bins, const double* edges,
                   int* out) {
  for (size_t i = 0; i < n; ++i) out[i] = eb::hist_bin_uniform(x[i], first, last, span, bins, edges);
}

// out[i] = the bin of x[i] under np.histogramdd's rule, or HIST_DROP
void probe_searched(const double* x, size_t n, const double* edges, int bins, int* out) {
  for (size_t i = 0; i < n; ++i) out[i] = eb::hist_bin_searched(x[i], edges, bins);
}

// the tile count of m positions in blocks of b: listed (hist2_tiles) and closed form (hist2_ntiles)
void probe_ntiles(int m, int b, uint64_t* listed, uint64_t* closed) {
  *listed = eb::hist2_tiles(m, b).size();
  *closed = eb::hist2_ntiles(m, b);
}

// x[rows, D] row-major; params[m]; edges[m, bins + 1]; hist[m (m - 1) / 2, bins, bins] (zeroed here).  The tiles
// are those of a shared-memory budget of hist_bytes, at most block_max positions per block.  Returns the number of
// tiles.
int probe_hist2(const double* x, uint64_t rows, int D, const uint32_t* params, int m, int bins, const double* edges,
                size_t hist_bytes, int block_max, uint64_t* hist) {
  using namespace eb;
  int b = hist2_block(m, bins, hist_bytes);
  if (b > block_max) b = block_max;
  const std::vector<HistTile> tiles = hist2_tiles(m, b);
  const size_t bb = (size_t)bins * bins;
  for (size_t i = 0; i < (size_t)m * (m - 1) / 2 * bb; ++i) hist[i] = 0;
  std::vector<int> idx;
  for (const HistTile& t : tiles) {
    const int K = (int)(t.na + t.nb);
    idx.assign((size_t)K, 0);
    for (uint64_t r = 0; r < rows; ++r) {
      for (int k = 0; k < K; ++k) {
        const uint32_t pos = k < (int)t.na ? t.a0 + k : t.b0 + (k - t.na);
        idx[k] = hist_bin_searched(x[r * D + params[pos]], edges + (size_t)pos * (bins + 1), bins);
      }
      for (uint32_t i = 0; i < t.na; ++i)
        for (uint32_t j = 0; j < t.nb; ++j) {
          if (t.a0 == t.b0 && i >= j) continue;
          const int xi = idx[i], yj = idx[t.na + j];
          if (xi < 0 || yj < 0) continue;
          hist[hist2_pair_index(t.a0 + i, t.b0 + j, (uint64_t)m) * bb + (size_t)xi * bins + yj]++;
        }
    }
  }
  return (int)tiles.size();
}
}
