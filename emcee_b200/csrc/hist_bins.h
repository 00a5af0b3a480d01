// Bin rules of the stored-chain histograms (histogram.cu, eb_chain_histogram / eb_chain_histogram2d) and the pair
// tiles of the 2-D kernel.  Builds for the host without CUDA, so that tests/helpers/histogram_host.cpp runs the same
// statements on the CPU; the rules are device functions too.
//
// hist_bin_uniform is np.histogram's fast path for uniform bins (numpy/lib/_histograms_impl.py, `histogram`), one
// statement for one, in float64; hist_bin_searched is np.histogramdd's (`searchsorted(side="right")`, the right
// edge moved into the last bin, the two outlier bins dropped).  The arithmetic is written with the _rn intrinsics
// on the device, so that no contraction or fast-math flag can change an index.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

#ifdef __CUDACC__
#define EB_HIST_HD __host__ __device__ __forceinline__
#else
#define EB_HIST_HD inline
#endif

namespace eb {

constexpr int HIST_BINS_MAX = 4096;   // eb_chain_histogram: bins per parameter
constexpr int HIST2_BINS_MAX = 128;   // eb_chain_histogram2d: a 64 KiB uint32 pair histogram
constexpr int HIST_DROP = -1;         // outside the range (or NaN): not counted, as numpy drops it
constexpr int HIST_BAD = -2;          // an index past numpy's edge array (np.histogram raises IndexError there)

EB_HIST_HD double hist_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
EB_HIST_HD double hist_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
EB_HIST_HD double hist_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

// np.histogram(a, n, range) for one value x: first / last are the outer edges (_get_outer_edges), span numpy's
// norm_denom = last - first (as numpy subtracts the range's own scalars), edges[n + 1] its linspace.  span can be
// smaller than the float64 last - first (a range of float32 scalars is subtracted in float32), so f can exceed n:
// numpy truncates it and moves n to n - 1 all the same, and only an index above n falls off its edge array.
EB_HIST_HD int hist_bin_uniform(double x, double first, double last, double span, int n, const double* edges) {
  if (!(x >= first && x <= last)) return HIST_DROP;             // keep = (a >= first_edge) & (a <= last_edge)
  const double f = hist_mul(hist_div(hist_sub(x, first), span), (double)n);  // ((a - first) / denom) * n
  if (!(f >= 0.0 && f < (double)n + 1.0)) return HIST_BAD;      // truncates above n (or NaN): IndexError
  int idx = (int)f;                                             // f_indices.astype(np.intp)
  if (idx == n) idx = n - 1;                                    // indices[indices == n] -= 1
  if (x < edges[idx]) --idx;                                    // decrement = a < bin_edges[indices]
  if (idx < 0) return HIST_BAD;
  if (x >= edges[idx + 1] && idx != n - 1) ++idx;               // increment = (a >= edges[idx + 1]) & (idx != n - 1)
  return idx;
}

// np.histogramdd's bin of x along one axis with edges[n + 1] (non-decreasing): idx = #(edges <= x)
// (searchsorted(side="right")), x == edges[n] moves to the last bin, idx 0 and n + 1 are the outliers.  NaN compares
// false everywhere and is dropped too.
EB_HIST_HD int hist_bin_searched(double x, const double* edges, int n) {
  int lo = 0, hi = n + 1;  // upper bound: the first edge > x
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (edges[mid] <= x) lo = mid + 1;
    else hi = mid;
  }
  int idx = lo;
  if (x == edges[n]) --idx;
  return (idx == 0 || idx == n + 1) ? HIST_DROP : idx - 1;
}

// ---- pair tiles of eb_chain_histogram2d ----------------------------------------------------------------------------
// The m parameters (positions 0 .. m - 1 of the caller's list) are cut into blocks of b positions; a tile is a pair of
// blocks (u <= v) and counts the pairs (i in u, j in v, i < j).  Its shared memory holds b * b pair histograms
// (the diagonal tile uses the cells with i < j), so b is the largest block whose b^2 histograms of bins^2 uint32 fit
// `hist_bytes`.  Pair (i, j) is output pair i m - i (i + 1) / 2 + j - i - 1, itertools.combinations' order.
struct HistTile {
  uint32_t a0, na, b0, nb;  // positions a0 .. a0 + na - 1 against b0 .. b0 + nb - 1
};

inline int hist2_block(int m, int bins, size_t hist_bytes) {
  const size_t per = (size_t)bins * bins * sizeof(uint32_t);
  int b = 1;
  while (b < m && (size_t)(b + 1) * (b + 1) * per <= hist_bytes) ++b;
  return b;
}

inline std::vector<HistTile> hist2_tiles(int m, int b) {
  std::vector<HistTile> t;
  for (int u = 0; u < m; u += b)
    for (int v = u; v < m; v += b) {
      const uint32_t na = (uint32_t)(m - u < b ? m - u : b), nb = (uint32_t)(m - v < b ? m - v : b);
      if (u == v && na < 2) continue;  // a one-position diagonal block holds no pair
      t.push_back(HistTile{(uint32_t)u, na, (uint32_t)v, nb});
    }
  return t;
}

// hist2_tiles(m, b).size() without building the list: every block pair u <= v, less the diagonal tiles of
// one-position blocks (all K of them when b == 1, the short last block when m % b == 1)
inline uint64_t hist2_ntiles(int m, int b) {
  const uint64_t K = ((uint64_t)m + b - 1) / b;
  const uint64_t single = b == 1 ? K : (m % b == 1 ? 1 : 0);
  return K * (K + 1) / 2 - single;
}

EB_HIST_HD uint64_t hist2_pair_index(uint64_t i, uint64_t j, uint64_t m) { return i * m - i * (i + 1) / 2 + j - i - 1; }

}  // namespace eb
