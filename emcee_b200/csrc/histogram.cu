// Histograms of a stored chain slice on the device: np.histogram of each parameter (eb_chain_histogram) and
// np.histogram2d of parameter pairs (eb_chain_histogram2d), with the bin rules of hist_bins.h and numpy's own edges
// (computed on the host).
//
// Both kernels read the slice once, in place, through a table of slot base pointers (one per stored step, as
// select.cu does): CTA x is a column block (1-D) or a tile of parameter pairs (2-D), CTA y a range of the slice's
// rows (stored step, walker).  A slot of nseg segments (ensembles, eb_chain_histogram_segments) of n = N / nseg rows
// is read as select.cu reads it: the 1-D kernel sees nseg * D columns of count * n rows, column c = k * D + d at
// offset k * n * D + w * D + d of a slot (a column block may span segments), and the 2-D grid holds one copy of the
// pair tiles per segment.  nseg = 1 is eb_chain_histogram itself.  Counts live in shared uint32 bins and are
// flushed, where non-zero, to 64-bit global counts; a CTA counts fewer than 2^32 rows.  Counts are integers, so the
// result does not depend on the order in which the atomics land.
#include <algorithm>
#include <vector>

#include "engine.cuh"
#include "hist_bins.h"

namespace eb {
namespace {

constexpr int HIST_THREADS = 256;
constexpr int HIST2_THREADS = 512;
constexpr int HIST2_ROWS = 256;                    // rows staged per round of the 2-D kernel
constexpr int HIST2_BLOCK_MAX = 32;                // positions per block of a pair tile
constexpr size_t HIST1_SMEM = 96 * 1024;           // 1-D: column blocks sized to this (one column may need 48 KiB)
constexpr size_t HIST2_SMEM_HIST = 160 * 1024;     // 2-D: pair histograms of one tile
constexpr uint64_t HIST_ROWS_PER_CTA_MAX = (uint64_t)1 << 31;

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// bytes of one column of the 1-D kernel's shared memory: its edges, (first, last, span) and uint32 bins
size_t hist1_col_bytes(int bins) { return (size_t)(bins + 1 + 3) * sizeof(double) + (size_t)bins * sizeof(uint32_t); }

// Column block x: columns x * W .. x * W + w - 1 of ncol = nseg * D; a slot row holds D values and segment k starts
// seg_stride = n * D values into the slot.  outer[ncol, 3] = (first, last, span), edges[ncol, bins + 1].
__global__ void __launch_bounds__(HIST_THREADS)
    hist1_kernel(const double* const* __restrict__ slots, uint32_t N, int D, uint64_t seg_stride, int ncol,
                 uint64_t nrows, uint64_t rows_per_cta, int W, int bins, const double* __restrict__ outer,
                 const double* __restrict__ edges, unsigned long long* __restrict__ hist,
                 unsigned int* __restrict__ bad) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int d0 = (int)blockIdx.x * W, w = min(W, ncol - d0);
  double* se = reinterpret_cast<double*>(smem);               // [w, bins + 1]
  double* so = se + (size_t)w * (bins + 1);                   // [w, 3]
  unsigned int* sh = reinterpret_cast<unsigned int*>(so + 3 * w);  // [w, bins]
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < w * (bins + 1); i += HIST_THREADS) se[i] = edges[(size_t)d0 * (bins + 1) + i];
  for (int i = tid; i < 3 * w; i += HIST_THREADS) so[i] = outer[(size_t)d0 * 3 + i];
  for (int i = tid; i < w * bins; i += HIST_THREADS) sh[i] = 0;
  __syncthreads();
  const int per = HIST_THREADS / w;  // rows per iteration
  const int c = tid % w, ro = tid / w;
  const bool col_ok = ro < per;
  const double first = so[3 * c], last = so[3 * c + 1], span = so[3 * c + 2];
  const double* e = se + (size_t)c * (bins + 1);
  const int kseg = (d0 + c) / D;
  const size_t cbase = (size_t)kseg * seg_stride + (size_t)(d0 + c - kseg * D);  // the column's offset in a slot
  const uint64_t r0 = (uint64_t)blockIdx.y * rows_per_cta;
  const uint64_t r1 = min(nrows, r0 + rows_per_cta);
  uint64_t R = r0 + (uint64_t)ro;
  uint64_t s = R / N;
  uint32_t wk = (uint32_t)(R - s * N);
  // every thread runs the same number of iterations, so that the warp-wide match below is uniform
  for (uint64_t base = r0; base < r1; base += (uint64_t)per) {
    int hs = -1;  // shared bin of this thread's value
    if (col_ok && R < r1) {
      const double v = slots[s][(size_t)wk * D + cbase];
      const int b = hist_bin_uniform(v, first, last, span, bins, e);
      if (b >= 0) hs = c * bins + b;
      else if (b == HIST_BAD) atomicOr(bad, 1u);
    }
    if (w < 32) {  // several lanes share a parameter: one atomic per distinct bin of the warp
      const unsigned int m = __match_any_sync(0xffffffffu, hs);
      if (hs >= 0 && __ffs(m) - 1 == lane) atomicAdd(sh + hs, (unsigned int)__popc(m));
    } else if (hs >= 0) {
      atomicAdd(sh + hs, 1u);
    }
    R += (uint64_t)per;
    wk += (uint32_t)per;
    if (wk >= N) {
      s += wk / N;
      wk %= N;
    }
  }
  __syncthreads();
  for (int i = tid; i < w * bins; i += HIST_THREADS)
    if (sh[i]) atomicAdd(hist + (size_t)d0 * bins + i, (unsigned long long)sh[i]);
}

struct Hist2Geom {
  int block = 1;       // positions per block
  size_t smem = 0;     // dynamic shared bytes of the largest tile
};

Hist2Geom hist2_geom(int m, int bins) {
  Hist2Geom g;
  g.block = std::min(hist2_block(m, bins, HIST2_SMEM_HIST), HIST2_BLOCK_MAX);
  const size_t b = (size_t)g.block;
  g.smem = 2 * b * (bins + 1) * sizeof(double) + b * b * (size_t)bins * bins * sizeof(uint32_t) +
           HIST2_ROWS * sizeof(const double*) + HIST2_ROWS * 2 * b;
  return g;
}

// CTA x: tile x % ntiles of segment k = x / ntiles, positions a0 .. a0 + na - 1 against b0 .. b0 + nb - 1 of
// params[m] (pairs i < j only).  Segment k's rows start seg_stride values into a slot; edges[nseg, m, bins + 1] in
// position order; hist[nseg, m (m - 1) / 2, bins, bins].  Each round stages HIST2_ROWS rows: every (row, position)
// value is binned once (idx, 0xff = outlier), then every (row, pair) adds one count.
__global__ void __launch_bounds__(HIST2_THREADS)
    hist2_kernel(const double* const* __restrict__ slots, uint32_t N, int D, uint64_t seg_stride, uint64_t nrows,
                 uint64_t rows_per_cta, const HistTile* __restrict__ tiles, uint32_t ntiles,
                 const uint32_t* __restrict__ params, uint32_t m, int bins, const double* __restrict__ edges,
                 unsigned long long* __restrict__ hist) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t kseg = blockIdx.x / ntiles;
  const HistTile t = tiles[blockIdx.x - kseg * ntiles];
  edges += (size_t)kseg * m * (bins + 1);
  hist += (uint64_t)kseg * ((uint64_t)m * (m - 1) / 2) * (uint64_t)bins * bins;
  const size_t seg_off = (size_t)kseg * seg_stride;
  const int na = (int)t.na, nb = (int)t.nb, K = na + nb, P = na * nb, bb = bins * bins;
  const bool diag = t.a0 == t.b0;
  double* se = reinterpret_cast<double*>(smem);                                // [K, bins + 1]
  const double** rowp = reinterpret_cast<const double**>(se + (size_t)K * (bins + 1));  // [HIST2_ROWS]
  unsigned int* sh = reinterpret_cast<unsigned int*>(rowp + HIST2_ROWS);        // [P, bins, bins]
  uint8_t* idx = reinterpret_cast<uint8_t*>(sh + (size_t)P * bb);               // [HIST2_ROWS, K]
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < K * (bins + 1); i += HIST2_THREADS) {
    const int k = i / (bins + 1);
    const uint32_t pos = k < na ? t.a0 + k : t.b0 + (k - na);
    se[i] = edges[(size_t)pos * (bins + 1) + (i - k * (bins + 1))];
  }
  for (int i = tid; i < P * bb; i += HIST2_THREADS) sh[i] = 0;
  // column of each staged position, and the pair work split: G row groups per pair when the tile has few pairs
  const int G = P >= HIST2_THREADS ? 1 : min(HIST2_THREADS / P, HIST2_ROWS);
  const int L = tid;  // this thread's (pair, group) slot in the first sweep
  const uint64_t r0 = (uint64_t)blockIdx.y * rows_per_cta;
  const uint64_t r1 = min(nrows, r0 + rows_per_cta);
  for (uint64_t base = r0; base < r1; base += HIST2_ROWS) {
    __syncthreads();  // the previous round's idx is consumed (and, on the first round, the tables are set)
    if (tid < HIST2_ROWS) {
      const uint64_t R = base + (uint64_t)tid;
      const double* p = nullptr;
      if (R < r1) {
        const uint64_t s = R / N;
        p = slots[s] + seg_off + (size_t)(R - s * N) * D;
      }
      rowp[tid] = p;
    }
    __syncthreads();
    for (int i = tid; i < HIST2_ROWS * K; i += HIST2_THREADS) {
      const int r = i / K, k = i - r * K;
      uint8_t b = 0xff;
      if (rowp[r]) {
        const uint32_t pos = k < na ? t.a0 + k : t.b0 + (k - na);
        const int bin = hist_bin_searched(rowp[r][params[pos]], se + (size_t)k * (bins + 1), bins);
        if (bin >= 0) b = (uint8_t)bin;
      }
      idx[i] = b;
    }
    __syncthreads();
    for (int L0 = 0; L0 < P * G; L0 += HIST2_THREADS) {  // uniform over the CTA
      const int Lq = L0 + L;
      const int q = Lq % P, g = Lq / P;
      const int i = q / nb, j = q - i * nb;
      const bool pair_ok = Lq < P * G && (!diag || i < j);
      for (int rr = 0; rr < HIST2_ROWS; rr += G) {  // uniform over the CTA
        const int r = rr + g;
        int cell = -1;
        if (pair_ok && r < HIST2_ROWS) {
          const uint8_t x = idx[r * K + i], y = idx[r * K + na + j];
          if (x != 0xff && y != 0xff) cell = q * bb + (int)x * bins + (int)y;
        }
        if (P < 32) {  // lanes share a pair: one atomic per distinct cell of the warp
          const unsigned int mk = __match_any_sync(0xffffffffu, cell);
          if (cell >= 0 && __ffs(mk) - 1 == lane) atomicAdd(sh + cell, (unsigned int)__popc(mk));
        } else if (cell >= 0) {
          atomicAdd(sh + cell, 1u);
        }
      }
    }
  }
  __syncthreads();
  for (int c = tid; c < P * bb; c += HIST2_THREADS) {
    if (!sh[c]) continue;
    const int q = c / bb, i = q / nb, j = q - i * nb;
    const uint64_t out = hist2_pair_index(t.a0 + i, t.b0 + j, m);
    atomicAdd(hist + out * bb + (c - q * bb), (unsigned long long)sh[c]);
  }
}

// rows of the slice split over grid y: about `ctas` CTAs in all, at least `min_rows` rows each, fewer than 2^31
void split_rows(uint64_t n, uint64_t nx, uint64_t ctas, uint64_t min_rows, uint64_t* ys, uint64_t* rows_per) {
  uint64_t y = (ctas + nx - 1) / nx;
  y = std::min<uint64_t>(y, std::max<uint64_t>(1, n / min_rows));
  y = std::max<uint64_t>(y, (n + HIST_ROWS_PER_CTA_MAX - 1) / HIST_ROWS_PER_CTA_MAX);
  y = std::min<uint64_t>(std::max<uint64_t>(y, 1), 65535);
  *rows_per = (n + y - 1) / y;
  *ys = (n + *rows_per - 1) / *rows_per;
}

}  // namespace

bool hist_rows_fit(uint64_t n) { return n <= 65535 * HIST_ROWS_PER_CTA_MAX; }

size_t hist1_scratch_bytes(uint64_t count, size_t ncol, int bins) {
  return align256(count * sizeof(double*)) + align256(ncol * 3 * sizeof(double)) +
         align256(ncol * (bins + 1) * sizeof(double)) + align256(ncol * bins * sizeof(uint64_t)) +
         align256(sizeof(uint32_t));
}

cudaError_t hist1_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int Dp, int bins,
                      const double* outer, const double* edges, uint64_t* hist, bool* bad, void* scratch, int sm_count,
                      cudaStream_t st) {
  const uint32_t sn = N / nseg;  // rows of a segment in one stored step
  const uint64_t n = count * (uint64_t)sn;
  const size_t D = (size_t)nseg * Dp;  // columns
  char* p = static_cast<char*>(scratch);
  auto take = [&](size_t bytes) {
    char* q = p;
    p += align256(bytes);
    return q;
  };
  const double** d_slots = reinterpret_cast<const double**>(take(count * sizeof(double*)));
  double* d_outer = reinterpret_cast<double*>(take(D * 3 * sizeof(double)));
  double* d_edges = reinterpret_cast<double*>(take(D * (bins + 1) * sizeof(double)));
  unsigned long long* d_hist = reinterpret_cast<unsigned long long*>(take(D * bins * sizeof(uint64_t)));
  unsigned int* d_bad = reinterpret_cast<unsigned int*>(take(sizeof(uint32_t)));
#define HE(call)                      \
  do {                                \
    cudaError_t _e = (call);          \
    if (_e != cudaSuccess) return _e; \
  } while (0)
  HE(cudaMemcpyAsync(d_slots, slots, count * sizeof(double*), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(d_outer, outer, D * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(d_edges, edges, D * (bins + 1) * sizeof(double), cudaMemcpyHostToDevice, st));
  HE(cudaMemsetAsync(d_hist, 0, D * bins * sizeof(uint64_t), st));
  HE(cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), st));
  // the widest column block (at most 32 columns) whose shared memory fits HIST1_SMEM; one column always fits
  const size_t col = hist1_col_bytes(bins);
  const int W = (int)std::max<size_t>(1, std::min<size_t>({(size_t)32, D, HIST1_SMEM / col}));
  const size_t smem = (size_t)W * col;
  HE(cudaFuncSetAttribute(hist1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const uint64_t nx = ((uint64_t)D + W - 1) / W;
  uint64_t ys = 1, rows_per = n;
  split_rows(n, nx, (uint64_t)sm_count * 8, (uint64_t)(HIST_THREADS / W) * 16, &ys, &rows_per);
  hist1_kernel<<<dim3((unsigned)nx, (unsigned)ys), HIST_THREADS, smem, st>>>(
      d_slots, sn, Dp, (uint64_t)sn * Dp, (int)D, n, rows_per, W, bins, d_outer, d_edges, d_hist, d_bad);
  HE(cudaGetLastError());
  uint32_t hb = 0;
  HE(cudaMemcpyAsync(hist, d_hist, D * bins * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  HE(cudaMemcpyAsync(&hb, d_bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  HE(cudaStreamSynchronize(st));
  *bad = hb != 0;
  return cudaSuccess;
}

uint64_t hist2_grid_x(uint32_t nseg, int m, int bins) {
  return (uint64_t)nseg * hist2_ntiles(m, hist2_geom(m, bins).block);
}

size_t hist2_scratch_bytes(uint64_t count, uint32_t nseg, int m, int bins) {
  const Hist2Geom g = hist2_geom(m, bins);
  const size_t ntiles = (size_t)hist2_ntiles(m, g.block);  // the tile list itself is built once the scratch fits
  const size_t npairs = (size_t)m * (m - 1) / 2;
  return align256(count * sizeof(double*)) + align256(ntiles * sizeof(HistTile)) +
         align256((size_t)m * sizeof(uint32_t)) + align256((size_t)nseg * m * (bins + 1) * sizeof(double)) +
         align256((size_t)nseg * npairs * bins * bins * sizeof(uint64_t));
}

cudaError_t hist2_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int D,
                      const uint32_t* params, int m, int bins, const double* edges, uint64_t* hist, void* scratch,
                      int sm_count, cudaStream_t st) {
  const uint32_t sn = N / nseg;  // rows of a segment in one stored step
  const uint64_t n = count * (uint64_t)sn;
  const Hist2Geom g = hist2_geom(m, bins);
  const std::vector<HistTile> tiles = hist2_tiles(m, g.block);
  const size_t npairs = (size_t)m * (m - 1) / 2, out = (size_t)nseg * npairs * bins * bins;
  const size_t nedges = (size_t)nseg * m * (bins + 1);
  char* p = static_cast<char*>(scratch);
  auto take = [&](size_t bytes) {
    char* q = p;
    p += align256(bytes);
    return q;
  };
  const double** d_slots = reinterpret_cast<const double**>(take(count * sizeof(double*)));
  HistTile* d_tiles = reinterpret_cast<HistTile*>(take(tiles.size() * sizeof(HistTile)));
  uint32_t* d_params = reinterpret_cast<uint32_t*>(take((size_t)m * sizeof(uint32_t)));
  double* d_edges = reinterpret_cast<double*>(take(nedges * sizeof(double)));
  unsigned long long* d_hist = reinterpret_cast<unsigned long long*>(take(out * sizeof(uint64_t)));
  HE(cudaMemcpyAsync(d_slots, slots, count * sizeof(double*), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(HistTile), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(d_params, params, (size_t)m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(d_edges, edges, nedges * sizeof(double), cudaMemcpyHostToDevice, st));
  HE(cudaMemsetAsync(d_hist, 0, out * sizeof(uint64_t), st));
  HE(cudaFuncSetAttribute(hist2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
  const uint64_t nx = (uint64_t)nseg * tiles.size();  // at most 2^31 - 1 (the caller checks hist2_grid_x)
  uint64_t ys = 1, rows_per = n;
  split_rows(n, nx, (uint64_t)sm_count * 2, (uint64_t)HIST2_ROWS * 4, &ys, &rows_per);
  hist2_kernel<<<dim3((unsigned)nx, (unsigned)ys), HIST2_THREADS, g.smem, st>>>(
      d_slots, sn, D, (uint64_t)sn * D, n, rows_per, d_tiles, (uint32_t)tiles.size(), d_params, (uint32_t)m, bins,
      d_edges, d_hist);
  HE(cudaGetLastError());
  HE(cudaMemcpyAsync(hist, d_hist, out * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  HE(cudaStreamSynchronize(st));
  return cudaSuccess;
}

// ---- running histograms of the live state ---------------------------------------------------------------------
// The same kernels over one "stored step": the engine's [N, D] coordinates (and [N] log-probabilities), read through
// a two-entry slot table uploaded once.  The counts and the bad flag persist across launches; a launch only adds.

namespace {

// the layout of LiveHist::mem: slot table, 1-D tables and counts, bad flag, then the 2-D tables and counts
struct LiveLayout {
  size_t slots, outer, edges, hist, bad, tiles, params, edges2, hist2, bytes;
};

LiveLayout live_layout(int D, int bins, int lp, int m, int bins2, uint64_t ntiles) {
  const size_t rows = (size_t)D + (size_t)lp, npairs = (size_t)m * (m > 0 ? m - 1 : 0) / 2;
  LiveLayout l;
  size_t at = 0;
  auto take = [&](size_t bytes) {
    const size_t q = at;
    at += align256(bytes);
    return q;
  };
  l.slots = take(2 * sizeof(double*));
  l.outer = take(rows * 3 * sizeof(double));
  l.edges = take(rows * (bins + 1) * sizeof(double));
  l.hist = take(rows * bins * sizeof(uint64_t));
  l.bad = take(sizeof(uint32_t));
  l.tiles = take(ntiles * sizeof(HistTile));
  l.params = take((size_t)m * sizeof(uint32_t));
  l.edges2 = take((size_t)m * (bins2 + 1) * sizeof(double));
  l.hist2 = take(npairs * bins2 * bins2 * sizeof(uint64_t));
  l.bytes = at;
  return l;
}

uint64_t live_ntiles(int m, int bins2) { return m >= 2 ? hist2_ntiles(m, hist2_geom(m, bins2).block) : 0; }

// column block width, shared bytes and grid of the 1-D kernel over D columns of N rows
void live_hist1_geom(uint32_t N, int D, int bins, int sm_count, int* W, size_t* smem, dim3* grid, uint64_t* rows_per) {
  const size_t col = hist1_col_bytes(bins);
  *W = (int)std::max<size_t>(1, std::min<size_t>({(size_t)32, (size_t)D, HIST1_SMEM / col}));
  *smem = (size_t)*W * col;
  const uint64_t nx = ((uint64_t)D + *W - 1) / *W;
  uint64_t ys = 1;
  split_rows(N, nx, (uint64_t)sm_count * 8, (uint64_t)(HIST_THREADS / *W) * 16, &ys, rows_per);
  *grid = dim3((unsigned)nx, (unsigned)ys);
}

}  // namespace

size_t live_hist_bytes(int D, int bins, int lp, int m, int bins2) {
  return live_layout(D, bins, lp, m, bins2, live_ntiles(m, bins2)).bytes;
}

cudaError_t live_hist_setup(LiveHist* h, void* mem, uint32_t N, int D, int bins, int lp, const double* outer,
                            const double* edges, const uint32_t* params, int m, int bins2, const double* edges2,
                            const double* coords, const double* logp, int sm_count, cudaStream_t st) {
  const std::vector<HistTile> tiles = m >= 2 ? hist2_tiles(m, hist2_geom(m, bins2).block) : std::vector<HistTile>();
  const LiveLayout l = live_layout(D, bins, lp, m, bins2, tiles.size());
  char* p = static_cast<char*>(mem);
  *h = LiveHist{};
  h->N = N;
  h->D = D;
  h->bins = bins;
  h->lp = lp;
  h->m = m;
  h->bins2 = bins2;
  h->mem = mem;
  h->slots = reinterpret_cast<const double**>(p + l.slots);
  h->outer = reinterpret_cast<double*>(p + l.outer);
  h->edges = reinterpret_cast<double*>(p + l.edges);
  h->hist = reinterpret_cast<unsigned long long*>(p + l.hist);
  h->bad = reinterpret_cast<unsigned int*>(p + l.bad);
  h->tiles = reinterpret_cast<HistTile*>(p + l.tiles);
  h->ntiles = (uint32_t)tiles.size();
  h->params = reinterpret_cast<uint32_t*>(p + l.params);
  h->edges2 = reinterpret_cast<double*>(p + l.edges2);
  h->hist2 = reinterpret_cast<unsigned long long*>(p + l.hist2);
  const size_t rows = (size_t)D + (size_t)lp, npairs = (size_t)m * (m > 0 ? m - 1 : 0) / 2;
  const double* table[2] = {coords, logp};
  HE(cudaMemcpyAsync(h->slots, table, sizeof(table), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(h->outer, outer, rows * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  HE(cudaMemcpyAsync(h->edges, edges, rows * (bins + 1) * sizeof(double), cudaMemcpyHostToDevice, st));
  HE(cudaMemsetAsync(h->hist, 0, rows * bins * sizeof(uint64_t), st));
  HE(cudaMemsetAsync(h->bad, 0, sizeof(uint32_t), st));
  live_hist1_geom(N, D, bins, sm_count, &h->W1, &h->smem1, &h->grid1, &h->rows1);
  live_hist1_geom(N, 1, bins, sm_count, &h->Wlp, &h->smemlp, &h->gridlp, &h->rowslp);
  if (m >= 2) {
    HE(cudaMemcpyAsync(h->tiles, tiles.data(), tiles.size() * sizeof(HistTile), cudaMemcpyHostToDevice, st));
    HE(cudaMemcpyAsync(h->params, params, (size_t)m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    HE(cudaMemcpyAsync(h->edges2, edges2, (size_t)m * (bins2 + 1) * sizeof(double), cudaMemcpyHostToDevice, st));
    HE(cudaMemsetAsync(h->hist2, 0, npairs * bins2 * bins2 * sizeof(uint64_t), st));
    h->smem2 = hist2_geom(m, bins2).smem;
    uint64_t ys = 1;
    split_rows(N, tiles.size(), (uint64_t)sm_count * 2, (uint64_t)HIST2_ROWS * 4, &ys, &h->rows2);
    h->grid2 = dim3((unsigned)tiles.size(), (unsigned)ys);
  }
  return cudaStreamSynchronize(st);
}

cudaError_t live_hist_launch(const LiveHist& h, cudaStream_t st, uint64_t& launches) {
  // the attribute is set at every launch: eb_chain_histogram sets the same kernels' limits to its own sizes
  HE(cudaFuncSetAttribute(hist1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                          (int)std::max(h.smem1, h.lp ? h.smemlp : 0)));
  hist1_kernel<<<h.grid1, HIST_THREADS, h.smem1, st>>>(h.slots, h.N, h.D, 0, h.D, h.N, h.rows1, h.W1, h.bins,
                                                       h.outer, h.edges, h.hist, h.bad);
  HE(cudaGetLastError());
  ++launches;
  if (h.lp) {  // the log-probabilities: row D of the tables, one column of stride 1
    hist1_kernel<<<h.gridlp, HIST_THREADS, h.smemlp, st>>>(h.slots + 1, h.N, 1, 0, 1, h.N, h.rowslp, h.Wlp, h.bins,
                                                           h.outer + 3 * (size_t)h.D,
                                                           h.edges + (size_t)h.D * (h.bins + 1),
                                                           h.hist + (size_t)h.D * h.bins, h.bad);
    HE(cudaGetLastError());
    ++launches;
  }
  if (h.m >= 2) {
    HE(cudaFuncSetAttribute(hist2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h.smem2));
    hist2_kernel<<<h.grid2, HIST2_THREADS, h.smem2, st>>>(h.slots, h.N, h.D, 0, h.N, h.rows2, h.tiles, h.ntiles,
                                                          h.params, (uint32_t)h.m, h.bins2, h.edges2, h.hist2);
    HE(cudaGetLastError());
    ++launches;
  }
  return cudaSuccess;
}

cudaError_t live_hist_read(const LiveHist& h, uint64_t* hist, uint64_t* hist2, bool* bad, cudaStream_t st) {
  const size_t rows = (size_t)h.D + (size_t)h.lp, npairs = (size_t)h.m * (h.m > 0 ? h.m - 1 : 0) / 2;
  uint32_t hb = 0;
  if (hist) HE(cudaMemcpyAsync(hist, h.hist, rows * h.bins * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (hist2 && h.m >= 2)
    HE(cudaMemcpyAsync(hist2, h.hist2, npairs * h.bins2 * h.bins2 * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  HE(cudaMemcpyAsync(&hb, h.bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  HE(cudaStreamSynchronize(st));
  *bad = hb != 0;
  return cudaSuccess;
}
#undef HE

}  // namespace eb
