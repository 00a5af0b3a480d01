// Exact order statistics of a stored chain slice on the device (eb_chain_select): what np.partition of each
// parameter's count * nwalkers values puts at the requested ranks, by MSB-first radix selection over
// order-preserving keys (select_keys.h).
//
// Every pass reads the whole slice once, in place (a table of slot base pointers, one per stored step), with one
// launch of select_pass_kernel: CTA x is a column block of at most SEL_WMAX parameters (SelTask), CTA y a range of
// the slice's rows (stored step, walker).  A slot of nseg segments (eb_chain_select_segments) of N rows is read as
// nseg * D columns of N rows: column c = k * D + d is parameter d of segment k, at offset k * N * D of the slot, so
// one plan selects for every segment in the same passes.  A value's key is matched to its parameter's live group; a histogram
// group counts the key's next digit in shared memory (flushed to 64-bit global counts at the end), a compaction
// group copies the key into its slice of the candidate buffer.  select_sort_kernel then sorts each compacted group
// (at most SEL_CAP keys, bitonic in shared memory) and gathers the ranks it answers.  The host refines the groups
// from the histograms between passes (SelPlan).  Counts are integers and the compacted candidates are sorted, so
// the result is deterministic whatever order the atomics land in.
#include <algorithm>
#include <vector>

#include "engine.cuh"
#include "select_keys.h"

namespace eb {
namespace {

constexpr int SEL_THREADS = 256;
constexpr int SORT_THREADS = 512;

__global__ void __launch_bounds__(SEL_THREADS)
    select_pass_kernel(const double* const* __restrict__ slots, uint32_t N, int D, uint64_t seg_stride, uint64_t nrows,
                       uint64_t rows_per_cta, const SelTask* __restrict__ tasks, const uint32_t* __restrict__ colrange,
                       const SelGroup* __restrict__ groups, int bits, unsigned long long* __restrict__ hist,
                       unsigned long long* __restrict__ cand, unsigned int* __restrict__ cand_cnt,
                       uint8_t* __restrict__ nanflag) {
  __shared__ unsigned int sh[SEL_HMAX * SEL_BINS];
  __shared__ int slot_group[SEL_HMAX];
  const SelTask t = tasks[blockIdx.x];
  const int W = (int)t.w, per = SEL_THREADS / W;  // rows per iteration
  const int tid = threadIdx.x, lane = tid & 31;
  const int c = tid % W, ro = tid / W;
  const bool col_ok = ro < per;
  const uint32_t glo = colrange[t.cr + 2 * c], ghi = colrange[t.cr + 2 * c + 1];
  const int col = (int)t.d0 + c;  // k * D + d
  const int kseg = col / D, d = col - kseg * D;
  const size_t cbase = (size_t)kseg * seg_stride + (size_t)d;  // the column's offset in a slot
  for (int i = tid; i < SEL_HMAX * SEL_BINS; i += SEL_THREADS) sh[i] = 0;
  if (tid < W)
    for (uint32_t g = glo; g < ghi; ++g)
      if (groups[g].hslot >= 0) slot_group[groups[g].hslot] = (int)g;
  __syncthreads();
  const uint64_t r0 = (uint64_t)blockIdx.y * rows_per_cta;
  const uint64_t r1 = min(nrows, r0 + rows_per_cta);
  uint64_t R = r0 + (uint64_t)ro;
  uint64_t s = R / N;
  uint32_t w = (uint32_t)(R - s * N);
  // every thread runs the same number of iterations, so that the warp-wide match below is uniform
  for (uint64_t base = r0; base < r1; base += (uint64_t)per) {
    int hs = -1;  // shared histogram bin of this thread's value
    if (col_ok && R < r1) {
      const double v = slots[s][(size_t)w * D + cbase];
      if (nanflag && isnan(v)) nanflag[col] = 1;
      const uint64_t key = order_key_bits((uint64_t)__double_as_longlong(v));
      const int g = find_group(groups, glo, ghi, key, bits);
      if (g >= 0) {
        const int slot = groups[g].hslot;
        if (slot >= 0) {
          hs = slot * SEL_BINS + key_digit(key, bits);
        } else {
          const unsigned int pos = atomicAdd(cand_cnt + g, 1u);
          if (pos < groups[g].count) cand[groups[g].cand_off + pos] = key;
        }
      }
    }
    if (W < 32) {  // several lanes share a parameter: one atomic per distinct bin of the warp
      const unsigned int m = __match_any_sync(0xffffffffu, hs);
      if (hs >= 0 && __ffs(m) - 1 == lane) atomicAdd(sh + hs, (unsigned int)__popc(m));
    } else if (hs >= 0) {
      atomicAdd(sh + hs, 1u);
    }
    R += (uint64_t)per;
    w += (uint32_t)per;
    if (w >= N) {
      s += w / N;
      w %= N;
    }
  }
  __syncthreads();
  int nslots = 0;
  for (uint32_t cc = 0; cc < t.w; ++cc) {
    const uint32_t lo = colrange[t.cr + 2 * cc], hi = colrange[t.cr + 2 * cc + 1];
    for (uint32_t g = lo; g < hi; ++g) nslots += groups[g].hslot >= 0;
  }
  for (int i = tid; i < nslots * SEL_BINS; i += SEL_THREADS)
    if (sh[i]) atomicAdd(hist + (size_t)slot_group[i / SEL_BINS] * SEL_BINS + (i % SEL_BINS), (unsigned long long)sh[i]);
}

// CTA j: sorts the candidates of compacted group cg[j] in place (bitonic, padded with ~0 to a power of two) and
// writes the keys at candidate indices pidx[poff[j] .. poff[j + 1]) to pkey.
__global__ void __launch_bounds__(SORT_THREADS)
    select_sort_kernel(const SelGroup* __restrict__ groups, const uint32_t* __restrict__ cg,
                       const uint32_t* __restrict__ poff, const uint64_t* __restrict__ pidx,
                       unsigned long long* __restrict__ cand, unsigned long long* __restrict__ pkey) {
  __shared__ unsigned long long s[SEL_CAP];
  const SelGroup g = groups[cg[blockIdx.x]];
  const int n = (int)g.count;
  int P = 1;
  while (P < n) P <<= 1;
  unsigned long long* src = cand + g.cand_off;
  for (int i = threadIdx.x; i < P; i += SORT_THREADS) s[i] = i < n ? src[i] : ~0ull;
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < P; i += SORT_THREADS) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = s[i], b = s[l];
          if (((i & k) == 0) == (a > b)) {
            s[i] = b;
            s[l] = a;
          }
        }
      }
    }
  __syncthreads();
  for (uint32_t i = poff[blockIdx.x] + threadIdx.x; i < poff[blockIdx.x + 1]; i += SORT_THREADS)
    pkey[i] = s[pidx[i] - g.cand_off];
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

// Device scratch of one selection: the slot table, per-parameter NaN flags, the plan of one batch of at most
// `batch` (parameter, rank) pairs (groups, tasks, histograms, pick lists) and a candidate buffer of `budget` keys.
SelectScratch select_scratch(uint64_t count, int D, size_t npairs) {
  SelectScratch z;
  z.batch = std::min(npairs, SELECT_PAIR_BATCH);
  z.budget = std::min((uint64_t)z.batch * SEL_CAP, SELECT_CAND_MAX);
  const size_t B = z.batch, T = B + (size_t)D;
  z.bytes = align256(count * sizeof(double*)) + align256((size_t)D) + align256(B * sizeof(SelGroup)) +
            align256(T * sizeof(SelTask)) + align256(2 * T * sizeof(uint32_t)) +
            align256(B * SEL_BINS * sizeof(uint64_t)) + align256(B * sizeof(uint32_t)) +
            align256(z.budget * sizeof(uint64_t)) + align256(B * sizeof(uint32_t)) +
            align256((B + 1) * sizeof(uint32_t)) + 2 * align256(B * sizeof(uint64_t));
  return z;
}

// See eb_chain_select_segments.  slots[count]: base of each stored step's [nseg, N, D] block (device pointers, rows
// D apart); ranks[nranks] < count * N.  out[nseg, nranks, D], has_nan[nseg, D] on the host; *passes counts full
// reads of the slice.  The planning runs over the nseg * D columns (select.cu's header).
cudaError_t select_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int Dp,
                       const uint64_t* ranks, size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes,
                       const SelectScratch& z, void* scratch, int sm_count, cudaStream_t st) {
  const uint64_t n = count * (uint64_t)N;
  const int D = (int)nseg * Dp;  // columns
  const uint64_t seg_stride = (uint64_t)N * (uint64_t)Dp;
  const size_t B = z.batch, T = B + (size_t)D;
  char* p = static_cast<char*>(scratch);
  auto take = [&](size_t bytes) {
    char* q = p;
    p += align256(bytes);
    return q;
  };
  const double** d_slots = reinterpret_cast<const double**>(take(count * sizeof(double*)));
  uint8_t* d_nan = reinterpret_cast<uint8_t*>(take((size_t)D));
  SelGroup* d_groups = reinterpret_cast<SelGroup*>(take(B * sizeof(SelGroup)));
  SelTask* d_tasks = reinterpret_cast<SelTask*>(take(T * sizeof(SelTask)));
  uint32_t* d_colrange = reinterpret_cast<uint32_t*>(take(2 * T * sizeof(uint32_t)));
  unsigned long long* d_hist = reinterpret_cast<unsigned long long*>(take(B * SEL_BINS * sizeof(uint64_t)));
  unsigned int* d_cnt = reinterpret_cast<unsigned int*>(take(B * sizeof(uint32_t)));
  unsigned long long* d_cand = reinterpret_cast<unsigned long long*>(take(z.budget * sizeof(uint64_t)));
  uint32_t* d_cg = reinterpret_cast<uint32_t*>(take(B * sizeof(uint32_t)));
  uint32_t* d_poff = reinterpret_cast<uint32_t*>(take((B + 1) * sizeof(uint32_t)));
  uint64_t* d_pidx = reinterpret_cast<uint64_t*>(take(B * sizeof(uint64_t)));
  unsigned long long* d_pkey = reinterpret_cast<unsigned long long*>(take(B * sizeof(uint64_t)));
#define SE(call)                              \
  do {                                        \
    cudaError_t _e = (call);                  \
    if (_e != cudaSuccess) return _e;         \
  } while (0)
  SE(cudaMemcpyAsync(d_slots, slots, count * sizeof(double*), cudaMemcpyHostToDevice, st));
  SE(cudaMemsetAsync(d_nan, 0, (size_t)D, st));
  std::vector<uint8_t> nan((size_t)D, 0), dropped((size_t)D, 0);
  *passes = 0;
  // (column, rank) pairs in (column, rank) order; pair i of column d = k * Dp + p answers out[k][r][p]
  std::vector<uint32_t> order(nranks);
  for (size_t r = 0; r < nranks; ++r) order[r] = (uint32_t)r;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ranks[a] < ranks[b]; });
  const size_t npairs = (size_t)D * nranks;
  std::vector<uint32_t> bd;
  std::vector<uint64_t> bk;
  std::vector<size_t> bo;
  std::vector<uint64_t> hist, pkey;
  SelPlan plan;
  for (size_t p0 = 0; p0 < npairs; p0 += B) {
    const size_t p1 = std::min(npairs, p0 + B);
    bd.clear();
    bk.clear();
    bo.clear();
    for (size_t i = p0; i < p1; ++i) {
      const uint32_t d = (uint32_t)(i / nranks);
      const uint32_t r = order[i % nranks];
      if (nan[d]) continue;  // a NaN seen by an earlier batch
      bd.push_back(d);
      bk.push_back(ranks[r]);
      bo.push_back(((size_t)(d / Dp) * nranks + r) * Dp + d % Dp);
    }
    plan.init(bd.data(), bk.data(), bd.size(), n);
    while (plan.live()) {
      plan.layout(z.budget);
      const size_t ng = plan.groups.size(), nt = plan.tasks.size();
      SE(cudaMemcpyAsync(d_groups, plan.groups.data(), ng * sizeof(SelGroup), cudaMemcpyHostToDevice, st));
      SE(cudaMemcpyAsync(d_tasks, plan.tasks.data(), nt * sizeof(SelTask), cudaMemcpyHostToDevice, st));
      SE(cudaMemcpyAsync(d_colrange, plan.colrange.data(), plan.colrange.size() * sizeof(uint32_t),
                         cudaMemcpyHostToDevice, st));
      SE(cudaMemsetAsync(d_hist, 0, ng * SEL_BINS * sizeof(uint64_t), st));
      SE(cudaMemsetAsync(d_cnt, 0, ng * sizeof(uint32_t), st));
      // rows of the slice split over grid y so that the pass fills the device with about 8 CTAs per SM
      const int per = SEL_THREADS / (int)SEL_WMAX;
      uint64_t ys = ((uint64_t)sm_count * 8 + nt - 1) / nt;
      ys = std::min<uint64_t>(ys, std::max<uint64_t>(1, n / ((uint64_t)per * 16)));
      ys = std::min<uint64_t>(std::max<uint64_t>(ys, 1), 65535);
      const uint64_t rows_per = (n + ys - 1) / ys;
      ys = (n + rows_per - 1) / rows_per;
      select_pass_kernel<<<dim3((unsigned)nt, (unsigned)ys), SEL_THREADS, 0, st>>>(
          d_slots, N, Dp, seg_stride, n, rows_per, d_tasks, d_colrange, d_groups, plan.bits, d_hist, d_cand, d_cnt, d_nan);
      SE(cudaGetLastError());
      ++*passes;
      const std::vector<uint64_t> pidx = plan.picks();
      pkey.assign(pidx.size(), 0);
      if (!pidx.empty()) {
        std::vector<uint32_t> cg, poff{0};
        for (size_t g = 0; g < ng; ++g)
          if (plan.groups[g].hslot < 0) {
            cg.push_back((uint32_t)g);
            poff.push_back(poff.back() + (uint32_t)plan.mem[g].size());
          }
        SE(cudaMemcpyAsync(d_cg, cg.data(), cg.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        SE(cudaMemcpyAsync(d_poff, poff.data(), poff.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        SE(cudaMemcpyAsync(d_pidx, pidx.data(), pidx.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
        select_sort_kernel<<<(unsigned)cg.size(), SORT_THREADS, 0, st>>>(d_groups, d_cg, d_poff, d_pidx, d_cand,
                                                                          d_pkey);
        SE(cudaGetLastError());
        SE(cudaMemcpyAsync(pkey.data(), d_pkey, pidx.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
      }
      hist.resize(ng * SEL_BINS);
      SE(cudaMemcpyAsync(hist.data(), d_hist, ng * SEL_BINS * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
      SE(cudaMemcpyAsync(nan.data(), d_nan, (size_t)D, cudaMemcpyDeviceToHost, st));
      SE(cudaStreamSynchronize(st));
      plan.refine(hist.data(), pkey.data());
      // a batch's first pass reads every value of its parameters: one holding a NaN is answered with NaN
      for (uint32_t d : bd)
        if (nan[d] && !dropped[d]) {
          plan.drop_param(d);
          dropped[d] = 1;
        }
    }
    for (size_t i = 0; i < bd.size(); ++i) out[bo[i]] = nan[bd[i]] ? NAN : key_value(plan.key[i]);
  }
#undef SE
  for (int d = 0; d < D; ++d) has_nan[d] = nan[(size_t)d];
  return cudaSuccess;
}

}  // namespace eb
