// Device chain storage (eb_step_store_chain, eb_chain_write, the running window): one launch per stored step.
#include "engine.cuh"

namespace eb {
namespace {

// cx[nx] = x[nx], clp[nl] = lp[nl], accepted[w] += acc[w] (backend.py:224-229) and cmask[w] = acc[w] (a running
// window's slot mask) in one launch; accepted and cmask are nullable.  The engine's arrays and every chain slot start
// 16 bytes aligned (slot pitches are even), so the copies move double2; an odd length leaves one scalar tail.  The
// chain is written with evict-first stores: the next step reads the state, not the chain.
__global__ void __launch_bounds__(256) chain_store_kernel(const double* __restrict__ x, const double* __restrict__ lp,
                                                          const uint8_t* __restrict__ acc, double* __restrict__ cx,
                                                          double* __restrict__ clp, double* __restrict__ accepted,
                                                          uint8_t* __restrict__ cmask, size_t nx, size_t nl,
                                                          int64_t N) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t nt = (size_t)gridDim.x * blockDim.x;
  const double2* x2 = reinterpret_cast<const double2*>(x);
  double2* cx2 = reinterpret_cast<double2*>(cx);
  for (size_t i = t; i < nx / 2; i += nt) __stcs(cx2 + i, x2[i]);
  const double2* lp2 = reinterpret_cast<const double2*>(lp);
  double2* clp2 = reinterpret_cast<double2*>(clp);
  for (size_t i = t; i < nl / 2; i += nt) __stcs(clp2 + i, lp2[i]);
  if (t == 0) {
    if (nx & 1) __stcs(cx + nx - 1, x[nx - 1]);
    if (nl & 1) __stcs(clp + nl - 1, lp[nl - 1]);
  }
  if (acc)
    for (size_t w = t; w < (size_t)N; w += nt) {
      if (accepted) accepted[w] += (double)acc[w];
      if (cmask) __stcs(cmask + w, acc[w]);
    }
}

// sums[w] = the sum over the slots s < nslots of mask[s, w], in slot order: one thread per walker, the slots' rows
// read coalesced across the walkers
__global__ void __launch_bounds__(256) mask_sum_kernel(const uint8_t* __restrict__ mask, uint64_t nslots, int64_t N,
                                                       double* __restrict__ sums) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= N) return;
  double s = 0.0;
  for (uint64_t k = 0; k < nslots; ++k) s += (double)mask[k * (uint64_t)N + (uint64_t)w];
  sums[w] = s;
}

}  // namespace

cudaError_t launch_chain_store(const double* x, const double* lp, const uint8_t* acc, double* cx, double* clp,
                               double* accepted, size_t nx, size_t nl, int64_t N, int sm_count, cudaStream_t st,
                               uint8_t* cmask) {
  size_t work = nx / 2;
  if (nl / 2 > work) work = nl / 2;
  if (acc && (size_t)N > work) work = (size_t)N;
  if (work == 0) work = 1;
  size_t blocks = (work + 255) / 256;
  const size_t cap = (size_t)sm_count * 8;
  if (blocks > cap) blocks = cap;
  chain_store_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, lp, acc, cx, clp, accepted, cmask, nx, nl, N);
  return cudaGetLastError();
}

cudaError_t launch_mask_sum(const uint8_t* mask, uint64_t nslots, int64_t N, double* sums, cudaStream_t st) {
  mask_sum_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(mask, nslots, N, sums);
  return cudaGetLastError();
}

}  // namespace eb
