// Blob selection of a callback model (eb_callback_blobs): after the accept launch of a half-step, the walkers that
// accepted their proposal take the proposal's blob record (moves/move.py:36-43 `old_state.blobs[m1] =
// new_state.blobs[m2]`); the others keep theirs.  A separate kernel, launched only for models with blobs, so the
// half-step kernels and their launch counts are those of a run without blobs.
//
// Records are packed (device stride = record size), so the live blobs reach the host layout [nwalkers, record] in one
// contiguous copy.  Buffers come from cudaMalloc (256-byte aligned), so every record starts at a multiple of the
// largest power of two dividing the record size: that is the vector width, and an aligned record needs no byte loop.
#include <algorithm>

#include "engine.cuh"

namespace eb {

namespace {

// one thread per vector of a record: t -> (active rank r, vector v); consecutive threads copy consecutive vectors
// of a record.  `accepted` is the mask the accept launch just wrote for this split's walkers.
template <class V>
__global__ void __launch_bounds__(256) blob_select_kernel(const int32_t* __restrict__ order, int a_start, int i_lo,
                                                          int64_t rows, const uint8_t* __restrict__ accepted,
                                                          const V* __restrict__ prop, V* __restrict__ live,
                                                          int64_t vpr) {
  const int64_t total = rows * vpr;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / vpr, v = t - r * vpr;
    const int64_t i = i_lo + r;
    const int64_t w = order ? (int64_t)order[a_start + i] : i;  // as in half_step_generic_kernel
    if (accepted[w]) live[w * vpr + v] = prop[t];
  }
}

template <class V>
cudaError_t launch_t(const int32_t* order, int a_start, int i_lo, int64_t rows, const uint8_t* accepted,
                     const void* prop, void* live, size_t record_bytes, cudaStream_t st) {
  const int64_t vpr = (int64_t)(record_bytes / sizeof(V));
  const int64_t total = rows * vpr;
  const unsigned grid = (unsigned)std::min<int64_t>((total + 255) / 256, 4096);
  blob_select_kernel<V><<<grid, 256, 0, st>>>(order, a_start, i_lo, rows, accepted, static_cast<const V*>(prop),
                                               static_cast<V*>(live), vpr);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_blob_select(const int32_t* order, int a_start, int i_lo, int i_hi, const uint8_t* accepted,
                               const void* prop, void* live, size_t record_bytes, cudaStream_t st) {
  const int64_t rows = (int64_t)i_hi - i_lo;
  if (rows <= 0 || record_bytes == 0) return cudaSuccess;
  if (record_bytes % 16 == 0) return launch_t<uint4>(order, a_start, i_lo, rows, accepted, prop, live, record_bytes, st);
  if (record_bytes % 8 == 0) return launch_t<uint2>(order, a_start, i_lo, rows, accepted, prop, live, record_bytes, st);
  if (record_bytes % 4 == 0) return launch_t<uint32_t>(order, a_start, i_lo, rows, accepted, prop, live, record_bytes, st);
  if (record_bytes % 2 == 0) return launch_t<uint16_t>(order, a_start, i_lo, rows, accepted, prop, live, record_bytes, st);
  return launch_t<uint8_t>(order, a_start, i_lo, rows, accepted, prop, live, record_bytes, st);
}

}  // namespace eb
