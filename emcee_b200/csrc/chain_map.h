// Stored index -> (segment, offset) of a device chain kept as a list of segments (eb_chain, context.h).  Host code
// only, without CUDA, so that tests/helpers/chain_map_host.cpp can build it for the CPU tests.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace eb {

// The slice first, first + stride, ..., first + (count - 1) * stride of a chain whose segment s holds the slots
// [start[s], start[s + 1]) (start[0] = 0, start[nseg] = capacity).  f(seg, off, k0, n) is called once per run of
// the slice inside one segment, in order: slice entries k0 .. k0 + n - 1 are the slots off, off + stride, ...,
// off + (n - 1) * stride of segment seg.  Returns false, calling nothing, when stride == 0 or a slot lies beyond
// the capacity.
template <class F>
bool for_each_chain_run(const uint64_t* start, size_t nseg, uint64_t first, uint64_t stride, uint64_t count, F&& f) {
  if (count == 0) return true;
  if (stride == 0) return false;
  if (count - 1 > (UINT64_MAX - first) / stride) return false;
  if (first + (count - 1) * stride >= start[nseg]) return false;
  size_t s = 0;
  for (uint64_t k = 0; k < count;) {
    const uint64_t slot = first + k * stride;
    while (slot >= start[s + 1]) ++s;
    uint64_t n = (start[s + 1] - 1 - slot) / stride + 1;  // entries left in this segment
    if (n > count - k) n = count - k;
    f(s, slot - start[s], k, n);
    k += n;
  }
  return true;
}

}  // namespace eb
