// Stored index -> (segment, offset) of a device chain kept as a list of segments (eb_chain, context.h).  Host code
// only, without CUDA, so that tests/helpers/chain_map_host.cpp and chain_ring_host.cpp can build it for the CPU tests.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace eb {

// The slice first, first + stride, ..., first + (count - 1) * stride of a chain whose segment s holds the slots
// [start[s], start[s + 1]) (start[0] = 0, start[nseg] = capacity), read from the ring origin `origin`: logical slot
// i is physical slot (origin + i) mod capacity (origin 0 for a chain that is not a ring).  f(seg, off, k0, n) is
// called once per run of the slice inside one segment, in order: slice entries k0 .. k0 + n - 1 are the physical
// slots off, off + stride, ..., off + (n - 1) * stride of segment seg.  A run ends at a segment's end, and so where
// the ring wraps (the end of the last segment).  Returns false, calling nothing, when stride == 0, a slot lies beyond
// the capacity or origin does not.
template <class F>
bool for_each_chain_run(const uint64_t* start, size_t nseg, uint64_t origin, uint64_t first, uint64_t stride,
                        uint64_t count, F&& f) {
  if (count == 0) return true;
  if (stride == 0) return false;
  const uint64_t cap = start[nseg];
  if (count - 1 > (UINT64_MAX - first) / stride) return false;
  if (first + (count - 1) * stride >= cap || origin >= cap) return false;
  const uint64_t tail = cap - origin;  // logical slots before the wrap
  size_t s = 0;
  for (uint64_t k = 0; k < count;) {
    const uint64_t logical = first + k * stride;
    const uint64_t slot = logical < tail ? origin + logical : logical - tail;
    if (slot < start[s]) s = 0;  // wrapped
    while (slot >= start[s + 1]) ++s;
    uint64_t n = (start[s + 1] - 1 - slot) / stride + 1;  // entries left in this segment
    if (n > count - k) n = count - k;
    f(s, slot - start[s], k, n);
    k += n;
  }
  return true;
}

// The same slice of a chain that is not a ring (origin 0).
template <class F>
bool for_each_chain_run(const uint64_t* start, size_t nseg, uint64_t first, uint64_t stride, uint64_t count, F&& f) {
  return for_each_chain_run(start, nseg, 0, first, stride, count, static_cast<F&&>(f));
}

}  // namespace eb
