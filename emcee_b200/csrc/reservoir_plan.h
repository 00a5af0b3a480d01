// The running reservoir's plan (reservoir.cu, eb_reservoir_config / eb_reservoir_read): which rows are kept, when the
// buffer is compacted, and how a compaction finds the rows to keep.  Everything here builds without CUDA, so
// tests/helpers/reservoir_host.cpp runs the same decisions on the host and checks them against np.lexsort.
//
//   kept      the K rows first in the order (key, step, walker) of all rows offered; key = reservoir_key
//             (philox.cuh, tag 10) of (seed, step, walker).  Bottom-K by random keys: a uniform sample without
//             replacement, and any prefix of the sorted rows is the reservoir of a smaller K.
//   buffer    cap = K + max(K, N) entries.  A recorded step appends the rows that pass res_passes; a compaction
//             keeps the K first and sets tau = the K-th key and full.
//   filter    a row passes while the buffer has never been full, or when its key is below tau.  A row whose key
//             equals tau loses: its step is later than that of every kept entry, so it comes after the K-th.  The
//             engine keeps that premise: eb_set_rng empties the reservoir when it changes the seed or moves the step
//             counter back, since the rows of a step offered again would come back with their old keys.
//   schedule  the host does not read the live count.  It keeps an upper bound of it (ResSchedule) and compacts
//             before a record that could overflow cap, and before every read.
//   select    MSB-first radix select over the live keys, RES_PASSES passes of RES_DIGIT_BITS bits: pass p counts the
//             digit p of the keys that match the digits chosen so far, and res_digit_holds picks the digit holding
//             the entry of rank K - 1.  After the last pass the prefix is the K-th key T, and `rank + 1` of the
//             entries with key T are kept: all of them when the group is that size (always, unless two 64-bit
//             keys collide), else the first by (step, walker, buffer index) (res_entry_before), so that exactly
//             K entries stay whatever the buffer holds.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define EB_RES_HD __host__ __device__ __forceinline__
#else
#define EB_RES_HD inline
#endif

namespace eb {

constexpr int RES_DIGIT_BITS = 8;
constexpr int RES_BINS = 1 << RES_DIGIT_BITS;
constexpr int RES_PASSES = 64 / RES_DIGIT_BITS;

EB_RES_HD uint64_t res_cap(uint64_t K, uint64_t N) { return K + (K > N ? K : N); }

// the filter of a recorded row
EB_RES_HD bool res_passes(bool full, uint64_t tau, uint64_t key) { return !full || key < tau; }

// digit `pass` of a key, most significant first
EB_RES_HD uint32_t res_digit(uint64_t key, int pass) {
  return (uint32_t)(key >> (64 - RES_DIGIT_BITS * (pass + 1))) & (RES_BINS - 1);
}

// the key agrees with `prefix` on the digits chosen before pass `pass`
EB_RES_HD bool res_in_prefix(uint64_t key, uint64_t prefix, int pass) {
  return pass == 0 || (key >> (64 - RES_DIGIT_BITS * pass)) == (prefix >> (64 - RES_DIGIT_BITS * pass));
}

// the state of a select: the digits chosen so far, and the rank of the wanted entry among the keys that match them
struct ResSelect {
  uint64_t prefix;
  uint64_t rank;
};

EB_RES_HD ResSelect res_select_start(uint64_t K) { return ResSelect{0, K - 1}; }

// digit d of a pass holds the wanted entry: `below` keys of the matching ones have a smaller digit, `here` have d
EB_RES_HD bool res_digit_holds(uint64_t below, uint64_t here, uint64_t rank) { return below <= rank && rank < below + here; }

EB_RES_HD void res_take_digit(ResSelect& s, int pass, uint32_t d, uint64_t below) {
  s.prefix |= (uint64_t)d << (64 - RES_DIGIT_BITS * (pass + 1));
  s.rank -= below;
}

// the order of the entries that tie on the key
EB_RES_HD bool res_row_before(uint64_t step_a, uint32_t walker_a, uint64_t step_b, uint32_t walker_b) {
  return step_a < step_b || (step_a == step_b && walker_a < walker_b);
}

// the order of the live entries a and b that tie on the key: (step, walker), then the buffer index, a strict order
// even for two entries of the same (step, walker)
EB_RES_HD bool res_entry_before(uint64_t step_a, uint32_t walker_a, uint64_t index_a, uint64_t step_b,
                                uint32_t walker_b, uint64_t index_b) {
  if (res_row_before(step_a, walker_a, step_b, walker_b)) return true;
  return step_a == step_b && walker_a == walker_b && index_a < index_b;
}

// sizes from this on are refused: entries are addressed with 32 bits
constexpr uint64_t RES_SIZE_LIMIT = (uint64_t)1 << 32;

// the host's view of the buffer: rows offered, and an upper bound of the live entries
struct ResSchedule {
  uint64_t K = 0, N = 0, cap = 0;
  uint64_t offered = 0;
  uint64_t bound = 0;

  ResSchedule() = default;
  ResSchedule(uint64_t k, uint64_t n) : K(k), N(n), cap(res_cap(k, n)) {}
  bool compact_before_record() const { return bound + N > cap; }
  bool compact_before_read() const { return bound > K; }
  uint64_t kept() const { return offered < K ? offered : K; }
  void compacted() { bound = kept(); }
  void recorded() {
    offered += N;
    bound += N;
  }
};

}  // namespace eb
