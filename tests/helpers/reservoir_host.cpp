// Host-side probe of the running reservoir: the tag-10 key of emcee_b200/csrc/philox.cuh, and the decisions of
// emcee_b200/csrc/reservoir_plan.h (filter, schedule, radix select, tie rule) in the order reservoir.cu's kernels take
// them, one entry at a time.  Built by tests/test_reservoir_keys_host.py with g++ and checked against numpy.
#include <cmath>
#include <cstdint>
#include <algorithm>
#include <vector>
using std::sqrt;
#include "../../emcee_b200/csrc/philox.cuh"
#include "../../emcee_b200/csrc/reservoir_plan.h"

namespace {

struct Buf {
  std::vector<uint64_t> key, step;
  std::vector<uint32_t> walker;
  uint64_t count = 0, tau = 0;
  bool full = false;
};

// res_begin_kernel .. res_move_kernel: keep the K first of the live entries (a no-op while no more than K are live)
void compact(Buf& b, uint64_t K) {
  if (b.count <= K) return;
  eb::ResSelect s = eb::res_select_start(K);
  uint64_t group = 0;
  for (int pass = 0; pass < eb::RES_PASSES; ++pass) {
    uint64_t hist[eb::RES_BINS] = {0};
    for (uint64_t i = 0; i < b.count; ++i)
      if (eb::res_in_prefix(b.key[i], s.prefix, pass)) ++hist[eb::res_digit(b.key[i], pass)];
    uint64_t below = 0;
    for (uint32_t d = 0; d < (uint32_t)eb::RES_BINS; ++d) {
      if (eb::res_digit_holds(below, hist[d], s.rank)) {
        eb::res_take_digit(s, pass, d, below);
        group = hist[d];
        break;
      }
      below += hist[d];
    }
  }
  const uint64_t T = s.prefix, need = s.rank + 1;
  std::vector<uint64_t> holes, movers, grouped;
  for (uint64_t i = 0; i < b.count; ++i) {
    const uint64_t k = b.key[i];
    const bool g = k == T && group != need;
    const bool kept = k < T || (k == T && group == need);
    if (g) grouped.push_back(i);
    else if (i < K && !kept) holes.push_back(i);
    else if (i >= K && kept) movers.push_back(i);
  }
  for (uint64_t e : grouped) {
    uint64_t before = 0;
    for (uint64_t f : grouped)
      before += eb::res_entry_before(b.step[f], b.walker[f], f, b.step[e], b.walker[e], e) ? 1 : 0;
    const bool kept = before < need;
    if (e < K && !kept) holes.push_back(e);
    if (e >= K && kept) movers.push_back(e);
  }
  for (size_t j = 0; j < std::min(movers.size(), holes.size()); ++j) {
    b.key[holes[j]] = b.key[movers[j]];
    b.step[holes[j]] = b.step[movers[j]];
    b.walker[holes[j]] = b.walker[movers[j]];
  }
  b.tau = T;
  b.full = true;
  b.count = K;
}

}  // namespace

extern "C" {

void probe_reservoir_keys(uint64_t seed, const uint64_t* step, const uint32_t* walker, int n, uint64_t* out) {
  for (int i = 0; i < n; ++i) out[i] = eb::reservoir_key(seed, step[i], walker[i]);
}

uint64_t probe_reservoir_cap(uint64_t K, uint64_t N) { return eb::res_cap(K, N); }

// one compaction of count entries: keep[i] = 1 for the entries it keeps
void probe_reservoir_compact(const uint64_t* key, const uint64_t* step, const uint32_t* walker, uint64_t count,
                             uint64_t K, uint8_t* keep) {
  Buf b;
  b.key.assign(key, key + count);
  b.step.assign(step, step + count);
  b.walker.assign(walker, walker + count);
  b.count = count;
  compact(b, K);
  for (uint64_t i = 0; i < count; ++i) keep[i] = 0;
  // the entries are told apart by (step, walker), distinct in the probe's input
  for (uint64_t j = 0; j < b.count; ++j)
    for (uint64_t i = 0; i < count; ++i)
      if (step[i] == b.step[j] && walker[i] == b.walker[j]) keep[i] = 1;
}

// R records of N rows (row w of record r has key keys[r * N + w], step steps[r], walker w) through the schedule, the
// filter and the compactions of the engine, then the read.  Writes the kept (key, step, walker) in buffer order and
// returns their number; stats = [compactions, largest bound, largest live count, cap, offered]
uint64_t probe_reservoir_stream(const uint64_t* keys, const uint64_t* steps, uint64_t R, uint64_t N, uint64_t K,
                                uint64_t* out_key, uint64_t* out_step, uint32_t* out_walker, uint64_t* stats) {
  eb::ResSchedule plan(K, N);
  Buf b;
  b.key.resize(plan.cap);
  b.step.resize(plan.cap);
  b.walker.resize(plan.cap);
  uint64_t ncompact = 0, max_bound = 0, max_count = 0;
  for (uint64_t r = 0; r < R; ++r) {
    if (plan.compact_before_record()) {
      compact(b, K);
      plan.compacted();
      ++ncompact;
    }
    for (uint64_t w = 0; w < N; ++w) {
      const uint64_t key = keys[r * N + w];
      if (!eb::res_passes(b.full, b.tau, key)) continue;
      if (b.count >= plan.cap) return ~(uint64_t)0;  // an overflow the schedule should have prevented
      b.key[b.count] = key;
      b.step[b.count] = steps[r];
      b.walker[b.count] = (uint32_t)w;
      ++b.count;
    }
    plan.recorded();
    if (b.count > plan.bound) return ~(uint64_t)0;  // the bound is not one
    max_bound = plan.bound > max_bound ? plan.bound : max_bound;
    max_count = b.count > max_count ? b.count : max_count;
  }
  if (plan.compact_before_read()) {
    compact(b, K);
    plan.compacted();
    ++ncompact;
  }
  if (b.count != plan.kept()) return ~(uint64_t)0;
  for (uint64_t j = 0; j < b.count; ++j) {
    out_key[j] = b.key[j];
    out_step[j] = b.step[j];
    out_walker[j] = b.walker[j];
  }
  stats[0] = ncompact;
  stats[1] = max_bound;
  stats[2] = max_count;
  stats[3] = plan.cap;
  stats[4] = plan.offered;
  return b.count;
}
}
