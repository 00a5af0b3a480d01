// Host-side probe of emcee_b200/csrc/select_keys.h, built by tests/test_chain_summary_host.py with g++: the key
// transform, and the whole selection of eb_chain_select run on the CPU with the same plan (SelPlan), the same
// CTA column blocks and group lookup as select_pass_kernel, and a sort of each compacted group.
#include <algorithm>
#include <cmath>
#include <vector>

#include "../../emcee_b200/csrc/select_keys.h"

namespace {
int max_column_tasks = 0;  // the most CTA column blocks one parameter took in a pass of the last probe_select
}

extern "C" {

int probe_select_max_column_tasks() { return max_column_tasks; }

void probe_keys(const double* x, size_t n, uint64_t* keys, double* back) {
  for (size_t i = 0; i < n; ++i) {
    keys[i] = eb::order_key(x[i]);
    back[i] = eb::key_value(keys[i]);
  }
}

// x[rows, D] row-major; ranks[nranks] sorted; out[nranks, D]; has_nan[D]; returns the passes, or -1 when a
// group was seen inconsistent (a count the histograms promised that the compaction did not find)
int probe_select(const double* x, uint64_t rows, int D, const uint64_t* ranks, size_t nranks, uint64_t cand_budget,
                 double* out, uint8_t* has_nan) {
  using namespace eb;
  std::vector<uint8_t> nan((size_t)D, 0);
  for (uint64_t r = 0; r < rows; ++r)
    for (int d = 0; d < D; ++d)
      if (x[r * D + d] != x[r * D + d]) nan[(size_t)d] = 1;
  std::vector<uint32_t> pd;
  std::vector<uint64_t> pk;
  for (int d = 0; d < D; ++d)
    for (size_t r = 0; r < nranks; ++r) {
      pd.push_back((uint32_t)d);
      pk.push_back(ranks[r]);
    }
  SelPlan plan;
  plan.init(pd.data(), pk.data(), pd.size(), rows);
  int passes = 0;
  std::vector<uint64_t> hist, cand;
  std::vector<uint32_t> cnt;
  bool first = true;
  max_column_tasks = 0;
  std::vector<int> col_tasks;
  while (plan.live()) {
    plan.layout(cand_budget);
    const size_t ng = plan.groups.size();
    hist.assign(ng * SEL_BINS, 0);
    cand.assign(plan.cand_used, 0);
    cnt.assign(ng, 0);
    col_tasks.assign((size_t)D, 0);
    for (const SelTask& t : plan.tasks)
      for (uint32_t c = 0; c < t.w && t.d0 + c < (uint32_t)D; ++c)
        max_column_tasks = std::max(max_column_tasks, ++col_tasks[t.d0 + c]);
    for (const SelTask& t : plan.tasks) {
      if (t.w == 0 || t.w > (uint32_t)SEL_WMAX) return -1;
      int slots = 0;
      for (uint32_t c = 0; c < t.w; ++c)
        for (uint32_t g = plan.colrange[t.cr + 2 * c]; g < plan.colrange[t.cr + 2 * c + 1]; ++g)
          if (plan.groups[g].hslot >= 0) {
            if (plan.groups[g].hslot >= SEL_HMAX) return -1;
            ++slots;
          }
      if (slots > SEL_HMAX) return -1;
      for (uint64_t r = 0; r < rows; ++r)
        for (uint32_t c = 0; c < t.w; ++c) {
          const int d = (int)(t.d0 + c);
          const uint64_t key = order_key(x[r * D + d]);
          const int g = find_group(plan.groups.data(), plan.colrange[t.cr + 2 * c], plan.colrange[t.cr + 2 * c + 1],
                                   key, plan.bits);
          if (g < 0) continue;
          const SelGroup& G = plan.groups[(size_t)g];
          if (!key_in_group(key, G.prefix, plan.bits) || G.d != (uint32_t)d) return -1;
          if (G.hslot >= 0) {
            hist[(size_t)g * SEL_BINS + key_digit(key, plan.bits)]++;
          } else if (cnt[(size_t)g] < G.count) {
            cand[G.cand_off + cnt[(size_t)g]++] = key;
          }
        }
    }
    ++passes;
    for (size_t g = 0; g < ng; ++g) {
      const SelGroup& G = plan.groups[g];
      if (G.hslot >= 0) {
        uint64_t tot = 0;
        for (int b = 0; b < SEL_BINS; ++b) tot += hist[g * SEL_BINS + b];
        if (tot != G.count && !nan[G.d]) return -1;
      } else {
        if (cnt[g] != G.count && !nan[G.d]) return -1;
        std::sort(cand.begin() + G.cand_off, cand.begin() + G.cand_off + G.count);
      }
    }
    const std::vector<uint64_t> pidx = plan.picks();
    std::vector<uint64_t> picked(pidx.size());
    for (size_t i = 0; i < pidx.size(); ++i) picked[i] = cand[pidx[i]];
    plan.refine(hist.data(), picked.data());
    if (first)
      for (int d = 0; d < D; ++d)
        if (nan[(size_t)d]) plan.drop_param((uint32_t)d);
    first = false;
  }
  for (size_t i = 0; i < pd.size(); ++i) {
    const size_t r = i % nranks;
    out[r * D + pd[i]] = nan[pd[i]] ? (double)NAN : key_value(plan.key[i]);
  }
  for (int d = 0; d < D; ++d) has_nan[d] = nan[(size_t)d];
  return passes;
}
}
