// Exact order statistics of a stored chain slice (select.cu, eb_chain_select): the order-preserving key of a
// float64 and the bookkeeping of the MSB-first radix selection.  Builds for the host without CUDA, so that
// tests/helpers/select_host.cpp can run the same plan on the CPU; the key helpers are device functions too.
//
// One selection finds, for every (parameter d, rank k) pair, the k-th smallest of that parameter's n values.  The
// pairs of one parameter whose candidates agree in their top `bits` key bits form a group; every pass over the
// slice refines each group by its next SEL_DIGIT bits (a per-group histogram of that digit), or, once the group
// holds at most SEL_CAP candidates, copies those candidates out (compaction) so that a sort finishes it.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#ifdef __CUDACC__
#define EB_SEL_HD __host__ __device__ __forceinline__
#else
#define EB_SEL_HD inline
#endif

namespace eb {

constexpr int SEL_DIGIT = 8;                 // bits resolved per histogram pass
constexpr int SEL_BINS = 1 << SEL_DIGIT;     // histogram bins per group
constexpr uint64_t SEL_CAP = 4096;           // a group of at most this many candidates is compacted and sorted
constexpr int SEL_HMAX = 40;                 // histogram groups per CTA: 40 x 256 uint32 = 40 KB of shared memory
constexpr int SEL_WMAX = 32;                 // parameters per CTA column block

// float64 -> uint64 with the same order: -0.0 becomes +0.0 first, negatives get every bit flipped, positives the
// sign bit set.  -inf < finite < +inf keep their order; NaN maps outside [-inf, +inf] (never selected: a
// parameter holding one is answered with NaN).
EB_SEL_HD uint64_t order_key_bits(uint64_t u) {
  const uint64_t sign = (uint64_t)1 << 63;
  if (u == sign) u = 0;  // -0.0
  return (u & sign) ? ~u : (u | sign);
}

EB_SEL_HD uint64_t key_to_bits(uint64_t key) {
  const uint64_t sign = (uint64_t)1 << 63;
  return (key & sign) ? (key & ~sign) : ~key;
}

inline uint64_t order_key(double v) {
  uint64_t u;
  memcpy(&u, &v, sizeof u);
  return order_key_bits(u);
}

inline double key_value(uint64_t key) {
  const uint64_t u = key_to_bits(key);
  double v;
  memcpy(&v, &u, sizeof v);
  return v;
}

// does `key` carry the group prefix of its top `bits` bits?
EB_SEL_HD bool key_in_group(uint64_t key, uint64_t prefix, int bits) {
  return bits == 0 || (key >> (64 - bits)) == prefix;
}

// the digit after the top `bits` bits
EB_SEL_HD int key_digit(uint64_t key, int bits) { return (int)((key >> (64 - SEL_DIGIT - bits)) & (SEL_BINS - 1)); }

// A group of one pass, as the device reads it (32 bytes).
struct SelGroup {
  uint64_t prefix;    // top `bits` bits of every candidate
  uint64_t count;     // candidates (values of parameter d with this prefix)
  uint64_t cand_off;  // compaction: first slot of the group in the candidate buffer
  int32_t hslot;      // histogram: slot in its CTA's shared histograms; -1: compaction
  uint32_t d;         // parameter
};

// A CTA column block of a pass: parameters d0 .. d0 + w - 1; the groups of parameter d0 + c it handles are
// [colrange[cr + c][0], colrange[cr + c][1]).
struct SelTask {
  uint32_t d0, w, cr, pad;
};

// index of the group among g[lo, hi) (sorted by prefix, one parameter) whose prefix `key` carries, or -1
EB_SEL_HD int find_group(const SelGroup* g, uint32_t lo, uint32_t hi, uint64_t key, int bits) {
  if (lo >= hi) return -1;
  const uint64_t p = bits == 0 ? 0 : key >> (64 - bits);
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (g[mid].prefix <= p) lo = mid;
    else hi = mid;
  }
  return g[lo].prefix == p ? (int)lo : -1;
}

// The digit holding rank k of a histogram of SEL_BINS counts; k becomes the rank within that digit's bin and
// *bin its count.  k < sum(hist).
inline int pick_digit(const uint64_t* hist, uint64_t& k, uint64_t* bin) {
  int b = 0;
  while (k >= hist[b]) k -= hist[b++];
  *bin = hist[b];
  return b;
}

// The host side of one selection over pairs (d[i], k[i]) of a slice with n values per parameter.
struct SelPlan {
  int bits = 0;                            // key bits every live group has resolved
  std::vector<SelGroup> groups;            // live groups of the next pass, sorted by (d, prefix)
  std::vector<std::vector<uint32_t>> mem;  // pairs of each live group
  std::vector<uint32_t> pd;                // per pair: parameter
  std::vector<uint64_t> pk;                // per pair: rank within its group
  std::vector<uint64_t> key;               // per pair: the selected key, once done
  std::vector<uint8_t> done;
  // layout of the next pass
  std::vector<SelTask> tasks;
  std::vector<uint32_t> colrange;  // [lo, hi) per task column
  uint64_t cand_used = 0;

  // pairs sorted by (parameter, rank); one group per parameter holds all its pairs
  void init(const uint32_t* d, const uint64_t* k, size_t npairs, uint64_t n) {
    bits = 0;
    pd.assign(d, d + npairs);
    pk.assign(k, k + npairs);
    key.assign(npairs, 0);
    done.assign(npairs, 0);
    groups.clear();
    mem.clear();
    for (size_t i = 0; i < npairs; ++i) {
      if (groups.empty() || groups.back().d != d[i]) {
        groups.push_back(SelGroup{0, n, 0, 0, d[i]});
        mem.emplace_back();
      }
      mem.back().push_back((uint32_t)i);
    }
  }

  bool live() const { return !groups.empty(); }

  // Modes and CTA blocks of the next pass: a group of at most SEL_CAP candidates is compacted while the candidate
  // buffer (cand_budget keys) has room; the others get histogram slots, at most SEL_HMAX per task, and a task
  // spans at most SEL_WMAX consecutive parameters.  A parameter with more histogram groups than one task holds is
  // split over several one-column tasks.
  void layout(uint64_t cand_budget) {
    tasks.clear();
    colrange.clear();
    cand_used = 0;
    for (SelGroup& g : groups) {
      if (g.count <= SEL_CAP && cand_used + g.count <= cand_budget) {
        g.hslot = -1;
        g.cand_off = cand_used;
        cand_used += g.count;
      } else {
        g.hslot = 0;
        g.cand_off = 0;
      }
    }
    size_t i = 0;
    int nh = 0;  // histogram slots of the open task
    auto open = [&](uint32_t d) {
      tasks.push_back(SelTask{d, 0, (uint32_t)colrange.size(), 0});
      nh = 0;
    };
    while (i < groups.size()) {
      const uint32_t d = groups[i].d;
      size_t j = i;
      int h = 0;
      while (j < groups.size() && groups[j].d == d) h += groups[j++].hslot >= 0;
      if (tasks.empty() || tasks.back().w == (uint32_t)SEL_WMAX || nh + h > SEL_HMAX ||
          tasks.back().d0 + tasks.back().w != d)
        open(d);
      if (h <= SEL_HMAX) {
        for (size_t m = i; m < j; ++m)
          if (groups[m].hslot >= 0) groups[m].hslot = nh++;
        colrange.push_back((uint32_t)i);
        colrange.push_back((uint32_t)j);
        tasks.back().w++;
      } else {  // one column per task, SEL_HMAX histogram groups each
        size_t m = i;
        while (m < j) {
          if (tasks.back().w != 0) open(d);
          const size_t lo = m;
          int c = 0;
          while (m < j && (c < SEL_HMAX || groups[m].hslot < 0)) {
            if (groups[m].hslot >= 0) groups[m].hslot = c++;
            ++m;
          }
          colrange.push_back((uint32_t)lo);
          colrange.push_back((uint32_t)m);
          tasks.back().w = 1;
          nh = SEL_HMAX + 1;  // nothing joins a split column's task
        }
      }
      i = j;
    }
  }

  // drop the groups of parameter d (it holds a NaN: its answers are NaN)
  void drop_param(uint32_t d) {
    size_t o = 0;
    for (size_t i = 0; i < groups.size(); ++i) {
      if (groups[i].d == d) {
        for (uint32_t p : mem[i]) done[p] = 1;
        continue;
      }
      if (o != i) {
        groups[o] = groups[i];
        mem[o] = std::move(mem[i]);
      }
      ++o;
    }
    groups.resize(o);
    mem.resize(o);
  }

  // Candidate-buffer indices of the ranks the compacted groups of the last layout answer, once their candidates
  // are sorted in place; refine() takes their keys in this order.
  std::vector<uint64_t> picks() const {
    std::vector<uint64_t> out;
    for (size_t i = 0; i < groups.size(); ++i)
      if (groups[i].hslot < 0)
        for (uint32_t p : mem[i]) out.push_back(groups[i].cand_off + pk[p]);
    return out;
  }

  // After a pass: `hist` holds SEL_BINS counts per live group (only the histogram groups' are read), `picked` the
  // keys at picks().  Compacted groups are finished; every histogram group is split by its next digit, and a
  // group whose prefix reaches 64 bits is finished too.
  void refine(const uint64_t* hist, const uint64_t* picked) {
    std::vector<SelGroup> ng;
    std::vector<std::vector<uint32_t>> nm;
    size_t q = 0;
    for (size_t i = 0; i < groups.size(); ++i) {
      const SelGroup& g = groups[i];
      if (g.hslot < 0) {
        for (uint32_t p : mem[i]) {
          key[p] = picked[q++];
          done[p] = 1;
        }
        continue;
      }
      const uint64_t* h = hist + i * SEL_BINS;
      // the pairs of a group ascend in rank, so their digits ascend and the new groups stay sorted
      for (uint32_t p : mem[i]) {
        uint64_t cnt = 0;
        const int b = pick_digit(h, pk[p], &cnt);
        const uint64_t prefix = (g.prefix << SEL_DIGIT) | (uint64_t)b;
        if (bits + SEL_DIGIT == 64) {
          key[p] = prefix;
          done[p] = 1;
          continue;
        }
        if (ng.empty() || ng.back().d != g.d || ng.back().prefix != prefix) {
          ng.push_back(SelGroup{prefix, cnt, 0, 0, g.d});
          nm.emplace_back();
        }
        nm.back().push_back(p);
      }
    }
    groups.swap(ng);
    mem.swap(nm);
    bits += SEL_DIGIT;
  }
};

}  // namespace eb
