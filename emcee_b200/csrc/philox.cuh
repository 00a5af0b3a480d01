// Counter-addressed draws (Philox4x32-10) -- CUDA/host statement of the draw
// specification in DESIGN.md; the numpy statement is oracle/philox.py and the
// two must agree bit for bit (tests/test_gpu_parity.py).
//
// counter = (index, step_lo, step_hi, (split << 8) | tag), key = (seed_lo, seed_hi)
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define EB_HD __host__ __device__ __forceinline__
#else
#define EB_HD inline
#endif
#ifdef __CUDA_ARCH__
#define EB_UNROLL _Pragma("unroll")
#else
#define EB_UNROLL
#endif

namespace eb {

enum : uint32_t {
  TAG_MOVE = 1,     // move of the step            (ensemble.py:406)
  TAG_SHUFFLE = 2,  // split-permutation round keys (red_blue.py:79-80)
  TAG_PROP_A = 3,   // proposal draw block A of active rank i
  TAG_PROP_B = 4,   // proposal draw block B of active rank i
  TAG_ACCEPT = 5,   // Metropolis uniform of active rank i (red_blue.py:100)
  TAG_NORMAL = 6,   // bulk standard normals of row i: block k = normals 2k, 2k+1 (walk.py:36, gaussian.py:97)
  TAG_SUBSET = 7,   // round keys of the helper-subset permutation of active rank i (walk.py:34)
  TAG_GRAPH = 9,    // draws of a captured proposal's row i: block k = draws 2k, 2k+1 (eb_move_set_proposal_graphs)
  TAG_RESERVOIR = 10  // the key of recorded row (step, walker i) of the running reservoir (eb_reservoir_config)
};

constexpr int FEISTEL_ROUNDS = 8;

struct u32x4 {
  uint32_t x, y, z, w;
};

EB_HD void mulhilo32(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
  lo = a * b;
  hi = __umulhi(a, b);
#else
  uint64_t p = (uint64_t)a * (uint64_t)b;
  lo = (uint32_t)p;
  hi = (uint32_t)(p >> 32);
#endif
}

EB_HD u32x4 philox4x32_10(u32x4 c, uint32_t k0, uint32_t k1) {
EB_UNROLL
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, lo0, hi1, lo1;
    mulhilo32(0xD2511F53u, c.x, hi0, lo0);
    mulhilo32(0xCD9E8D57u, c.z, hi1, lo1);
    u32x4 n;
    n.x = hi1 ^ c.y ^ k0;
    n.y = lo1;
    n.z = hi0 ^ c.w ^ k1;
    n.w = lo0;
    c = n;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

EB_HD u32x4 draw_words(uint64_t seed, uint64_t step, uint32_t split, uint32_t tag, uint32_t index) {
  u32x4 c;
  c.x = index;
  c.y = (uint32_t)step;
  c.z = (uint32_t)(step >> 32);
  c.w = ((split & 0xFFFFFFu) << 8) | (tag & 0xFFu);
  return philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// uniform on [0,1): top 53 bits of hi:lo times 2^-53
EB_HD double u53(uint32_t lo, uint32_t hi) {
  uint64_t x = ((uint64_t)hi << 32) | (uint64_t)lo;
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}

// the Box-Muller pair of a block's words (draw specification, tag 6): r cos t, r sin t with r = sqrt(-2 log(1 -
// u53(w0, w1))), t = 2 pi u53(w2, w3).  Tag 6 (normal_pair, draws.cuh) and tag 9 ("normal") both decode with it.
EB_HD void box_muller_pair(const u32x4& w, double& n0, double& n1) {
  const double r = sqrt(-2.0 * log(1.0 - u53(w.x, w.y)));
  double sn, cs;
#ifdef __CUDA_ARCH__
  sincos(6.283185307179586 * u53(w.z, w.w), &sn, &cs);
#else
  const double th = 6.283185307179586 * u53(w.z, w.w);
  sn = sin(th);
  cs = cos(th);
#endif
  n0 = r * cs;
  n1 = r * sn;
}

// draws 2k and 2k + 1 of a captured proposal's row from the words w of its TAG_GRAPH block k: two uniforms, or
// (normal != 0) the Box-Muller pair of these words
EB_HD void graph_draw_pair(const u32x4& w, int normal, double& d0, double& d1) {
  if (normal) {
    box_muller_pair(w, d0, d1);
    return;
  }
  d0 = u53(w.x, w.y);
  d1 = u53(w.z, w.w);
}

// the reservoir key of walker w's row recorded at step counter `step`: (w1 << 32) | w0 of block (step, 0, TAG_RESERVOIR,
// w); a separate purpose, so that recording rows changes no other draw
EB_HD uint64_t reservoir_key(uint64_t seed, uint64_t step, uint32_t walker) {
  const u32x4 w = draw_words(seed, step, 0, TAG_RESERVOIR, walker);
  return ((uint64_t)w.y << 32) | (uint64_t)w.x;
}

// integer on [0,n): high 64 bits of (hi:lo) * n
EB_HD uint64_t bounded64(uint32_t lo, uint32_t hi, uint64_t n) {
  uint64_t x = ((uint64_t)hi << 32) | (uint64_t)lo;
#ifdef __CUDA_ARCH__
  return __umul64hi(x, n);
#else
  return (uint64_t)(((unsigned __int128)x * (unsigned __int128)n) >> 64);
#endif
}

EB_HD uint32_t fmix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

struct FeistelKeys {
  uint32_t k[FEISTEL_ROUNDS];
};

EB_HD FeistelKeys feistel_keys(uint64_t seed, uint64_t step) {
  FeistelKeys fk;
EB_UNROLL
  for (int i = 0; i < FEISTEL_ROUNDS / 4; ++i) {
    u32x4 w = draw_words(seed, step, 0, TAG_SHUFFLE, (uint32_t)i);
    fk.k[4 * i + 0] = w.x;
    fk.k[4 * i + 1] = w.y;
    fk.k[4 * i + 2] = w.z;
    fk.k[4 * i + 3] = w.w;
  }
  return fk;
}

EB_HD int feistel_half_bits(uint64_t n) {
  int bits = 0;
  uint64_t v = n - 1;
  while (v) {
    ++bits;
    v >>= 1;
  }
  if (bits < 2) bits = 2;
  return (bits + 1) / 2;
}

// pi(w): balanced Feistel on 2*h bits, cycle-walked into [0,n)
EB_HD uint64_t split_permute(uint64_t w, uint64_t n, int h, const FeistelKeys& fk) {
  const uint64_t mask = ((uint64_t)1 << h) - 1;
  uint64_t x = w;
  do {
    uint64_t left = x >> h, right = x & mask;
EB_UNROLL
    for (int r = 0; r < FEISTEL_ROUNDS; ++r) {
      uint64_t f = (uint64_t)fmix32((uint32_t)right ^ fk.k[r]) & mask;
      uint64_t nl = right;
      right = left ^ f;
      left = nl;
    }
    x = (left << h) | right;
  } while (x >= n);
  return x;
}

// row m of the ordered-pair table of DEMove (de.py:67-77), decoded
// analytically: m < T -> (r, col) of the m-th strictly-lower-triangular entry
// in row-major order, else the same entry with the two swapped.
EB_HD void de_pair_decode(uint64_t m, uint64_t n, uint64_t& p0, uint64_t& p1) {
  const uint64_t T = n * (n - 1) / 2;
  const bool upper = m >= T;
  const uint64_t k = upper ? m - T : m;
  uint64_t r = (uint64_t)((1.0 + sqrt(1.0 + 8.0 * (double)k)) * 0.5);
  if (r * (r - 1) / 2 > k) --r;
  if ((r + 1) * r / 2 <= k) ++r;
  const uint64_t col = k - r * (r - 1) / 2;
  p0 = upper ? col : r;
  p1 = upper ? r : col;
}

}  // namespace eb
