// Decoding of the per-walker draws (DESIGN.md §2, tags 3-6) and the proposal and Metropolis arithmetic built on
// them -- the CUDA statement for every device move, beside the numpy statement oracle/philox.py.  Every half-step
// and proposal kernel calls these, so the draw taps (which run the generic kernel) test the code the fast kernels
// run.  Each function keeps the rounding of the expression it states: __dadd_rn / __dmul_rn where numpy rounds
// each operation and an FMA contraction would change the result, plain operators and fma where the kernels use them.
#pragma once
#include <math.h>

#include "philox.cuh"

namespace eb {

// index into order[] of complement rank r: the complement is order[0, a_start) followed by
// order[a_start + a_count, N) (red_blue.py:85-87).  The bounds are taken by reference: the lookup reads them from
// the caller's argument block itself, which leaves the callers' generated code as it is with the expression inline.
__device__ __forceinline__ int64_t complement_slot(int64_t r, const int& a_start, const int& a_count) {
  return r < a_start ? r : r + a_count;
}

// split field of a draw with a sub-index k (oracle/philox.py sub_split)
__device__ __forceinline__ uint32_t sub_split(uint32_t split, uint32_t k) { return (split & 0x3Fu) | (k << 6); }

// the two proposal blocks of active rank i (tags 3 and 4); the decoders below take their words, so a kernel
// places each Philox block where it wants it in its own instruction stream
__device__ __forceinline__ u32x4 prop_a(uint64_t seed, uint64_t step, uint32_t split, uint32_t i) {
  return draw_words(seed, step, split, TAG_PROP_A, i);
}
__device__ __forceinline__ u32x4 prop_b(uint64_t seed, uint64_t step, uint32_t split, uint32_t i) {
  return draw_words(seed, step, split, TAG_PROP_B, i);
}

// ---- StretchMove --------------------------------------------------------------------------------------------
// stretch.py:30  zz = ((a - 1) * u + 1) ** 2 / a (each op rounded once)
__device__ __forceinline__ double stretch_zz(const u32x4& A, double a) {
  const double t = __dadd_rn(__dmul_rn(__dsub_rn(a, 1.0), u53(A.x, A.y)), 1.0);
  return __ddiv_rn(__dmul_rn(t, t), a);
}

// stretch.py:32  rint: the complement rank of the partner
__device__ __forceinline__ int64_t stretch_rank(const u32x4& A, int64_t Nc) {
  return (int64_t)bounded64(A.z, A.w, (uint64_t)Nc);
}

// stretch.py:31  factor = (ndim - 1) * log(zz), given dm1 = ndim - 1.0
__device__ __forceinline__ double stretch_factor(double dm1, double zz) { return __dmul_rn(dm1, log(zz)); }

// stretch.py:33  q = c - (c - s) * zz (each op rounded once)
__device__ __forceinline__ double stretch_q(double s, double c, double zz) {
  return __dsub_rn(c, __dmul_rn(__dsub_rn(c, s), zz));
}

// ---- DEMove -------------------------------------------------------------------------------------------------
// de.py:49  pair index m of the Nc (Nc - 1) ordered pairs, :67-77 decoded: the complement ranks of c[p0], c[p1]
__device__ __forceinline__ void de_pair(const u32x4& A, int64_t Nc, int64_t& r0, int64_t& r1) {
  uint64_t p0, p1;
  de_pair_decode(bounded64(A.x, A.y, (uint64_t)Nc * (uint64_t)(Nc - 1)), (uint64_t)Nc, p0, p1);
  r0 = (int64_t)p0;
  r1 = (int64_t)p1;
}

// de.py:56  gamma = g0 * (1 + sigma * normal), the normal by Box-Muller from block B
__device__ __forceinline__ double de_gamma(const u32x4& B, double g0, double sigma) {
  const double n = sqrt(-2.0 * log(1.0 - u53(B.x, B.y))) * cos(6.283185307179586 * u53(B.z, B.w));
  return __dmul_rn(g0, __dadd_rn(1.0, __dmul_rn(sigma, n)));
}

// de.py:53,62  q = s + gamma * (c[p1] - c[p0])
__device__ __forceinline__ double de_q(double s, double c0, double c1, double gamma) {
  return __dadd_rn(s, __dmul_rn(gamma, __dsub_rn(c1, c0)));
}

// ---- DESnookerMove ------------------------------------------------------------------------------------------
// de_snooker.py:38  one pick from each of the three other sets (c_start, c_count: their slots in order[]), :39  the
// shuffle of the three rows, one of 6 orders.  id(slot) loads a walker id in the caller's flavour; the ids come back
// as z, z1, z2.
template <class Id, class Load>
__device__ __forceinline__ void snooker_partners(const u32x4& A, const u32x4& B, const int (&c_start)[3],
                                                 const int (&c_count)[3], Load id, Id (&pw)[3]) {
  const Id c0 = id(c_start[0] + (int64_t)bounded64(A.x, A.y, (uint64_t)c_count[0]));
  const Id c1 = id(c_start[1] + (int64_t)bounded64(A.z, A.w, (uint64_t)c_count[1]));
  const Id c2 = id(c_start[2] + (int64_t)bounded64(B.x, B.y, (uint64_t)c_count[2]));
  const int p = (int)bounded64(B.z, B.w, 6);
  const int i0 = p >> 1;                        // 0,0,1,1,2,2
  const int rest0 = (i0 == 0) ? 1 : 0;          // smaller of the remaining two
  const int rest1 = (i0 == 2) ? 1 : 2;          // larger of the remaining two
  const int i1 = (p & 1) ? rest1 : rest0;
  const int i2 = (p & 1) ? rest0 : rest1;
  pw[0] = i0 == 0 ? c0 : (i0 == 1 ? c1 : c2);
  pw[1] = i1 == 0 ? c0 : (i1 == 1 ? c1 : c2);
  pw[2] = i2 == 0 ? c0 : (i2 == 1 ? c1 : c2);
}

// de_snooker.py:41  delta = s - z
__device__ __forceinline__ double snooker_delta(double s, double z) { return __dsub_rn(s, z); }

// de_snooker.py:43  u = delta / norm
__device__ __forceinline__ double snooker_u(double delta, double norm) { return __ddiv_rn(delta, norm); }

// de_snooker.py:44  q = s + u * gammas * (u.z1 - u.z2), with dd = u.z1 - u.z2
__device__ __forceinline__ double snooker_q(double s, double u, double gammas, double dd) {
  return __dadd_rn(s, __dmul_rn(__dmul_rn(u, gammas), dd));
}

// de_snooker.py:45-46  factor = (ndim - 1) * (log(|q - z|) - log(|s - z|)), given dm1 = ndim - 1.0
__device__ __forceinline__ double snooker_factor(double dm1, double qn, double norm) {
  return __dmul_rn(dm1, __dsub_rn(log(qn), log(norm)));
}

// ---- KDEMove, GaussianMove ----------------------------------------------------------------------------------
// kde.py:41 (gaussian_kde.resample): choice(nc, p=uniform) -> complement rank of the kernel centre of proposal i
__device__ __forceinline__ int64_t kde_centre_rank(const u32x4& A, int64_t nc) {
  return (int64_t)bounded64(A.x, A.y, (uint64_t)nc);
}

// gaussian.py:100  mode "random": the one dimension walker w moves (block B of index w, split 0)
__device__ __forceinline__ int gaussian_random_dim(const u32x4& B, int D) {
  return (int)bounded64(B.x, B.y, (uint64_t)D);
}

// ---- normals and the Metropolis test ------------------------------------------------------------------------
// the pair of standard normals (2k, 2k+1) of row `index` (walk.py:36, gaussian.py:97,116, kde.py:41): Box-Muller
__device__ __forceinline__ void normal_pair(uint64_t seed, uint64_t step, uint32_t split, uint32_t k, uint32_t index,
                                            double& n0, double& n1) {
  box_muller_pair(draw_words(seed, step, sub_split(split, k), TAG_NORMAL, index), n0, n1);
}

// red_blue.py:100, mh.py:58  the accept uniform of active rank (or MHMove walker) i
__device__ __forceinline__ double accept_uniform(uint64_t seed, uint64_t step, uint32_t split, uint32_t i) {
  const u32x4 U = draw_words(seed, step, split, TAG_ACCEPT, i);
  return u53(U.x, U.y);
}

// red_blue.py:99  lnpdiff = f + lp_new - lp_old, left to right
__device__ __forceinline__ double lnpdiff_red_blue(double f, double lp_new, double lp_old) {
  return __dsub_rn(__dadd_rn(f, lp_new), lp_old);
}

// mh.py:57  lnpdiff = lp_new - lp_old + f: a user MHMove's order, which rounds differently once f != 0
__device__ __forceinline__ double lnpdiff_mh(double f, double lp_new, double lp_old) {
  return __dadd_rn(__dsub_rn(lp_new, lp_old), f);
}

}  // namespace eb
