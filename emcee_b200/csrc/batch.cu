// Batch contexts (eb_create_batch): the split tables and the half-step of K independent ensembles stacked as the rows
// of one engine, each drawing under its own Philox key.  Every ensemble gets the draws, partners, proposals and
// accept decisions the generic kernel (kernels.cu) gives a single ensemble of that key: the per-walker body below is
// half_step_generic_kernel's, built from the same decoders (draws.cuh) and row operations (rowops.cuh), with the
// ensemble's row offset and key in place of the engine's.
#include <math.h>

#include <algorithm>

#include "draws.cuh"
#include "engine.cuh"
#include "rowops.cuh"

namespace eb {

// ===========================================================================
// split tables: block (k, s) = ensemble k at step step0 + s
// ===========================================================================
// split_table_kernel's stable partition of the walkers by inds[w] = (randomize ? pi_step(w) : w) % P under seeds[k],
// with as many warps as the n walkers need (at most 32): a warp scans the per-warp counts of sets warp, warp + nwarps..
__global__ void __launch_bounds__(TABLE_THREADS) batch_split_table_kernel(int32_t* __restrict__ order_base,
                                                                          const StepInfo* __restrict__ info, int64_t n,
                                                                          int64_t K, const uint64_t* __restrict__ seeds,
                                                                          uint64_t step0) {
  __shared__ int base[MAX_SPLITS];
  __shared__ int chunk_tot[MAX_SPLITS];
  __shared__ int warp_off[MAX_SPLITS][32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int64_t k = blockIdx.x;
  const uint64_t step = step0 + blockIdx.y;
  const int P = info[blockIdx.y].nsplits;
  const bool randomize = info[blockIdx.y].randomize != 0;
  int32_t* order = order_base + ((size_t)blockIdx.y * (size_t)K + (size_t)k) * (size_t)n;

  if (tid < P) {
    int64_t s = 0;
    for (int j = 0; j < tid; ++j) s += (n - j + P - 1) / P;
    base[tid] = (int)s;
  }
  const FeistelKeys fk = feistel_keys(seeds[k], step);
  const int h = feistel_half_bits((uint64_t)n);
  __syncthreads();

  for (int64_t c0 = 0; c0 < n; c0 += blockDim.x) {
    const int64_t w = c0 + tid;
    const bool valid = w < n;
    int sid = -1;
    if (valid) sid = (int)((randomize ? split_permute((uint64_t)w, (uint64_t)n, h, fk) : (uint64_t)w) % (uint64_t)P);
    int my_prefix = 0;
    for (int j = 0; j < P; ++j) {
      const unsigned b = __ballot_sync(0xffffffffu, sid == j);
      if (sid == j) my_prefix = __popc(b & ((1u << lane) - 1u));
      if (lane == 0) warp_off[j][warp] = __popc(b);
    }
    __syncthreads();
    for (int j = warp; j < P; j += nwarps) {
      const int v = lane < nwarps ? warp_off[j][lane] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      warp_off[j][lane] = incl - v;
      if (lane == 31) chunk_tot[j] = incl;
    }
    __syncthreads();
    if (valid) order[base[sid] + warp_off[sid][warp] + my_prefix] = (int32_t)w;
    __syncthreads();
    if (tid < P) base[tid] += chunk_tot[tid];
    __syncthreads();
  }
}

cudaError_t launch_batch_split_tables(int32_t* order, const StepInfo* info_dev, int nsteps_chunk, int64_t n, int64_t K,
                                      const uint64_t* seeds, uint64_t step0, cudaStream_t st) {
  const int threads = (int)std::min<int64_t>(TABLE_THREADS, (n + 31) / 32 * 32);
  batch_split_table_kernel<<<dim3((unsigned)K, (unsigned)nsteps_chunk), threads, 0, st>>>(order, info_dev, n, K, seeds,
                                                                                          step0);
  return cudaGetLastError();
}

// ===========================================================================
// half-step: active rank t of the batch = rank i = t mod a_count of ensemble k = t / a_count
// ===========================================================================
template <int MOVE, int MODEL>
__global__ void __launch_bounds__(256) batch_half_step_kernel(const BatchArgs a, const int G, const ExternalBufs ext) {
  extern __shared__ double smem[];
  constexpr int NROWS = (MOVE == EB_MOVE_SNOOKER ? 4 : 1) + (MODEL == EB_MODEL_GAUSS_DENSE ? 1 : 0);
  constexpr bool PRE = MOVE == MOVE_PRECOMPUTED;  // the accept phase of a callback model
  const int D = a.D;
  const int groups = blockDim.x / G;
  const int gid = threadIdx.x / G, g = threadIdx.x % G;
  const int lane = threadIdx.x & 31;
  const unsigned mask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
  const int64_t t = (int64_t)blockIdx.x * groups + gid;  // row of the [K, a_count] staging blocks
  if (t >= a.K * a.a_count) return;  // whole groups leave together
  const int64_t k = t / a.a_count;
  const int64_t i = t - k * a.a_count;
  const int64_t row0 = k * a.n;  // ensemble k's first row
  const int32_t* order = a.order + row0;
  const uint64_t seed = a.seeds[k];

  double* q = smem + (size_t)gid * NROWS * D;
  double* xc = q + (size_t)(NROWS - 1) * D;  // centred row (dense model only)
  const int64_t w = row0 + order[a.a_start + i];
  const double* s_row = a.coords + (size_t)w * D;

  const u32x4 A = prop_a(seed, a.step, (uint32_t)a.split, (uint32_t)i);
  double factor = 0.0;

  if (MOVE == EB_MOVE_STRETCH) {
    const int64_t Nc = a.n - a.a_count;
    const double zz = stretch_zz(A, a.p0);
    const double* c_row = a.coords + (size_t)(row0 + order[complement_slot(stretch_rank(A, Nc), a.a_start, a.a_count)]) * D;
    for (int e = g; e < D; e += G) {
      const double v = stretch_q(s_row[e], c_row[e], zz);
      q[e] = v;
      if (!isfinite(v)) flag_nonfinite(v, a.status);
    }
    factor = stretch_factor((double)D - 1.0, zz);
  } else if (MOVE == EB_MOVE_DE) {
    const double gamma = de_gamma(prop_b(seed, a.step, (uint32_t)a.split, (uint32_t)i), a.p0, a.p1);
    int64_t r0, r1;
    de_pair(A, a.n - a.a_count, r0, r1);
    const int64_t w0 = row0 + order[complement_slot(r0, a.a_start, a.a_count)];
    const int64_t w1 = row0 + order[complement_slot(r1, a.a_start, a.a_count)];
    const double* c0 = a.coords + (size_t)w0 * D;
    const double* c1 = a.coords + (size_t)w1 * D;
    for (int e = g; e < D; e += G) {
      const double v = de_q(s_row[e], c0[e], c1[e], gamma);
      q[e] = v;
      if (!isfinite(v)) flag_nonfinite(v, a.status);
    }
  } else if (PRE) {
    const double* qrow = a.qbuf + (size_t)t * D;
    for (int e = g; e < D; e += G) {
      const double v = qrow[e];
      q[e] = v;
      if (!isfinite(v)) flag_nonfinite(v, a.status);
    }
    factor = ext.f[t];
  } else {  // EB_MOVE_SNOOKER
    const u32x4 B = prop_b(seed, a.step, (uint32_t)a.split, (uint32_t)i);
    int64_t pw[3];
    snooker_partners(A, B, a.c_start, a.c_count, [&](int64_t slot) -> int64_t { return row0 + order[slot]; }, pw);
    double* sS = q + (size_t)1 * D;  // rows: q | s | z | (z1 - z2 is streamed)
    double* sZ = q + (size_t)2 * D;
    double* sU = q + (size_t)3 * D;
    const double* z = a.coords + (size_t)pw[0] * D;
    const double* z1 = a.coords + (size_t)pw[1] * D;
    const double* z2 = a.coords + (size_t)pw[2] * D;
    double n2 = 0.0;
    for (int e = g; e < D; e += G) {
      const double s = s_row[e], zz_ = z[e];
      const double d = snooker_delta(s, zz_);
      sS[e] = s;
      sZ[e] = zz_;
      sU[e] = d;
      n2 = fma(d, d, n2);
    }
    const double norm = sqrt(group_sum(n2, G, mask));  // de_snooker.py:42
    double d1 = 0.0, d2 = 0.0;
    for (int e = g; e < D; e += G) {
      const double u = snooker_u(sU[e], norm);
      sU[e] = u;
      d1 = fma(u, z1[e], d1);
      d2 = fma(u, z2[e], d2);
    }
    d1 = group_sum(d1, G, mask);
    d2 = group_sum(d2, G, mask);
    const double dd = __dsub_rn(d1, d2);
    double m2 = 0.0;
    for (int e = g; e < D; e += G) {
      const double v = snooker_q(sS[e], sU[e], a.p0, dd);
      q[e] = v;
      if (!isfinite(v)) flag_nonfinite(v, a.status);
      const double dq = __dsub_rn(v, sZ[e]);
      m2 = fma(dq, dq, m2);
    }
    const double qn = sqrt(group_sum(m2, G, mask));
    factor = snooker_factor((double)D - 1.0, qn, norm);
  }
  __syncwarp(mask);

  if (MODEL == MODEL_EXTERNAL && !PRE) {
    // propose phase: the staged row and its factor go to row t of the [K, a_count] block the function receives
    double* dst = ext.q + (size_t)t * D;
    for (int e = g; e < D; e += G) dst[e] = q[e];
    if (g == 0) ext.f[t] = factor;
    return;
  }

  double lp_new;
  if (MODEL == MODEL_EXTERNAL) {
    lp_new = ext.lp[t];  // NaN was refused before this launch
  } else {
    lp_new = model_logprob<MODEL>(q, xc, D, g, G, mask, a.model);
    if (a.model.lo != nullptr && !row_in_box(q, D, g, G, mask, a.model)) lp_new = -INFINITY;
    if (isnan(lp_new) && g == 0) atomicOr(a.status, FLAG_NAN_LOGPROB);
  }

  const double u_acc = accept_uniform(seed, a.step, (uint32_t)a.split, (uint32_t)i);
  const bool acc = lnpdiff_red_blue(factor, lp_new, a.logp[w]) > log(u_acc);
  if (acc) {
    double* dst = a.coords + (size_t)w * D;
    for (int e = g; e < D; e += G) dst[e] = q[e];
  }
  if (g == 0) {
    if (acc) {
      a.logp[w] = lp_new;
      a.nacc[w] += 1ull;
    }
    a.accepted[w] = acc ? 1 : 0;
  }
}

template <int MOVE, int MODEL>
static cudaError_t launch_batch_t(const BatchArgs& a, const ExternalBufs& ext, cudaStream_t st) {
  const int G = lanes_per_walker(a.D);
  constexpr int NROWS = (MOVE == EB_MOVE_SNOOKER ? 4 : 1) + (MODEL == EB_MODEL_GAUSS_DENSE ? 1 : 0);
  int threads = 256;
  size_t smem = (size_t)(threads / G) * NROWS * a.D * sizeof(double);
  while (smem > 200 * 1024 && threads > G) {
    threads >>= 1;
    smem = (size_t)(threads / G) * NROWS * a.D * sizeof(double);
  }
  if (smem > 200 * 1024) return cudaErrorInvalidConfiguration;
  const int groups = threads / G;
  const int64_t count = a.K * a.a_count;
  if (count <= 0) return cudaSuccess;
  auto kern = batch_half_step_kernel<MOVE, MODEL>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<(unsigned)((count + groups - 1) / groups), threads, smem, st>>>(a, G, ext);
  return cudaGetLastError();
}

template <int MOVE>
static cudaError_t launch_batch_m(const BatchArgs& a, const ExternalBufs& ext, cudaStream_t st) {
  switch (a.model.kind) {
    case EB_MODEL_GAUSS_ISO:
      return launch_batch_t<MOVE, EB_MODEL_GAUSS_ISO>(a, ext, st);
    case EB_MODEL_GAUSS_DENSE:
      return launch_batch_t<MOVE, EB_MODEL_GAUSS_DENSE>(a, ext, st);
    case EB_MODEL_ROSENBROCK:
      return launch_batch_t<MOVE, EB_MODEL_ROSENBROCK>(a, ext, st);
    case EB_MODEL_RING:
      return launch_batch_t<MOVE, EB_MODEL_RING>(a, ext, st);
    case MODEL_EXTERNAL:
      return launch_batch_t<MOVE, MODEL_EXTERNAL>(a, ext, st);
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_batch_half_step(int move_kind, const BatchArgs& a, const ExternalBufs& ext, cudaStream_t st) {
  switch (move_kind) {
    case EB_MOVE_STRETCH:
      return launch_batch_m<EB_MOVE_STRETCH>(a, ext, st);
    case EB_MOVE_DE:
      return launch_batch_m<EB_MOVE_DE>(a, ext, st);
    case EB_MOVE_SNOOKER:
      return launch_batch_m<EB_MOVE_SNOOKER>(a, ext, st);
    case MOVE_PRECOMPUTED:
      if (a.model.kind == MODEL_EXTERNAL) return launch_batch_t<MOVE_PRECOMPUTED, MODEL_EXTERNAL>(a, ext, st);
  }
  return cudaErrorInvalidValue;
}

}  // namespace eb
