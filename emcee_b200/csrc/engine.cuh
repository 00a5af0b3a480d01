// Internal types shared by the kernels and the C ABI (not part of the boundary).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/emcee_b200.h"
#include "acf_grid.h"
#include "philox.cuh"

namespace eb {

constexpr int MAX_SPLITS = 32;      // split_table_kernel uses one warp per set
constexpr int TABLE_THREADS = 1024;
// dense_dmma timeline buffer shape: per tile record 0 tile id, 1..5 and 9 consumer stamps, 6..8, 10 and 11 producer
// stamps (dense_dmma.cu)
constexpr int TL_TILES = 8, TL_EVENTS = 12;

// device status flags (OR-ed by kernels, read back after every call)
enum : int {
  FLAG_NAN_LOGPROB = 1,
  FLAG_INF_PARAM = 2,
  FLAG_NAN_PARAM = 4,
  FLAG_COMM_TIMEOUT = 8,
  FLAG_WAIT_TIMEOUT = 16,  // a warp gave up on an in-kernel hand-off (shared-memory barrier) of its own CTA
  FLAG_NAN_INITIAL = 32,   // a NaN in an initial log_prob given in device memory (eb_set_state_from)
  FLAG_KDE_SINGULAR = 64,  // KDEMove: the complement covariance of a split has a zero pivot (kde.cu)
};

struct ModelDev {
  int kind;
  const double* params;  // device: gauss_dense mu[D], A[D*D]; else unused
  const double* chol;    // device: gauss_dense packed factor for the DMMA kernel (or null)
  double s0, s1;         // rosenbrock a,b ; ring R,sigma
  // device: the prior's support lo[D] <= x <= hi[D] (eb_model_set_bounds); null when unbounded.  Outside it the
  // log-probability is -inf; every kernel tests the box on a warp-uniform branch on lo != nullptr
  const double* lo;
  const double* hi;
};

// per-step split description handed to split_table_kernel
struct StepInfo {
  int32_t nsplits;
  int32_t randomize;
};

// everything one half-step (one split of one step) needs
struct HalfStepArgs {
  double* coords;            // [N, D] row-major, live state
  double* logp;              // [N]
  uint8_t* accepted;         // [N] accept mask of the current step
  unsigned long long* nacc;  // [N] accepted-proposal counters
  int* status;               // flags
  const int32_t* order;      // [N] walker ids grouped by set, ascending inside a set
  const double* const* peer_coords;  // P2P mode: [nranks] peer-mapped coords (or null)
  int64_t rows_per_rank;     // P2P mode: owner(w) = w / rows_per_rank
  // P2P mode, barrier fused into the kernel (dense_dmma): producers wait until every peer has
  // published p2p_wait before touching the state; the last CTA to finish publishes p2p_signal
  unsigned* const* p2p_peer_flags;  // [nranks] peer-mapped flag arrays (null: no fused barrier)
  const unsigned* p2p_my_flags;     // [nranks] this rank's flag array (written by the peers)
  unsigned* p2p_done;               // CTA-completion counter of this rank
  int p2p_rank, p2p_nranks;
  unsigned p2p_wait, p2p_signal;
  int dmma_stagger;  // dense_dmma: pairs 4..7 request their first tile only when pairs 0..3's rows have landed
  // dense_dmma, one half-step per launch on one GPU: the launch is the programmatic dependent of a launch that
  // ran only earlier splits of the same step, so its own rows and log-probs may be read before griddepcontrol.wait
  int dmma_early_own;
  int64_t N;
  int D;
  int split;
  int a_start, a_count;  // active set = order[a_start .. a_start + a_count)
  int i_lo, i_hi;        // active ranks processed by this GPU (an upper bound for grid sizing when `range` is set)
  const int2* range;     // multi-GPU: device-resident [i_lo, i_hi) of this rank for this (step, split), or null
  // multi-GPU (P2P, dense_dmma): per (step, split) the owned active ranks with LOCAL partners first -- tile t
  // takes active ranks aperm[a_start + i_lo + 8 t ..]; null: natural order.  Same layout as `order`.
  const int32_t* aperm;
  int c_start[3], c_count[3];  // snooker: the three complement sets (ascending j != split)
  uint64_t seed, step;
  double p0, p1;  // stretch: a | de: g0, sigma | snooker: gammas
  ModelDev model;
  // optional taps (null unless debugging is enabled)
  int64_t* tap_partners;  // [3, N]
  double* tap_scalar;     // [N]
  double* tap_u;          // [N]
  int64_t* tap_active;    // [N]
  long long* timeline;    // dense_dmma instrumentation: [SM][consumer][tile<=TL_TILES][TL_EVENTS] cycles, or null
  const double* qbuf;     // MOVE_PRECOMPUTED: proposals [a_count, D] written by a proposal kernel (moves_extra.cu)
};

// internal move kind of half_step_generic_kernel: the proposal of active rank i is row i of HalfStepArgs::qbuf and
// the Hastings factor is 0 (WalkMove walk.py:37, GaussianMove gaussian.py:104); order == nullptr: walker id = i
constexpr int MOVE_PRECOMPUTED = 100;

// internal model kind of half_step_generic_kernel: the log-probabilities come from outside the kernel (a host or
// CUDA-array callback, eb_model_set_callback).  A half-step runs as two launches around the callback:
//   propose  <STRETCH | DE | SNOOKER, MODEL_EXTERNAL>: the proposal code of the fused kernel, then row i of the
//            staged proposal -> ExternalBufs::q[i - i_lo] and its Hastings factor -> f[i - i_lo]; nothing else
//   accept   <MOVE_PRECOMPUTED, MODEL_EXTERNAL>: lp_new = lp[i - i_lo], factor = f[i - i_lo] (0 when f is null:
//            WalkMove / GaussianMove), then the accept draw and update of the fused kernel
constexpr int MODEL_EXTERNAL = 100;
struct ExternalBufs {
  double* q;         // propose: [a_count, D] proposals (the accept launch reads them back through HalfStepArgs::qbuf)
  double* f;         // [a_count] Hastings factors, or null
  const double* lp;  // accept: [a_count] log-probabilities of the proposals
};

// one half-step of every ensemble of a batch context (batch.cu): K ensembles of n walkers stacked as K n rows.  Set
// sizes depend on n and the split count only, so every ensemble has the same active set [a_start, a_start + a_count)
// of its own segment of the split table, and the half-step covers K a_count active ranks.
struct BatchArgs {
  double* coords;  // [K n, D]
  double* logp;    // [K n]
  uint8_t* accepted;
  unsigned long long* nacc;
  int* status;
  const int32_t* order;   // [K, n] this step's split tables: ensemble k's walker ids (0 .. n - 1) at k n
  const uint64_t* seeds;  // [K] the Philox key of each ensemble
  int64_t n;
  int64_t K;
  int D;
  int split;
  int a_start, a_count;
  int c_start[3], c_count[3];  // snooker: the three complement sets
  uint64_t step;
  double p0, p1;  // as HalfStepArgs
  ModelDev model;
  const double* qbuf;  // accept phase of MODEL_EXTERNAL: [K a_count, D] the proposals the propose phase staged
};

// ---- kernel launchers (implemented in the .cu files) ----------------------
// batch.cu: the split tables of nsteps_chunk steps of a batch, [nsteps_chunk, K, n]; block (k, s) runs
// split_table_kernel's permutation of ensemble k under seeds[k] at step step0 + s
cudaError_t launch_batch_split_tables(int32_t* order, const StepInfo* info_dev, int nsteps_chunk, int64_t n, int64_t K,
                                      const uint64_t* seeds, uint64_t step0, cudaStream_t st);
// batch.cu: half_step_generic_kernel's per-walker body for the K a_count active ranks of a batch half-step.  A
// registered model runs move_kind STRETCH / DE / SNOOKER fused; MODEL_EXTERNAL runs them as the propose phase (row
// k a_count + i of ext.q, ext.f) and MOVE_PRECOMPUTED as the accept phase (a.qbuf, ext.f, ext.lp)
cudaError_t launch_batch_half_step(int move_kind, const BatchArgs& a, const ExternalBufs& ext, cudaStream_t st);
// ranges (nullable): [nsteps_chunk, MAX_SPLITS] int2 = active ranks of each set owned by walkers [w_lo, w_hi)
cudaError_t launch_split_tables(int32_t* order, const StepInfo* info_dev, int nsteps_chunk, int64_t N,
                                uint64_t seed, uint64_t step0, int64_t w_lo, int64_t w_hi, int2* ranges,
                                cudaStream_t st);
// multi-GPU: for every (step, split) of the chunk, the active ranks [i_lo, i_hi) this rank owns with up to
// front_cap walkers whose stretch partner lives on this rank moved to the front (stable) -- tiles built from the
// front need no NVLink traffic and no peer barrier, so a half-step starts computing while the barrier and the
// first remote rows are still in flight
cudaError_t launch_locality_tables(const int32_t* order, const StepInfo* info_dev, const int2* ranges, int nsteps_chunk,
                                   int64_t N, uint64_t seed, uint64_t step0, int64_t rows_per_rank, int rank,
                                   int front_cap, int32_t* aperm, cudaStream_t st);
cudaError_t launch_half_step_generic(int move_kind, const HalfStepArgs& a, cudaStream_t st);
// the two launches of a half-step of a callback model (MODEL_EXTERNAL above): move_kind STRETCH / DE / SNOOKER
// runs the propose phase, MOVE_PRECOMPUTED the accept phase
cudaError_t launch_half_step_external(int move_kind, const HalfStepArgs& a, const ExternalBufs& ext, cudaStream_t st);
// blobs of a callback model (blobs.cu): for each active rank i in [i_lo, i_hi), walker w = order ? order[a_start + i]
// : i takes record i - i_lo of prop[rows, record_bytes] into live[w] when accepted[w] is set (packed records)
cudaError_t launch_blob_select(const int32_t* order, int a_start, int i_lo, int i_hi, const uint8_t* accepted,
                               const void* prop, void* live, size_t record_bytes, cudaStream_t st);
// user proposals (eb_move_set_proposal).  Accept launch of a half-step whose proposals a user function wrote: row i
// - i_lo of HalfStepArgs::qbuf, Hastings factor f[i - i_lo].  move_kind EB_MOVE_USER: a device model, red-blue
// order (f + lp_new) - lp_old (red_blue.py:99); EB_MOVE_USER_MH: a device model or MODEL_EXTERNAL (lp from ext.lp),
// mh.py:57 order (lp_new - lp_old) + f, uniform indexed by walker (order == nullptr)
cudaError_t launch_half_step_user(int move_kind, const HalfStepArgs& a, const ExternalBufs& ext, cudaStream_t st);
// user_moves.cu: out[r] = coords row of walker order[a_start + r] for r < a_count, then the other sets in set order
// (order[r - a_count] for the sets before, order[r] for the sets after): the rows s | c of red_blue.py:85-87
cudaError_t launch_split_gather(const double* coords, const int32_t* order, int64_t N, int D, int a_start, int a_count,
                                double* out, cudaStream_t st);
// status |= FLAG_NAN_LOGPROB if any of x[n] is NaN (logprob != 0), else the non-finite parameter flags of x[n]
cudaError_t launch_scan_nonfinite(const double* x, size_t n, int logprob, int* status, cudaStream_t st);
// cuda_arrays.cu: status |= flag if any of x[n] is NaN
cudaError_t launch_flag_nan(const double* x, size_t n, int flag, int* status, cudaStream_t st);
// graph_fn.cu, around a captured log-probability graph (eb_model_set_graphs).  The first error of a call is recorded
// once in *err as graph_err_word(flags, split, step); `tag` is graph_err_word(0, split, step) of the running half-step.
constexpr int GRAPH_RESULT_THREADS = 512;
constexpr unsigned GRAPH_NO_SPLIT = 0xff;  // the split field of an evaluation outside a step (initial state, compute)
inline unsigned long long graph_err_word(int flags, unsigned split, uint64_t step) {
  return (unsigned long long)(flags & 0xff) | ((unsigned long long)(split & 0xff) << 8) | ((unsigned long long)step << 16);
}
// x[r, :] (row stride x_stride_bytes) = src[min(r, rows - 1), :] for r < m, unless *status holds an error: then
// nothing is copied and the error is recorded
cudaError_t launch_graph_stage(const double* src, int64_t rows, int64_t m, int D, double* x, int64_t x_stride_bytes,
                               const int* status, unsigned long long* err, unsigned long long tag, cudaStream_t st);
// out[i] = lp[i] (stride lp_stride_bytes) for i < rows; a NaN raises and records FLAG_NAN_LOGPROB; after a NaN, or
// when *status held an error already, every out[i] is NaN
cudaError_t launch_graph_result(const double* lp, int64_t lp_stride_bytes, int64_t rows, double* out, int* status,
                                unsigned long long* err, unsigned long long tag, cudaStream_t st);
// graph_moves.cu, around a captured proposal graph (eb_move_set_proposal_graphs).  Strides are in doubles.
struct GraphMoveBufs {
  double* s;
  int64_t s_stride;
  double* c;  // null: an MHMove, whose s is every walker
  int64_t c_stride;
  double* draws;
  int64_t draws_stride;
  const double* q;
  int64_t q_stride;
  const double* f;
  int64_t f_stride;
};
// rows r < N of the live state into s (r < a_count) and c, walker order[a_start + r] / order[r - a_count] /
// order[r] as launch_split_gather (order null: walker r, a_count = N), and draws[i, 0 .. ndraws) for i < a_count from
// TAG_GRAPH blocks (index i, sub-index k) at (seed, step, split); unless *status holds an error: then nothing is
// written and the error is recorded in *err as `tag` | flags
cudaError_t launch_graph_move_stage(const double* coords, const int32_t* order, int64_t N, int D, int a_start,
                                    int a_count, const GraphMoveBufs& b, int normal, int64_t ndraws, uint64_t seed,
                                    uint64_t step, uint32_t split, const int* status, unsigned long long* err,
                                    unsigned long long tag, cudaStream_t st);
// qbuf[ns, D] = q, f[ns] = factors; a non-finite q raises FLAG_INF_PARAM / FLAG_NAN_PARAM (ensemble.py:476-479).
// After the launch's last block sees an error in *status (raised now or earlier) it records it and sets every f[i]
// to NaN.  `ticket` is a zeroed counter the launch leaves zeroed.
cudaError_t launch_graph_move_result(const GraphMoveBufs& b, int64_t ns, int D, double* qbuf, double* f, int* status,
                                     unsigned* ticket, unsigned long long* err, unsigned long long tag,
                                     cudaStream_t st);
// the cell of the tma_rows kernel a launch chose (eb_last_kernel_variant)
struct TmaVariant {
  int R;        // walkers per tile (G = 32 / R lanes per walker)
  int epl;      // 8: register path, 0: strided path
  int own_reg;  // stretch register path with the own row in registers
  int warps;    // warps per CTA
};
// TMA row-gather variant for the HBM-bound models (tma_rows.cu); *used == false: not applicable, use the generic one
// (long_rows: also take rows so long that only one walker per tile fits; own_reg: stretch rows of <= 512 bytes keep
// the own row in registers -- plain loads / stores -- and stage only the partner rows).  *variant (nullable) gets
// the cell when *used.
cudaError_t launch_half_step_tma(int move_kind, const HalfStepArgs& a, int sm_count, bool long_rows, bool own_reg,
                                 cudaStream_t st, bool* used, TmaVariant* variant = nullptr);
cudaError_t launch_logprob_generic(const ModelDev& m, const double* x, int64_t rows, int D, double* out,
                                   int* status, cudaStream_t st);
// specialised: stretch + dense Gaussian on FP64 tensor cores (DMMA).  Returns
// cudaErrorNotSupported when the shape is outside its envelope.
bool dense_dmma_supported(int D);
size_t dense_dmma_factor_doubles(int D);
void dense_dmma_pack_factor(const double* L, int D, double* packed);  // host
// log-probability of dense-Gaussian rows on the tensor pipe (same arithmetic as the half-step kernel)
cudaError_t launch_logprob_dense_dmma(const ModelDev& m, int D, const double* x, int64_t rows, double* out,
                                      int* status, int sm_count, cudaStream_t st);
// one half-step of a persistent dense_dmma launch
struct HalfDesc {
  uint64_t step;       // sampler step index (Philox counter)
  int32_t order_step;  // which split table of the chunk (also indexes `range`)
  int32_t split;
  int32_t a_start, a_count;
};
// runs `nhalf` consecutive half-steps in ONE cooperative launch (grid barrier between them);
// a.order / a.range point at the chunk's table bases; d0 == descs[0] travels by value.  max_count bounds the active ranks per
// half-step (grid sizing).  gbar is a monotonic global counter, gbar_base its value at launch.
// `pdl`: launch as a programmatic dependent of the previous kernel in the stream (nhalf == 1 only; the caller
// guarantees that kernel is a dense_dmma launch of the same run).
cudaError_t launch_dense_dmma(const HalfStepArgs& a, const HalfDesc& d0, const HalfDesc* descs_dev, int nhalf,
                              int max_count,
                              unsigned long long* gbar, unsigned long long gbar_base, int sm_count, bool pdl,
                              int* grid_out, cudaStream_t st);

// ---- proposal generators of WalkMove / GaussianMove (moves_extra.cu) ----------------------------
// acc = [S1 | S2] moment sums about a shift over n rows -> cov (np.cov) -> thresholded lower Cholesky factor L
cudaError_t launch_cov_chol(const double* acc, double n, int D, double* cov, double* L, cudaStream_t st);
cudaError_t launch_walk_shared_propose(const HalfStepArgs& a, const double* L, double* qbuf, cudaStream_t st);
bool walk_subset_supported(int D, int s0);
cudaError_t launch_walk_subset_propose(const HalfStepArgs& a, int s0, double* qbuf, cudaStream_t st);
cudaError_t launch_gaussian_shift(const double* L, int D, double f, uint64_t seed, uint64_t step, double* v,
                                  cudaStream_t st);
cudaError_t launch_gaussian_propose(const double* x0, int64_t row0, int64_t nrows, int D, int form, const double* scale,
                                    double f, int mode, int seq_dim, uint64_t seed, uint64_t step, double* qbuf,
                                    cudaStream_t st);

// ---- KDEMove (kde.cu) ---------------------------------------------------------------------------
// launch geometry of the log-density kernel: ptiles point tiles of 64 (2 ns points: the s rows, then the q rows) x
// nchunks chunks of tpc centre tiles of 64
struct KdePlan {
  int64_t ptiles;
  int tpc, nchunks;
};
KdePlan kde_plan(int64_t ns, int64_t nc, int sm_count);
// doubles of the partial (max, sum) buffer every plan of an N-walker engine fits in
size_t kde_partial_doubles(int64_t N, int sm_count);
// L of cov_chol over nc complement rows with moment sums acc about shift -> minv = (bw L)^-1, mean = the complement
// mean; a zero pivot of L sets FLAG_KDE_SINGULAR in status and writes nothing
cudaError_t launch_kde_factor(const double* L, const double* acc, const double* shift, double nc, int D, double bw,
                              double* minv, double* mean, int* status, cudaStream_t st);
// the proposals qbuf[ns, D], whitened points yp[2 ns, D] (s rows, then q rows), whitened complement yc[nc, D] and
// the walker id of each proposal's kernel centre jw[ns] of half-step a
cudaError_t launch_kde_prepare(const HalfStepArgs& a, const double* L, const double* minv, const double* mean,
                               double bw, double* qbuf, double* yp, double* yc, int64_t* jw, cudaStream_t st);
// f[ns] = LSE_c(-|y_s - y_c|^2 / 2) - LSE_c(-|y_q - y_c|^2 / 2); part: kde_partial_doubles scratch
cudaError_t launch_kde_factors(const double* yp, const double* yc, int64_t ns, int64_t nc, int D, const KdePlan& p,
                               double* part, double* f, cudaStream_t st);

// ---- chain analysis (analysis.cu) ------------------------------------------------------------
// column means of X[nrows, D] (fixed summation order); status (nullable) gets the non-finite flags
cudaError_t launch_colmean(const double* X, int64_t nrows, int D, double* mean, int* status, cudaStream_t st);
// acc[D + D*D] += [sum(x - shift), (x - shift)^T (x - shift)] over the rows of X (DMMA; D <= 1024);
// partial: scratch of moments_partial_bytes(D, sm_count)
size_t moments_partial_bytes(int D, int sm_count);
// rowidx (nullable): row r of the set is walker rowidx[r < skip_start ? r : r + skip_count]
cudaError_t launch_moments(const double* X, int64_t nrows, int D, const double* shift, double* partial, double* acc,
                           int sm_count, cudaStream_t st, const int32_t* rowidx = nullptr, int skip_start = 0,
                           int skip_count = 0);

// segmented moments of a stored slice (eb_chain_moments_segments): nseg segments of N walkers per stored step,
// slots a device table of count step bases; shift[nseg, D], acc[nseg, D + D*D] (sums about shift) and
// partial[nchunks, nseg, D + D*D] of scratch, nchunks = moments_seg_chunks(count, nseg, D)
uint64_t moments_seg_chunks(uint64_t count, int64_t nseg, int D);
cudaError_t launch_moments_segments(const double* const* slots, uint64_t count, int64_t nseg, int64_t N, int D,
                                    uint64_t nchunks, double* shift, double* partial, double* acc, cudaStream_t st);

// walker-averaged normalised autocorrelation function (autocorr.py:21-46,101-107), slab by slab (geometry:
// acf_grid.h)
cudaError_t launch_acf_twiddles(double2* tw, int M, cudaStream_t st);
// the slab is walkers [w0, w0 + wb) of a chain of segments of seg_w walkers; f[segment][nd][n_t]
cudaError_t launch_acf_slab(const double* xin, int n_t, int wb, int nd, int M, const double2* tw, double2* z,
                            double* mean, double* f, int64_t seg_w, int64_t w0, cudaStream_t st);
cudaError_t launch_acf_scale(double* f, size_t n, double scale, cudaStream_t st);

// ---- device chain storage (chain.cu) ----------------------------------------------------------
// one stored step: cx[nx] = x[nx], clp[nl] = lp[nl], accepted[N] += acc[N] and cmask[N] = acc[N] (acc, accepted
// and cmask nullable; nx = nl = 0: only the accept counts).  x, lp, cx, clp 16-byte aligned.
cudaError_t launch_chain_store(const double* x, const double* lp, const uint8_t* acc, double* cx, double* clp,
                               double* accepted, size_t nx, size_t nl, int64_t N, int sm_count, cudaStream_t st,
                               uint8_t* cmask = nullptr);
// sums[N] (device) = the per-walker sums of the accept masks mask[nslots, N], in slot order
cudaError_t launch_mask_sum(const uint8_t* mask, uint64_t nslots, int64_t N, double* sums, cudaStream_t st);

// ---- exact order statistics of a stored slice (select.cu, eb_chain_select) ----------------------------------
constexpr size_t SELECT_PAIR_BATCH = 16384;          // (parameter, rank) pairs planned at once
constexpr uint64_t SELECT_CAND_MAX = (uint64_t)1 << 23;  // compacted candidates held at once (64 MiB)
struct SelectScratch {
  size_t batch = 0;     // pairs per batch
  uint64_t budget = 0;  // candidate keys
  size_t bytes = 0;     // device scratch select_run needs
};
SelectScratch select_scratch(uint64_t count, int D, size_t npairs);
// slots[count] (host array of device pointers): each stored step's [nseg, N, D] block, nseg segments of N rows.
// out[nseg, nranks, D] and has_nan[nseg, D] on the host; *passes = full reads of the slice.  scratch: z.bytes of
// device memory, z = select_scratch(count, nseg * D, nseg * D * nranks).
cudaError_t select_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int D,
                       const uint64_t* ranks, size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes,
                       const SelectScratch& z, void* scratch, int sm_count, cudaStream_t st);

// ---- histograms of a stored slice (histogram.cu, eb_chain_histogram[2d]_segments) ---------------------------------
// A slot holds nseg segments (ensembles) of N / nseg rows of D values each; nseg = 1 is the whole slot.
// can count * (N / nseg) rows be split over grid y with fewer than 2^32 counted by one CTA?
bool hist_rows_fit(uint64_t n);
size_t hist1_scratch_bytes(uint64_t count, size_t ncol, int bins);
// slots[count] (host array of device pointers); outer[nseg * D, 3] = (first, last, span), edges[nseg * D, bins + 1]
// and hist[nseg * D, bins] on the host, column k * D + d; *bad: some value's bin index fell outside the edges
cudaError_t hist1_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int D, int bins,
                      const double* outer, const double* edges, uint64_t* hist, bool* bad, void* scratch, int sm_count,
                      cudaStream_t st);
// CTAs along grid x of the 2-D kernel: one copy of the pair tiles per segment
uint64_t hist2_grid_x(uint32_t nseg, int m, int bins);
size_t hist2_scratch_bytes(uint64_t count, uint32_t nseg, int m, int bins);
// params[m] distinct columns; edges[nseg, m, bins + 1] and hist[nseg, m (m - 1) / 2, bins, bins] on the host
cudaError_t hist2_run(const double* const* slots, uint64_t count, uint32_t nseg, uint32_t N, int D,
                      const uint32_t* params, int m, int bins, const double* edges, uint64_t* hist, void* scratch,
                      int sm_count, cudaStream_t st);

// ---- running histograms of the live state (histogram.cu, eb_histograms_config / eb_histograms) -------------------
struct HistTile;
// one configuration: device tables and persistent counts inside `mem` (live_hist_bytes of it), launch geometry
struct LiveHist {
  uint32_t N = 0;
  int D = 0, bins = 0, lp = 0;  // lp: row D of the 1-D tables counts the log-probabilities
  int m = 0, bins2 = 0;         // 2-D: m parameters (m >= 2), bins2 per axis
  void* mem = nullptr;
  const double** slots = nullptr;  // [coords, logp]
  double* outer = nullptr;         // [D + lp, 3]
  double* edges = nullptr;         // [D + lp, bins + 1]
  unsigned long long* hist = nullptr;  // [D + lp, bins]
  unsigned int* bad = nullptr;
  HistTile* tiles = nullptr;
  uint32_t ntiles = 0;
  uint32_t* params = nullptr;           // [m]
  double* edges2 = nullptr;             // [m, bins2 + 1]
  unsigned long long* hist2 = nullptr;  // [m (m - 1) / 2, bins2, bins2]
  int W1 = 1, Wlp = 1;
  size_t smem1 = 0, smemlp = 0, smem2 = 0;
  dim3 grid1, gridlp, grid2;
  uint64_t rows1 = 0, rowslp = 0, rows2 = 0;
};
size_t live_hist_bytes(int D, int bins, int lp, int m, int bins2);
// uploads the tables, zeroes the counts and synchronises; m < 2: no 2-D counts
cudaError_t live_hist_setup(LiveHist* h, void* mem, uint32_t N, int D, int bins, int lp, const double* outer,
                            const double* edges, const uint32_t* params, int m, int bins2, const double* edges2,
                            const double* coords, const double* logp, int sm_count, cudaStream_t st);
// adds the current state to the counts: kernels only, on `st` (launches += their number)
cudaError_t live_hist_launch(const LiveHist& h, cudaStream_t st, uint64_t& launches);
// hist[(D + lp) * bins], hist2 (nullable) to the host; *bad: some value fell past numpy's edge array
cudaError_t live_hist_read(const LiveHist& h, uint64_t* hist, uint64_t* hist2, bool* bad, cudaStream_t st);

// ---- running trace of the live state (trace.cu, eb_trace_config / eb_trace_read / eb_trace_best) -----------------
struct TraceBest {
  double log_prob;
  unsigned long long step, walker;
  unsigned long long have;  // 0 until a step has been recorded
};
// the fixed part of a trace inside `mem` (live_trace_fixed_bytes of it); the rows are the engine's to grow
struct LiveTrace {
  uint32_t N = 0;
  int D = 0;
  const double* coords = nullptr;
  const double* logp = nullptr;
  const uint8_t* accepted = nullptr;
  void* mem = nullptr;
  double* partial = nullptr;      // [trace_nchunks(N), 2 D + 4] chunk sums, folded in place
  TraceBest* best = nullptr;
  double* best_coords = nullptr;  // [D]
};
size_t live_trace_fixed_bytes(uint32_t N, int D);
// lays the pointers out, clears the best sample and synchronises
cudaError_t live_trace_setup(LiveTrace* t, void* mem, uint32_t N, int D, const double* coords, const double* logp,
                             const uint8_t* accepted, cudaStream_t st);
// row[2 D + 4] (device) = the statistics of the current state, recorded as `step`: two kernels on `st`
cudaError_t live_trace_launch(const LiveTrace& t, double* row, uint64_t step, cudaStream_t st, uint64_t& launches);
// the best sample so far to the host (coords nullable); synchronises
cudaError_t live_trace_best(const LiveTrace& t, TraceBest* best, double* coords, cudaStream_t st);

// ---- running autocorrelation function (running_acf.cu, eb_running_acf_config / eb_running_acf_read) -------------
// the sums of N D series over lags 0 .. max_lag inside one allocation of live_racf_bytes (running_acf.h)
struct LiveRacf {
  uint32_t N = 0;
  int D = 0;
  uint64_t max_lag = 0;
  const double* coords = nullptr;
  double* x0 = nullptr;       // [N D] first recorded value of every series
  double* ring = nullptr;     // [max_lag + RACF_B, N D] the last recorded values, shifted by x0
  double* head = nullptr;     // [max_lag, N D] the first recorded values, shifted
  double* s_hi = nullptr;     // [max_lag + 1, N D] lag sums of the folded blocks (double-double)
  double* s_lo = nullptr;
  double* y_hi = nullptr;     // [N D] sum of the folded blocks' values (double-double)
  double* y_lo = nullptr;
  double* partial = nullptr;  // [walker chunks, max_lag + 1, D] of a read
  double* rho = nullptr;      // [max_lag + 1, D] of a read
};
// bytes of the sums of an N x D ensemble up to max_lag (SIZE_MAX when a size_t cannot hold them)
size_t live_racf_bytes(uint32_t N, int D, uint64_t max_lag);
// lays the pointers out, zeroes the sums and synchronises
cudaError_t live_racf_setup(LiveRacf* r, void* mem, uint32_t N, int D, uint64_t max_lag, const double* coords,
                            cudaStream_t st);
// records the current state as recorded step n (0-based), and folds the block it completes: kernels only, on `st`
cudaError_t live_racf_record(const LiveRacf& r, uint64_t n, cudaStream_t st, uint64_t& launches);
// rho[min(n, max_lag + 1), D] (host) after n recorded steps; nothing the later reads use changes; synchronises
cudaError_t live_racf_read(const LiveRacf& r, uint64_t n, double* rho, cudaStream_t st);

// ---- running reservoir of recorded rows (reservoir.cu, eb_reservoir_config / eb_reservoir_read) ------------------
struct ResCtl;  // the device's live count, tau, full flag and radix-select state
// a reservoir of K rows inside `mem` (live_reservoir_bytes of it); cap = res_cap(K, N) entries (reservoir_plan.h)
struct LiveReservoir {
  uint32_t N = 0;
  int D = 0;
  uint64_t K = 0, cap = 0;
  int sm_count = 0;
  const double* coords = nullptr;
  const double* logp = nullptr;
  double* x = nullptr;                // [cap, D]
  double* lp = nullptr;               // [cap]
  unsigned long long* key = nullptr;  // [cap]
  unsigned long long* step = nullptr;  // [cap]
  uint32_t* walker = nullptr;         // [cap]
  uint32_t* group = nullptr;          // [cap] the boundary group of a compaction, or the order of a read
  uint32_t* holes = nullptr;          // [K] entries below K that a compaction drops
  uint32_t* movers = nullptr;         // [K] entries from K on that it keeps
  ResCtl* ctl = nullptr;
};
// bytes of a reservoir of K rows; cap must be below 2^32
size_t live_reservoir_bytes(uint64_t K, uint32_t N, int D);
// lays the pointers out, empties the reservoir and synchronises
cudaError_t live_reservoir_setup(LiveReservoir* r, void* mem, uint64_t K, uint32_t N, int D, const double* coords,
                                 const double* logp, int sm_count, cudaStream_t st);
// offers the current state's N rows, recorded as `step`: one kernel on `st`; the caller has made room for N entries
cudaError_t live_reservoir_record(const LiveReservoir& r, uint64_t seed, uint64_t step, cudaStream_t st,
                                  uint64_t& launches);
// keeps the K first of at most `bound` live entries: kernels only, on `st` (no-ops while no more than K are live)
cudaError_t live_reservoir_compact(const LiveReservoir& r, uint64_t bound, cudaStream_t st, uint64_t& launches);
// the `kept` entries of a compacted reservoir in the order (key, step, walker): coords[kept, D] and lp[kept] to the
// host, or (device_out) to device memory; step and walker to the host.  Any output may be null; synchronises
cudaError_t live_reservoir_read(const LiveReservoir& r, uint64_t kept, double* coords, double* lp, uint64_t* step,
                                int64_t* walker, bool device_out, cudaStream_t st);

inline int lanes_per_walker(int D) {
  int g = 4;
  while (g < 32 && g * 4 < D) g <<= 1;
  return g;
}

}  // namespace eb
