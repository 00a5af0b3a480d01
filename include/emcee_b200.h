/*
 * emcee_b200.h -- C ABI of the H100-native ensemble-MCMC walker-update engine.
 *
 * This is the drop-in boundary for the hot path of dfm/emcee (reference @ 8ab6c0f,
 * pure Python, no FFI of its own).  Each entry point below names the reference
 * interface it replaces (file:line relative to the reference root).  The Python
 * host side (emcee_b200/ensemble.py, moves/, state.py) binds these with ctypes
 * and mirrors EnsembleSampler / moves.Move / State; INTEGRATION.md shows the
 * stub a reference maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes; host buffers are caller-owned, C-contiguous
 *     float64 (numpy); device memory is owned by the library.
 *   - every call returns 0 (EB_OK) or a negative eb_status; eb_last_error()
 *     gives the message.  Nothing throws across the boundary.
 *   - one host thread per context; calls are synchronous at return.
 *   - there is no CPU fallback: without a CUDA device eb_create fails.
 */
#ifndef EMCEE_B200_H
#define EMCEE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EB_ABI_VERSION 2

typedef enum eb_status {
  EB_OK = 0,
  EB_ERR_INVALID = -1,      /* bad argument / shape            -> ValueError  */
  EB_ERR_CUDA = -2,         /* CUDA runtime failure            -> RuntimeError */
  EB_ERR_COMM = -3,         /* NCCL / peer-memory failure      -> RuntimeError */
  EB_ERR_STATE = -4,        /* call order (no model, no state) -> RuntimeError */
  EB_ERR_UNSUPPORTED = -5,  /*                                 -> NotImplementedError */
  EB_ERR_NOMEM = -6,        /* device allocation failed or would not fit -> MemoryError */
  EB_ERR_CALLBACK = -7,     /* the log-probability callback failed -> re-raise the caller's exception */
  /* device-detected conditions the reference raises as exceptions */
  EB_ERR_NAN_LOGPROB = -10, /* ensemble.py:550-551 "Probability function returned NaN" */
  EB_ERR_INF_PARAM = -11,   /* ensemble.py:476-477 "At least one parameter value was infinite" */
  EB_ERR_NAN_PARAM = -12,   /* ensemble.py:478-479 "At least one parameter value was NaN" */
  EB_ERR_FEW_WALKERS = -13, /* moves/red_blue.py:64-70 RuntimeError (nwalkers < 2*ndim) */
  EB_ERR_NAN_INITIAL = -14, /* ensemble.py:357-358 "The initial log_prob was NaN" */
  EB_ERR_SINGULAR = -15     /* EB_MOVE_KDE: a complement covariance is singular (gaussian_kde's LinAlgError) */
} eb_status;

/* registered device-side log-probability models (replace the Python callable
 * log_prob_fn of ensemble.py:79-83 / _FunctionWrapper ensemble.py:626-650) */
typedef enum eb_model_kind {
  EB_MODEL_GAUSS_ISO = 0,   /* -0.5*sum(x^2); params: none                                    */
  EB_MODEL_GAUSS_DENSE = 1, /* -0.5*(x-mu)^T A (x-mu); params: mu[D] then A[D*D] row-major    */
  EB_MODEL_ROSENBROCK = 2,  /* -sum b(x[i+1]-x[i]^2)^2+(a-x[i])^2; params: a, b               */
  EB_MODEL_RING = 3         /* -(|x|-R)^2/(2 s^2); params: R, s                               */
} eb_model_kind;

/* red-blue moves (moves/stretch.py, moves/de.py, moves/de_snooker.py) */
typedef enum eb_move_kind {
  EB_MOVE_STRETCH = 0, /* p0 = a        (stretch.py:22)                         */
  EB_MOVE_DE = 1,      /* p0 = sigma, p1 = gamma0 or NaN for 2.38/sqrt(2 ndim) (de.py:28,33-38) */
  EB_MOVE_SNOOKER = 2, /* p0 = gammas   (de_snooker.py:26); nsplits must be 4 (:28) */
  EB_MOVE_WALK = 3,    /* p0 = s, the number of helper walkers, or NaN for the whole complement (walk.py:24,32) */
  EB_MOVE_GAUSSIAN = 4 /* MHMove with a Gaussian proposal (mh.py:35-65, gaussian.py:32-119): `mode`, p1 = factor
                          or NaN, `cov`/`ncov` = the cov argument (1 scalar, ndim vector, ndim*ndim matrix);
                          not a red-blue move: nsplits / randomize_split are ignored */
} eb_move_kind;

/* user-written proposals (eb_move_set_proposal below); not members of eb_move_kind so that the enum keeps its
 * ABI 2 range */
#define EB_MOVE_USER 5    /* red-blue move with a user proposal (red_blue.py:47,90); p0 = proposal slot;
                             mode = EB_USER_SETUP: call the function once per step with the whole ensemble first */
#define EB_MOVE_USER_MH 6 /* MHMove with a user proposal_function (mh.py:31-33,52); p0 = proposal slot;
                             nsplits / randomize_split are ignored */
#define EB_USER_SETUP 1

/* KDEMove (moves/kde.py: scipy.stats.gaussian_kde of the complement, resample + logpdf ratio); not a member of
 * eb_move_kind for the same reason.  p0 = the bandwidth rule: NaN Scott (n ** (-1 / (d + 4))), EB_KDE_SILVERMAN
 * ((n (d + 2) / 4) ** (-1 / (d + 4))), EB_KDE_SCALAR: p1 is the bandwidth (finite, > 0); n = the complement size.
 * A split whose complement has fewer rows than ndim is refused before any update (EB_ERR_INVALID, scipy's
 * message); a singular complement covariance (a Cholesky pivot <= 1e-12 max(diag)) stops the call at that
 * half-step with EB_ERR_SINGULAR, earlier splits applied.  ndim <= 1024; sharded engines: EB_ERR_UNSUPPORTED. */
#define EB_MOVE_KDE 7
#define EB_KDE_SILVERMAN 1.0
#define EB_KDE_SCALAR 2.0

typedef enum eb_gaussian_mode { /* gaussian.py:63,99-104 */
  EB_GAUSS_VECTOR = 0, EB_GAUSS_RANDOM = 1, EB_GAUSS_SEQUENTIAL = 2
} eb_gaussian_mode;

/* one entry of the move schedule (ensemble.py:115-129) with the RedBlueMove
 * constructor arguments (moves/red_blue.py:37-42) */
typedef struct eb_move {
  int32_t kind;             /* eb_move_kind */
  int32_t nsplits;          /* red_blue.py:40 */
  int32_t randomize_split;  /* red_blue.py:42 */
  int32_t live_dangerously; /* red_blue.py:41 */
  double weight;            /* un-normalised; normalised as ensemble.py:128-129 */
  double p0;
  double p1;
  /* ABI 2: GaussianMove only (zero / NULL otherwise) */
  int32_t mode;             /* eb_gaussian_mode */
  int32_t reserved;
  int64_t seq_index;        /* mode "sequential": the proposal's `index` (gaussian.py:64) when the call starts */
  const double* cov;        /* host pointer, read during the call */
  uint64_t ncov;
} eb_move;

typedef struct eb_ctx eb_ctx;

/* ---- lifetime ---------------------------------------------------------- */
int eb_abi_version(void);
/* number of visible CUDA devices (0 when the driver is absent). */
int eb_device_count(void);
/* replaces EnsembleSampler.__init__'s state set-up (ensemble.py:131-167): an
 * engine for an [nwalkers, ndim] float64 ensemble on CUDA device `device`, its
 * Philox key = seed, step counter = 0. */
int eb_create(int device, int64_t nwalkers, int64_t ndim, uint64_t seed, eb_ctx** out);
/* a batch context: nbatch independent [nwalkers, ndim] ensembles stacked as the nbatch * nwalkers rows of one
 * engine, ensemble k in rows [k nwalkers, (k + 1) nwalkers), with Philox key seeds[k] (host, read during the call)
 * and one step counter.  Ensemble k of a batch advances exactly as an eb_create engine of key seeds[k] running the
 * generic kernel.  Every call that takes or returns rows (eb_set_state, eb_get_state, eb_compute_log_prob,
 * eb_step, eb_step_store, eb_get_naccepted, ...) sees the nbatch * nwalkers rows; a callback model is called once
 * per half-step with the [nbatch, m] block of all ensembles' proposals, ensemble-major (m = the split's size).
 * The schedule is one EB_MOVE_STRETCH / EB_MOVE_DE / EB_MOVE_SNOOKER entry (EB_ERR_UNSUPPORTED otherwise).  Calls
 * without a meaning for a batch return EB_ERR_UNSUPPORTED: device chains, running statistics, options and debug
 * taps, user proposals, graphs, blobs, CUDA-array state and results, eb_set_rng and communicators.
 * EB_ERR_INVALID for nbatch * nwalkers >= 2^31; EB_ERR_NOMEM when the rows do not fit in free device memory. */
int eb_create_batch(int device, int64_t nbatch, int64_t nwalkers, int64_t ndim, const uint64_t* seeds, eb_ctx** out);
/* the Philox keys seeds[nbatch] and the step counter of a batch context (either output may be NULL); setting them
 * resumes the batch there.  EB_ERR_UNSUPPORTED on a single-ensemble context. */
int eb_batch_rng_get(const eb_ctx* ctx, uint64_t* seeds, uint64_t* step);
int eb_batch_rng_set(eb_ctx* ctx, const uint64_t* seeds, uint64_t step);
int eb_destroy(eb_ctx* ctx);
/* message of the last failing call on ctx (ctx == NULL: last eb_create failure
 * of this thread).  Pointer valid until the next call on the same ctx. */
const char* eb_last_error(const eb_ctx* ctx);

/* ---- model ------------------------------------------------------------- */
/* replaces passing log_prob_fn/args/kwargs (ensemble.py:79-98,169-171). */
int eb_model_set(eb_ctx* ctx, int kind, const double* params, size_t nparams);
/* the prior's support, a closed box: lower[ndim], upper[ndim] (host, read during
 * the call).  The log-probability of x becomes the model's value when
 * lower[k] <= x[k] <= upper[k] for every k and exactly -inf otherwise, on every
 * kernel (the `if not in box: return -np.inf` of a log_prior).  -inf / +inf
 * bounds give one-sided boxes; NaN bounds and lower[k] >= upper[k] are refused
 * (EB_ERR_INVALID).  NULL, NULL clears the box.  Needs a model (EB_ERR_STATE);
 * eb_model_set clears the box.  A callback model has no box (EB_ERR_UNSUPPORTED). */
int eb_model_set_bounds(eb_ctx* ctx, const double* lower, const double* upper);

/* a user log-probability function, called once per half-step on the [m, ndim]
 * block of proposals of one split (red_blue.py:90-93 -> ensemble.py:458-553):
 * rows in ascending walker order, m = the split's size (nwalkers for
 * GaussianMove and for the initial state).  It writes lp[m] and returns 0, or
 * returns non-zero to stop the calling ABI function with EB_ERR_CALLBACK. */
#define EB_CALLBACK_HOST 0   /* x, lp are host pointers (pinned staging owned by the engine), stream = NULL */
#define EB_CALLBACK_DEVICE 1 /* x, lp are device pointers, x complete when fn is called; stream = the engine's
                                cudaStream_t (idle during the call) */
/* In both modes x is the engine's copy of the proposals: the function may overwrite it, the update reads the
 * proposals from elsewhere.  x and lp are valid only during the call. */
typedef int (*eb_logprob_fn)(void* user, const double* x, int64_t m, int64_t ndim, double* lp, void* stream);
/* replaces the model, like eb_model_set, by fn (`user` is passed back unchanged;
 * both must stay valid while the model is set).  Each half-step then runs:
 *   1. the proposal kernel(s) of the move;  2. a stream synchronisation;
 *   3. a non-finite proposal stops the call with EB_ERR_INF_PARAM / EB_ERR_NAN_PARAM
 *      before fn sees it (ensemble.py:476-479);
 *   4. host mode: the proposals are copied to the host;  5. fn;
 *   6. host mode: lp is copied back;
 *   7. a NaN in lp stops the call with EB_ERR_NAN_LOGPROB before the update
 *      (ensemble.py:550-551);
 *   8. the accept + update kernel (red_blue.py:96-104).
 * eb_set_state(coords, NULL) and eb_compute_log_prob call fn too, with the same
 * guards.  When a call stops inside a step, the step counter is that step, the
 * splits of it that ran before stay applied, and every completed step is fully
 * stored.  Inside fn, every other call on the same context returns EB_ERR_STATE
 * ("engine is inside a log-probability callback").  Sharded engines
 * (eb_comm_init) are refused with EB_ERR_UNSUPPORTED, both ways round. */
int eb_model_set_callback(eb_ctx* ctx, eb_logprob_fn fn, void* user, int where);
/* EB_CALLBACK_DEVICE, from inside fn: copy m float64 values, stride_bytes apart
 * (> 0, a multiple of 8), from src (device or host memory) into fn's lp, ordered
 * after the work on src_stream (CUDA Array Interface v3 encoding: 0 = none,
 * 1 = legacy default stream, 2 = per-thread default stream, else a
 * cudaStream_t), or after all work on the device for EB_STREAM_UNKNOWN (a
 * producer that names no stream, such as an interface v2 object).  The copy
 * has completed when the call returns. */
#define EB_STREAM_UNKNOWN UINT64_MAX
int eb_callback_result(eb_ctx* ctx, double* lp, const void* src, int64_t stride_bytes, int64_t m, uint64_t src_stream);
/* Blobs (ensemble.py:498-547 splits them off the function's results; moves/move.py:36-43 carries them with each
 * accepted walker; backends/backend.py:157-231 stores them).  From inside fn, either mode, at most once per call:
 * m (= fn's m) records of record_bytes bytes, stride_bytes apart (>= record_bytes), from src (host or device
 * memory), ordered on src_stream as eb_callback_result orders its copy.  The engine keeps fixed-width records
 * packed, one per walker; what they hold is the caller's business.
 *   - inside eb_set_state(coords, NULL): the records become the state's blobs and fix the live layout
 *     (record_bytes); a function that delivers none leaves the state without blobs;
 *   - inside a step: record_bytes must equal the live layout (EB_ERR_INVALID otherwise, before any update); each
 *     walker that accepts its proposal takes the proposal's record, on the device, behind the accept launch;
 *     a state without blobs (eb_set_state given log_prob, no eb_set_state_blobs) refuses them with the message of
 *     moves/move.py:38-42, and a state with blobs refuses a call that delivers none;
 *   - inside eb_compute_log_prob_blobs: record_bytes must equal the live layout if there is one.
 * Host mode copies the records to pinned staging here; they reach the device beside lp (step 6), without a
 * synchronisation of their own.  Device mode copies them before returning. */
int eb_callback_blobs(eb_ctx* ctx, const void* src, int64_t record_bytes, int64_t stride_bytes, int64_t m,
                      uint64_t src_stream);

/* A user log-probability function captured as CUDA graphs, one per row count m: the graph reads m rows from its
 * static input x[m, ndim] (float64, rows contiguous, x_row_stride_bytes apart) and writes m values to its static
 * output lp[m] (lp_stride_bytes apart).  exec is a cudaGraphExec_t instantiated on the engine's device. */
#define EB_CALLBACK_GRAPH 2
typedef struct {
  int64_t m;
  uint64_t exec;
  void* x;
  int64_t x_row_stride_bytes;
  void* lp;
  int64_t lp_stride_bytes;
} eb_graph;
/* replaces the model, like eb_model_set_callback, by n captured graphs (callback mode EB_CALLBACK_GRAPH).  Every
 * log-probability is then evaluated on the engine's stream without the host: a half-step of m rows enqueues the
 * non-finite scan of the rows when the move's kernels do not raise it themselves, a copy of the rows into the x of
 * the graph for m, cudaGraphLaunch, and a copy of its lp into the engine with the NaN scan.  The initial state and
 * eb_compute_log_prob run the graph for nwalkers rows in chunks, the last chunk padded with copies of its last row.
 * Errors (EB_ERR_INF_PARAM, EB_ERR_NAN_PARAM, EB_ERR_NAN_LOGPROB) are found on the device: from the first one on,
 * nothing is copied into x and every proposal is rejected.  The host reads them where a stepping call synchronises
 * anyway (the start of each chunk of steps, KDEMove's per-half-step check, user proposals), before each stored step
 * and each step a running statistic records, and at the end of the call; it then reports the first error, with the
 * step counter, the stored steps and the statistics where eb_model_set_callback leaves them.  Refused
 * (EB_ERR_INVALID): no graph for m = nwalkers, m outside [1, nwalkers], a repeated m, exec = 0, null buffers, strides
 * that are not positive multiples of 8 (x: at least a row), and buffers that are not device memory of the engine's
 * device.  Sharded engines are refused with EB_ERR_UNSUPPORTED.  The engine does not own the graphs or the
 * buffers: they must stay valid, and unused by anything else, while the model is set.  eb_model_set and
 * eb_model_set_callback clear the set. */
int eb_model_set_graphs(eb_ctx* ctx, const eb_graph* graphs, size_t n);

/* ---- user proposals (moves/red_blue.py:47,82-93; moves/mh.py:31-33,52) ------------------------------------ */
/* A user proposal, called once per half-step of a schedule entry of kind EB_MOVE_USER / EB_MOVE_USER_MH:
 *   EB_MOVE_USER (RedBlueMove.get_proposal(s, c, random), red_blue.py:85-90): split = the active set; s[ns, ndim]
 *     is that set's walkers in ascending walker order; c holds the nsets = nsplits - 1 other sets back to back, in
 *     set order, each in ascending walker order, c_counts[nsets] their sizes (red_blue.py:85-87);
 *   EB_MOVE_USER_MH (proposal_function(coords, random), mh.py:52): split = 0, s = the whole ensemble in walker
 *     order (ns = nwalkers), c = c_counts = NULL, nsets = 0;
 *   setup call (EB_MOVE_USER with mode = EB_USER_SETUP; RedBlueMove.setup(coords), red_blue.py:73): once per step
 *     before its splits, split = -1, s = the whole ensemble in walker order, c = c_counts = q = factors = NULL.
 * The function writes q[ns, ndim] and factors[ns] (the log Hastings ratios) and returns 0, or returns non-zero to
 * stop the calling ABI function with EB_ERR_CALLBACK.  `step` is the sampler step, so (seed, step, split) names the
 * call for a generator of the caller's own (DESIGN.md "Draw specification", purpose 8).  Host mode (`where` =
 * EB_CALLBACK_HOST): every pointer is pinned host staging owned by the engine, stream = NULL.  Device mode: s and
 * c are device scratch, complete when fn is called; q and factors are the engine's device buffers, which fn fills
 * with eb_proposal_result (or with work of its own on `stream`, the engine's cudaStream_t).  All pointers are valid
 * only during the call. */
typedef int (*eb_proposal_fn)(void* user, uint64_t step, int32_t split, const double* s, int64_t ns,
                              const double* c, const int64_t* c_counts, int32_t nsets, int64_t ndim, double* q,
                              double* factors, void* stream);
#define EB_MAX_PROPOSAL_SLOTS 64
/* register fn as proposal slot `slot` (0 <= slot < EB_MAX_PROPOSAL_SLOTS); fn == NULL clears it.  `user` is passed back unchanged;
 * both must stay valid while the slot is set.  A half-step of a user move runs:
 *   1. the gather of s and c from the live state, in one kernel (red_blue.py:85-87);
 *   2. host mode: one copy to the host, then a stream synchronisation;  3. fn;
 *   4. host mode: q and factors are copied to the device;
 *   5. a non-finite q stops the call with EB_ERR_INF_PARAM / EB_ERR_NAN_PARAM before any log-probability is
 *      evaluated (ensemble.py:476-479); NaN factors are no error: the comparison rejects them (red_blue.py:100);
 *   6. the log-probability of q -- the device model, fused with the accept + update kernel, or the callback of
 *      eb_model_set_callback with its own guards -- then the accept + update (red_blue.py:96-104, mh.py:57-62).
 * A schedule naming an unset slot is refused with EB_ERR_INVALID.  Failures of fn stop the call inside a step
 * exactly as a failing log-probability callback does; inside fn every other call on the context returns
 * EB_ERR_STATE.  Sharded engines are refused with EB_ERR_UNSUPPORTED. */
int eb_move_set_proposal(eb_ctx* ctx, int32_t slot, eb_proposal_fn fn, void* user, int where);
/* device mode, from inside fn: copy m (= fn's ns) rows of ndim float64 values, q_row_stride_bytes apart (contiguous
 * inside a row), from q, and m factors, f_stride_bytes apart, from factors (device or host memory) into fn's q and
 * factors, ordered on src_stream as eb_callback_result orders its copy.  Complete when the call returns. */
int eb_proposal_result(eb_ctx* ctx, const void* q, int64_t q_row_stride_bytes, const void* factors,
                       int64_t f_stride_bytes, int64_t m, uint64_t src_stream);

/* A user proposal captured as CUDA graphs, one per split of the moves that use its slot: launched, the graph reads
 * the active set s[ns, ndim], the other sets c[N - ns, ndim] back to back in set order (NULL for an MHMove, whose
 * s is the whole ensemble in walker order and whose split is 0) and ndraws draws per row draws[ns, ndraws], and
 * writes q[ns, ndim] and factors[ns].  Every buffer is float64 device memory of the engine's device with contiguous
 * rows; the *_stride_bytes are the distances between rows (factors: between entries).  Splits that see the same
 * shapes may share one graph and its buffers.  exec is a cudaGraphExec_t instantiated on the engine's device. */
typedef struct {
  int32_t split;
  int64_t ns;
  uint64_t exec;
  void* s;
  int64_t s_row_stride_bytes;
  void* c;
  int64_t c_row_stride_bytes;
  void* draws;
  int64_t draws_row_stride_bytes;
  void* q;
  int64_t q_row_stride_bytes;
  void* factors;
  int64_t factors_stride_bytes;
} eb_proposal_graph;
#define EB_DRAW_UNIFORM 0 /* draws 2k, 2k+1 of row i: u53(w0, w1), u53(w2, w3) of block (i, sub-index k, purpose 9) */
#define EB_DRAW_NORMAL 1  /* the same words through purpose 6's Box-Muller pair */
#define EB_MAX_GRAPH_DRAWS (1 << 19) /* the 18-bit sub-index field of the counter holds k < 2^18 */
/* make n captured graphs proposal slot `slot` (callback mode EB_CALLBACK_GRAPH); eb_move_set_proposal on the same
 * slot clears them.  A half-step of a schedule entry of kind EB_MOVE_USER / EB_MOVE_USER_MH naming the slot enqueues,
 * with no host synchronisation:
 *   1. one kernel that gathers s and c from the live state into the graph's buffers (red_blue.py:85-87) and fills
 *      draws from purpose 9 of the draw specification (DESIGN.md §2) at the sampler's (seed, step, split);
 *   2. cudaGraphLaunch;
 *   3. one kernel that copies q and factors into the engine and raises EB_ERR_INF_PARAM / EB_ERR_NAN_PARAM for a
 *      non-finite q (ensemble.py:476-479); NaN factors are no error;
 *   4. step 6 of eb_move_set_proposal: the log-probability and the accept + update.
 * Errors stay on the device as under eb_model_set_graphs: from the first one on, nothing is copied into the graphs'
 * inputs and every factor is NaN, so every later proposal is rejected; the host reports the first error where a
 * stepping call synchronises, with the step counter, the stored steps and the statistics where eb_move_set_proposal
 * leaves them.  Refused (EB_ERR_INVALID): draw_kind other than EB_DRAW_UNIFORM / EB_DRAW_NORMAL, ndraws < 0, a split
 * outside [0, 32) or given twice, ns outside [1, nwalkers], exec = 0, null buffers (c: an MHMove passes none; draws:
 * none when ndraws = 0), strides that are not positive multiples of 8 or shorter than a row, buffers that are not
 * device memory of the engine's device; ndraws > EB_MAX_GRAPH_DRAWS and sharded engines: EB_ERR_UNSUPPORTED.  A
 * schedule whose entry needs a split the slot lacks, or a split of another size, or EB_USER_SETUP, is refused by
 * eb_step.  The engine does not own the graphs or the buffers: they must stay valid, and unused by anything else,
 * while the slot is set. */
int eb_move_set_proposal_graphs(eb_ctx* ctx, int32_t slot, int draw_kind, int64_t ndraws,
                                const eb_proposal_graph* graphs, size_t n);

/* ---- state (state.py:10-45) ------------------------------------------- */
/* State(initial_state, copy=True) + the initial compute_log_prob
 * (ensemble.py:312,350-358): copies coords[nwalkers*ndim] to the device;
 * log_prob == NULL -> evaluated on the device.  Non-finite coords / NaN
 * log-prob give the reference's errors. */
int eb_set_state(eb_ctx* ctx, const double* coords, const double* log_prob);
/* device -> host copy of the live state; either pointer may be NULL.
 * Sharded ensembles (after eb_comm_init): eb_set_state reads only the rows this
 * rank owns from the (globally indexed) host arrays, and eb_get_state returns
 * the GLOBAL state -- it replicates the other ranks' rows first and is
 * therefore COLLECTIVE (every rank calls it at the same point), as are
 * eb_get_naccepted, eb_step with accepted_last != NULL and eb_step_store. */
int eb_get_state(eb_ctx* ctx, double* coords, double* log_prob);
/* rows [row0, row0 + nrows) this context owns: the whole ensemble on one GPU,
 * the rank's row block after eb_comm_init. */
int eb_owned_rows(const eb_ctx* ctx, int64_t* row0, int64_t* nrows);
/* device -> host copy of rows [row0, row0 + nrows) of the live state into
 * coords[nrows * ndim] / log_prob[nrows] (either may be NULL).  Not collective:
 * on a sharded ensemble only the owned block (or any rows after a collective
 * read) is valid; other rows are refused with EB_ERR_STATE. */
int eb_get_state_rows(eb_ctx* ctx, int64_t row0, int64_t nrows, double* coords, double* log_prob);
/* State(coords, log_prob, blobs) of a callback model (state.py:10-45, ensemble.py:344-349): after an eb_set_state
 * given log_prob, upload blobs[nwalkers * record_bytes] (host) as the state's blobs and fix the live layout.
 * NULL, 0 clears them.  Device blob memory is checked before allocation (EB_ERR_NOMEM, as eb_chain_grow). */
int eb_set_state_blobs(eb_ctx* ctx, const void* blobs, size_t record_bytes);
/* the state's blobs (State.blobs, moves/move.py:36-43): out[nwalkers * record_bytes] (host); EB_ERR_STATE when the
 * state has none. */
int eb_get_blobs(eb_ctx* ctx, void* out);

/* ---- log-probability (ensemble.py:458-553) ------------------------------ */
/* EnsembleSampler.compute_log_prob(coords[m, ndim]) -> out[m], with the
 * isinf/isnan guards on the input (:476-479) and the NaN guard on the output
 * (:550-551). */
int eb_compute_log_prob(eb_ctx* ctx, const double* coords, size_t m, double* out);
/* compute_log_prob returning blobs (ensemble.py:458-553 `return log_prob, blob`) for a callback model: as
 * eb_compute_log_prob, and *blobs_out receives page-locked host memory holding the m records the function
 * delivered, *record_bytes their size (free it with eb_host_free); NULL and 0 when it delivered none. */
int eb_compute_log_prob_blobs(eb_ctx* ctx, const double* coords, size_t m, double* out, void** blobs_out,
                              size_t* record_bytes);

/* ---- random state (ensemble.py:216-238) --------------------------------- */
/* The engine's "random_state" is (seed, step): every draw is a pure function
 * of (seed, step, split, active rank, purpose) -- see DESIGN.md "Draw
 * specification".  A new seed, or a step counter below the current one,
 * empties the running reservoir (eb_reservoir_config): the rows of a step
 * offered again would come back with their old keys. */
int eb_set_rng(eb_ctx* ctx, uint64_t seed, uint64_t step);
int eb_get_rng(const eb_ctx* ctx, uint64_t* seed, uint64_t* step);

/* ---- the hot path ------------------------------------------------------- */
/* nsteps iterations of the sample() inner loop (ensemble.py:403-419): per step
 * draw one move from the schedule (:406), then Move.propose = the RedBlueMove
 * split cycle (moves/red_blue.py:52-106): split assignment (:76-80), per split
 * proposal (stretch.py:26-33 / de.py:40-64 / de_snooker.py:31-46), log-prob of
 * the proposals (:93), Metropolis accept (:96-101) and in-place update
 * (:103-104 -> moves/move.py:29-34).  accepted_last (nullable, nwalkers bytes)
 * receives the accept mask of the last step (the `accepted` propose returns).
 * Per-walker accept counts accumulate on the device (backend.py:229). */
int eb_step(eb_ctx* ctx, const eb_move* moves, size_t nmoves, uint64_t nsteps,
            uint8_t* accepted_last);
/* like eb_step with store=True (ensemble.py:416-417 -> backend.py:214-231):
 * every thin_by-th step's coords / log_prob are appended to the host arrays
 * chain[nstore, nwalkers, ndim], log_prob[nstore, nwalkers] (nstore =
 * nsteps / thin_by) and accepted[nwalkers] (float64, backend.py:31) is
 * incremented per accepted proposal of the stored steps' windows. */
int eb_step_store(eb_ctx* ctx, const eb_move* moves, size_t nmoves, uint64_t nsteps,
                  uint64_t thin_by, double* chain, double* log_prob, double* accepted);
/* eb_step_store that also stores the state's blobs (backend.py:226-227): each stored step's records go to
 * blobs[nstore, nwalkers, record_bytes] (host), through the same double-buffered pinned staging and drain as
 * coords and log_prob, so a call stopped by the function leaves the blobs of every completed stored step in
 * place.  blobs == NULL is eb_step_store; non-NULL needs a state with blobs (EB_ERR_STATE). */
int eb_step_store_blobs(eb_ctx* ctx, const eb_move* moves, size_t nmoves, uint64_t nsteps,
                        uint64_t thin_by, double* chain, double* log_prob, double* accepted, void* blobs);

/* ---- device chain storage (backends/backend.py:12-237 kept in HBM) ----- */
/* A stored chain on one device: coords[slots, nwalkers, ndim], log_prob[slots,
 * nwalkers] and accepted[nwalkers] (float64, backend.py:31), with its own
 * stream and error string.  It belongs to no engine: any engine of the same
 * shape on the same device may store into it (a second sampler on an already
 * initialised backend appends, ensemble.py:137-162).  Storage is a list of
 * segments, one per eb_chain_grow; growing never copies stored steps. */
typedef struct eb_chain eb_chain;
/* Backend.reset (backend.py:20-36): an empty chain, accepted = 0. */
int eb_chain_create(int device, int64_t nwalkers, int64_t ndim, eb_chain** out);
int eb_chain_destroy(eb_chain* ch);
/* message of the last failing call on ch (ch == NULL: last eb_chain_create
 * failure of this thread). */
const char* eb_chain_last_error(const eb_chain* ch);
/* Backend.grow (backend.py:164-185): capacity becomes nslots by one new segment
 * for exactly the missing slots (no-op when it already holds nslots).  More than
 * the device's total memory is refused before any allocation, a failed
 * allocation leaves the chain as it was: both EB_ERR_NOMEM, naming the requested
 * and the free bytes. */
int eb_chain_grow(eb_chain* ch, uint64_t nslots);
/* slots allocated, and the device bytes the chain holds. */
int eb_chain_capacity(const eb_chain* ch, uint64_t* nslots, uint64_t* bytes);
/* eb_step_store into a device chain (ensemble.py:416-417 -> backend.py:214-231):
 * every thin_by-th step's coords / log_prob go to slots slot0, slot0 + 1, ...
 * (nsteps / thin_by of them) and its accept mask is added to the chain's
 * accepted, each by one kernel behind the step on the engine's stream; the call
 * synchronises once, at its end.  The chain must match the engine's shape and
 * device (for a batch context, nbatch * nwalkers rows: ensemble k is segment k
 * of the chain); sharded engines are refused (EB_ERR_UNSUPPORTED). */
int eb_step_store_chain(eb_ctx* ctx, const eb_move* moves, size_t nmoves, uint64_t nsteps,
                        uint64_t thin_by, eb_chain* ch, uint64_t slot0);
/* Backend.save_step (backend.py:214-231): host coords[nwalkers*ndim] /
 * log_prob[nwalkers] into slot `slot`, accepted (nullable, nwalkers bytes of 0/1)
 * added to the chain's counts. */
int eb_chain_write(eb_chain* ch, uint64_t slot, const double* coords, const double* log_prob,
                   const uint8_t* accepted);
/* Backend.get_value (backend.py:42-58): the slots first + k * stride, k < count,
 * into host coords[count, nwalkers, ndim] / log_prob[count, nwalkers] (either
 * may be NULL); stride >= 1. */
int eb_chain_read(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count,
                  double* coords, double* log_prob);
/* Backend.accepted (backend.py:31,229): accepted[nwalkers] to the host. */
int eb_chain_accepted(eb_chain* ch, double* accepted);
/* eb_autocorr of the stored slice first + k * stride, k < count, read where it
 * is stored: acf[ndim, count], bit-identical to eb_autocorr of the same slice
 * copied to the host. */
int eb_chain_autocorr(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* acf);
/* Exact order statistics of the stored slice first + k * stride, k < count, read
 * where it is stored: for each parameter (what = EB_CHAIN_COORDS: ndim of them;
 * EB_CHAIN_LOG_PROB: one) out[r * D + d] is the value np.partition puts at
 * 0-based rank ranks[r] (nranks >= 1; each < count * nwalkers; any order, repeats allowed) of
 * that parameter's count * nwalkers values, with -0.0 returned as +0.0.
 * has_nan[D] flags the parameters holding a NaN; their entries of out are NaN.
 * *passes (nullable) = full reads of the slice the call made (radix passes of
 * SEL_DIGIT bits, select_keys.h).  Device scratch is bounded (about 100 MiB at
 * most) and checked against the free memory first: EB_ERR_NOMEM. */
#define EB_CHAIN_COORDS 0
#define EB_CHAIN_LOG_PROB 1
int eb_chain_select(eb_chain* ch, int what, uint64_t first, uint64_t stride, uint64_t count,
                    const uint64_t* ranks, size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes);
/* eb_moments of the stored slice: mean[ndim], cov[ndim*ndim] (np.mean /
 * np.cov(rowvar=False, ddof=1) of get_chain(flat=True)) and their sample count
 * count * nwalkers; the sums run about the column mean of the slice's first
 * stored step, one accumulation per stored step in slot order.  ndim <= 1024
 * (EB_ERR_UNSUPPORTED beyond); an empty slice gives NaN.  Scratch is checked
 * against the free memory first: EB_ERR_NOMEM. */
int eb_chain_moments(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* mean, double* cov,
                     uint64_t* n);
/* Segmented analyses: the chain's nwalkers are nseg segments (ensembles, the
 * rows of a batch context, eb_create_batch) of nw = nwalkers / nseg walkers,
 * segment k being walkers [k * nw, (k + 1) * nw) of every stored step.  nseg >= 1
 * must divide nwalkers (EB_ERR_INVALID otherwise); nseg = 1 is the whole chain.
 *
 * eb_chain_autocorr of each segment: acf[nseg, ndim, count], row k bit-identical
 * to eb_chain_autocorr of segment k stored alone. */
int eb_chain_autocorr_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                               double* acf);
/* eb_chain_select of each segment: out[nseg, nranks, D] and has_nan[nseg, D],
 * ranks < count * nw; every segment's parameters are refined in the same passes
 * (nseg * D columns), so *passes does not grow with nseg. */
int eb_chain_select_segments(eb_chain* ch, int64_t nseg, int what, uint64_t first, uint64_t stride, uint64_t count,
                             const uint64_t* ranks, size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes);
/* eb_chain_moments of each segment: mean[nseg, ndim], cov[nseg, ndim, ndim] and
 * *n = count * nw, the sums of segment k about the column mean of its first
 * stored step, in (step, walker) order with a fixed chunking of the steps (three
 * launches for the whole slice).  ndim <= 1024; scratch checked: EB_ERR_NOMEM. */
int eb_chain_moments_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                              double* mean, double* cov, uint64_t* n);
/* eb_chain_read_to in the per-segment layout: coords_dst[nseg, count * nw, ndim]
 * and log_prob_dst[nseg, count * nw] (either may be NULL), device to device. */
int eb_chain_read_segments_to(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                              double* coords_dst, double* log_prob_dst);
/* np.histogram of each parameter (what = EB_CHAIN_COORDS: ndim of them;
 * EB_CHAIN_LOG_PROB: one) of the stored slice first + k * stride, k < count, read
 * where it is stored, with numpy's edges given by the caller: outer[D * 3] holds
 * each parameter's (first_edge, last_edge, norm_denom) and edges[D * (bins + 1)]
 * its linspace, as np.histogram forms them.  hist[D * bins] gets the counts of
 * numpy's uniform-bin rule (values outside [first_edge, last_edge] and NaN are
 * dropped).  1 <= bins <= 4096 (EB_ERR_UNSUPPORTED beyond); a value whose
 * truncated index ((x - first) / span) * bins is above bins (numpy indexes past
 * its edges there and raises IndexError) gives EB_ERR_INVALID; count == 0 gives
 * zero counts.  Scratch is checked against the
 * free memory first: EB_ERR_NOMEM. */
int eb_chain_histogram(eb_chain* ch, int what, uint64_t first, uint64_t stride, uint64_t count, uint32_t bins,
                       const double* outer, const double* edges, uint64_t* hist);
/* np.histogram2d of every pair of the nparams >= 2 distinct coordinates
 * params[] (each < ndim) of the stored slice: pair p is the p-th of
 * itertools.combinations(params, 2) and hist[p * bins * bins + x * bins + y]
 * counts its values in bin x of params[i] and bin y of params[j], with
 * np.histogramdd's rule (searchsorted right, the last edge in the last bin,
 * outliers and NaN dropped) against edges[k * (bins + 1) ...], the edges of
 * params[k].  1 <= bins <= 128 (EB_ERR_UNSUPPORTED beyond); count == 0 gives
 * zero counts.  hist holds nparams (nparams - 1) / 2 * bins^2 counts, all in
 * device scratch at once, checked against the free memory first: EB_ERR_NOMEM. */
int eb_chain_histogram2d(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, const uint32_t* params,
                         size_t nparams, uint32_t bins, const double* edges, uint64_t* hist);
/* eb_chain_histogram of each segment (nseg divides nwalkers; segment k is
 * walkers k * nw .. (k + 1) * nw - 1, nw = nwalkers / nseg): column k * D + d
 * is parameter d of segment k, with outer[nseg * D * 3], edges[nseg * D *
 * (bins + 1)] and hist[nseg * D * bins] in that column order.  Every column is
 * counted in the same read of the slice; eb_chain_histogram is nseg = 1. */
int eb_chain_histogram_segments(eb_chain* ch, int64_t nseg, int what, uint64_t first, uint64_t stride, uint64_t count,
                                uint32_t bins, const double* outer, const double* edges, uint64_t* hist);
/* eb_chain_histogram2d of each segment: edges[nseg * nparams * (bins + 1)]
 * holds segment k's edges of params[] at k * nparams * (bins + 1) and hist
 * [nseg * npairs * bins^2] its pair counts at k * npairs * bins^2.  The counts of
 * every segment are held in device scratch at once (EB_ERR_NOMEM when they do
 * not fit); eb_chain_histogram2d is nseg = 1. */
int eb_chain_histogram2d_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                                  const uint32_t* params, size_t nparams, uint32_t bins, const double* edges,
                                  uint64_t* hist);

/* ---- device memory in and out (CUDA Array Interface) --------------------- */
/* The device twins of the state, log-probability and chain transfers above, for callers that keep their arrays
 * in GPU memory (torch, CuPy, Numba, ...).  Sources are ordered after the producer's work on src_stream with the
 * encoding of eb_callback_result (CUDA Array Interface v3: 0 = none, 1 = legacy default stream, 2 = per-thread
 * default stream, else a cudaStream_t; EB_STREAM_UNKNOWN = after all work on the device).  Rows must be
 * contiguous; only the first axis may be strided (a positive multiple of 8 bytes, at least a row).  Every call
 * is complete when it returns.  Device pointers must be device (or managed) memory of the context's or chain's
 * device: another device, or host memory, gives EB_ERR_INVALID.  Sharded engines (eb_comm_init) are refused
 * with EB_ERR_UNSUPPORTED.  The data moves on the copy engines (cudaMemcpy2DAsync, cudaMemcpyDefault). */
/* device memory for arrays the caller hands out: bytes on device `device` (0 gives NULL, touching no
 * device).  More than the device's total memory is refused before cudaMalloc, and a failed allocation is
 * refused too: both EB_ERR_NOMEM (as eb_chain_grow).  Messages of these three calls: eb_last_error(NULL). */
int eb_device_alloc(int device, size_t bytes, void** out);
/* frees what eb_device_alloc returned (NULL is a no-op). */
int eb_device_free(int device, void* p);
/* rows of width bytes, src_pitch apart in src (memory of `device`, or host memory), packed into dst (host or
 * device memory), ordered after src_stream: a CUDA array read back (DeviceArray.get, the host check of an
 * initial state given on the device), copied or uploaded. */
int eb_device_copy(int device, void* dst, const void* src, int64_t width, int64_t src_pitch, int64_t rows,
                   uint64_t src_stream);
/* eb_set_state from device memory (State(initial_state, copy=True) + the initial compute_log_prob,
 * ensemble.py:312,350-358; state.py:10-45): coords[nwalkers] rows coords_row_stride_bytes apart, log_prob
 * (nullable) lp_stride_bytes apart.  log_prob == NULL: evaluated on the device with eb_set_state's guards and
 * callback / blob behaviour.  A given log_prob is checked for NaN on the device (EB_ERR_NAN_INITIAL, "The
 * initial log_prob was NaN", ensemble.py:357-358). */
int eb_set_state_from(eb_ctx* ctx, const void* coords, int64_t coords_row_stride_bytes, const void* log_prob,
                      int64_t lp_stride_bytes, uint64_t src_stream);
/* eb_get_state into device memory: coords_dst[nwalkers * ndim], log_prob_dst[nwalkers], either may be NULL
 * (state.py:10-45, the State yielded by ensemble.py:403-424). */
int eb_get_state_to(eb_ctx* ctx, double* coords_dst, double* log_prob_dst);
/* eb_compute_log_prob (ensemble.py:458-553) of m rows of device memory, row_stride_bytes apart, into
 * out_dst[m] (device), with the same guards on the input (:476-479) and the output (:550-551); m == 0 is a
 * no-op. */
int eb_compute_log_prob_from(eb_ctx* ctx, const void* coords, int64_t row_stride_bytes, int64_t m, double* out_dst,
                             uint64_t src_stream);
/* eb_chain_read into device memory (Backend.get_value, backend.py:42-58): the slots first + k * stride, k <
 * count, into coords_dst[count, nwalkers, ndim] / log_prob_dst[count, nwalkers] (either may be NULL), device to
 * device. */
int eb_chain_read_to(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* coords_dst,
                     double* log_prob_dst);

/* per-walker number of accepted proposals since creation / eb_reset_counters
 * (numerator of acceptance_fraction, ensemble.py:555-558). */
int eb_get_naccepted(eb_ctx* ctx, uint64_t* naccepted);
/* how many steps of the LAST eb_step / eb_step_store call ran each entry of its move schedule
 * (picks[nmoves]): the host mirror of a stateful move (GaussianMove mode "sequential",
 * gaussian.py:102-103) advances its index by this count. */
int eb_move_picks(const eb_ctx* ctx, uint64_t* picks, size_t nmoves);
int eb_reset_counters(eb_ctx* ctx);

/* ---- chain analysis on the device --------------------------------------- */
/* Running moments of the chain for store=False runs (ensemble.py:287-291 keeps
 * nothing; a caller who wants the chain mean / covariance would otherwise need
 * a D2H of the state every step).  Enabled by eb_set_option("moments_every", n):
 * after every n-th step the rows this context owns are folded into device
 * accumulators (sum and outer-product sum on the FP64 tensor pipe).  Returns
 * mean[ndim], cov[ndim*ndim] (= np.mean / np.cov(rowvar=False, ddof=1) over
 * the accumulated (step, walker) samples), their number, and the total number
 * of accepted proposals of the owned walkers; any output may be NULL.  On a
 * sharded ensemble the values are per rank (the host combines them). */
int eb_moments(eb_ctx* ctx, double* mean, double* cov, uint64_t* count, uint64_t* naccepted_total);
/* Running histograms of the chain for store=False runs: eb_chain_histogram /
 * eb_chain_histogram2d of the steps a store with thin_by = every would keep,
 * without storing them.  After every step whose counter is a multiple of
 * `every` (the cadence of "moments_every"), each walker's coordinates are
 * counted into device counts by kernels behind the step on the engine's stream
 * (no synchronisation or copy per count); every == 0 counts nothing.
 * 1-D: outer[(ndim + log_prob) * 3] and edges[(ndim + log_prob) * (bins + 1)]
 * as eb_chain_histogram takes them, one row per parameter and, when log_prob is
 * non-zero, a last row for the log-probabilities; 1 <= bins <= 4096.  2-D
 * (nparams2d == 0: none): the 2 <= nparams2d <= ndim distinct params2d[] with
 * edges2d[nparams2d * (bins2d + 1)], as eb_chain_histogram2d takes them;
 * 1 <= bins2d <= 128.  Each call replaces the configuration and zeroes the
 * counts.  The tables are uploaded and the uint64 counts allocated here, checked
 * against the free memory first (EB_ERR_NOMEM); the 2-D counts take
 * nparams2d (nparams2d - 1) / 2 * bins2d^2 * 8 bytes.  Sharded engines are
 * refused with EB_ERR_UNSUPPORTED, both ways round (eb_comm_init). */
int eb_histograms_config(eb_ctx* ctx, uint64_t every, uint32_t bins, const double* outer, const double* edges,
                         int log_prob, const uint32_t* params2d, size_t nparams2d, uint32_t bins2d,
                         const double* edges2d);
/* the counts since eb_histograms_config: hist[(ndim + log_prob) * bins] and
 * hist2d[npairs * bins2d^2] in eb_chain_histogram / eb_chain_histogram2d's
 * layout (either may be NULL), and the number of samples counted per parameter
 * (*count: counted steps * nwalkers).  EB_ERR_STATE before any configuration; a
 * value whose truncated index is above bins (see eb_chain_histogram) gives
 * EB_ERR_INVALID, with the counts written. */
int eb_histograms(eb_ctx* ctx, uint64_t* hist, uint64_t* hist2d, uint64_t* count);
/* Running trace for store=False runs: the time axis that eb_moments and
 * eb_histograms pool away.  After every step whose counter is a multiple of
 * `every` (the cadence of eb_histograms_config) one row of 2 ndim + 4 doubles is
 * recorded in device memory by two kernels behind the step on the engine's
 * stream: the mean and the ddof = 1 variance of each parameter over the
 * ensemble, the mean and the maximum of the log-probabilities, the number of
 * walkers that accepted their proposal in that step, and the lowest walker
 * holding the maximum.  The sums are taken in a fixed order that depends on
 * nwalkers alone (csrc/trace_sum.h), so a row does not depend on how the steps
 * were launched.  The largest log-probability of all recorded steps is kept
 * with its coordinates (eb_trace_best).  every > 0 drops the rows and the best
 * sample recorded so far; every == 0 records nothing more and leaves them
 * readable.  The rows are not allocated here: each stepping call knows how many
 * it will add and makes room once before its first launch, checked against the
 * free memory (EB_ERR_NOMEM, with nothing enqueued); recorded rows survive the
 * growth.  Nothing is allocated, copied to the host, cleared or synchronised per
 * recorded step.  Sharded engines are refused with EB_ERR_UNSUPPORTED, both ways
 * round (eb_comm_init). */
int eb_trace_config(eb_ctx* ctx, uint64_t every);
/* rows recorded since the last eb_trace_config with every > 0; EB_ERR_STATE
 * before any configuration (as eb_trace_read and eb_trace_best) */
int eb_trace_count(eb_ctx* ctx, uint64_t* rows);
/* rows first .. first + count - 1 in one download: step[count] their step
 * counters and rows_out[count * (2 ndim + 4)], a row being mean[ndim],
 * var[ndim], log_prob_mean, log_prob_max, accepted, argmax walker (the last two
 * whole numbers).  Either output may be NULL; a range past eb_trace_count gives
 * EB_ERR_INVALID. */
int eb_trace_read(eb_ctx* ctx, uint64_t first, uint64_t count, uint64_t* step, double* rows_out);
/* the largest log-probability among the recorded steps: coords[ndim], its
 * value, the step counter and the walker; ties go to the earliest step, then
 * the lowest walker.  Any output may be NULL; EB_ERR_STATE while no step has
 * been recorded. */
int eb_trace_best(eb_ctx* ctx, double* coords, double* log_prob, uint64_t* step, uint64_t* walker);
/* Running reservoir for store=False runs: a uniform sample without
 * replacement of `size` (K) of the (step, walker) rows recorded after every
 * step whose counter is a multiple of `every` (the cadence of
 * eb_histograms_config), in device memory of a fixed size however long the
 * run is.  Every recorded row gets the key (w1 << 32) | w0 of draw block
 * (seed, step, split 0, tag 10, index = walker) of the draw specification, and
 * the reservoir keeps the K rows first in the order (key, step, walker): a
 * pure function of the seed and the recorded states, independent of how the
 * steps were cut into calls; no other draw changes.  Rows pass a filter kernel
 * behind the step on the engine's stream (key below the K-th kept key) into a
 * buffer of K + max(K, nwalkers) entries of 8 ndim + 32 bytes, which a radix
 * select on the device cuts back to K before a record that could overflow it
 * and before every read (csrc/reservoir_plan.h); nothing is copied to the host
 * or synchronised per recorded step.  The buffers are allocated here,
 * checked against the free memory first (EB_ERR_NOMEM, with nothing
 * changed); so is size >= 2^32, past the entries the reservoir addresses.
 * size >= 1 (EB_ERR_INVALID).  every > 0 drops what was kept;
 * every == 0 records nothing more and leaves the contents (and their size)
 * readable.  eb_set_rng with a new seed, or a step counter moved back, empties
 * the reservoir and keeps its configuration.  Blobs are not kept.  Sharded engines are refused with
 * EB_ERR_UNSUPPORTED, both ways round (eb_comm_init). */
int eb_reservoir_config(eb_ctx* ctx, uint64_t size, uint64_t every);
/* rows offered since the last eb_reservoir_config with every > 0 (nwalkers
 * times the recorded steps) and rows kept, min(size, offered); either output
 * may be NULL.  EB_ERR_STATE before any configuration (as the reads). */
int eb_reservoir_count(eb_ctx* ctx, uint64_t* offered, uint64_t* kept);
/* the kept rows (eb_reservoir_count) in the order (key, step, walker), so that
 * any prefix of length k is the reservoir of the same run with size k:
 * coords[kept * ndim], log_prob[kept], step[kept] (the step counter the row
 * was recorded at) and walker[kept], all host memory; any output may be NULL. */
int eb_reservoir_read(eb_ctx* ctx, double* coords, double* log_prob, uint64_t* step, int64_t* walker);
/* eb_reservoir_read with coords_dst[kept * ndim] and log_prob_dst[kept] in
 * device memory (gathered on the device; any 8-byte aligned pointers); step
 * and walker stay host memory. */
int eb_reservoir_read_to(eb_ctx* ctx, double* coords_dst, double* log_prob_dst, uint64_t* step, int64_t* walker);
/* Running autocorrelation function for store=False runs: the walker-averaged
 * normalised autocorrelation function of every parameter at lags 0 ..
 * max_lag (autocorr.py:49-104 of the reference's estimator) of the states
 * recorded after every step whose counter is a multiple of `every` (the
 * cadence of eb_trace_config), in device memory of a fixed size however long
 * the run is: about 8 nwalkers ndim (4 max_lag + 64) bytes.  Each (walker,
 * parameter) series is shifted by its first recorded value; every recorded
 * step writes the state into a ring, and every 64 recorded steps one kernel
 * adds the block's lag products into double-double lag sums
 * (csrc/running_acf.h), so the result is a pure function of the recorded
 * states, independent of how the steps were cut into calls.  The buffers are
 * allocated here, checked against the free memory first (EB_ERR_NOMEM, with
 * nothing changed).  max_lag >= 1 (EB_ERR_INVALID).  every > 0 drops what
 * was recorded; every == 0 records nothing more and leaves the result
 * readable.  Sharded engines are refused with EB_ERR_UNSUPPORTED, both ways
 * round (eb_comm_init). */
int eb_running_acf_config(eb_ctx* ctx, uint64_t max_lag, uint64_t every);
/* steps recorded since the last eb_running_acf_config with every > 0.
 * EB_ERR_STATE before any configuration (as the read). */
int eb_running_acf_count(eb_ctx* ctx, uint64_t* n);
/* rho[min(n, max_lag + 1) * ndim] (host memory): rho[tau, d] is the mean over
 * the walkers of c_w(tau) / c_w(0), c_w the autocovariance of walker w's
 * parameter d about its mean over the n recorded steps (NaN for a walker
 * whose series is constant).  Values of an unfinished block are folded into
 * copies of the sums, so a read changes nothing a later read returns. */
int eb_running_acf_read(eb_ctx* ctx, double* rho);
/* Running window for store=False runs: the states after the last `size`
 * steps whose counter is a multiple of `every` (the cadence of
 * eb_trace_config), kept in device memory as a ring chain that every
 * eb_chain_* reader takes: size * nwalkers * (ndim + 1) * 8 bytes of states
 * and size * nwalkers bytes of accept masks.  A recorded step copies the
 * coords, log-probabilities and the step's accept mask into physical slot
 * (recorded mod size) with one kernel behind the step; once the ring is full,
 * logical slot 0 (the oldest step) is physical slot (recorded mod size).  The
 * ring is allocated here, checked against the free memory first (EB_ERR_NOMEM,
 * with nothing changed); size >= 1 (EB_ERR_INVALID).  every > 0 drops what
 * was recorded; every == 0 records nothing more and leaves the contents
 * readable.  Sharded engines are refused with EB_ERR_UNSUPPORTED, both ways
 * round (eb_comm_init). */
int eb_window_config(eb_ctx* ctx, uint64_t size, uint64_t every);
/* steps recorded since the last eb_window_config with every > 0, and the slots
 * they fill: min(recorded, size).  EB_ERR_STATE before any configuration (as
 * the other eb_window_* calls). */
int eb_window_count(eb_ctx* ctx, uint64_t* recorded, uint64_t* filled);
/* for each filled slot in logical order (oldest first): steps[filled] the step
 * counter after the recorded step, seeds[filled] the Philox key it ran with
 * (either nullable); (seed, step) is the random state that resumes the run
 * from that slot's state. */
int eb_window_steps(eb_ctx* ctx, uint64_t* steps, uint64_t* seeds);
/* *ring = the window's ring, a borrowed eb_chain of `size` slots whose slot k
 * is the k-th oldest filled slot.  eb_chain_read, _read_to, _autocorr,
 * _select, _moments, _histogram and _histogram2d take it with slices of the
 * filled slots; eb_chain_accepted gives the per-walker sums of the accept
 * masks of the filled slots (summed on the device); eb_chain_capacity counts
 * the masks too.  eb_chain_grow, eb_chain_write, eb_chain_destroy and
 * eb_step_store_chain refuse it (EB_ERR_INVALID).  The handle is valid until
 * the next eb_window_config or the engine's destruction.  This call
 * synchronises the engine's stream: reads through the handle see every step
 * recorded before it. */
int eb_window_chain(eb_ctx* ctx, eb_chain** ring);
/* walkers_independent (ensemble.py:653-663) on the device: gram[ndim*ndim] =
 * C^T C of the centred, column-normalised coords[rows, ndim] (:656-661), whose
 * extreme eigenvalues give cond(C)^2.  *flags: bit 0 = non-finite coordinate
 * (:655), bit 1 = a column with zero span (:659-660), bit 2 (additive: earlier
 * builds of ABI 2 never set it) = some column's sum of squares about its mean is not a positive,
 * finite, normal double, or an entry overflowed: the Gram matrix is unreliable
 * (its entries in such columns are 0) and the caller should decide on the host.
 * Bits 1 and 2 are tested on the sums about the device's column mean, not the
 * reference's: a caller that wants the reference's zero-span test applies it
 * itself, and hands over coordinates of a moderate scale.  The D x D symmetric
 * eigen-solve stays on the host (numpy). */
int eb_walkers_gram(eb_ctx* ctx, const double* coords, size_t rows, double* gram, int* flags);
/* The device part of autocorr.integrated_time (autocorr.py:49-123, called from
 * backends/backend.py:130-150 on the stored chain): for chain[n_step, n_walker,
 * n_param] (host, C order) acf[n_param, n_step] = the walker average of the
 * normalised autocorrelation functions function_1d(chain[:, k, d])
 * (autocorr.py:21-46: FFT of the mean-subtracted series zero-padded to
 * 2*next_pow_two(n_step), power spectrum, inverse FFT, / acf[0]; :101-106).
 * Sokal's window search on acf (:107-109) is O(n_step * n_param) and stays
 * on the host.  Independent of the context's ensemble shape. */
int eb_autocorr(eb_ctx* ctx, const double* chain, size_t n_step, size_t n_walker, size_t n_param, double* acf);

/* ---- measurement / test taps ------------------------------------------- */
/* device time (ms, CUDA events on the engine's stream) of the last eb_step /
 * eb_step_store / eb_step_store_chain call, first launch to last, and the
 * number of kernels it launched for the steps (the store kernels of
 * eb_step_store_chain are not counted, so both store calls report the same).
 * With a callback model the span includes the time the stream waits for the
 * callbacks (and their copies). */
int eb_last_step_timing(const eb_ctx* ctx, double* ms, uint64_t* launches);
/* draws of the LAST half-step executed (known-answer tests): for each active
 * rank i of that split, partner walker ids (up to 3 per walker: stretch uses
 * [0]; DE [0]=p0,[1]=p1; snooker z,z1,z2), the proposal scalar (stretch zz,
 * DE gamma, snooker |s-z|) and the accept uniform.  Arrays sized nwalkers
 * (x3 for partners); *nactive returns the count. */
int eb_debug_taps(eb_ctx* ctx, int64_t* partners, double* scalar, double* u_accept,
                  int64_t* active, int64_t* nactive);
/* per-tile cycle stamps of the dense_dmma consumers during the LAST half-step
 * launched (option "dmma_timeline"): [SM][8 consumers][8 tiles][12 events]
 * (0..5 and 9 consumer, 6..8, 10 and 11 producer). */
int eb_debug_timeline(eb_ctx* ctx, int64_t* out, size_t capacity, size_t* written);
/* engine options: "debug_taps" (0/1: record the draws of each half-step for
 * eb_debug_taps; forces the generic kernel), "dense_dmma" (0/1: allow the
 * FP64 tensor-core kernel for stretch + gauss_dense; default 1), "tma_rows" (0/1/2: the TMA row-gather kernel
 * for the HBM-bound models: off / rows short enough for several walkers per tile / any even ndim; default 2), "dmma_stagger" (0/1: staggered
 * first tiles at launch start; default 1), "dmma_group" (n >= 1: half-steps
 * fused into one persistent cooperative launch of that kernel, separated by an
 * in-kernel grid barrier -- and, on a P2P-sharded ensemble, a peer-flag barrier; default 1), "pdl" (0/1/2: consecutive dense_dmma launches chain as programmatic
 * dependent launches so a launch's prologue overlaps its predecessor's tail; 1 = on one GPU (default), 2 = on sharded ensembles too), "tma_own_reg" (0/1: tma_rows with the stretch move and rows of at most 512 bytes keeps the own row
 * in registers and stages only the partner rows; default 1), "dmma_local_first" (0/1/2: sharded dense_dmma -- build the first round of tiles from walkers whose
 * partner is local and take the peer barrier behind them; 0 never (default: the measured effect changes sign with the
 * number of GPUs), 1 when a consumer warp has at most two tiles per half-step, 2 always), "moments_every" (n >= 0: see
 * eb_moments; setting it resets the accumulators), "dmma_timeline" (0/1/2: record consumer cycle stamps
 * for eb_debug_timeline in a separately compiled, instrumented kernel; 1 keeps those of the last launch of a call,
 * 2 those of the last launch that starts a step, i.e. runs its first split), "l2_flush"
 * (0/1: benchmark hygiene -- write a 256 MiB buffer before every step and time
 * each step with its own CUDA-event pair, so eb_last_step_timing excludes the
 * flush). */
int eb_set_option(eb_ctx* ctx, const char* name, int64_t value);
/* name of the kernel variant the last eb_step used for its half-steps
 * ("generic", "dense_dmma", ...). */
const char* eb_last_kernel_name(const eb_ctx* ctx);
/* the cell of that kernel the last half-step launch ran, with the parameters its launcher chose:
 * "tma_rows R=<walkers per tile> epl=<8 register path | 0 strided> own_reg=<0|1> warps=<per CTA>",
 * "dense_dmma nhalf_max=<most half-steps of one launch in the call> grid=<CTAs>", "generic G=<lanes per
 * walker>", "walk", "gaussian", "callback G=<lanes per walker> where=host|device|graph" (eb_last_kernel_name
 * "callback": any move with a callback model), "user_move where=host|device|graph" (eb_last_kernel_name "user_move": a
 * user proposal, with any model) or "none". */
const char* eb_last_kernel_variant(const eb_ctx* ctx);

/* device micro-benchmarks that anchor the FP64 roofline: what = 0 DFMA, 1 DMMA m8n8k4, 2 DMMA m16n8k8,
 * 3 DMMA m16n8k16 (result in TFLOP/s), 4 HBM copy (GB/s).  Current device. */
int eb_microbench(int what, int warps_per_sm, double* result);
/* page-locked host memory for callers that want full-speed H2D/D2H of the
 * arrays they hand to eb_set_state / eb_get_state / eb_step_store. */
int eb_host_alloc(size_t bytes, void** out);
int eb_host_free(void* ptr);

/* ---- multi-GPU: one process per GPU, walkers sharded by row block ------- */
#define EB_COMM_ID_BYTES 128
/* rank 0 creates the id (ncclGetUniqueId), the host side broadcasts it. */
int eb_comm_id(char id[EB_COMM_ID_BYTES]);
/* join the communicator.  After this, nwalkers is the GLOBAL ensemble size,
 * rank r owns walkers [r*N/R, (r+1)*N/R) and eb_step exchanges the updated
 * rows after every split (one ncclAllGather, or peer-memory loads when
 * mode == EB_COMM_P2P). */
#define EB_COMM_ALLGATHER 0
#define EB_COMM_P2P 1
int eb_comm_init(eb_ctx* ctx, const char id[EB_COMM_ID_BYTES], int rank, int nranks, int mode);
/* peer-memory set-up for EB_COMM_P2P: export this rank's handles, then import
 * all ranks' (the host side all-gathers the blobs between the two calls). */
#define EB_IPC_BLOB_BYTES 256
int eb_comm_export(eb_ctx* ctx, char blob[EB_IPC_BLOB_BYTES]);
int eb_comm_import(eb_ctx* ctx, const char* blobs /* nranks * EB_IPC_BLOB_BYTES */);

/* measurement: GB/s of reading rank `peer`'s walker array (own rank = local HBM) with
 * what = 0 streaming 16-byte loads, 1 random whole rows (16-byte loads), 2 random whole rows
 * through TMA bulk copies (the dense_dmma producers' pattern). */
int eb_comm_probe(eb_ctx* ctx, int peer, int what, double* gbs);

#ifdef __cplusplus
}
#endif
#endif /* EMCEE_B200_H */
