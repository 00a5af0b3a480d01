// Private to the engine's C ABI: the engine and device-chain objects, the error macros, and the helpers that
// the ABI (capi.cu), the step driver (step.cu) and the running statistics (running.cu) share.
#pragma once

#include <stdio.h>

#include <memory>
#include <string>
#include <vector>

#include "comm.h"
#include "engine.cuh"
#include "owners.h"
#include "running.h"

using namespace eb;

// Every buffer, event and stream of an engine or a chain is held by an owner (owners.h), so deleting the object
// releases them.  A group of buffers that is tested through one of its members is allocated into local owners and
// moved in only once the whole group exists: a failed call never leaves half a group behind.

// a stored chain in device memory (eb_chain_*): segments of [n, N, D] coords and [n, N] log-probs, one per grow
struct ChainSeg {
  DevPtr<double> x;
  DevPtr<double> lp;
};

struct eb_chain {
  int device = 0;
  int sm_count = 0;
  int64_t N = 0;
  int D = 0;
  size_t xs = 0, ls = 0;  // slot pitches in doubles: N * D and N rounded up to even (16-byte aligned slots)
  size_t max_pitch = 0;   // cudaMemcpy2D limit; larger strides are copied row by row
  StreamPtr st;           // declared first among the owners: destroyed after the memory
  std::vector<ChainSeg> segs;
  std::vector<uint64_t> start{0};  // segment s holds slots [start[s], start[s + 1])
  DevPtr<double> accepted;         // [N] float64 (backend.py:31)
  DevPtr<uint8_t> mask;            // [N] eb_chain_write's accept mask
  // a running window's ring (eb_window_chain): one segment owned by an engine, read from logical slot 0 at physical
  // slot `origin` (chain_map.h); eb_chain_accepted sums the accept masks of its `filled` slots
  bool ring = false;
  uint64_t origin = 0, filled = 0;
  DevPtr<uint8_t> slot_mask;  // ring: [capacity, N] the accept mask of the step each slot holds
  std::string err;
};

struct eb_ctx {
  int device = 0;
  int sm_count = 0;
  int64_t N = 0;
  int D = 0;
  uint64_t seed = 0, step = 0;
  // a batch context (eb_create_batch): nbatch independent ensembles of bn walkers stacked as the N = nbatch * bn
  // rows of the live state, ensemble k in rows [k bn, (k + 1) bn), each drawing under its own key seeds[k] (the
  // step counter is shared); 0 for a single ensemble
  int64_t nbatch = 0, bn = 0;
  std::vector<uint64_t> seeds;
  StreamPtr st;  // declared first among the owners: destroyed after the events and the memory
  DevPtr<uint64_t> seeds_dev;  // [nbatch]
  EventPtr ev0, ev1;

  DevPtr<double> coords;  // [N, D], then the peer-memory barrier flags (exported to the peers, comm.h)
  DevPtr<double> logp;
  DevPtr<uint8_t> accepted;
  DevPtr<unsigned long long> nacc;
  DevPtr<int> status_dev;
  HostPtr<int> status_host;

  ModelDev model{};
  DevPtr<double> model_params;
  DevPtr<double> model_chol;
  DevPtr<double> model_box;  // [lo[D] | hi[D]] of eb_model_set_bounds, or null
  bool have_model = false, have_state = false;

  DevPtr<int32_t> order;  // [table_cap, N]
  size_t table_cap = 0;
  DevPtr<StepInfo> info_dev;
  HostPtr<StepInfo> info_host;
  DevPtr<HalfDesc> descs_dev;  // [table_cap * MAX_SPLITS] half-step descriptors of a chunk (dense_dmma)
  HostPtr<HalfDesc> descs_host;
  DevPtr<unsigned long long> gbar;  // grid-barrier counter of the persistent dense_dmma kernel
  unsigned long long gbar_count = 0;   // arrivals issued so far
  // split tables already on the device: steps [tbl_step0, tbl_step0 + tbl_n) of key tbl_seed, built with tbl_info
  uint64_t tbl_seed = 0, tbl_step0 = 0;
  size_t tbl_n = 0;
  std::vector<StepInfo> tbl_info;

  DevPtr<double> scratch_x;
  DevPtr<double> scratch_lp;
  size_t scratch_rows = 0;

  // pinned staging for eb_step_store
  HostPtr<double> stage[2];
  HostPtr<uint8_t> stage_acc[2];
  EventPtr stage_ev[2];

  bool debug = false;
  DevPtr<int64_t> tap_partners;
  DevPtr<double> tap_scalar;
  DevPtr<double> tap_u;
  DevPtr<int64_t> tap_active;
  int64_t tap_count = 0;
  DevPtr<long long> timeline;  // dense_dmma instrumentation buffer (option "dmma_timeline")
  bool timeline_first_split = false;  // option "dmma_timeline" = 2: stamp only launches that start a step

  // optional L2 flush between steps (benchmark hygiene): per-step event pairs
  bool l2_flush = false;
  DevPtr<void> flush_buf;
  size_t flush_bytes = (size_t)256 << 20;
  std::vector<EventPtr> ev_pool;

  double last_ms = 0.0;
  uint64_t last_launches = 0;
  const char* last_kernel = "none";
  char last_variant[96] = "none";  // eb_last_kernel_variant: the parameters the last half-step launch chose
  int dmma_nhalf_max = 0;          // most half-steps one dense_dmma launch ran in the current stepping call
  bool allow_dmma = true;
  int allow_tma = 2;  // TMA row-gather kernel for the HBM-bound models: 0 off, 1 short rows only, 2 long rows too
  bool tma_own_reg = true;  // tma_rows, stretch rows <= 512 B: own rows through registers instead of the TMA unit
  bool fused_last = false;  // the last dense_dmma launch carried the P2P barrier itself
  int dmma_stagger = 1;
  int dmma_group = 1;  // half-steps per persistent dense_dmma launch (1: a launch per half-step)
  int pdl = 1;           // dense_dmma launches chain as programmatic dependents (1: one GPU only, 2: sharded too)
  int local_first = 0;  // sharded dense_dmma: local-partner tiles first, peer barrier behind them (0 never, 1 auto, 2 always)
  // multi-GPU: log_prob / accept mask / counters (and, P2P, coords) of rows owned by OTHER ranks are stale
  // on this rank until the next collective read (eb_get_state, eb_get_naccepted, ...) replicates them
  bool replicas_dirty = false;

  RunningStats run;  // the running statistics (running.h)
  DevPtr<double> mom_partial;  // per-CTA partials of one moment accumulation (launch_moments)

  // WalkMove / GaussianMove scratch (moves_extra.cu)
  DevPtr<double> qbuf;       // [N, D] proposals
  DevPtr<double> walk_work;  // [D shift | D + D*D moment sums | D*D cov | D*D L]
  DevPtr<double> gauss_dev;  // per schedule entry: scale / factor L of GaussianMove
  size_t gauss_cap = 0;
  std::vector<uint64_t> picks;  // per schedule entry: steps of the last call that ran it
  // KDEMove scratch (kde.cu), allocated together on its first half-step
  DevPtr<double> kde_y;     // [ns + ns + nc <= N + N / 2 + 1, D] whitened s | q rows, then complement rows
  DevPtr<double> kde_f;     // [N] Hastings factors
  DevPtr<int64_t> kde_j;    // [N] walker id of each proposal's kernel centre (debug taps)
  DevPtr<double> kde_part;  // kde_partial_doubles: partial (max, sum) pairs of the log-sum-exps
  DevPtr<double> kde_mat;   // [D * D] (bw L)^-1, then [D] the complement mean

  Comm comm;  // multi-GPU (comm.h)

  // log-probability callback (eb_model_set_callback; model.kind == MODEL_EXTERNAL)
  eb_logprob_fn cb_fn = nullptr;
  void* cb_user = nullptr;
  int cb_where = EB_CALLBACK_HOST;
  bool in_callback = false;        // every other call on the context is refused while fn runs
  HostPtr<double> cb_x;            // host mode: pinned [cb_rows, D] proposals
  HostPtr<double> cb_lp;           // host mode: pinned [cb_rows] results
  DevPtr<double> cb_xdev;          // device mode: [cb_rows, D] copy of the rows, the function's to overwrite
  size_t cb_rows = 0;
  DevPtr<double> ext_f;            // device [N] Hastings factors of the propose phase
  DevPtr<double> ext_lp;           // device [N] the callback's log-probabilities
  int cb_phase = 0;                // CB_STEP / CB_SET_STATE / CB_COMPUTE: what the running callback evaluates
  int64_t cb_m = 0;                // rows of the running callback
  int cb_split = 0;                // CB_STEP: the split of the running half-step

  // captured log-probability graphs (eb_model_set_graphs; cb_where == EB_CALLBACK_GRAPH), one per row count
  struct Graph {
    int64_t m;
    cudaGraphExec_t exec;
    double* x;
    int64_t x_stride;  // bytes
    const double* lp;
    int64_t lp_stride;  // bytes
  };
  std::vector<Graph> graphs;
  DevPtr<unsigned long long> graph_err;       // the first error since the last check, graph_err_word (engine.cuh)
  HostPtr<unsigned long long> graph_err_host;  // read back beside the status word
  // run_steps in graph mode: the steps [graph_step0, step) enqueued since the last clean check, and the schedule
  // entry of each, so that an error found later can put the step counter and the picks back to its step
  bool graph_run = false;
  uint64_t graph_step0 = 0;
  std::vector<size_t> graph_picks;

  // blobs of a callback model (eb_callback_blobs): packed records of blob_bytes bytes, one per walker
  size_t blob_bytes = 0;           // the live layout (0: none)
  bool blobs_live = false;         // blob_live holds the records of the current state
  DevPtr<uint8_t> blob_live;       // device [N, blob_bytes]
  DevPtr<uint8_t> blob_prop;       // device [N, blob_bytes] the records of the running half-step's proposals
  HostPtr<uint8_t> blob_host;      // host mode: pinned [N, blob_bytes] staging of the function's records
  size_t blob_cap = 0;             // bytes of each of the three buffers
  int64_t cb_blob_rows = -1;       // records the running callback delivered (-1: none)
  size_t cb_blob_bytes = 0;        // their size
  uint8_t* cb_blob_dst = nullptr;  // host mode: where run_callback copies blob_host to, next to the lp copy-back
  HostPtr<uint8_t> cmp_blobs;      // CB_COMPUTE: pinned [m, record] records handed to the caller
  HostPtr<uint8_t> stage_blob[2];  // eb_step_store_blobs: pinned [N, blob_bytes] staging
  size_t stage_blob_cap = 0;

  // user proposals (eb_move_set_proposal), indexed by slot
  struct ProposalSlot {
    eb_proposal_fn fn = nullptr;
    void* user = nullptr;
    int where = EB_CALLBACK_HOST;
  };
  std::vector<ProposalSlot> props;
  // captured proposal graphs (eb_move_set_proposal_graphs; props[slot].where == EB_CALLBACK_GRAPH), indexed by slot,
  // one graph per split; empty for the other slots
  struct ProposalGraph {
    int split;
    int64_t ns;
    cudaGraphExec_t exec;
    GraphMoveBufs b;
  };
  struct ProposalGraphs {
    std::vector<ProposalGraph> graphs;
    int draw_kind = EB_DRAW_UNIFORM;
    int64_t ndraws = 0;
  };
  std::vector<ProposalGraphs> prop_graphs;
  bool in_proposal = false;   // every other call on the context is refused while a proposal runs
  int up_where = EB_CALLBACK_HOST;  // mode of the running proposal
  int64_t up_m = 0;           // rows the running proposal returns
  DevPtr<double> up_x;        // device [N, D] rows handed to the proposal (s | c, or the ensemble)
  DevPtr<double> up_f;        // device [N] its Hastings factors
  HostPtr<double> up_hx;      // host mode: pinned [N, D] copy of up_x's rows
  HostPtr<double> up_hq;      // host mode: pinned [N, D] proposals
  HostPtr<double> up_hf;      // host mode: pinned [N] factors
  DevPtr<unsigned> gm_ticket;  // captured proposals: the block counter of graph_move_result (zero between launches)
  // a captured proposal's half-step was enqueued since the status was last read: its error freezes only the captured
  // moves (and a graph model's evaluations), so run_steps reads the status before it enqueues any other move
  bool gm_unchecked = false;

  std::string err;
};

// what a running log-probability callback evaluates: a half-step's proposals, the state of eb_set_state(coords,
// NULL), or the rows of eb_compute_log_prob -- it decides where eb_callback_blobs puts the records
enum { CB_STEP = 0, CB_SET_STATE = 1, CB_COMPUTE = 2 };

#define NOT_IN_CALLBACK(ctx)                                                      \
  do {                                                                            \
    if ((ctx)->in_callback || (ctx)->in_proposal) {                               \
      (ctx)->err = (ctx)->in_callback ? "engine is inside a log-probability callback" \
                                      : "engine is inside a user proposal";       \
      return EB_ERR_STATE;                                                        \
    }                                                                             \
  } while (0)

// an entry point without a meaning for a batch context (eb_create_batch)
#define NOT_BATCH(ctx, who)                                                                               \
  do {                                                                                                    \
    if ((ctx)->nbatch > 0) FAIL(ctx, EB_ERR_UNSUPPORTED, "%s is not available on a batch context", who); \
  } while (0)

#define FAIL(ctx, code, ...)                      \
  do {                                            \
    char _b[512];                                 \
    snprintf(_b, sizeof(_b), __VA_ARGS__);        \
    (ctx)->err = _b;                              \
    return (code);                                \
  } while (0)

#define CK(ctx, call)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (call);                                                               \
    if (_e != cudaSuccess) {                                                               \
      cudaGetLastError();                                                                  \
      FAIL(ctx, EB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, \
           __LINE__);                                                                      \
    }                                                                                      \
  } while (0)

// an allocation into an owner (dev_alloc / host_alloc) that fails makes the call fail with EB_ERR_NOMEM; the
// message may name the CUDA error as cudaGetErrorString(alloc_err)
#define CK_NOMEM(ctx, call, ...)            \
  do {                                      \
    const cudaError_t alloc_err = (call);   \
    if (alloc_err != cudaSuccess) {         \
      cudaGetLastError();                   \
      FAIL(ctx, EB_ERR_NOMEM, __VA_ARGS__); \
    }                                       \
  } while (0)

// `bytes` of device memory must fit in what is free, else the call fails with EB_ERR_NOMEM: "<who>: <n> bytes of
// <what>, <free> bytes free".  Obj is an engine or a chain.
template <class Obj>
int check_free(Obj* c, const char* who, const char* what, size_t bytes) {
  size_t free_b = 0, total_b = 0;
  CK(c, cudaMemGetInfo(&free_b, &total_b));
  if (bytes > free_b) FAIL(c, EB_ERR_NOMEM, "%s: %zu bytes of %s, %zu bytes free", who, bytes, what, free_b);
  return EB_OK;
}

// allocate `bytes` of device memory into `out`, refused by check_free before anything is allocated
template <class Obj, class T>
int dev_alloc_checked(Obj* c, const char* who, const char* what, size_t bytes, DevPtr<T>& out) {
  const int rc = check_free(c, who, what, bytes);
  if (rc) return rc;
  CK_NOMEM(c, dev_alloc(out, bytes), "%s: allocating %zu bytes of %s failed (%s)", who, bytes, what,
           cudaGetErrorString(alloc_err));
  return EB_OK;
}

// an empty chain of nwalkers x ndim on `device`: its stream and its [N] accept buffers (eb_chain_create, and the ring
// of eb_window_config); synchronises
cudaError_t chain_init(eb_chain* ch, int device, int64_t nwalkers, int ndim);
// mean[D], cov[D * D] of m samples from the sums acc = [S1 | S2] about `shift` (eb_moments, eb_chain_moments):
// mean = shift + S1 / m, cov = (S2 - S1 S1^T / m) / (m - 1)   (np.cov(flatchain, rowvar=False)); NaN when m == 0
void finish_moments(const double* acc, const double* shift, uint64_t count, size_t D, double* mean, double* cov);

// a graph model (eb_model_set_graphs): its half-steps report errors through graph_err, read by fetch_status
inline bool graph_mode(const eb_ctx* c) { return c->model.kind == MODEL_EXTERNAL && c->cb_where == EB_CALLBACK_GRAPH; }
// a proposal slot holds captured graphs (eb_move_set_proposal_graphs)
inline bool proposal_graphs(const eb_ctx* c) {
  for (const eb_ctx::ProposalGraphs& p : c->prop_graphs)
    if (!p.graphs.empty()) return true;
  return false;
}
// the captured graphs of proposal slot `slot`, or null
inline const eb_ctx::ProposalGraphs* slot_graphs(const eb_ctx* c, size_t slot) {
  return slot < c->prop_graphs.size() && !c->prop_graphs[slot].graphs.empty() ? &c->prop_graphs[slot] : nullptr;
}
// half-steps report errors through graph_err: a graph model, or a captured proposal
inline bool graph_errors(const eb_ctx* c) { return graph_mode(c) || proposal_graphs(c); }
int check_status(eb_ctx* c);  // map (and clear) the status word read back last
int fetch_status(eb_ctx* c);  // read the status word back, then check_status
int enqueue_status_read(eb_ctx* c);  // the read-back of fetch_status, without its synchronisation
int run_callback(eb_ctx* c, const double* x, int64_t m, double* lp, bool scan_x);
void owned_rows(const eb_ctx* c, int64_t& r0, int64_t& r1);
int sync_replicas(eb_ctx* c);
