// The host-side step driver of the C ABI: the move schedule, the half-step launches of every move kind, the
// dense_dmma grouping, the calls into the running statistics (running.cu), and eb_step / eb_step_store /
// eb_step_store_blobs / eb_step_store_chain.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "context.h"

// ---- the hot path --------------------------------------------------------------
namespace {

struct Schedule {
  std::vector<eb_move> moves;
  std::vector<double> cdf;
  // GaussianMove: form (0 scalar, 1 diagonal, 2 full) and where its scale / Cholesky factor sits in gauss_dev
  std::vector<int> gform;
  std::vector<size_t> goff;
};

// thresholded lower Cholesky factor (the draw specification's multivariate_normal; oracle/philox.py chol_psd)
void chol_psd_host(const double* A, int D, std::vector<double>& L) {
  L.assign((size_t)D * D, 0.0);
  double m = 0.0;
  for (int j = 0; j < D; ++j) m = std::max(m, A[(size_t)j * D + j]);
  const double tol = 1e-12 * m;
  for (int j = 0; j < D; ++j) {
    double d = A[(size_t)j * D + j];
    for (int k = 0; k < j; ++k) d -= L[(size_t)j * D + k] * L[(size_t)j * D + k];
    if (!(d > tol)) continue;
    const double piv = sqrt(d);
    L[(size_t)j * D + j] = piv;
    for (int i = j + 1; i < D; ++i) {
      double v = A[(size_t)i * D + j];
      for (int k = 0; k < j; ++k) v -= L[(size_t)i * D + k] * L[(size_t)j * D + k];
      L[(size_t)i * D + j] = v / piv;
    }
  }
}

void split_starts(int64_t N, int P, int* start);  // below

// the captured graph of split `split` of a proposal slot, or null
const eb_ctx::ProposalGraph* find_proposal_graph(const eb_ctx::ProposalGraphs& p, int split) {
  for (const eb_ctx::ProposalGraph& g : p.graphs)
    if (g.split == split) return &g;
  return nullptr;
}

// a schedule entry whose proposal runs as captured graphs (eb_move_set_proposal_graphs)
bool captured_proposal(const eb_ctx* c, const eb_move& m) {
  return (m.kind == EB_MOVE_USER || m.kind == EB_MOVE_USER_MH) && slot_graphs(c, (size_t)m.p0) != nullptr;
}

// a schedule entry whose slot holds captured graphs (eb_move_set_proposal_graphs): a graph of the right size for
// every half-step it runs, and no setup call
int check_proposal_graphs(eb_ctx* c, const eb_move& m) {
  const eb_ctx::ProposalGraphs& p = *slot_graphs(c, (size_t)m.p0);
  if (m.kind == EB_MOVE_USER_MH) {
    const eb_ctx::ProposalGraph* g = find_proposal_graph(p, 0);
    if (!g || g->ns != c->N)
      FAIL(c, EB_ERR_INVALID, "eb_step: proposal slot %g has no captured graph of split 0 for all %lld walkers", m.p0,
           (long long)c->N);
    return EB_OK;
  }
  if (m.mode == EB_USER_SETUP) FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: a captured proposal has no setup call");
  if (m.nsplits < 2 || m.nsplits > MAX_SPLITS || m.nsplits > c->N) return EB_OK;  // refused below
  int start[MAX_SPLITS + 1];
  split_starts(c->N, m.nsplits, start);
  for (int j = 0; j < m.nsplits; ++j) {
    const eb_ctx::ProposalGraph* g = find_proposal_graph(p, j);
    const int64_t ns = start[j + 1] - start[j];
    if (!g || g->ns != ns || !g->b.c)
      FAIL(c, EB_ERR_INVALID, "eb_step: proposal slot %g has no captured graph of split %d for %lld rows", m.p0, j,
           (long long)ns);
  }
  return EB_OK;
}

int build_schedule(eb_ctx* c, const eb_move* moves, size_t nmoves, Schedule& s) {
  if (!moves || nmoves == 0) FAIL(c, EB_ERR_INVALID, "eb_step: empty move schedule");
  if (c->nbatch > 0) {
    // one red-blue move for every ensemble: a schedule would pick a move, and with it a split count, per ensemble
    const eb_move& m = moves[0];
    if (nmoves != 1 || (m.kind != EB_MOVE_STRETCH && m.kind != EB_MOVE_DE && m.kind != EB_MOVE_SNOOKER))
      FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: a batch runs exactly one StretchMove, DEMove or DESnookerMove");
    if (m.nsplits < 2 || m.nsplits > MAX_SPLITS || m.nsplits > c->bn)
      FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: nsplits must be in [2, min(%d, nwalkers)] (got %d)", MAX_SPLITS, m.nsplits);
    if (m.kind == EB_MOVE_DE && c->bn - (c->bn + m.nsplits - 1) / m.nsplits < 2)
      FAIL(c, EB_ERR_INVALID, "eb_step: DEMove needs at least 2 complement walkers");
  }
  s.moves.assign(moves, moves + nmoves);
  double tot = 0.0;
  s.gform.assign(nmoves, 0);
  s.goff.assign(nmoves, 0);
  std::vector<double> ghost;  // host image of gauss_dev
  for (size_t mi = 0; mi < nmoves; ++mi) {
    eb_move& m = s.moves[mi];
    if (m.kind == EB_MOVE_USER || m.kind == EB_MOVE_USER_MH) {
      if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "user proposals are not sharded across GPUs");
      if (c->debug) FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: debug taps do not cover user proposals");
      if (!(m.p0 >= 0.0 && m.p0 < (double)c->props.size()) || m.p0 != floor(m.p0) ||
          (!c->props[(size_t)m.p0].fn && !slot_graphs(c, (size_t)m.p0)))
        FAIL(c, EB_ERR_INVALID, "eb_step: proposal slot %g is not set (eb_move_set_proposal)", m.p0);
      if (!(m.weight >= 0.0) || !isfinite(m.weight)) FAIL(c, EB_ERR_INVALID, "eb_step: bad move weight");
      if (slot_graphs(c, (size_t)m.p0)) {
        const int rc = check_proposal_graphs(c, m);
        if (rc) return rc;
      }
      if (m.kind == EB_MOVE_USER_MH) {
        m.nsplits = 1;  // the split table of such a step is never read
        m.randomize_split = 0;
        tot += m.weight;
        continue;
      }
      if (m.mode != 0 && m.mode != EB_USER_SETUP) FAIL(c, EB_ERR_INVALID, "eb_step: unknown user-move mode %d", m.mode);
    } else if ((m.kind < EB_MOVE_STRETCH || m.kind > EB_MOVE_GAUSSIAN) && m.kind != EB_MOVE_KDE) {
      FAIL(c, EB_ERR_INVALID, "eb_step: unknown move kind %d", m.kind);
    }
    if (m.kind == EB_MOVE_KDE) {
      if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: KDEMove is not sharded across GPUs");
      if (c->D > 1024) FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: KDEMove is limited to ndim <= 1024");
      if (!isnan(m.p0) && m.p0 != EB_KDE_SILVERMAN && m.p0 != EB_KDE_SCALAR)
        FAIL(c, EB_ERR_INVALID, "eb_step: unknown KDEMove bandwidth rule %g", m.p0);
      if (m.p0 == EB_KDE_SCALAR && !(m.p1 > 0.0 && isfinite(m.p1)))
        FAIL(c, EB_ERR_INVALID, "eb_step: a KDEMove bandwidth must be finite and > 0 (got %g)", m.p1);
      // the smallest complement, that of the first split (scipy/stats/_kde.py gaussian_kde.__init__)
      if (m.nsplits >= 2 && m.nsplits <= MAX_SPLITS && m.nsplits <= c->N &&
          (int64_t)c->D > c->N - (c->N + m.nsplits - 1) / m.nsplits)
        FAIL(c, EB_ERR_INVALID,
             "Number of dimensions is greater than number of samples. This results in a singular data covariance "
             "matrix, which cannot be treated using the algorithms implemented in `gaussian_kde`. Note that "
             "`gaussian_kde` interprets each *column* of `dataset` to be a point; consider transposing the input to "
             "`dataset`.");
    }
    if ((m.kind == EB_MOVE_WALK || m.kind == EB_MOVE_GAUSSIAN) && c->comm.nranks > 1)
      FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: WalkMove / GaussianMove are not sharded across GPUs yet");
    if ((m.kind == EB_MOVE_WALK || m.kind == EB_MOVE_GAUSSIAN) && c->debug)
      FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: debug taps do not cover WalkMove / GaussianMove");
    if (m.kind == EB_MOVE_GAUSSIAN) {
      const size_t D = (size_t)c->D;
      if (!m.cov || (m.ncov != 1 && m.ncov != D && m.ncov != D * D) || (D == 1 && m.ncov != 1))
        FAIL(c, EB_ERR_INVALID, "Invalid proposal scale dimensions");  // gaussian.py:53-54
      if (m.mode < EB_GAUSS_VECTOR || m.mode > EB_GAUSS_SEQUENTIAL)
        FAIL(c, EB_ERR_INVALID, "eb_step: unknown GaussianMove mode %d", m.mode);
      if (!isnan(m.p1) && m.p1 < 1.0) FAIL(c, EB_ERR_INVALID, "'factor' must be >= 1.0");  // gaussian.py:69-70
      if (!(m.weight >= 0.0) || !isfinite(m.weight)) FAIL(c, EB_ERR_INVALID, "eb_step: bad move weight");
      s.goff[mi] = ghost.size();
      if (m.ncov == D * D && D > 1) {
        if (m.mode != EB_GAUSS_VECTOR)
          FAIL(c, EB_ERR_INVALID, "a full proposal covariance only supports mode 'vector'");  // gaussian.py:110-111
        s.gform[mi] = 2;
        std::vector<double> L;
        chol_psd_host(m.cov, c->D, L);
        ghost.insert(ghost.end(), L.begin(), L.end());
        ghost.resize(ghost.size() + D);  // the shared shift v[D] of a step lives behind its factor
      } else {
        s.gform[mi] = m.ncov == 1 ? 0 : 1;
        for (size_t k = 0; k < m.ncov; ++k) {
          if (!(m.cov[k] >= 0.0)) FAIL(c, EB_ERR_INVALID, "GaussianMove: variances must be >= 0");
          ghost.push_back(sqrt(m.cov[k]));  // gaussian.py:45,58
        }
      }
      m.nsplits = 1;  // the split table of such a step is never read
      m.randomize_split = 0;
      tot += m.weight;
      continue;
    }
    if (m.kind == EB_MOVE_WALK && !isnan(m.p0)) {
      const int64_t nc_min = c->N - (c->N + m.nsplits - 1) / std::max(m.nsplits, 1);
      if (m.p0 != floor(m.p0) || m.p0 < 2 || (m.nsplits >= 2 && m.p0 > (double)nc_min))
        FAIL(c, EB_ERR_INVALID, "eb_step: WalkMove needs 2 <= s <= size of the smallest complement (got %g)", m.p0);
      // launch_step_walk picks the kernel per split: a split whose own complement is larger than s runs the
      // helper-subset kernel, even when s equals the smallest complement (nwalkers not divisible by nsplits).
      // Complements grow with the split index, so the first and the last split cover every size.
      const int P = std::max(m.nsplits, 1);
      const int64_t nc_max = c->N - c->N / P;
      const bool subset = (int64_t)m.p0 != nc_min || (int64_t)m.p0 != nc_max;
      if (subset && !walk_subset_supported(c->D, (int)m.p0))
        FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: WalkMove with a helper subset is limited to ndim <= 64 and s <= 4096");
    }
    if (m.kind == EB_MOVE_WALK && c->D > 1024) FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: WalkMove is limited to ndim <= 1024");
    if (m.nsplits < 2 || m.nsplits > MAX_SPLITS || m.nsplits > c->N)
      FAIL(c, EB_ERR_UNSUPPORTED, "eb_step: nsplits must be in [2, min(%d, nwalkers)] (got %d)", MAX_SPLITS,
           m.nsplits);
    if (m.kind == EB_MOVE_SNOOKER && m.nsplits != 4)
      FAIL(c, EB_ERR_INVALID, "eb_step: DESnookerMove uses nsplits = 4 (de_snooker.py:28)");
    if (m.kind == EB_MOVE_DE && c->N - (c->N + m.nsplits - 1) / m.nsplits < 2)
      FAIL(c, EB_ERR_INVALID, "eb_step: DEMove needs at least 2 complement walkers");
    if (!(m.weight >= 0.0) || !isfinite(m.weight)) FAIL(c, EB_ERR_INVALID, "eb_step: bad move weight");
    if (m.kind == EB_MOVE_STRETCH && !(m.p0 > 0.0)) FAIL(c, EB_ERR_INVALID, "eb_step: stretch scale a must be > 0");
    tot += m.weight;
  }
  if (!(tot > 0.0)) FAIL(c, EB_ERR_INVALID, "eb_step: move weights sum to zero");
  if (!ghost.empty()) {
    if (ghost.size() > c->gauss_cap) {
      CK(c, cudaStreamSynchronize(c->st.get()));
      CK(c, dev_alloc(c->gauss_dev, ghost.size() * sizeof(double)));
      c->gauss_cap = ghost.size();
    }
    CK(c, cudaMemcpyAsync(c->gauss_dev.get(), ghost.data(), ghost.size() * sizeof(double), cudaMemcpyHostToDevice,
                          c->st.get()));
    CK(c, cudaStreamSynchronize(c->st.get()));  // ghost is a local
  }
  c->picks.assign(nmoves, 0);
  // ensemble.py:128-129 then RandomState.choice(p=...): cdf = cumsum(p); cdf /= cdf[-1]
  s.cdf.resize(nmoves);
  double run = 0.0;
  for (size_t k = 0; k < nmoves; ++k) {
    run += s.moves[k].weight / tot;
    s.cdf[k] = run;
  }
  for (size_t k = 0; k < nmoves; ++k) s.cdf[k] /= run;
  return EB_OK;
}

// ensemble.py:406 -- one move per step for the whole ensemble
size_t choose_move(const eb_ctx* c, const Schedule& s, uint64_t step) {
  if (s.moves.size() == 1) return 0;
  const u32x4 w = draw_words(c->seed, step, 0, TAG_MOVE, 0);
  const double u = u53(w.x, w.y);
  size_t idx = 0;
  while (idx + 1 < s.cdf.size() && !(s.cdf[idx] > u)) ++idx;  // searchsorted(side="right")
  return idx;
}

void split_starts(int64_t N, int P, int* start) {
  start[0] = 0;
  for (int j = 0; j < P; ++j) start[j + 1] = start[j] + (int)((N - j + P - 1) / P);
}

// the arguments every half-step of move mv shares: the engine's buffers, model and options, the move's parameters
HalfStepArgs move_args(const eb_ctx* c, const eb_move& mv) {
  HalfStepArgs a{};
  a.coords = c->coords.get();
  a.logp = c->logp.get();
  a.accepted = c->accepted.get();
  a.nacc = c->nacc.get();
  a.status = c->status_dev.get();
  a.N = c->N;
  a.D = c->D;
  a.seed = c->seed;
  a.model = c->model;
  if (c->debug) {
    a.tap_partners = c->tap_partners.get();
    a.tap_scalar = c->tap_scalar.get();
    a.tap_u = c->tap_u.get();
    a.tap_active = c->tap_active.get();
  }
  switch (mv.kind) {
    case EB_MOVE_STRETCH:
      a.p0 = mv.p0;
      break;
    case EB_MOVE_DE:
      a.p0 = isnan(mv.p1) ? 2.38 / sqrt(2.0 * (double)c->D) : mv.p1;  // de.py:33-38
      a.p1 = mv.p0;                                                    // sigma
      break;
    default:
      a.p0 = mv.p0;  // gammas
  }
  a.timeline = c->timeline.get();
  a.dmma_stagger = c->dmma_stagger;
  comm_fill_args(c->comm, a);
  return a;
}

// half-step `split` of move mv at `step`, whose split table is table `tbl` of the chunk and whose splits start at
// start[0 .. nsplits] (split_starts).  The snooker complement sets are the other splits in ascending order.
HalfStepArgs split_args(const eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, const int* start, int split) {
  HalfStepArgs a = move_args(c, mv);
  a.order = c->order.get() + tbl * (size_t)c->N;
  a.step = step;
  a.split = split;
  a.a_start = start[split];
  a.a_count = start[split + 1] - start[split];
  int k = 0;
  for (int j = 0; j < mv.nsplits && k < 3; ++j) {
    if (j == split) continue;
    a.c_start[k] = start[j];
    a.c_count[k] = start[j + 1] - start[j];
    ++k;
  }
  comm_active_range(c->comm, a, tbl);  // i_lo / i_hi for this rank
  a.qbuf = c->qbuf.get();
  return a;
}

// the one half-step of a step that moves every walker at once, in walker order (GaussianMove, a user MHMove)
HalfStepArgs ensemble_args(const eb_ctx* c, const eb_move& mv, uint64_t step) {
  HalfStepArgs a = move_args(c, mv);
  a.step = step;
  a.a_count = (int)c->N;
  a.i_hi = (int)c->N;
  a.qbuf = c->qbuf.get();
  return a;
}

// eb_last_kernel_name / eb_last_kernel_variant: the kernel of the last half-step and the parameters it chose
__attribute__((format(printf, 3, 4))) void note_kernel(eb_ctx* c, const char* name, const char* fmt, ...) {
  c->last_kernel = name;
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(c->last_variant, sizeof(c->last_variant), fmt, ap);
  va_end(ap);
}

void note_callback(eb_ctx* c) {
  note_kernel(c, "callback", "callback G=%d where=%s", lanes_per_walker(c->D),
              c->cb_where == EB_CALLBACK_HOST ? "host" : c->cb_where == EB_CALLBACK_GRAPH ? "graph" : "device");
}

bool dmma_eligible(const eb_ctx* c, const eb_move& mv) {
  return c->allow_dmma && mv.kind == EB_MOVE_STRETCH && c->model.kind == EB_MODEL_GAUSS_DENSE &&
         c->model.chol != nullptr && !c->debug;
}

int check_walker_count(eb_ctx* c, const eb_move& mv) {
  if ((c->nbatch > 0 ? c->bn : c->N) < 2 * (int64_t)c->D && !mv.live_dangerously)  // red_blue.py:64-70
    FAIL(c, EB_ERR_FEW_WALKERS,
         "It is unadvisable to use a red-blue move with fewer walkers than twice the number of dimensions.");
  return EB_OK;
}

// the accept of a half-step whose proposals are in qbuf, with Hastings factors f (or none), under a
// log-probability function (eb_model_set_callback): the function, the accept launch -- a user MHMove's (kind
// EB_MOVE_USER_MH) or the callback model's --, then the blob select when the state has blobs.  The fused kernel's
// propose phase (factors in ext_f) raises the non-finite flags of its rows itself; every other proposal is scanned.
int external_accept(eb_ctx* c, int kind, const HalfStepArgs& a, double* f, uint64_t& launches) {
  const ExternalBufs ext{c->qbuf.get(), f, c->ext_lp.get()};
  c->cb_phase = CB_STEP;
  c->cb_split = a.split;
  const int rc = run_callback(c, c->qbuf.get(), (int64_t)a.i_hi - a.i_lo, c->ext_lp.get(), f != c->ext_f.get());
  if (rc) return rc;
  if (kind == EB_MOVE_USER_MH)
    CK(c, launch_half_step_user(EB_MOVE_USER_MH, a, ext, c->st.get()));
  else
    CK(c, launch_half_step_external(MOVE_PRECOMPUTED, a, ext, c->st.get()));
  ++launches;
  if (c->blobs_live) {  // accepted walkers take their proposal's record (moves/move.py:36-43)
    CK(c, launch_blob_select(a.order, a.a_start, a.i_lo, a.i_hi, a.accepted, c->blob_prop.get(), c->blob_live.get(),
                             c->blob_bytes, c->st.get()));
    ++launches;
  }
  return EB_OK;
}

// the accept of the proposals a move's own kernels left in qbuf (WalkMove, GaussianMove)
int accept_precomputed(eb_ctx* c, const HalfStepArgs& a, uint64_t& launches) {
  if (c->model.kind == MODEL_EXTERNAL) {
    const int rc = external_accept(c, MOVE_PRECOMPUTED, a, nullptr, launches);
    if (rc) return rc;
    note_callback(c);
    return EB_OK;
  }
  CK(c, launch_half_step_generic(MOVE_PRECOMPUTED, a, c->st.get()));
  ++launches;
  return EB_OK;
}

// launch the P half-steps of one step with the generic kernels (one launch per split); under a log-probability
// function each is the fused kernel's propose phase, then the function and the accept
int launch_step_generic(eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, uint64_t& launches) {
  int rc = check_walker_count(c, mv);
  if (rc) return rc;
  int start[MAX_SPLITS + 1];
  split_starts(c->N, mv.nsplits, start);
  for (int split = 0; split < mv.nsplits; ++split) {
    const HalfStepArgs a = split_args(c, mv, step, tbl, start, split);
    if (c->fused_last) {
      // the previous launch was a dense_dmma kernel that carried the peer barrier itself (signal at its end);
      // this kernel does not wait on its own, so the ranks meet explicitly before it reads peer rows
      if (comm_barrier(c->comm, c->st.get(), c->status_dev.get(), launches))
        FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
      c->fused_last = false;
    }
    if (c->model.kind == MODEL_EXTERNAL) {
      CK(c, launch_half_step_external(mv.kind, a, ExternalBufs{c->qbuf.get(), c->ext_f.get(), c->ext_lp.get()},
                                      c->st.get()));
      ++launches;
      rc = external_accept(c, mv.kind, a, c->ext_f.get(), launches);
      if (rc) return rc;
      note_callback(c);
      c->tap_count = a.a_count;
      continue;
    }
    bool used_tma = false;
    TmaVariant tv{};
    if (c->allow_tma && !c->debug)
      CK(c, launch_half_step_tma(mv.kind, a, c->sm_count, c->allow_tma >= 2, c->tma_own_reg, c->st.get(), &used_tma,
                                 &tv));
    if (used_tma) {
      note_kernel(c, "tma_rows", "tma_rows R=%d epl=%d own_reg=%d warps=%d", tv.R, tv.epl, tv.own_reg, tv.warps);
    } else {
      CK(c, launch_half_step_generic(mv.kind, a, c->st.get()));
      note_kernel(c, "generic", "generic G=%d", lanes_per_walker(c->D));
    }
    ++launches;
    c->tap_count = a.a_count;
    if (comm_after_split(c->comm, c->st.get(), c->status_dev.get(), launches))
      FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  }
  return EB_OK;
}

// the P half-steps of one step of every ensemble of a batch context: one launch each, or under a log-probability
// function the propose launch, the function on the [K, a_count] block, and the accept launch
int launch_step_batch(eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, uint64_t& launches) {
  int rc = check_walker_count(c, mv);
  if (rc) return rc;
  int start[MAX_SPLITS + 1];
  split_starts(c->bn, mv.nsplits, start);
  const HalfStepArgs m = move_args(c, mv);
  const bool external = c->model.kind == MODEL_EXTERNAL;
  const ExternalBufs ext{c->qbuf.get(), c->ext_f.get(), c->ext_lp.get()};
  for (int split = 0; split < mv.nsplits; ++split) {
    BatchArgs a{};
    a.coords = c->coords.get();
    a.logp = c->logp.get();
    a.accepted = c->accepted.get();
    a.nacc = c->nacc.get();
    a.status = c->status_dev.get();
    a.order = c->order.get() + tbl * (size_t)c->N;
    a.seeds = c->seeds_dev.get();
    a.n = c->bn;
    a.K = c->nbatch;
    a.D = c->D;
    a.split = split;
    a.a_start = start[split];
    a.a_count = start[split + 1] - start[split];
    int k = 0;
    for (int j = 0; j < mv.nsplits && k < 3; ++j) {
      if (j == split) continue;
      a.c_start[k] = start[j];
      a.c_count[k] = start[j + 1] - start[j];
      ++k;
    }
    a.step = step;
    a.p0 = m.p0;
    a.p1 = m.p1;
    a.model = c->model;
    a.qbuf = c->qbuf.get();
    CK(c, launch_batch_half_step(mv.kind, a, ext, c->st.get()));
    ++launches;
    if (!external) continue;
    c->cb_phase = CB_STEP;
    c->cb_split = split;
    rc = run_callback(c, c->qbuf.get(), c->nbatch * a.a_count, c->ext_lp.get(), false);
    if (rc) return rc;
    CK(c, launch_batch_half_step(MOVE_PRECOMPUTED, a, ext, c->st.get()));
    ++launches;
  }
  if (external)
    note_callback(c);
  else
    note_kernel(c, "batch", "batch G=%d K=%lld", lanes_per_walker(c->D), (long long)c->nbatch);
  return EB_OK;
}

int ensure_move_scratch(eb_ctx* c) {
  const size_t D = (size_t)c->D;
  if (!c->qbuf) CK(c, dev_alloc(c->qbuf, (size_t)c->N * D * sizeof(double)));
  if (!c->walk_work && D <= 1024) CK(c, dev_alloc(c->walk_work, (2 * D + 3 * D * D) * sizeof(double)));
  if (!c->mom_partial && D <= 1024) CK(c, dev_alloc(c->mom_partial, moments_partial_bytes(c->D, c->sm_count)));
  return EB_OK;
}

// WalkMove (walk.py:27-37): per split a proposal kernel writes q[a_count, D], then the fused
// log-prob + accept + update kernel consumes it
int launch_step_walk(eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, uint64_t& launches) {
  int rc = check_walker_count(c, mv);
  if (rc) return rc;
  rc = ensure_move_scratch(c);
  if (rc) return rc;
  int start[MAX_SPLITS + 1];
  split_starts(c->N, mv.nsplits, start);
  const size_t D = (size_t)c->D;
  double* shift = c->walk_work.get();
  double* acc = shift + D;
  double* cov = acc + D + D * D;
  double* L = cov + D * D;
  for (int split = 0; split < mv.nsplits; ++split) {
    const HalfStepArgs a = split_args(c, mv, step, tbl, start, split);
    const int64_t Nc = c->N - a.a_count;
    const int64_t s0 = isnan(mv.p0) ? Nc : (int64_t)mv.p0;  // walk.py:32
    if (s0 == Nc) {
      // every walker of the split draws from the covariance of the WHOLE complement (walk.py:34-35 with a
      // permutation of all Nc rows): computed once -- moment sums on the tensor pipe, then a D x D factorisation
      // any shift will do: the ensemble mean
      CK(c, launch_colmean(c->coords.get(), c->N, c->D, shift, nullptr, c->st.get()));
      CK(c, cudaMemsetAsync(acc, 0, (D + D * D) * sizeof(double), c->st.get()));
      CK(c, launch_moments(c->coords.get(), Nc, c->D, shift, c->mom_partial.get(), acc, c->sm_count, c->st.get(),
                           a.order, a.a_start, a.a_count));
      CK(c, launch_cov_chol(acc, (double)Nc, c->D, cov, L, c->st.get()));
      CK(c, launch_walk_shared_propose(a, L, c->qbuf.get(), c->st.get()));
      launches += 5;
    } else {
      CK(c, launch_walk_subset_propose(a, (int)s0, c->qbuf.get(), c->st.get()));
      ++launches;
    }
    rc = accept_precomputed(c, a, launches);
    if (rc) return rc;
  }
  if (c->model.kind != MODEL_EXTERNAL) note_kernel(c, "walk", "walk");
  return EB_OK;
}

// scipy's bandwidth factor of a KDE of n uniformly weighted points (gaussian_kde.scotts_factor / silverman_factor;
// neff = n)
double kde_bandwidth(const eb_move& mv, int64_t n, int D) {
  if (mv.p0 == EB_KDE_SCALAR) return mv.p1;
  const double neff = (double)n;
  if (mv.p0 == EB_KDE_SILVERMAN) return pow(neff * (D + 2.0) / 4.0, -1.0 / (D + 4));
  return pow(neff, -1.0 / (D + 4));
}

int ensure_kde_scratch(eb_ctx* c) {
  if (c->kde_y) return EB_OK;
  const size_t N = (size_t)c->N, D = (size_t)c->D;
  DevPtr<double> y, f, part, mat;
  DevPtr<int64_t> j;
  CK(c, dev_alloc(y, (N + N / 2 + 1) * D * sizeof(double)));
  CK(c, dev_alloc(f, N * sizeof(double)));
  CK(c, dev_alloc(j, N * sizeof(int64_t)));
  CK(c, dev_alloc(part, kde_partial_doubles(c->N, c->sm_count) * sizeof(double)));
  CK(c, dev_alloc(mat, (D * D + D) * sizeof(double)));
  c->kde_y = std::move(y);
  c->kde_f = std::move(f);
  c->kde_j = std::move(j);
  c->kde_part = std::move(part);
  c->kde_mat = std::move(mat);
  return EB_OK;
}

// KDEMove (kde.py:39-43): per split the complement covariance and factor as the whole-complement WalkMove's, then
// kde.cu's kernels write the proposals and their Hastings factors, and the accept of precomputed rows takes them.
// A singular factor stops the call here, before this split's update: the status read synchronises once per split.
int launch_step_kde(eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, uint64_t& launches) {
  int rc = check_walker_count(c, mv);
  if (rc) return rc;
  rc = ensure_move_scratch(c);
  if (rc) return rc;
  rc = ensure_kde_scratch(c);
  if (rc) return rc;
  int start[MAX_SPLITS + 1];
  split_starts(c->N, mv.nsplits, start);
  const size_t D = (size_t)c->D;
  double* shift = c->walk_work.get();
  double* acc = shift + D;
  double* cov = acc + D + D * D;
  double* L = cov + D * D;
  double* minv = c->kde_mat.get();
  double* mean = minv + D * D;
  KdePlan plan{};
  for (int split = 0; split < mv.nsplits; ++split) {
    const HalfStepArgs a = split_args(c, mv, step, tbl, start, split);
    const int64_t ns = a.a_count, nc = c->N - a.a_count;
    const double bw = kde_bandwidth(mv, nc, c->D);
    CK(c, launch_colmean(c->coords.get(), c->N, c->D, shift, nullptr, c->st.get()));
    CK(c, cudaMemsetAsync(acc, 0, (D + D * D) * sizeof(double), c->st.get()));
    CK(c, launch_moments(c->coords.get(), nc, c->D, shift, c->mom_partial.get(), acc, c->sm_count, c->st.get(),
                         a.order, a.a_start, a.a_count));
    CK(c, launch_cov_chol(acc, (double)nc, c->D, cov, L, c->st.get()));
    CK(c, launch_kde_factor(L, acc, shift, (double)nc, c->D, bw, minv, mean, c->status_dev.get(), c->st.get()));
    launches += 5;
    rc = fetch_status(c);
    if (rc) return rc;
    double* yp = c->kde_y.get();
    double* yc = yp + (size_t)2 * ns * D;
    CK(c, launch_kde_prepare(a, L, minv, mean, bw, c->qbuf.get(), yp, yc, c->kde_j.get(), c->st.get()));
    plan = kde_plan(ns, nc, c->sm_count);
    CK(c, launch_kde_factors(yp, yc, ns, nc, c->D, plan, c->kde_part.get(), c->kde_f.get(), c->st.get()));
    launches += 3;
    if (c->model.kind == MODEL_EXTERNAL) {
      rc = external_accept(c, MOVE_PRECOMPUTED, a, c->kde_f.get(), launches);
      if (rc) return rc;
      note_callback(c);
    } else {
      CK(c, launch_half_step_user(EB_MOVE_USER, a, ExternalBufs{c->qbuf.get(), c->kde_f.get(), nullptr}, c->st.get()));
      ++launches;
    }
    if (c->debug) {  // the accept wrote the uniforms and walkers; the centres and factors are this move's
      CK(c, cudaMemcpyAsync(c->tap_partners.get(), c->kde_j.get(), (size_t)ns * sizeof(int64_t),
                            cudaMemcpyDeviceToDevice, c->st.get()));
      CK(c, cudaMemcpyAsync(c->tap_scalar.get(), c->kde_f.get(), (size_t)ns * sizeof(double), cudaMemcpyDeviceToDevice,
                            c->st.get()));
      c->tap_count = a.a_count;
    }
  }
  if (c->model.kind != MODEL_EXTERNAL)
    note_kernel(c, "kde", "kde tpc=%d nchunks=%d", plan.tpc, plan.nchunks);
  return EB_OK;
}

// MHMove with the Gaussian proposal (mh.py:35-65, gaussian.py:72-119): every walker is proposed at once
int launch_step_gaussian(eb_ctx* c, const Schedule& s, size_t mi, uint64_t step, uint64_t& launches) {
  const eb_move& mv = s.moves[mi];
  int rc = ensure_move_scratch(c);
  if (rc) return rc;
  const int D = c->D;
  double f = 1.0;
  if (!isnan(mv.p1)) {  // gaussian.py:88-91  exp(uniform(-log f, log f))
    const u32x4 w = draw_words(c->seed, step, 0, TAG_MOVE, 1);
    const double lf = log(mv.p1);
    f = exp(-lf + (lf - (-lf)) * u53(w.x, w.y));
  }
  const int seq_dim = (int)(((uint64_t)mv.seq_index + c->picks[mi]) % (uint64_t)D);  // gaussian.py:102-103
  const double* dev = c->gauss_dev.get() + s.goff[mi];
  const int form = s.gform[mi];
  const double* scale = dev;
  if (form == 2) {
    double* v = c->gauss_dev.get() + s.goff[mi] + (size_t)D * D;
    CK(c, launch_gaussian_shift(dev, D, f, c->seed, step, v, c->st.get()));
    scale = v;
    ++launches;
  }
  CK(c, launch_gaussian_propose(c->coords.get(), 0, c->N, D, form, scale, f, mv.mode, seq_dim, c->seed, step,
                                c->qbuf.get(), c->st.get()));
  ++launches;
  rc = accept_precomputed(c, ensemble_args(c, mv, step), launches);
  if (rc) return rc;
  if (c->model.kind != MODEL_EXTERNAL) note_kernel(c, "gaussian", "gaussian");
  return EB_OK;
}

// ---- user proposals (eb_move_set_proposal) ----------------------------------------------------------
int ensure_user_scratch(eb_ctx* c, bool host) {
  const size_t N = (size_t)c->N, D = (size_t)c->D;
  if (!c->qbuf) CK(c, dev_alloc(c->qbuf, N * D * sizeof(double)));
  if (!c->up_x) CK(c, dev_alloc(c->up_x, N * D * sizeof(double)));
  if (!c->up_f) CK(c, dev_alloc(c->up_f, N * sizeof(double)));
  if (host && !c->up_hf) {
    HostPtr<double> hx, hq, hf;
    CK(c, host_alloc(hx, N * D * sizeof(double)));
    CK(c, host_alloc(hq, N * D * sizeof(double)));
    CK(c, host_alloc(hf, N * sizeof(double)));
    c->up_hx = std::move(hx);
    c->up_hq = std::move(hq);
    c->up_hf = std::move(hf);
  }
  return EB_OK;
}

// steps 2-5 of a user half-step (include/emcee_b200.h): rows[N, D] (device; s then c, or the ensemble) are
// enqueued.  ns > 0: the proposal of ns rows lands in qbuf / up_f; ns == 0: the setup call, which returns nothing
int user_proposal_call(eb_ctx* c, const eb_ctx::ProposalSlot& p, uint64_t step, int split, const double* rows,
                       int64_t ns, const int64_t* counts, int nsets) {
  const size_t N = (size_t)c->N, D = (size_t)c->D;
  const bool host = p.where == EB_CALLBACK_HOST;
  // the function gets its own copy of the rows
  if (host)
    CK(c, cudaMemcpyAsync(c->up_hx.get(), rows, N * D * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
  else if (rows != c->up_x.get())
    CK(c, cudaMemcpyAsync(c->up_x.get(), rows, N * D * sizeof(double), cudaMemcpyDeviceToDevice, c->st.get()));
  // complete before fn runs (a device consumer may ignore the stream it is given); the errors of a graph model or a
  // captured proposal so far stop the call here, so that the function never sees the state past one
  if (graph_errors(c)) {
    const int rc = fetch_status(c);
    if (rc) return rc;
  } else {
    CK(c, cudaStreamSynchronize(c->st.get()));
  }
  const double* s = host ? c->up_hx.get() : c->up_x.get();
  const double* cset = nsets > 0 ? s + (size_t)ns * D : nullptr;
  double* q = ns > 0 ? (host ? c->up_hq.get() : c->qbuf.get()) : nullptr;
  double* f = ns > 0 ? (host ? c->up_hf.get() : c->up_f.get()) : nullptr;
  c->up_m = ns;
  c->up_where = p.where;
  c->in_proposal = true;
  const int r = p.fn(p.user, step, (int32_t)split, s, ns > 0 ? ns : (int64_t)N, cset, nsets > 0 ? counts : nullptr,
                     nsets, (int64_t)D, q, f, host ? nullptr : (void*)c->st.get());
  c->in_proposal = false;
  c->up_m = 0;
  if (r != 0) {
    cudaStreamSynchronize(c->st.get());  // whatever the function enqueued before it failed
    FAIL(c, EB_ERR_CALLBACK, "the user proposal failed (returned %d)", r);
  }
  if (ns == 0) return EB_OK;
  if (host) {
    CK(c, cudaMemcpyAsync(c->qbuf.get(), c->up_hq.get(), (size_t)ns * D * sizeof(double), cudaMemcpyHostToDevice,
                          c->st.get()));
    CK(c, cudaMemcpyAsync(c->up_f.get(), c->up_hf.get(), (size_t)ns * sizeof(double), cudaMemcpyHostToDevice,
                          c->st.get()));
  }
  if (c->model.kind == MODEL_EXTERNAL) return EB_OK;  // run_callback scans the rows before the function sees them
  // ensemble.py:476-479: a non-finite proposal stops the call before any log-probability is evaluated
  CK(c, launch_scan_nonfinite(c->qbuf.get(), (size_t)ns * D, 0, c->status_dev.get(), c->st.get()));
  return fetch_status(c);
}

// step 6: the log-probability of qbuf's rows and the accept + update (kind EB_MOVE_USER / EB_MOVE_USER_MH)
int user_accept(eb_ctx* c, const eb_ctx::ProposalSlot& p, int kind, const HalfStepArgs& a, uint64_t& launches) {
  if (c->model.kind == MODEL_EXTERNAL) {
    const int rc = external_accept(c, kind, a, c->up_f.get(), launches);
    if (rc) return rc;
  } else {
    CK(c, launch_half_step_user(kind, a, ExternalBufs{c->qbuf.get(), c->up_f.get(), c->ext_lp.get()}, c->st.get()));
    ++launches;
  }
  note_kernel(c, "user_move", "user_move where=%s",
              p.where == EB_CALLBACK_HOST ? "host" : p.where == EB_CALLBACK_GRAPH ? "graph" : "device");
  return EB_OK;
}

// steps 1-3 of a captured proposal's half-step (eb_move_set_proposal_graphs), all enqueued: the gather of s and c
// (split table `order`; null: an MHMove, every walker in walker order) with the draws, the graph, the read of q and
// the factors into qbuf / up_f
int graph_proposal(eb_ctx* c, const eb_ctx::ProposalGraphs& p, const HalfStepArgs& a, const int32_t* order,
                   uint64_t& launches) {
  const eb_ctx::ProposalGraph& g = *find_proposal_graph(p, a.split);  // build_schedule checked it is there
  const unsigned long long tag = graph_err_word(0, (unsigned)a.split, a.step);
  CK(c, launch_graph_move_stage(c->coords.get(), order, c->N, c->D, a.a_start, a.a_count, g.b,
                                p.draw_kind == EB_DRAW_NORMAL, p.ndraws, c->seed, a.step, (uint32_t)a.split,
                                c->status_dev.get(), c->graph_err.get(), tag, c->st.get()));
  CK(c, cudaGraphLaunch(g.exec, c->st.get()));
  CK(c, launch_graph_move_result(g.b, a.a_count, c->D, c->qbuf.get(), c->up_f.get(), c->status_dev.get(),
                                 c->gm_ticket.get(), c->graph_err.get(), tag, c->st.get()));
  launches += 3;
  c->gm_unchecked = true;
  return EB_OK;
}

// a RedBlueMove with a user get_proposal (red_blue.py:52-106): per split the gather, the function, the accept
int launch_step_user(eb_ctx* c, const eb_move& mv, uint64_t step, size_t tbl, uint64_t& launches) {
  int rc = check_walker_count(c, mv);
  if (rc) return rc;
  if (const eb_ctx::ProposalGraphs* g = slot_graphs(c, (size_t)mv.p0)) {  // captured graphs: no host work per half-step
    int start[MAX_SPLITS + 1];
    split_starts(c->N, mv.nsplits, start);
    for (int split = 0; split < mv.nsplits; ++split) {
      const HalfStepArgs a = split_args(c, mv, step, tbl, start, split);
      rc = graph_proposal(c, *g, a, a.order, launches);
      if (!rc) rc = user_accept(c, c->props[(size_t)mv.p0], EB_MOVE_USER, a, launches);
      if (rc) return rc;
    }
    return EB_OK;
  }
  const eb_ctx::ProposalSlot p = c->props[(size_t)mv.p0];
  rc = ensure_user_scratch(c, p.where == EB_CALLBACK_HOST);
  if (rc) return rc;
  if (mv.mode == EB_USER_SETUP) {  // red_blue.py:73 setup(state.coords), once per step before the splits
    rc = user_proposal_call(c, p, step, -1, c->coords.get(), 0, nullptr, 0);
    if (rc) return rc;
  }
  const int P = mv.nsplits;
  int start[MAX_SPLITS + 1];
  split_starts(c->N, P, start);
  for (int split = 0; split < P; ++split) {
    const HalfStepArgs a = split_args(c, mv, step, tbl, start, split);
    int64_t counts[MAX_SPLITS];
    int k = 0;
    for (int j = 0; j < P; ++j)
      if (j != split) counts[k++] = start[j + 1] - start[j];
    CK(c, launch_split_gather(c->coords.get(), a.order, c->N, c->D, a.a_start, a.a_count, c->up_x.get(),
                              c->st.get()));
    ++launches;
    rc = user_proposal_call(c, p, step, split, c->up_x.get(), a.a_count, counts, P - 1);
    if (rc) return rc;
    rc = user_accept(c, p, EB_MOVE_USER, a, launches);
    if (rc) return rc;
  }
  return EB_OK;
}

// MHMove with a user proposal_function (mh.py:35-65): the whole ensemble in walker order, one accept launch
int launch_step_user_mh(eb_ctx* c, const eb_move& mv, uint64_t step, uint64_t& launches) {
  if (const eb_ctx::ProposalGraphs* g = slot_graphs(c, (size_t)mv.p0)) {  // a captured graph
    const HalfStepArgs a = ensemble_args(c, mv, step);
    const int rc = graph_proposal(c, *g, a, nullptr, launches);
    return rc ? rc : user_accept(c, c->props[(size_t)mv.p0], EB_MOVE_USER_MH, a, launches);
  }
  const eb_ctx::ProposalSlot p = c->props[(size_t)mv.p0];
  int rc = ensure_user_scratch(c, p.where == EB_CALLBACK_HOST);
  if (rc) return rc;
  rc = user_proposal_call(c, p, step, 0, c->coords.get(), c->N, nullptr, 0);
  if (rc) return rc;
  return user_accept(c, p, EB_MOVE_USER_MH, ensemble_args(c, mv, step), launches);
}

constexpr int DMMA_TILE_SLOTS = 8;  // consumer warps per SM of the dense_dmma kernel

// a run of consecutive half-steps handed to ONE persistent dense_dmma launch
struct DmmaGroup {
  size_t first = 0;  // index into the chunk's HalfDesc array
  int nhalf = 0;
  int max_count = 0;
};

// The dense_dmma launches of one stepping call.  `live` holds while the last operation enqueued on the stream is a
// dense_dmma launch of this call: only then may the next launch be its programmatic dependent (PDL), and only then
// do `first` / `last`, the first and last half-step of that launch, tell which rows it may still be writing.
// run_steps clears `live` behind everything else it enqueues.
struct DmmaChain {
  bool live = false;
  HalfDesc first{}, last{};
};

int flush_dmma(eb_ctx* c, const eb_move& mv, DmmaGroup& grp, DmmaChain& chain, uint64_t& launches) {
  if (grp.nhalf == 0) return EB_OK;
  HalfStepArgs a = move_args(c, mv);
  a.order = c->order.get();  // chunk base; HalfDesc::order_step selects the table
  a.range = c->comm.nranks > 1 ? c->comm.ranges : nullptr;
  int bound = grp.max_count;
  if (c->comm.nranks > 1 && c->comm.rows_per_rank < bound) bound = (int)c->comm.rows_per_rank;
  // Locality-sorted tiles hide the peer barrier and the first remote fetch behind local work, but move the
  // remote burst to the second round: the gain or loss depends on the GPU count -- hence off by default; "auto"
  // (option value 1) enables it when a consumer warp has at most ~2 tiles per half-step.
  const bool few_tiles = (bound + 7) / 8 <= 2 * DMMA_TILE_SLOTS * c->sm_count;
  a.aperm = (c->comm.nranks > 1 && (c->local_first == 2 || (c->local_first == 1 && few_tiles))) ? c->comm.aperm : nullptr;
  // P2P: the peer barrier rides inside the kernel (wait at its start, between its half-steps, signal at its end)
  const bool fused = comm_fuse_barrier(c->comm, a, grp.nhalf);
  c->fused_last = fused;
  // (sharded ensembles: measured slower with the dependent launch -- the early CTAs only add pollers on the
  // peer flags -- so it is opt-in there: option "pdl" = 2)
  const bool pdl = chain.live && grp.nhalf == 1 && (c->comm.nranks > 1 ? c->pdl >= 2 : c->pdl >= 1);
  // The predecessor ran only earlier splits of the same step, the last one being split - 1: they write only
  // their own active walkers, so this split's rows may be requested before the predecessor has finished.
  // Not across a step boundary (a randomised split can write any row), not sharded (peer GPUs write rows too).
  const HalfDesc& d0 = c->descs_host.get()[grp.first];
  a.dmma_early_own = pdl && c->comm.nranks == 1 && d0.split > 0 && chain.first.step == d0.step &&
                     chain.first.order_step == d0.order_step && chain.last.step == d0.step &&
                     chain.last.split == d0.split - 1;
  // "dmma_timeline" = 2: the other launches run uninstrumented, so the stamps left are those of a first split
  if (c->timeline_first_split && d0.split != 0) a.timeline = nullptr;
  int grid = 0;
  CK(c, launch_dense_dmma(a, c->descs_host.get()[grp.first], c->descs_dev.get() + grp.first, grp.nhalf, bound,
                          c->gbar.get(), c->gbar_count, c->sm_count, pdl, &grid, c->st.get()));
  c->gbar_count += (unsigned long long)(grp.nhalf - 1) * (unsigned long long)grid;
  c->dmma_nhalf_max = std::max(c->dmma_nhalf_max, grp.nhalf);
  note_kernel(c, "dense_dmma", "dense_dmma nhalf_max=%d grid=%d", c->dmma_nhalf_max, grid);
  chain.live = grid > 0;
  chain.first = c->descs_host.get()[grp.first];
  chain.last = c->descs_host.get()[grp.first + grp.nhalf - 1];
  ++launches;
  grp = DmmaGroup{};
  return EB_OK;
}

// the steps [c->step, c->step + pick.size()) of one chunk
struct Chunk {
  std::vector<size_t> pick;  // the schedule entry of each step
  size_t off = 0;            // the split table of the first step, in c->order
  size_t build = 0;          // split tables to build from info_host before the first step (0: cached ones cover it)
  size_t ndesc = 0;          // dense_dmma half-step descriptors in descs_host
};

// Picks the moves of the next n steps, finds their split tables on the device or plans their build, and writes
// the dense_dmma descriptors.  Waits for the stream first: info_host / descs_host are reused per chunk.
int prepare_chunk(eb_ctx* c, const Schedule& s, size_t n, Chunk& ch) {
  CK(c, cudaStreamSynchronize(c->st.get()));
  ch.pick.resize(n);
  for (size_t k = 0; k < n; ++k) {
    ch.pick[k] = choose_move(c, s, c->step + k);
    const eb_move& mv = s.moves[ch.pick[k]];
    c->info_host.get()[k].nsplits = mv.nsplits;
    c->info_host.get()[k].randomize = mv.randomize_split;
  }
  // Split tables depend only on (seed, step, nsplits, randomize): reuse the ones already on the
  // device when they cover this chunk, else build them -- looking ahead with the same schedule, so
  // a caller that steps one iteration per call pays for one table launch every 64 calls, not one each.
  ch.off = 0;
  ch.build = 0;
  bool hit = c->tbl_n > 0 && c->tbl_seed == c->seed && c->step >= c->tbl_step0 && c->step + n <= c->tbl_step0 + c->tbl_n;
  if (hit) {
    ch.off = (size_t)(c->step - c->tbl_step0);
    for (size_t k = 0; k < n && hit; ++k)
      hit = c->tbl_info[ch.off + k].nsplits == c->info_host.get()[k].nsplits &&
            c->tbl_info[ch.off + k].randomize == c->info_host.get()[k].randomize;
  }
  if (!hit) {
    ch.off = 0;
    ch.build = std::min<size_t>(c->table_cap, std::max<size_t>(n, 64));
    for (size_t k = n; k < ch.build; ++k) {
      const eb_move& mv = s.moves[choose_move(c, s, c->step + k)];
      c->info_host.get()[k].nsplits = mv.nsplits;
      c->info_host.get()[k].randomize = mv.randomize_split;
    }
    c->tbl_seed = c->seed;
    c->tbl_step0 = c->step;
    c->tbl_n = ch.build;
    c->tbl_info.assign(c->info_host.get(), c->info_host.get() + ch.build);
  }
  ch.ndesc = 0;
  for (size_t k = 0; k < n; ++k) {
    const eb_move& mv = s.moves[ch.pick[k]];
    if (!dmma_eligible(c, mv)) continue;
    int start[MAX_SPLITS + 1];
    split_starts(c->N, mv.nsplits, start);
    for (int split = 0; split < mv.nsplits; ++split) {
      HalfDesc& d = c->descs_host.get()[ch.ndesc++];
      d.step = c->step + k;
      d.order_step = (int32_t)(ch.off + k);
      d.split = split;
      d.a_start = start[split];
      d.a_count = start[split + 1] - start[split];
    }
  }
  return EB_OK;
}

// the uploads of a chunk, charged to its first step: the dense_dmma descriptors and the split tables to build
int upload_chunk(eb_ctx* c, const Chunk& ch, uint64_t& launches) {
  if (ch.ndesc)
    CK(c, cudaMemcpyAsync(c->descs_dev.get(), c->descs_host.get(), ch.ndesc * sizeof(HalfDesc), cudaMemcpyHostToDevice,
                          c->st.get()));
  if (ch.build) {
    CK(c, cudaMemcpyAsync(c->info_dev.get(), c->info_host.get(), ch.build * sizeof(StepInfo), cudaMemcpyHostToDevice,
                          c->st.get()));
    const Comm& cm = c->comm;
    if (c->nbatch > 0) {
      CK(c, launch_batch_split_tables(c->order.get(), c->info_dev.get(), (int)ch.build, c->bn, c->nbatch,
                                      c->seeds_dev.get(), c->step, c->st.get()));
      ++launches;
      return EB_OK;
    }
    CK(c, launch_split_tables(c->order.get(), c->info_dev.get(), (int)ch.build, c->N, c->seed, c->step,
                              cm.rows_per_rank * cm.rank, cm.rows_per_rank * (cm.rank + 1),
                              cm.nranks > 1 ? cm.ranges : nullptr, c->st.get()));
    ++launches;
    if (cm.nranks > 1 && cm.aperm) {
      // front group = one tile (8 walkers) for each of the 8 consumer warps of every SM: the first round
      CK(c, launch_locality_tables(c->order.get(), c->info_dev.get(), cm.ranges, (int)ch.build, c->N, c->seed,
                                   c->step, cm.rows_per_rank, cm.rank, 64 * c->sm_count, cm.aperm, c->st.get()));
      ++launches;
    }
  }
  return EB_OK;
}

// graph mode (eb_model_set_graphs, eb_move_set_proposal_graphs): run_steps logs the steps it enqueues for
// check_status while it runs
struct GraphRun {
  eb_ctx* c;
  explicit GraphRun(eb_ctx* ctx) : c(ctx) {
    c->graph_run = graph_errors(c);
    c->graph_step0 = c->step;
    c->graph_picks.clear();
  }
  ~GraphRun() { c->graph_run = false; }
};

// run nsteps steps.  `after_step(k)` is called with the work of step k enqueued and may
// enqueue copies on the stream; `sync_every` > 0 tells how often it actually does (every
// sync_every-th step), so that steps in between can share one persistent launch.
template <class F>
int run_steps(eb_ctx* c, const Schedule& s, uint64_t nsteps, uint64_t sync_every, F&& after_step) {
  uint64_t launches = 0;
  const GraphRun graph_run(c);
  const bool perstep = c->l2_flush;  // flush L2 before every step, time each step on its own
  if (perstep) {
    if (nsteps > 16384) FAIL(c, EB_ERR_INVALID, "l2_flush mode times each step separately; use nsteps <= 16384");
    if (!c->flush_buf) CK(c, dev_alloc(c->flush_buf, c->flush_bytes));
    while (c->ev_pool.size() < 2 * nsteps) {
      EventPtr e;
      CK(c, event_create(e));
      c->ev_pool.push_back(std::move(e));
    }
  }
  if (const int rc = running_prepare(c, nsteps)) return rc;
  c->dmma_nhalf_max = 0;
  CK(c, cudaEventRecord(c->ev0.get(), c->st.get()));
  if (comm_begin(c->comm, c->st.get(), c->status_dev.get(), launches)) FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  c->fused_last = false;
  const bool multi = c->comm.nranks > 1;
  // sharded ensembles run one half-step per launch: NCCL exchanges whole row blocks after every split, and the
  // P2P peer barrier rides on the kernel boundary (a persistent launch with the peer barrier between its
  // half-steps measured no faster and was dropped)
  const bool one_per_launch = multi;
  const bool exchange_each = multi && c->comm.mode == EB_COMM_ALLGATHER;
  DmmaChain chain;
  Chunk ch;
  uint64_t done = 0;
  while (done < nsteps) {
    const size_t chunk = (size_t)std::min<uint64_t>(nsteps - done, c->table_cap);
    int rc = EB_OK;
    if (c->graph_run && done > 0) rc = fetch_status(c);  // prepare_chunk waits for the stream anyway
    if (!rc) rc = prepare_chunk(c, s, chunk, ch);
    if (rc) return rc;
    DmmaGroup grp;
    size_t desc_cursor = 0;
    const eb_move* grp_move = nullptr;
    for (size_t k = 0; k < chunk; ++k) {
      const eb_move& mv = s.moves[ch.pick[k]];
      // Only a captured proposal's own kernels, and a graph model's, stop at an error the device has recorded; every
      // other move would go on updating the state.  So after a captured proposal has run, the status is read before
      // any other move is enqueued (a graph model freezes every move itself).
      if (c->gm_unchecked && !graph_mode(c) && !captured_proposal(c, mv)) {
        rc = fetch_status(c);
        if (rc) return rc;
      }
      const bool due = running_due(c, c->step + 1);
      const bool stored = sync_every > 0 && (done + k + 1) % sync_every == 0;  // after_step enqueues copies
      if (perstep) {
        CK(c, cudaMemsetAsync(c->flush_buf.get(), (int)(k & 0xff), c->flush_bytes, c->st.get()));
        CK(c, cudaEventRecord(c->ev_pool[2 * (done + k)].get(), c->st.get()));
        chain.live = false;
      }
      if (k == 0 && (ch.ndesc || ch.build)) {
        rc = upload_chunk(c, ch, launches);
        if (rc) return rc;
        chain.live = false;
      }
      if (dmma_eligible(c, mv)) {
        rc = check_walker_count(c, mv);
        if (rc) return rc;
        if (grp_move && grp_move != &mv) {  // a different move object: its parameters differ
          rc = flush_dmma(c, *grp_move, grp, chain, launches);
          if (rc) return rc;
        }
        grp_move = &mv;
        for (int split = 0; split < mv.nsplits; ++split) {
          const HalfDesc& d = c->descs_host.get()[desc_cursor];
          if (grp.nhalf == 0) grp.first = desc_cursor;
          grp.nhalf += 1;
          grp.max_count = std::max(grp.max_count, (int)d.a_count);
          ++desc_cursor;
          if (one_per_launch || (grp.nhalf >= c->dmma_group && split + 1 < mv.nsplits)) {
            rc = flush_dmma(c, mv, grp, chain, launches);
            if (rc) return rc;
            if (exchange_each) {
              chain.live = false;
              if (comm_after_split(c->comm, c->st.get(), c->status_dev.get(), launches))
                FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
            }
          }
        }
        // a group ends where the host or a statistic reads the state
        if (perstep || due || stored || k + 1 == chunk || grp.nhalf >= c->dmma_group) {
          rc = flush_dmma(c, mv, grp, chain, launches);
          if (rc) return rc;
        }
      } else {
        if (grp_move) {
          rc = flush_dmma(c, *grp_move, grp, chain, launches);
          if (rc) return rc;
        }
        chain.live = false;
        const size_t tbl = ch.off + k;
        switch (mv.kind) {
          case EB_MOVE_WALK:
            rc = launch_step_walk(c, mv, c->step, tbl, launches);
            break;
          case EB_MOVE_KDE:
            rc = launch_step_kde(c, mv, c->step, tbl, launches);
            break;
          case EB_MOVE_GAUSSIAN:
            rc = launch_step_gaussian(c, s, ch.pick[k], c->step, launches);
            break;
          case EB_MOVE_USER:
            rc = launch_step_user(c, mv, c->step, tbl, launches);
            break;
          case EB_MOVE_USER_MH:
            rc = launch_step_user_mh(c, mv, c->step, launches);
            break;
          default:
            rc = c->nbatch > 0 ? launch_step_batch(c, mv, c->step, tbl, launches)
                               : launch_step_generic(c, mv, c->step, tbl, launches);
        }
        if (rc) return rc;
      }
      c->picks[ch.pick[k]] += 1;
      c->step += 1;
      if (c->graph_run) {
        c->graph_picks.push_back(ch.pick[k]);
        // a graph model's error stops the call before a statistic or a stored step records a state past it
        if (due || stored) {
          rc = fetch_status(c);
          if (rc) return rc;
        }
      }
      if (due) {
        rc = running_record(c, launches);
        if (rc) return rc;
        chain.live = false;
      }
      if (perstep) {
        CK(c, cudaEventRecord(c->ev_pool[2 * (done + k) + 1].get(), c->st.get()));
        chain.live = false;
      }
      rc = after_step(done + k);
      if (rc) return rc;
      if (stored) chain.live = false;
    }
    done += chunk;
  }
  CK(c, cudaEventRecord(c->ev1.get(), c->st.get()));
  // multi-GPU: the rows of other ranks are NOT replicated here; collective readers (eb_get_state,
  // eb_get_naccepted, the accept mask of eb_step) do that on demand, sharded readers never need it
  if (multi) c->replicas_dirty = true;
  int rc = enqueue_status_read(c);
  if (rc) return rc;
  CK(c, cudaStreamSynchronize(c->st.get()));
  float ms = 0.f;
  if (perstep) {
    double tot = 0.0;
    for (uint64_t k = 0; k < nsteps; ++k) {
      CK(c, cudaEventElapsedTime(&ms, c->ev_pool[2 * k].get(), c->ev_pool[2 * k + 1].get()));
      tot += ms;
    }
    c->last_ms = tot;
  } else {
    CK(c, cudaEventElapsedTime(&ms, c->ev0.get(), c->ev1.get()));
    c->last_ms = ms;
  }
  c->last_launches = launches;
  return check_status(c);
}

int step_preflight(eb_ctx* c) {
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_step: no model set");
  if (!c->have_state) FAIL(c, EB_ERR_STATE, "eb_step: no state set");
  CK(c, cudaSetDevice(c->device));
  return EB_OK;
}

}  // namespace

extern "C" {

int eb_step(eb_ctx* c, const eb_move* moves, size_t nmoves, uint64_t nsteps, uint8_t* accepted_last) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  int rc = step_preflight(c);
  if (rc) return rc;
  Schedule s;
  rc = build_schedule(c, moves, nmoves, s);
  if (rc) return rc;
  if (nsteps > 0) {
    rc = run_steps(c, s, nsteps, 0, [](uint64_t) { return EB_OK; });
    if (rc) return rc;
  }
  if (accepted_last) {
    rc = sync_replicas(c);  // multi-GPU: the mask of every rank's rows (collective)
    if (rc) return rc;
    CK(c, cudaMemcpyAsync(accepted_last, c->accepted.get(), (size_t)c->N, cudaMemcpyDeviceToHost, c->st.get()));
    CK(c, cudaStreamSynchronize(c->st.get()));
  }
  return EB_OK;
}

int eb_step_store(eb_ctx* c, const eb_move* moves, size_t nmoves, uint64_t nsteps, uint64_t thin_by,
                  double* chain, double* log_prob, double* accepted) {
  return eb_step_store_blobs(c, moves, nmoves, nsteps, thin_by, chain, log_prob, accepted, nullptr);
}

int eb_step_store_blobs(eb_ctx* c, const eb_move* moves, size_t nmoves, uint64_t nsteps, uint64_t thin_by,
                        double* chain, double* log_prob, double* accepted, void* blobs) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (thin_by == 0) FAIL(c, EB_ERR_INVALID, "Invalid thinning argument");  // ensemble.py:380-381
  if (!chain || !log_prob) FAIL(c, EB_ERR_INVALID, "eb_step_store: null output buffer");
  if (blobs && !c->blobs_live) FAIL(c, EB_ERR_STATE, "eb_step_store_blobs: the state has no blobs");
  int rc = step_preflight(c);
  if (rc) return rc;
  Schedule s;
  rc = build_schedule(c, moves, nmoves, s);
  if (rc) return rc;
  const size_t N = (size_t)c->N, D = (size_t)c->D;
  const size_t row = N * D + N;  // coords then log_prob, staged together
  for (int k = 0; k < 2; ++k) {
    if (c->stage[k]) continue;
    HostPtr<double> x;
    HostPtr<uint8_t> acc;
    EventPtr ev;
    CK(c, host_alloc(x, row * sizeof(double)));
    CK(c, host_alloc(acc, N));
    CK(c, event_create(ev, cudaEventDisableTiming));
    c->stage[k] = std::move(x);
    c->stage_acc[k] = std::move(acc);
    c->stage_ev[k] = std::move(ev);
  }
  const size_t blob_row = blobs ? N * c->blob_bytes : 0;  // the blob records of a stored step, staged beside them
  if (blob_row > c->stage_blob_cap) {
    for (HostPtr<uint8_t>& b : c->stage_blob) b.reset();
    c->stage_blob_cap = 0;
    for (HostPtr<uint8_t>& b : c->stage_blob) CK(c, host_alloc(b, blob_row));
    c->stage_blob_cap = blob_row;
  }
  uint8_t* blob_out = static_cast<uint8_t*>(blobs);
  // double-buffered pinned staging: the D2H of stored step k overlaps the
  // kernels of the following steps; the host drains slot k-1 while k is in flight
  uint64_t stored = 0;
  int64_t pending[2] = {-1, -1};
  auto drain = [&](int slot) -> int {
    if (pending[slot] < 0) return EB_OK;
    CK(c, cudaEventSynchronize(c->stage_ev[slot].get()));
    const size_t k = (size_t)pending[slot];
    memcpy(chain + k * N * D, c->stage[slot].get(), N * D * sizeof(double));          // backend.py:224
    memcpy(log_prob + k * N, c->stage[slot].get() + N * D, N * sizeof(double));        // backend.py:225
    if (blob_out) memcpy(blob_out + k * blob_row, c->stage_blob[slot].get(), blob_row);  // backend.py:226-227
    if (accepted)
      for (size_t w = 0; w < N; ++w) accepted[w] += (double)c->stage_acc[slot].get()[w];  // backend.py:229
    pending[slot] = -1;
    return EB_OK;
  };
  rc = run_steps(c, s, nsteps, thin_by, [&](uint64_t k) -> int {
    if ((k + 1) % thin_by != 0) return EB_OK;  // ensemble.py:416
    const int slot = (int)(stored & 1);
    int r = drain(slot);
    if (r) return r;
    if (c->comm.nranks > 1) {
      // a stored step holds EVERY walker: replicate the other ranks' rows (log_prob, accept mask and, in
      // P2P mode, coords) before the copy -- the in-run exchange only moves what the kernels need
      uint64_t l = 0;
      if (comm_sync_state(c->comm, c->st.get(), c->status_dev.get(), c->logp.get(), c->accepted.get(), nullptr, l))
        FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
      c->fused_last = false;
    }
    CK(c, cudaMemcpyAsync(c->stage[slot].get(), c->coords.get(), N * D * sizeof(double), cudaMemcpyDeviceToHost,
                          c->st.get()));
    CK(c, cudaMemcpyAsync(c->stage[slot].get() + N * D, c->logp.get(), N * sizeof(double), cudaMemcpyDeviceToHost,
                          c->st.get()));
    CK(c, cudaMemcpyAsync(c->stage_acc[slot].get(), c->accepted.get(), N, cudaMemcpyDeviceToHost, c->st.get()));
    if (blob_out) CK(c, cudaMemcpyAsync(c->stage_blob[slot].get(), c->blob_live.get(), blob_row, cudaMemcpyDeviceToHost,
                                        c->st.get()));
    CK(c, cudaEventRecord(c->stage_ev[slot].get(), c->st.get()));
    pending[slot] = (int64_t)stored;
    ++stored;
    return EB_OK;
  });
  int r0 = drain((int)(stored & 1));
  int r1 = drain((int)((stored + 1) & 1));
  if (rc) return rc;
  if (r0) return r0;
  return r1;
}

int eb_step_store_chain(eb_ctx* c, const eb_move* moves, size_t nmoves, uint64_t nsteps, uint64_t thin_by,
                        eb_chain* ch, uint64_t slot0) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (thin_by == 0) FAIL(c, EB_ERR_INVALID, "Invalid thinning argument");  // ensemble.py:380-381
  if (!ch) FAIL(c, EB_ERR_INVALID, "eb_step_store_chain: null chain");
  if (ch->ring) FAIL(c, EB_ERR_INVALID, "eb_step_store_chain: a running window's ring is written by its engine only");
  if (ch->device != c->device || ch->N != c->N || ch->D != c->D)
    FAIL(c, EB_ERR_INVALID, "eb_step_store_chain: the chain is [%lld, %d] on device %d, the engine [%lld, %d] on device %d",
         (long long)ch->N, ch->D, ch->device, (long long)c->N, c->D, c->device);
  if (c->comm.nranks > 1)
    FAIL(c, EB_ERR_UNSUPPORTED,
         "eb_step_store_chain: a stored step holds every walker, and sharded ensembles replicate the other ranks' "
         "rows before each stored step only for host chains (eb_step_store); device chains are not sharded");
  const uint64_t nstore = nsteps / thin_by;
  if (nstore > 0 && (slot0 >= ch->start.back() || nstore > ch->start.back() - slot0))
    FAIL(c, EB_ERR_INVALID, "eb_step_store_chain: slots [%llu, %llu) out of range (capacity %llu slots)",
         (unsigned long long)slot0, (unsigned long long)(slot0 + nstore), (unsigned long long)ch->start.back());
  int rc = step_preflight(c);
  if (rc) return rc;
  Schedule s;
  rc = build_schedule(c, moves, nmoves, s);
  if (rc) return rc;
  const size_t nx = (size_t)c->N * c->D;
  uint64_t slot = slot0;
  size_t seg = 0;
  // no host synchronisation per stored step: the store kernel is enqueued behind the step on the engine's
  // stream, and run_steps synchronises once at its end
  return run_steps(c, s, nsteps, thin_by, [&](uint64_t k) -> int {
    if ((k + 1) % thin_by != 0) return EB_OK;  // ensemble.py:416
    while (slot >= ch->start[seg + 1]) ++seg;
    const uint64_t off = slot - ch->start[seg];
    CK(c, launch_chain_store(c->coords.get(), c->logp.get(), c->accepted.get(), ch->segs[seg].x.get() + off * ch->xs,
                             ch->segs[seg].lp.get() + off * ch->ls, ch->accepted.get(), nx, (size_t)c->N, c->N,
                             c->sm_count, c->st.get()));
    ++slot;
    return EB_OK;
  });
}

}  // extern "C"
