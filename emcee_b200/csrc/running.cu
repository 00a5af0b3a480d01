// The running statistics of an engine (running.h): their configuration and read-out entry points of the C ABI, and
// the hooks through which the step driver records them.  Every statistic records the live state after every `every`-th
// step; within a step they record in the order of RunningStats, behind the step on the engine's stream.
#include <algorithm>
#include <vector>

#include "context.h"

namespace {

// the refusals of a sharded ensemble, from the configuration and from eb_comm_init
const char* const HIST_NOT_SHARDED = "running histograms are not sharded across GPUs";
const char* const TRACE_NOT_SHARDED = "the running trace is not sharded across GPUs";
const char* const RESERVOIR_NOT_SHARDED = "the running reservoir is not sharded across GPUs";
const char* const ACF_NOT_SHARDED = "the running autocorrelation is not sharded across GPUs";
const char* const WINDOW_NOT_SHARDED = "the running window is not sharded across GPUs";

// the opening of eb_histograms_config, eb_trace_config, eb_reservoir_config, eb_running_acf_config and
// eb_window_config: a single ensemble outside a callback, not sharded, and the steps recorded so far done before the
// configuration changes the buffers they write
int config_prologue(eb_ctx* c, const char* who, const char* not_sharded) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, who);
  NOT_IN_CALLBACK(c);
  if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "%s", not_sharded);
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

// trace, reservoir, autocorrelation and window: the first configuration, and every one with every > 0, starts from
// scratch (start()); every == 0 after a configuration keeps what was recorded readable and records nothing more
template <class Start>
int reconfigure(uint64_t& every_of, bool on, uint64_t every, Start&& start) {
  if (every > 0 || !on) {
    const int rc = start();
    if (rc) return rc;
  }
  every_of = every;
  return EB_OK;
}

// the result of a statistic's setup call, named after `who`
int setup_result(eb_ctx* c, const char* who, cudaError_t s) {
  if (s == cudaSuccess) return EB_OK;
  cudaGetLastError();
  FAIL(c, EB_ERR_CUDA, "%s: %s", who, cudaGetErrorString(s));
}

// empty the reservoir of K rows in its buffers (the same size, a new seed or an earlier step)
int reservoir_restart(eb_ctx* c, const char* who, uint64_t K) {
  RunReservoir& r = c->run.reservoir;
  r.plan = ResSchedule(K, (uint64_t)c->N);
  return setup_result(c, who, live_reservoir_setup(&r.live, r.mem.get(), K, (uint32_t)c->N, c->D, c->coords.get(),
                                                   c->logp.get(), c->sm_count, c->st.get()));
}

// ---- recording -----------------------------------------------------------------------------------------------------
// fold the rows this rank owns of the CURRENT state into the accumulators (enqueued on the stream)
int record_moments(eb_ctx* c, uint64_t& launches) {
  RunMoments& m = c->run.moments;
  int64_t r0, r1;
  owned_rows(c, r0, r1);
  const double* X = c->coords.get() + (size_t)r0 * c->D;
  if (!m.have_shift) {
    // shift = the ensemble mean at the first accumulation: keeps the raw second moments well conditioned
    CK(c, launch_colmean(X, r1 - r0, c->D, m.shift.get(), nullptr, c->st.get()));
    m.have_shift = true;
    ++launches;
  }
  CK(c, launch_moments(X, r1 - r0, c->D, m.shift.get(), c->mom_partial.get(), m.acc.get(), c->sm_count,
                       c->st.get()));
  launches += 2;
  m.count += (unsigned long long)(r1 - r0);
  return EB_OK;
}

// count the CURRENT state into the histograms
int record_histograms(eb_ctx* c, uint64_t& launches) {
  CK(c, live_hist_launch(c->run.hist.live, c->st.get(), launches));
  c->run.hist.count += (unsigned long long)c->N;
  return EB_OK;
}

// Room for the rows the next `nsteps` steps record, made before the first launch: the rows already recorded move
// into a larger allocation (half as large again when that fits, so that a run of many short calls grows a few times).
int reserve_trace(eb_ctx* c, uint64_t nsteps) {
  RunTrace& t = c->run.trace;
  const uint64_t add = (c->step + nsteps) / t.every - c->step / t.every;
  const uint64_t have = t.steps.size(), need = have + add;
  if (need <= t.cap) return EB_OK;
  const size_t row = (2 * (size_t)c->D + TRACE_EXTRA) * sizeof(double);
  const char* who = "the running trace";
  DevPtr<double> rows;
  uint64_t cap = std::max(need, t.cap + t.cap / 2);
  int rc = cap > need ? dev_alloc_checked(c, who, "rows", (size_t)cap * row, rows) : EB_ERR_NOMEM;
  if (rc == EB_ERR_NOMEM) {
    cap = need;
    rc = dev_alloc_checked(c, who, "rows", need <= SIZE_MAX / row ? (size_t)need * row : SIZE_MAX, rows);
  }
  if (rc) return rc;
  if (have)
    CK(c, cudaMemcpyAsync(rows.get(), t.rows.get(), (size_t)have * row, cudaMemcpyDeviceToDevice, c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  t.rows = std::move(rows);
  t.cap = cap;
  t.steps.reserve((size_t)cap);
  return EB_OK;
}

// record the CURRENT state as one row of the trace
int record_trace(eb_ctx* c, uint64_t& launches) {
  RunTrace& t = c->run.trace;
  double* row = t.rows.get() + t.steps.size() * (2 * (size_t)c->D + TRACE_EXTRA);
  CK(c, live_trace_launch(t.live, row, c->step, c->st.get(), launches));
  t.steps.push_back(c->step);
  return EB_OK;
}

// offer the CURRENT state's rows to the reservoir, behind a compaction when the rows could overflow its buffer
int record_reservoir(eb_ctx* c, uint64_t& launches) {
  RunReservoir& r = c->run.reservoir;
  if (r.plan.compact_before_record()) {
    CK(c, live_reservoir_compact(r.live, r.plan.bound, c->st.get(), launches));
    r.plan.compacted();
  }
  CK(c, live_reservoir_record(r.live, c->seed, c->step, c->st.get(), launches));
  r.plan.recorded();
  return EB_OK;
}

// write the CURRENT state into the autocorrelation ring, and fold the block of lag sums it completes
int record_autocorr(eb_ctx* c, uint64_t& launches) {
  CK(c, live_racf_record(c->run.acf.live, c->run.acf.n, c->st.get(), launches));
  c->run.acf.n += 1;
  return EB_OK;
}

// copy the CURRENT state and the step's accept mask into the window's ring, at physical slot n mod size (one
// kernel); once the ring is full the oldest slot moves on with every record
int record_window(eb_ctx* c, uint64_t& launches) {
  RunWindow& win = c->run.window;
  eb_chain* w = win.ring.get();
  const uint64_t size = w->start.back(), slot = win.n % size;
  CK(c, launch_chain_store(c->coords.get(), c->logp.get(), c->accepted.get(), w->segs[0].x.get() + slot * w->xs,
                           w->segs[0].lp.get() + slot * w->ls, nullptr, (size_t)c->N * c->D, (size_t)c->N, c->N,
                           c->sm_count, c->st.get(), w->slot_mask.get() + slot * (uint64_t)c->N));
  ++launches;
  win.steps[(size_t)slot] = c->step;
  win.seeds[(size_t)slot] = c->seed;
  win.n += 1;
  w->filled = std::min(win.n, size);
  w->origin = win.n >= size ? win.n % size : 0;
  return EB_OK;
}

bool due_at(uint64_t every, uint64_t n) { return every > 0 && n % every == 0; }

int reservoir_read(eb_ctx* c, double* coords, double* log_prob, uint64_t* step, int64_t* walker, bool device_out) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  RunReservoir& r = c->run.reservoir;
  if (!r.on) FAIL(c, EB_ERR_STATE, "eb_reservoir_read: configure the reservoir with eb_reservoir_config first");
  CK(c, cudaSetDevice(c->device));
  if (r.plan.compact_before_read()) {
    uint64_t launches = 0;
    CK(c, live_reservoir_compact(r.live, r.plan.bound, c->st.get(), launches));
    r.plan.compacted();
  }
  CK(c, live_reservoir_read(r.live, r.plan.kept(), coords, log_prob, step, walker, device_out, c->st.get()));
  return EB_OK;
}

}  // namespace

// ---- hooks ---------------------------------------------------------------------------------------------------------
int running_prepare(eb_ctx* c, uint64_t nsteps) { return c->run.trace.every > 0 ? reserve_trace(c, nsteps) : EB_OK; }

bool running_due(const eb_ctx* c, uint64_t n) {
  const RunningStats& r = c->run;
  return due_at(r.moments.every, n) || due_at(r.hist.every, n) || due_at(r.trace.every, n) ||
         due_at(r.reservoir.every, n) || due_at(r.acf.every, n) || due_at(r.window.every, n);
}

int running_record(eb_ctx* c, uint64_t& launches) {
  const RunningStats& r = c->run;
  const uint64_t n = c->step;
  int rc = EB_OK;
  if (due_at(r.moments.every, n)) rc = record_moments(c, launches);
  if (!rc && due_at(r.hist.every, n)) rc = record_histograms(c, launches);
  if (!rc && due_at(r.trace.every, n)) rc = record_trace(c, launches);
  if (!rc && due_at(r.reservoir.every, n)) rc = record_reservoir(c, launches);
  if (!rc && due_at(r.acf.every, n)) rc = record_autocorr(c, launches);
  if (!rc && due_at(r.window.every, n)) rc = record_window(c, launches);
  return rc;
}

int running_check_sharding(eb_ctx* c, int nranks) {
  if (nranks <= 1) return EB_OK;
  const RunningStats& r = c->run;
  if (r.hist.on) FAIL(c, EB_ERR_UNSUPPORTED, "%s", HIST_NOT_SHARDED);
  if (r.trace.on) FAIL(c, EB_ERR_UNSUPPORTED, "%s", TRACE_NOT_SHARDED);
  if (r.reservoir.on) FAIL(c, EB_ERR_UNSUPPORTED, "%s", RESERVOIR_NOT_SHARDED);
  if (r.acf.on) FAIL(c, EB_ERR_UNSUPPORTED, "%s", ACF_NOT_SHARDED);
  if (r.window.ring) FAIL(c, EB_ERR_UNSUPPORTED, "%s", WINDOW_NOT_SHARDED);
  return EB_OK;
}

// the rows of a step offered again would come back with their old keys, and a new seed draws other keys: either
// starts the reservoir again, so that it stays the sample of one stream of steps (reservoir_plan.h)
int running_set_rng(eb_ctx* c, uint64_t seed, uint64_t step) {
  if (!c->run.reservoir.on || (seed == c->seed && step >= c->step)) return EB_OK;
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return reservoir_restart(c, "eb_set_rng", c->run.reservoir.live.K);
}

// every call zeroes the sums, every == 0 included
int moments_config(eb_ctx* c, uint64_t every) {
  RunMoments& m = c->run.moments;
  CK(c, cudaSetDevice(c->device));
  if (every > 0 && c->D > 1024) FAIL(c, EB_ERR_UNSUPPORTED, "chain moments are limited to ndim <= 1024");
  const size_t n = (size_t)c->D + (size_t)c->D * c->D;
  if (every > 0 && !m.acc) {
    DevPtr<double> acc, shift, partial;
    CK(c, dev_alloc(acc, n * sizeof(double)));
    CK(c, dev_alloc(shift, (size_t)c->D * sizeof(double)));
    if (!c->mom_partial) CK(c, dev_alloc(partial, moments_partial_bytes(c->D, c->sm_count)));
    m.acc = std::move(acc);
    m.shift = std::move(shift);
    if (partial) c->mom_partial = std::move(partial);
  }
  if (m.acc) CK(c, cudaMemsetAsync(m.acc.get(), 0, n * sizeof(double), c->st.get()));
  m.count = 0;
  m.have_shift = false;
  m.every = every;
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

extern "C" {

// ---- moments -------------------------------------------------------------------------------------------------------
int eb_moments(eb_ctx* c, double* mean, double* cov, uint64_t* count, uint64_t* naccepted_total) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  const RunMoments& m = c->run.moments;
  if (!m.acc) FAIL(c, EB_ERR_STATE, "eb_moments: enable with eb_set_option(\"moments_every\", n) before stepping");
  CK(c, cudaSetDevice(c->device));
  const size_t D = (size_t)c->D, n = D + D * D;
  std::vector<double> acc(n), shift(D);
  CK(c, cudaMemcpyAsync(acc.data(), m.acc.get(), n * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
  CK(c, cudaMemcpyAsync(shift.data(), m.shift.get(), D * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
  std::vector<unsigned long long> nacc;
  int64_t r0, r1;
  owned_rows(c, r0, r1);
  if (naccepted_total) {
    nacc.resize((size_t)(r1 - r0));
    CK(c, cudaMemcpyAsync(nacc.data(), c->nacc.get() + r0, nacc.size() * sizeof(unsigned long long),
                          cudaMemcpyDeviceToHost, c->st.get()));
  }
  CK(c, cudaStreamSynchronize(c->st.get()));
  if (count) *count = m.count;
  if (naccepted_total) {
    unsigned long long tot = 0;
    for (unsigned long long v : nacc) tot += v;
    *naccepted_total = tot;
  }
  finish_moments(acc.data(), shift.data(), m.count, D, mean, cov);
  return EB_OK;
}

// ---- histograms ----------------------------------------------------------------------------------------------------
int eb_histograms_config(eb_ctx* c, uint64_t every, uint32_t bins, const double* outer, const double* edges,
                         int log_prob, const uint32_t* params2d, size_t nparams2d, uint32_t bins2d,
                         const double* edges2d) {
  const char* who = "eb_histograms_config";
  int rc = config_prologue(c, who, HIST_NOT_SHARDED);
  if (rc) return rc;
  if (bins == 0 || !outer || !edges) FAIL(c, EB_ERR_INVALID, "eb_histograms_config: bins == 0 or null buffer");
  if (bins > (uint32_t)HIST_BINS_MAX)
    FAIL(c, EB_ERR_UNSUPPORTED, "running histograms are limited to bins <= %d on the device, got %u", HIST_BINS_MAX,
         bins);
  if (nparams2d > 0) {
    if (!params2d || !edges2d || bins2d == 0)
      FAIL(c, EB_ERR_INVALID, "eb_histograms_config: bins2d == 0 or null 2-D buffer");
    if (bins2d > (uint32_t)HIST2_BINS_MAX)
      FAIL(c, EB_ERR_UNSUPPORTED, "running 2-D histograms are limited to bins <= %d on the device, got %u",
           HIST2_BINS_MAX, bins2d);
    if (nparams2d < 2 || nparams2d > (size_t)c->D)
      FAIL(c, EB_ERR_INVALID, "eb_histograms_config: need 2 <= nparams2d <= ndim = %d, got %zu", c->D, nparams2d);
    std::vector<uint8_t> seen((size_t)c->D, 0);
    for (size_t k = 0; k < nparams2d; ++k) {
      if (params2d[k] >= (uint32_t)c->D || seen[params2d[k]])
        FAIL(c, EB_ERR_INVALID, "eb_histograms_config: params2d must be distinct and < ndim = %d (params2d[%zu] = %u)",
             c->D, k, params2d[k]);
      seen[params2d[k]] = 1;
    }
  }
  // the old configuration goes first: its memory counts towards what the new one may take
  RunHistograms& h = c->run.hist;
  h = RunHistograms{};
  const int lp = log_prob ? 1 : 0, m = nparams2d > 0 ? (int)nparams2d : 0;
  DevPtr<void> mem;
  rc = dev_alloc_checked(c, who, "counts and tables", live_hist_bytes(c->D, (int)bins, lp, m, (int)bins2d), mem);
  if (rc) return rc;
  rc = setup_result(c, who, live_hist_setup(&h.live, mem.get(), (uint32_t)c->N, c->D, (int)bins, lp, outer, edges,
                                            params2d, m, (int)bins2d, edges2d, c->coords.get(), c->logp.get(),
                                            c->sm_count, c->st.get()));
  if (rc) {
    h.live = LiveHist{};
    return rc;
  }
  h.mem = std::move(mem);
  h.on = true;
  h.every = every;
  return EB_OK;
}

int eb_histograms(eb_ctx* c, uint64_t* hist, uint64_t* hist2d, uint64_t* count) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  const RunHistograms& h = c->run.hist;
  if (!h.on) FAIL(c, EB_ERR_STATE, "eb_histograms: configure them with eb_histograms_config first");
  CK(c, cudaSetDevice(c->device));
  bool bad = false;
  CK(c, live_hist_read(h.live, hist, hist2d, &bad, c->st.get()));
  if (count) *count = h.count;
  if (bad)
    FAIL(c, EB_ERR_INVALID, "eb_histograms: a value's truncated bin index is above bins (np.histogram raises "
         "IndexError there); the span does not fit the edges");
  return EB_OK;
}

// ---- trace ---------------------------------------------------------------------------------------------------------
int eb_trace_config(eb_ctx* c, uint64_t every) {
  const char* who = "eb_trace_config";
  if (const int rc = config_prologue(c, who, TRACE_NOT_SHARDED)) return rc;
  RunTrace& t = c->run.trace;
  return reconfigure(t.every, t.on, every, [&]() -> int {
    t.rows.reset();
    t.cap = 0;
    t.steps.clear();
    if (!t.on) {
      const int rc = dev_alloc_checked(c, who, "partial sums", live_trace_fixed_bytes((uint32_t)c->N, c->D), t.mem);
      if (rc) return rc;
    }
    const int rc = setup_result(c, who, live_trace_setup(&t.live, t.mem.get(), (uint32_t)c->N, c->D, c->coords.get(),
                                                         c->logp.get(), c->accepted.get(), c->st.get()));
    if (!rc) t.on = true;
    return rc;
  });
}

int eb_trace_count(eb_ctx* c, uint64_t* rows) {
  if (!c || !rows) return EB_ERR_INVALID;
  if (!c->run.trace.on) FAIL(c, EB_ERR_STATE, "eb_trace_count: configure the trace with eb_trace_config first");
  *rows = c->run.trace.steps.size();
  return EB_OK;
}

int eb_trace_read(eb_ctx* c, uint64_t first, uint64_t count, uint64_t* step, double* rows_out) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  const RunTrace& t = c->run.trace;
  if (!t.on) FAIL(c, EB_ERR_STATE, "eb_trace_read: configure the trace with eb_trace_config first");
  const uint64_t have = t.steps.size();
  if (first > have || count > have - first)
    FAIL(c, EB_ERR_INVALID, "eb_trace_read: rows %llu .. %llu + %llu of %llu recorded", (unsigned long long)first,
         (unsigned long long)first, (unsigned long long)count, (unsigned long long)have);
  if (count == 0) return EB_OK;
  if (step) std::copy(t.steps.begin() + first, t.steps.begin() + first + count, step);
  if (rows_out) {
    const size_t W = 2 * (size_t)c->D + TRACE_EXTRA;
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaMemcpyAsync(rows_out, t.rows.get() + first * W, (size_t)count * W * sizeof(double),
                          cudaMemcpyDeviceToHost, c->st.get()));
    CK(c, cudaStreamSynchronize(c->st.get()));
  }
  return EB_OK;
}

int eb_trace_best(eb_ctx* c, double* coords, double* log_prob, uint64_t* step, uint64_t* walker) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  const RunTrace& t = c->run.trace;
  if (!t.on) FAIL(c, EB_ERR_STATE, "eb_trace_best: configure the trace with eb_trace_config first");
  if (t.steps.empty()) FAIL(c, EB_ERR_STATE, "eb_trace_best: no step has been recorded yet");
  CK(c, cudaSetDevice(c->device));
  TraceBest b;
  CK(c, live_trace_best(t.live, &b, coords, c->st.get()));
  if (log_prob) *log_prob = b.log_prob;
  if (step) *step = b.step;
  if (walker) *walker = b.walker;
  return EB_OK;
}

// ---- reservoir -----------------------------------------------------------------------------------------------------
int eb_reservoir_config(eb_ctx* c, uint64_t size, uint64_t every) {
  const char* who = "eb_reservoir_config";
  if (const int rc = config_prologue(c, who, RESERVOIR_NOT_SHARDED)) return rc;
  if (size == 0) FAIL(c, EB_ERR_INVALID, "eb_reservoir_config: size must be >= 1");
  if (size >= RES_SIZE_LIMIT)
    FAIL(c, EB_ERR_NOMEM, "eb_reservoir_config: size %llu is not below 2^32, the entries the reservoir can address",
         (unsigned long long)size);
  RunReservoir& r = c->run.reservoir;
  return reconfigure(r.every, r.on, every, [&]() -> int {
    if (!r.on || r.live.K != size) {  // the same size empties the buffers in place
      // entries are addressed with 32 bits; the old buffers stay until the new ones exist
      const uint64_t cap = res_cap(size, (uint64_t)c->N);  // size < 2^32: no wrap
      const size_t bytes = cap < RES_SIZE_LIMIT ? live_reservoir_bytes(size, (uint32_t)c->N, c->D) : SIZE_MAX;
      DevPtr<void> mem;
      const int rc = dev_alloc_checked(c, who, "entries", bytes, mem);
      if (rc) return rc;
      r.mem = std::move(mem);
    }
    const int rc = reservoir_restart(c, who, size);
    if (!rc) r.on = true;
    return rc;
  });
}

int eb_reservoir_count(eb_ctx* c, uint64_t* offered, uint64_t* kept) {
  if (!c) return EB_ERR_INVALID;
  const RunReservoir& r = c->run.reservoir;
  if (!r.on) FAIL(c, EB_ERR_STATE, "eb_reservoir_count: configure the reservoir with eb_reservoir_config first");
  if (offered) *offered = r.plan.offered;
  if (kept) *kept = r.plan.kept();
  return EB_OK;
}

int eb_reservoir_read(eb_ctx* c, double* coords, double* log_prob, uint64_t* step, int64_t* walker) {
  return reservoir_read(c, coords, log_prob, step, walker, false);
}

int eb_reservoir_read_to(eb_ctx* c, double* coords_dst, double* log_prob_dst, uint64_t* step, int64_t* walker) {
  return reservoir_read(c, coords_dst, log_prob_dst, step, walker, true);
}

// ---- autocorrelation -----------------------------------------------------------------------------------------------
int eb_running_acf_config(eb_ctx* c, uint64_t max_lag, uint64_t every) {
  const char* who = "eb_running_acf_config";
  if (const int rc = config_prologue(c, who, ACF_NOT_SHARDED)) return rc;
  if (max_lag == 0) FAIL(c, EB_ERR_INVALID, "eb_running_acf_config: max_lag must be >= 1");
  RunAutocorr& a = c->run.acf;
  return reconfigure(a.every, a.on, every, [&]() -> int {
    if (!a.on || a.live.max_lag != max_lag) {  // the same lags zero the sums in place
      // the old sums stay until the new ones exist
      DevPtr<void> mem;
      const int rc = dev_alloc_checked(c, who, "lag sums", live_racf_bytes((uint32_t)c->N, c->D, max_lag), mem);
      if (rc) return rc;
      a.mem = std::move(mem);
    }
    a.n = 0;
    const int rc = setup_result(c, who, live_racf_setup(&a.live, a.mem.get(), (uint32_t)c->N, c->D, max_lag,
                                                        c->coords.get(), c->st.get()));
    if (!rc) a.on = true;
    return rc;
  });
}

int eb_running_acf_count(eb_ctx* c, uint64_t* n) {
  if (!c) return EB_ERR_INVALID;
  if (!c->run.acf.on)
    FAIL(c, EB_ERR_STATE, "eb_running_acf_count: configure the autocorrelation with eb_running_acf_config first");
  if (n) *n = c->run.acf.n;
  return EB_OK;
}

int eb_running_acf_read(eb_ctx* c, double* rho) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  const RunAutocorr& a = c->run.acf;
  if (!a.on)
    FAIL(c, EB_ERR_STATE, "eb_running_acf_read: configure the autocorrelation with eb_running_acf_config first");
  CK(c, cudaSetDevice(c->device));
  CK(c, live_racf_read(a.live, a.n, rho, c->st.get()));
  return EB_OK;
}

// ---- window --------------------------------------------------------------------------------------------------------
int eb_window_config(eb_ctx* c, uint64_t size, uint64_t every) {
  const char* who = "eb_window_config";
  if (const int rc = config_prologue(c, who, WINDOW_NOT_SHARDED)) return rc;
  if (size == 0) FAIL(c, EB_ERR_INVALID, "eb_window_config: size must be >= 1");
  RunWindow& win = c->run.window;
  return reconfigure(win.every, (bool)win.ring, every, [&]() -> int {
    if (!win.ring || win.ring->start.back() != size) {  // the same size reuses the ring
      // the whole ring is checked against the free memory before anything changes; the old ring stays until the new
      // one exists
      const size_t N = (size_t)c->N, xs = (N * (size_t)c->D + 1) & ~(size_t)1, ls = (N + 1) & ~(size_t)1;
      const size_t per_slot = (xs + ls) * sizeof(double) + N, fixed = N * (sizeof(double) + 1);
      const size_t bytes = size <= (SIZE_MAX - fixed) / per_slot ? (size_t)size * per_slot + fixed : SIZE_MAX;
      int rc = check_free(c, who, "ring", bytes);
      if (rc) return rc;
      std::unique_ptr<eb_chain> ring(new eb_chain());
      cudaError_t e = chain_init(ring.get(), c->device, c->N, c->D);
      if (e == cudaSuccess) {
        ChainSeg seg;
        e = dev_alloc(seg.x, (size_t)size * xs * sizeof(double));
        if (e == cudaSuccess) e = dev_alloc(seg.lp, (size_t)size * ls * sizeof(double));
        if (e == cudaSuccess) e = dev_alloc(ring->slot_mask, (size_t)size * N);
        ring->segs.push_back(std::move(seg));
        ring->start.push_back(size);
      }
      CK_NOMEM(c, e, "eb_window_config: %llu slots of %zu bytes: allocation failed (%s)", (unsigned long long)size,
               per_slot, cudaGetErrorString(alloc_err));
      std::vector<uint64_t> steps((size_t)size), seeds((size_t)size);
      ring->ring = true;
      win.ring = std::move(ring);
      win.steps.swap(steps);
      win.seeds.swap(seeds);
    }
    win.ring->origin = 0;
    win.ring->filled = 0;
    win.n = 0;
    return EB_OK;
  });
}

int eb_window_count(eb_ctx* c, uint64_t* recorded, uint64_t* filled) {
  if (!c) return EB_ERR_INVALID;
  const RunWindow& win = c->run.window;
  if (!win.ring) FAIL(c, EB_ERR_STATE, "eb_window_count: configure the window with eb_window_config first");
  if (recorded) *recorded = win.n;
  if (filled) *filled = win.ring->filled;
  return EB_OK;
}

int eb_window_steps(eb_ctx* c, uint64_t* steps, uint64_t* seeds) {
  if (!c) return EB_ERR_INVALID;
  const RunWindow& win = c->run.window;
  if (!win.ring) FAIL(c, EB_ERR_STATE, "eb_window_steps: configure the window with eb_window_config first");
  const uint64_t size = win.ring->start.back();
  for (uint64_t k = 0; k < win.ring->filled; ++k) {
    const size_t slot = (size_t)((win.ring->origin + k) % size);
    if (steps) steps[k] = win.steps[slot];
    if (seeds) seeds[k] = win.seeds[slot];
  }
  return EB_OK;
}

int eb_window_chain(eb_ctx* c, eb_chain** ring) {
  if (!c || !ring) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->run.window.ring) FAIL(c, EB_ERR_STATE, "eb_window_chain: configure the window with eb_window_config first");
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaStreamSynchronize(c->st.get()));  // the ring's reads run on its own stream, behind the steps' stores
  *ring = c->run.window.ring.get();
  return EB_OK;
}

}  // extern "C"
