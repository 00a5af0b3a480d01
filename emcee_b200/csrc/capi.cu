// C ABI of the engine (include/emcee_b200.h): context, state / model transfer, error mapping; the step driver
// is in step.cu.  No torch, no CPU fallback.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "chain_map.h"
#include "context.h"

static thread_local std::string g_create_err;

static const char* const MSG_BLOBS_WITH_LOG_PROB =  // moves/move.py:38-42
    "If you start sampling with a given log_prob, you also need to provide the current list of blobs at that "
    "position.";

// map (and clear) the device status word to the reference's exceptions, in the
// order compute_log_prob raises them (ensemble.py:476-479, 550-551)
int check_status(eb_ctx* c) {
  int f = *c->status_host;
  c->gm_unchecked = false;
  // a graph model or a captured proposal: the first error its half-steps recorded, which later ones may have added
  // flags to
  const unsigned long long g = graph_errors(c) ? *c->graph_err_host : 0ull;
  if (g != 0) {
    *c->graph_err_host = 0;
    cudaMemsetAsync(c->graph_err.get(), 0, sizeof(unsigned long long), c->st.get());
    f = (int)(g & 0xff);
    const uint64_t es = g >> 16;
    // inside a stepping call: back to the step that failed, as if the call had stopped there
    if (((g >> 8) & 0xff) != GRAPH_NO_SPLIT && c->graph_run && es >= c->graph_step0 && es <= c->step) {
      for (uint64_t s = es; s < c->step; ++s) c->picks[c->graph_picks[(size_t)(s - c->graph_step0)]] -= 1;
      c->step = es;
    }
  } else if (f == 0 && c->graph_run) {
    c->graph_step0 = c->step;  // every step enqueued so far completed without an error
    c->graph_picks.clear();
  }
  if (f == 0) return EB_OK;
  *c->status_host = 0;
  cudaMemsetAsync(c->status_dev.get(), 0, sizeof(int), c->st.get());
  cudaStreamSynchronize(c->st.get());
  if (f & FLAG_COMM_TIMEOUT) FAIL(c, EB_ERR_COMM, "peer-memory barrier timed out: another rank did not arrive");
  if (f & FLAG_WAIT_TIMEOUT) FAIL(c, EB_ERR_CUDA, "kernel stalled: a warp waited ~2 minutes for a hand-off in its block");
  if (f & FLAG_KDE_SINGULAR)  // scipy/stats/_kde.py, gaussian_kde.__init__'s LinAlgError
    FAIL(c, EB_ERR_SINGULAR,
         "The data appears to lie in a lower-dimensional subspace of the space in which it is expressed. This has "
         "resulted in a singular data covariance matrix, which cannot be treated using the algorithms implemented in "
         "`gaussian_kde`. Consider performing principal component analysis / dimensionality reduction and using "
         "`gaussian_kde` with the transformed data.");
  if (f & FLAG_NAN_INITIAL) FAIL(c, EB_ERR_NAN_INITIAL, "The initial log_prob was NaN");  // ensemble.py:357-358
  if (f & FLAG_INF_PARAM) FAIL(c, EB_ERR_INF_PARAM, "At least one parameter value was infinite");
  if (f & FLAG_NAN_PARAM) FAIL(c, EB_ERR_NAN_PARAM, "At least one parameter value was NaN");
  FAIL(c, EB_ERR_NAN_LOGPROB, "Probability function returned NaN");
}

int enqueue_status_read(eb_ctx* c) {
  CK(c, cudaMemcpyAsync(c->status_host.get(), c->status_dev.get(), sizeof(int), cudaMemcpyDeviceToHost, c->st.get()));
  if (graph_errors(c))
    CK(c, cudaMemcpyAsync(c->graph_err_host.get(), c->graph_err.get(), sizeof(unsigned long long),
                          cudaMemcpyDeviceToHost, c->st.get()));
  return EB_OK;
}

int fetch_status(eb_ctx* c) {
  const int rc = enqueue_status_read(c);
  if (rc) return rc;
  CK(c, cudaStreamSynchronize(c->st.get()));
  return check_status(c);
}

// the arguments eb_create and eb_chain_create (`who`) share
static int check_create_args(const char* who, int device, int64_t nwalkers, int64_t ndim) {
  if (nwalkers < 2 || ndim < 1 || nwalkers > (int64_t)0x7fffffff || ndim > 16384) {
    g_create_err = std::string(who) + ": need 2 <= nwalkers < 2^31 and 1 <= ndim <= 16384";
    return EB_ERR_INVALID;
  }
  int ndev = 0;
  const cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    g_create_err =
        std::string(who) + ": no CUDA device (" + cudaGetErrorString(e) + "); this engine has no CPU fallback";
    return EB_ERR_CUDA;
  }
  if (device < 0 || device >= ndev) {
    g_create_err = std::string(who) + ": device index out of range";
    return EB_ERR_INVALID;
  }
  return EB_OK;
}

// a failed step of eb_create / eb_chain_create; the owner the object is built in frees what exists of it
#define CREATE_CK(call)                                                                       \
  do {                                                                                        \
    const cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                                  \
      cudaGetLastError();                                                                     \
      g_create_err = std::string(__func__) + ": " + #call + ": " + cudaGetErrorString(_e);    \
      return EB_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

extern "C" {

int eb_abi_version(void) { return EB_ABI_VERSION; }

int eb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

const char* eb_last_error(const eb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int eb_create(int device, int64_t nwalkers, int64_t ndim, uint64_t seed, eb_ctx** out) {
  if (!out) return EB_ERR_INVALID;
  *out = nullptr;
  const int rc = check_create_args("eb_create", device, nwalkers, ndim);
  if (rc) return rc;
  std::unique_ptr<eb_ctx> c(new eb_ctx());
  c->device = device;
  c->N = nwalkers;
  c->D = (int)ndim;
  c->seed = seed;
  if (const char* e = getenv("EMCEE_B200_TMA_ROWS")) c->allow_tma = atoi(e);  // developer override
  CREATE_CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CREATE_CK(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  CREATE_CK(stream_create(c->st, cudaStreamNonBlocking));
  CREATE_CK(event_create(c->ev0));
  CREATE_CK(event_create(c->ev1));
  cudaStream_t st = c->st.get();
  const size_t nd = (size_t)nwalkers * (size_t)ndim;
  // the tail holds the peer-memory barrier flags so one IPC handle exports both
  CREATE_CK(dev_alloc(c->coords, nd * sizeof(double) + MAX_RANKS * sizeof(unsigned)));
  CREATE_CK(dev_alloc(c->logp, (size_t)nwalkers * sizeof(double)));
  CREATE_CK(dev_alloc(c->accepted, (size_t)nwalkers));
  CREATE_CK(dev_alloc(c->nacc, (size_t)nwalkers * sizeof(unsigned long long)));
  CREATE_CK(dev_alloc(c->status_dev, sizeof(int)));
  CREATE_CK(host_alloc(c->status_host, sizeof(int)));
  *c->status_host = 0;
  CREATE_CK(cudaMemsetAsync(c->status_dev.get(), 0, sizeof(int), st));
  CREATE_CK(cudaMemsetAsync(c->accepted.get(), 0, (size_t)nwalkers, st));
  CREATE_CK(cudaMemsetAsync(c->nacc.get(), 0, (size_t)nwalkers * sizeof(unsigned long long), st));
  // split tables for a chunk of steps: <= 64 MiB, 1..512 steps
  size_t cap = (64u << 20) / ((size_t)nwalkers * sizeof(int32_t));
  cap = std::max<size_t>(1, std::min<size_t>(cap, 512));
  c->table_cap = cap;
  CREATE_CK(dev_alloc(c->order, cap * (size_t)nwalkers * sizeof(int32_t)));
  CREATE_CK(dev_alloc(c->info_dev, cap * sizeof(StepInfo)));
  CREATE_CK(host_alloc(c->info_host, cap * sizeof(StepInfo)));
  CREATE_CK(dev_alloc(c->descs_dev, cap * MAX_SPLITS * sizeof(HalfDesc)));
  CREATE_CK(host_alloc(c->descs_host, cap * MAX_SPLITS * sizeof(HalfDesc)));
  CREATE_CK(dev_alloc(c->gbar, sizeof(unsigned long long)));
  CREATE_CK(cudaMemsetAsync(c->gbar.get(), 0, sizeof(unsigned long long), st));
  CREATE_CK(cudaStreamSynchronize(st));
  *out = c.release();
  return EB_OK;
}

int eb_create_batch(int device, int64_t nbatch, int64_t nwalkers, int64_t ndim, const uint64_t* seeds,
                    eb_ctx** out) {
  if (!out) return EB_ERR_INVALID;
  *out = nullptr;
  if (!seeds || nbatch < 1 || nwalkers < 2 || nbatch > (int64_t)0x7fffffff / nwalkers) {
    g_create_err = "eb_create_batch: need nbatch >= 1, nwalkers >= 2, seeds, and nbatch * nwalkers < 2^31 (the int32 "
                   "split tables)";
    return EB_ERR_INVALID;
  }
  const int64_t rows = nbatch * nwalkers;
  int rc = check_create_args("eb_create_batch", device, rows, ndim);
  if (rc) return rc;
  // what eb_create allocates for the rows (state, counters, split tables up to 64 MiB), against the free memory
  CREATE_CK(cudaSetDevice(device));
  size_t free_b = 0, total_b = 0;
  CREATE_CK(cudaMemGetInfo(&free_b, &total_b));
  const double need = (double)rows * ((double)ndim * 8.0 + 8.0 + 1.0 + 8.0 + 4.0) + (double)(64u << 20);
  if (need > (double)free_b) {
    char b[256];
    snprintf(b, sizeof(b), "eb_create_batch: %lld ensembles of %lld x %lld need about %.0f bytes, %zu bytes free",
             (long long)nbatch, (long long)nwalkers, (long long)ndim, need, free_b);
    g_create_err = b;
    return EB_ERR_NOMEM;
  }
  eb_ctx* c = nullptr;
  rc = eb_create(device, rows, ndim, 0, &c);
  if (rc) return rc;
  std::unique_ptr<eb_ctx> owner(c);
  c->nbatch = nbatch;
  c->bn = nwalkers;
  c->seeds.assign(seeds, seeds + nbatch);
  c->allow_dmma = false;  // a batch runs batch_half_step_kernel, and the initial log-probabilities the generic kernel
  c->allow_tma = 0;
  CREATE_CK(dev_alloc(c->seeds_dev, (size_t)nbatch * sizeof(uint64_t)));
  CREATE_CK(cudaMemcpy(c->seeds_dev.get(), seeds, (size_t)nbatch * sizeof(uint64_t), cudaMemcpyHostToDevice));
  *out = owner.release();
  return EB_OK;
}

int eb_batch_rng_get(const eb_ctx* c, uint64_t* seeds, uint64_t* step) {
  if (!c || c->nbatch == 0) return c ? EB_ERR_UNSUPPORTED : EB_ERR_INVALID;
  if (seeds) std::copy(c->seeds.begin(), c->seeds.end(), seeds);
  if (step) *step = c->step;
  return EB_OK;
}

int eb_batch_rng_set(eb_ctx* c, const uint64_t* seeds, uint64_t step) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (c->nbatch == 0) FAIL(c, EB_ERR_UNSUPPORTED, "eb_batch_rng_set: not a batch context (eb_set_rng)");
  if (!seeds) FAIL(c, EB_ERR_INVALID, "eb_batch_rng_set: null seeds");
  if (!std::equal(c->seeds.begin(), c->seeds.end(), seeds)) {
    CK(c, cudaSetDevice(c->device));
    CK(c, cudaStreamSynchronize(c->st.get()));  // the split-table launches still read seeds_dev
    CK(c, cudaMemcpy(c->seeds_dev.get(), seeds, (size_t)c->nbatch * sizeof(uint64_t), cudaMemcpyHostToDevice));
    c->seeds.assign(seeds, seeds + c->nbatch);
    c->tbl_n = 0;  // the cached split tables were built under the old keys
  }
  c->step = step;
  return EB_OK;
}

int eb_destroy(eb_ctx* c) {
  if (!c) return EB_OK;
  NOT_IN_CALLBACK(c);
  cudaSetDevice(c->device);
  comm_destroy(c->comm);  // before any free: coords is exported to the peers
  cudaStreamSynchronize(c->st.get());
  delete c;  // the owners release the buffers, then the events and the stream
  cudaGetLastError();
  return EB_OK;
}

// ---- model -----------------------------------------------------------------
// Lower Cholesky factor of the symmetric part of A, packed for the DMMA kernel
// (dense_dmma.cu).  Returns false when A is not numerically positive definite.
static bool cholesky_lower(const double* A, int D, std::vector<double>& L) {
  L.assign((size_t)D * D, 0.0);
  for (int j = 0; j < D; ++j) {
    double d = 0.5 * (A[(size_t)j * D + j] + A[(size_t)j * D + j]);
    for (int k = 0; k < j; ++k) d -= L[(size_t)j * D + k] * L[(size_t)j * D + k];
    if (!(d > 0.0) || !isfinite(d)) return false;
    const double ljj = sqrt(d);
    L[(size_t)j * D + j] = ljj;
    for (int i = j + 1; i < D; ++i) {
      double s = 0.5 * (A[(size_t)i * D + j] + A[(size_t)j * D + i]);
      for (int k = 0; k < j; ++k) s -= L[(size_t)i * D + k] * L[(size_t)j * D + k];
      L[(size_t)i * D + j] = s / ljj;
    }
  }
  return true;
}

int eb_model_set(eb_ctx* c, int kind, const double* params, size_t nparams) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  const size_t D = (size_t)c->D;
  ModelDev m{};
  m.kind = kind;
  std::vector<double> host;
  switch (kind) {
    case EB_MODEL_GAUSS_ISO:
      if (nparams != 0) FAIL(c, EB_ERR_INVALID, "gauss_iso takes no parameters");
      break;
    case EB_MODEL_GAUSS_DENSE:
      if (nparams != D + D * D || !params)
        FAIL(c, EB_ERR_INVALID, "gauss_dense takes mu[D] followed by A[D*D] (got %zu doubles)", nparams);
      for (size_t k = 0; k < nparams; ++k)
        if (!isfinite(params[k])) FAIL(c, EB_ERR_INVALID, "gauss_dense parameters must be finite");
      host.assign(params, params + nparams);
      for (size_t k = 0; k < D; ++k)
        if (params[k] != 0.0) m.s0 = 1.0;  // non-zero mean (dense_dmma.cu picks its variant by this)
      break;
    case EB_MODEL_ROSENBROCK:
    case EB_MODEL_RING:
      if (nparams != 2 || !params) FAIL(c, EB_ERR_INVALID, "model takes exactly 2 parameters");
      if (kind == EB_MODEL_RING && !(params[1] > 0.0)) FAIL(c, EB_ERR_INVALID, "ring sigma must be > 0");
      if (kind == EB_MODEL_ROSENBROCK && D < 2) FAIL(c, EB_ERR_INVALID, "rosenbrock needs ndim >= 2");
      m.s0 = params[0];
      m.s1 = params[1];
      break;
    default:
      FAIL(c, EB_ERR_INVALID, "unknown model kind %d", kind);
  }
  CK(c, cudaStreamSynchronize(c->st.get()));
  DevPtr<double> dparams, dchol;
  if (!host.empty()) {
    CK(c, dev_alloc(dparams, host.size() * sizeof(double)));
    CK(c, cudaMemcpy(dparams.get(), host.data(), host.size() * sizeof(double), cudaMemcpyHostToDevice));
    m.params = dparams.get();
    if (kind == EB_MODEL_GAUSS_DENSE && dense_dmma_supported(c->D)) {
      std::vector<double> L;
      if (cholesky_lower(host.data() + D, c->D, L)) {
        std::vector<double> packed(dense_dmma_factor_doubles(c->D));
        dense_dmma_pack_factor(L.data(), c->D, packed.data());
        CK(c, dev_alloc(dchol, packed.size() * sizeof(double)));
        CK(c, cudaMemcpy(dchol.get(), packed.data(), packed.size() * sizeof(double), cudaMemcpyHostToDevice));
        m.chol = dchol.get();
      }
    }
  }
  c->model_params = std::move(dparams);
  c->model_chol = std::move(dchol);
  c->model_box.reset();  // a new model starts unbounded
  c->model = m;
  c->have_model = true;
  c->cb_fn = nullptr;
  c->cb_user = nullptr;
  c->graphs.clear();
  c->blob_bytes = 0;
  c->blobs_live = false;
  return EB_OK;
}

int eb_model_set_callback(eb_ctx* c, eb_logprob_fn fn, void* user, int where) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!fn) FAIL(c, EB_ERR_INVALID, "eb_model_set_callback: null function");
  if (where != EB_CALLBACK_HOST && where != EB_CALLBACK_DEVICE)
    FAIL(c, EB_ERR_INVALID, "eb_model_set_callback: where must be EB_CALLBACK_HOST or EB_CALLBACK_DEVICE (got %d)", where);
  if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "log-probability callbacks are not sharded across GPUs");
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaStreamSynchronize(c->st.get()));
  if (!c->ext_f) CK(c, dev_alloc(c->ext_f, (size_t)c->N * sizeof(double)));
  if (!c->ext_lp) CK(c, dev_alloc(c->ext_lp, (size_t)c->N * sizeof(double)));
  if (!c->qbuf) CK(c, dev_alloc(c->qbuf, (size_t)c->N * c->D * sizeof(double)));
  c->model_params.reset();
  c->model_chol.reset();
  c->model_box.reset();
  c->model = ModelDev{};
  c->model.kind = MODEL_EXTERNAL;
  c->cb_fn = fn;
  c->cb_user = user;
  c->cb_where = where;
  c->graphs.clear();
  c->have_model = true;
  c->blob_bytes = 0;
  c->blobs_live = false;
  return EB_OK;
}

// device buffers for records of `record_bytes` (live + one call's proposals, and the host-mode staging): the size
// is checked against the free device memory before any allocation, as eb_chain_grow does
static int ensure_blob_buffers(eb_ctx* c, size_t record_bytes) {
  const size_t N = (size_t)c->N;
  const bool host = c->cb_where == EB_CALLBACK_HOST;
  if (record_bytes > ((size_t)1 << 40) / N)
    FAIL(c, EB_ERR_NOMEM, "blob records of %zu bytes for %zu walkers do not fit in device memory", record_bytes, N);
  const size_t need = N * record_bytes;
  if (need <= c->blob_cap && (!host || c->blob_host)) return EB_OK;
  CK(c, cudaStreamSynchronize(c->st.get()));
  size_t free_b = 0, total_b = 0;
  CK(c, cudaMemGetInfo(&free_b, &total_b));
  const size_t held = 2 * c->blob_cap;  // freed below before the new buffers are allocated
  if (2 * need > free_b + held)
    FAIL(c, EB_ERR_NOMEM, "blob buffers need %zu bytes of device memory, %zu are free", 2 * need, free_b + held);
  c->blob_live.reset();
  c->blob_prop.reset();
  c->blob_host.reset();
  c->blob_cap = 0;
  c->blobs_live = false;
  DevPtr<uint8_t> live, prop;
  HostPtr<uint8_t> staging;
  cudaError_t e = dev_alloc(live, need);
  if (e == cudaSuccess) e = dev_alloc(prop, need);
  if (e == cudaSuccess && host) e = host_alloc(staging, need);
  CK_NOMEM(c, e, "allocating %zu bytes of blob buffers failed", 2 * need);
  c->blob_live = std::move(live);
  c->blob_prop = std::move(prop);
  c->blob_host = std::move(staging);
  c->blob_cap = need;
  return EB_OK;
}

}  // extern "C"

// m records of `width` bytes, `spitch` apart in src (device or host memory), packed into dst on stream st
// (eb_callback_result, eb_callback_blobs, the device-memory transfers): ordered after the producer's work, complete
// when this returns.  Obj: anything with an `err` string (FAIL / CK)
template <class Obj>
static int copy_ordered(Obj* c, cudaStream_t st, void* dst, const void* src, size_t width, size_t spitch, size_t m,
                        uint64_t src_stream) {
  if (src_stream == EB_STREAM_UNKNOWN) {
    // a producer that names no stream (CUDA Array Interface v2, e.g. torch): its last kernel may be on any
    // stream of the device, so wait for all of them
    CK(c, cudaDeviceSynchronize());
  } else if (src_stream != 0) {
    // the producer's work on its stream comes first (CUDA Array Interface v3 stream encoding)
    cudaStream_t s = src_stream == 1 ? cudaStreamLegacy
                     : src_stream == 2 ? cudaStreamPerThread
                                       : reinterpret_cast<cudaStream_t>((uintptr_t)src_stream);
    EventPtr ev;
    CK(c, event_create(ev, cudaEventDisableTiming));
    CK(c, cudaEventRecord(ev.get(), s));
    CK(c, cudaStreamWaitEvent(st, ev.get(), 0));
  }
  if (spitch == width || m == 1)
    CK(c, cudaMemcpyAsync(dst, src, width * m, cudaMemcpyDefault, st));
  else
    CK(c, cudaMemcpy2DAsync(dst, width, src, spitch, width, m, cudaMemcpyDefault, st));
  CK(c, cudaStreamSynchronize(st));  // the caller may free or reuse src as soon as this returns
  return EB_OK;
}

static int copy_records(eb_ctx* c, void* dst, const void* src, size_t width, size_t spitch, size_t m,
                        uint64_t src_stream) {
  return copy_ordered(c, c->st.get(), dst, src, width, spitch, m, src_stream);
}

// a pointer the device-memory transfers take (eb_set_state_from, ...): device or managed memory of `device`
template <class Obj>
static int check_device_ptr(Obj* c, int device, const void* p, const char* who, const char* what) {
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    FAIL(c, EB_ERR_INVALID, "%s: %s is not CUDA memory (%s)", who, what, cudaGetErrorString(e));
  }
  if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
    FAIL(c, EB_ERR_INVALID, "%s: %s is not device memory", who, what);
  if (a.device != device) FAIL(c, EB_ERR_INVALID, "%s: %s is on device %d, not on device %d", who, what, a.device, device);
  return EB_OK;
}

// the first-axis stride of m rows of `row` bytes in device memory: a positive multiple of 8, at least a row
static bool row_stride_ok(int64_t stride, int64_t row, int64_t m) {
  return m <= 1 || (stride >= row && stride % 8 == 0);
}

extern "C" {

int eb_callback_blobs(eb_ctx* c, const void* src, int64_t record_bytes, int64_t stride_bytes, int64_t m,
                      uint64_t src_stream) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_callback_blobs");
  if (!c->in_callback) FAIL(c, EB_ERR_STATE, "eb_callback_blobs: only from inside a log-probability callback");
  if (c->cb_blob_rows >= 0) FAIL(c, EB_ERR_INVALID, "eb_callback_blobs: this call's blobs were already delivered");
  if (m != c->cb_m)
    FAIL(c, EB_ERR_INVALID, "the function returned %lld blob records for %lld rows", (long long)m, (long long)c->cb_m);
  if (record_bytes <= 0) FAIL(c, EB_ERR_INVALID, "eb_callback_blobs: records must have at least one byte");
  if (m > 1 && stride_bytes < record_bytes)
    FAIL(c, EB_ERR_INVALID, "eb_callback_blobs: the stride (%lld bytes) is shorter than a record (%lld bytes)",
         (long long)stride_bytes, (long long)record_bytes);
  if (m > 0 && !src) FAIL(c, EB_ERR_INVALID, "eb_callback_blobs: null records");
  const size_t R = (size_t)record_bytes;
  uint8_t* dst = nullptr;
  bool to_host = c->cb_where == EB_CALLBACK_HOST;
  switch (c->cb_phase) {
    case CB_SET_STATE: {  // the initial evaluation fixes the live layout
      int rc = ensure_blob_buffers(c, R);
      if (rc) return rc;
      dst = c->blob_live.get();
      break;
    }
    case CB_STEP:
      if (!c->blobs_live) FAIL(c, EB_ERR_INVALID, "%s", MSG_BLOBS_WITH_LOG_PROB);
      if (R != c->blob_bytes)
        FAIL(c, EB_ERR_INVALID, "the function returned blob records of %zu bytes; the state's records have %zu", R,
             c->blob_bytes);
      dst = c->blob_prop.get();
      break;
    default:  // CB_COMPUTE: straight to the caller's pinned buffer
      if (c->blob_bytes && R != c->blob_bytes)
        FAIL(c, EB_ERR_INVALID, "the function returned blob records of %zu bytes; the state's records have %zu", R,
             c->blob_bytes);
      c->cmp_blobs.reset();
      CK_NOMEM(c, host_alloc(c->cmp_blobs, std::max<size_t>(1, (size_t)m * R)),
               "allocating %zu bytes of pinned host memory for blobs failed", (size_t)m * R);
      dst = c->cmp_blobs.get();
      to_host = false;  // copied below, whatever the mode
  }
  if (m > 0) {
    if (to_host) {
      // host mode: into the pinned staging; run_callback copies it to dst next to the lp copy-back
      const uint8_t* s = static_cast<const uint8_t*>(src);
      if ((size_t)stride_bytes == R)
        memcpy(c->blob_host.get(), s, (size_t)m * R);
      else
        for (int64_t r = 0; r < m; ++r) memcpy(c->blob_host.get() + (size_t)r * R, s + (size_t)r * stride_bytes, R);
      c->cb_blob_dst = dst;
    } else {
      int rc = copy_records(c, dst, src, R, (size_t)stride_bytes, (size_t)m, src_stream);
      if (rc) return rc;
      c->cb_blob_dst = nullptr;
    }
  }
  c->cb_blob_rows = m;
  c->cb_blob_bytes = R;
  return EB_OK;
}

int eb_callback_result(eb_ctx* c, double* lp, const void* src, int64_t stride_bytes, int64_t m, uint64_t src_stream) {
  if (!c) return EB_ERR_INVALID;
  if (!c->in_callback || c->cb_where != EB_CALLBACK_DEVICE)
    FAIL(c, EB_ERR_STATE, "eb_callback_result: only from inside a device-mode log-probability callback");
  if (m < 0 || (m > 0 && (!lp || !src))) FAIL(c, EB_ERR_INVALID, "eb_callback_result: null buffer");
  if (stride_bytes <= 0 || stride_bytes % (int64_t)sizeof(double) != 0)
    FAIL(c, EB_ERR_INVALID, "eb_callback_result: the stride must be a positive multiple of 8 bytes (got %lld)",
         (long long)stride_bytes);
  if (m == 0) return EB_OK;
  return copy_records(c, lp, src, sizeof(double), (size_t)stride_bytes, (size_t)m, src_stream);
}

// the device word of the first error of a graph model's or a captured proposal's half-steps (graph_err_word)
static int ensure_graph_err(eb_ctx* c) {
  if (c->graph_err) return EB_OK;
  DevPtr<unsigned long long> err;
  HostPtr<unsigned long long> err_host;
  CK(c, dev_alloc(err, sizeof(unsigned long long)));
  CK(c, host_alloc(err_host, sizeof(unsigned long long)));
  CK(c, cudaMemset(err.get(), 0, sizeof(unsigned long long)));
  *err_host = 0;
  c->graph_err = std::move(err);
  c->graph_err_host = std::move(err_host);
  return EB_OK;
}

int eb_model_set_graphs(eb_ctx* c, const eb_graph* graphs, size_t n) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_model_set_graphs");
  NOT_IN_CALLBACK(c);
  if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "log-probability graphs are not sharded across GPUs");
  if (!graphs || n == 0) FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: no graphs");
  const int64_t row = (int64_t)c->D * (int64_t)sizeof(double);
  std::vector<eb_ctx::Graph> set;
  bool have_n = false;
  CK(c, cudaSetDevice(c->device));
  for (size_t k = 0; k < n; ++k) {
    const eb_graph& g = graphs[k];
    if (g.m < 1 || g.m > c->N)
      FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: graph %zu has %lld rows; a graph takes 1 to %lld rows", k,
           (long long)g.m, (long long)c->N);
    for (const eb_ctx::Graph& h : set)
      if (h.m == g.m) FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: two graphs for %lld rows", (long long)g.m);
    if (g.exec == 0) FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: graph %zu has no executable graph", k);
    if (!g.x || !g.lp) FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: graph %zu has a null buffer", k);
    if (g.x_row_stride_bytes <= 0 || g.x_row_stride_bytes % 8 != 0 || (g.m > 1 && g.x_row_stride_bytes < row))
      FAIL(c, EB_ERR_INVALID,
           "eb_model_set_graphs: the row stride of x must be a multiple of 8 bytes, at least %lld (got %lld)",
           (long long)row, (long long)g.x_row_stride_bytes);
    if (g.lp_stride_bytes <= 0 || g.lp_stride_bytes % 8 != 0)
      FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: the stride of lp must be a positive multiple of 8 bytes (got %lld)",
           (long long)g.lp_stride_bytes);
    int rc = check_device_ptr(c, c->device, g.x, "eb_model_set_graphs", "x");
    if (!rc) rc = check_device_ptr(c, c->device, g.lp, "eb_model_set_graphs", "lp");
    if (rc) return rc;
    set.push_back(eb_ctx::Graph{g.m, reinterpret_cast<cudaGraphExec_t>((uintptr_t)g.exec), static_cast<double*>(g.x),
                                g.x_row_stride_bytes, static_cast<const double*>(g.lp), g.lp_stride_bytes});
    have_n |= g.m == c->N;
  }
  if (!have_n)
    FAIL(c, EB_ERR_INVALID, "eb_model_set_graphs: no graph for nwalkers = %lld rows", (long long)c->N);
  CK(c, cudaStreamSynchronize(c->st.get()));
  if (!c->ext_f) CK(c, dev_alloc(c->ext_f, (size_t)c->N * sizeof(double)));
  if (!c->ext_lp) CK(c, dev_alloc(c->ext_lp, (size_t)c->N * sizeof(double)));
  if (!c->qbuf) CK(c, dev_alloc(c->qbuf, (size_t)c->N * c->D * sizeof(double)));
  const int rc = ensure_graph_err(c);
  if (rc) return rc;
  c->model_params.reset();
  c->model_chol.reset();
  c->model_box.reset();
  c->model = ModelDev{};
  c->model.kind = MODEL_EXTERNAL;
  c->cb_fn = nullptr;
  c->cb_user = nullptr;
  c->cb_where = EB_CALLBACK_GRAPH;
  c->graphs = std::move(set);
  c->have_model = true;
  c->blob_bytes = 0;
  c->blobs_live = false;
  return EB_OK;
}

int eb_move_set_proposal(eb_ctx* c, int32_t slot, eb_proposal_fn fn, void* user, int where) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_move_set_proposal");
  NOT_IN_CALLBACK(c);
  if (slot < 0 || slot >= EB_MAX_PROPOSAL_SLOTS)
    FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal: slot must be in [0, %d) (got %d)", EB_MAX_PROPOSAL_SLOTS, slot);
  if (fn && where != EB_CALLBACK_HOST && where != EB_CALLBACK_DEVICE)
    FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal: where must be EB_CALLBACK_HOST or EB_CALLBACK_DEVICE (got %d)", where);
  if (fn && c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "user proposals are not sharded across GPUs");
  if ((size_t)slot >= c->props.size()) c->props.resize((size_t)slot + 1);
  c->props[(size_t)slot].fn = fn;
  c->props[(size_t)slot].user = fn ? user : nullptr;
  c->props[(size_t)slot].where = where;
  if ((size_t)slot < c->prop_graphs.size()) c->prop_graphs[(size_t)slot] = eb_ctx::ProposalGraphs{};
  return EB_OK;
}

// a buffer of rows `rows` long of `width` doubles each, row_stride bytes apart
static int check_graph_rows(eb_ctx* c, size_t k, const char* what, const void* p, int64_t row_stride, int64_t rows,
                            int64_t width) {
  if (!p) FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: graph %zu has a null %s", k, what);
  const int64_t row = width * (int64_t)sizeof(double);
  if (row_stride <= 0 || row_stride % 8 != 0 || (rows > 1 && row_stride < row))
    FAIL(c, EB_ERR_INVALID,
         "eb_move_set_proposal_graphs: the row stride of %s must be a positive multiple of 8 bytes, at least %lld "
         "(got %lld)",
         what, (long long)row, (long long)row_stride);
  return check_device_ptr(c, c->device, p, "eb_move_set_proposal_graphs", what);
}

int eb_move_set_proposal_graphs(eb_ctx* c, int32_t slot, int draw_kind, int64_t ndraws, const eb_proposal_graph* graphs,
                                size_t n) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_move_set_proposal_graphs");
  NOT_IN_CALLBACK(c);
  if (slot < 0 || slot >= EB_MAX_PROPOSAL_SLOTS)
    FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: slot must be in [0, %d) (got %d)", EB_MAX_PROPOSAL_SLOTS,
         slot);
  if (c->comm.nranks > 1) FAIL(c, EB_ERR_UNSUPPORTED, "user proposals are not sharded across GPUs");
  if (draw_kind != EB_DRAW_UNIFORM && draw_kind != EB_DRAW_NORMAL)
    FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: draw_kind must be EB_DRAW_UNIFORM or EB_DRAW_NORMAL (got %d)",
         draw_kind);
  if (ndraws < 0) FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: ndraws must be >= 0 (got %lld)", (long long)ndraws);
  if (ndraws > EB_MAX_GRAPH_DRAWS)
    FAIL(c, EB_ERR_UNSUPPORTED, "a captured proposal takes at most %d draws per row (got %lld)", EB_MAX_GRAPH_DRAWS,
         (long long)ndraws);
  if (!graphs || n == 0) FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: no graphs");
  std::vector<eb_ctx::ProposalGraph> set;
  CK(c, cudaSetDevice(c->device));
  for (size_t k = 0; k < n; ++k) {
    const eb_proposal_graph& g = graphs[k];
    if (g.split < 0 || g.split >= MAX_SPLITS)
      FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: graph %zu has split %d; a split is in [0, %d)", k,
           (int)g.split, MAX_SPLITS);
    for (const eb_ctx::ProposalGraph& h : set)
      if (h.split == g.split)
        FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: two graphs for split %d", (int)g.split);
    if (g.ns < 1 || g.ns > c->N)
      FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: graph %zu has %lld rows; a graph takes 1 to %lld rows", k,
           (long long)g.ns, (long long)c->N);
    if (g.exec == 0) FAIL(c, EB_ERR_INVALID, "eb_move_set_proposal_graphs: graph %zu has no executable graph", k);
    const int64_t nc = c->N - g.ns;
    int rc = check_graph_rows(c, k, "s", g.s, g.s_row_stride_bytes, g.ns, c->D);
    if (!rc && nc > 0) rc = check_graph_rows(c, k, "c", g.c, g.c_row_stride_bytes, nc, c->D);
    if (!rc && ndraws > 0) rc = check_graph_rows(c, k, "draws", g.draws, g.draws_row_stride_bytes, g.ns, ndraws);
    if (!rc) rc = check_graph_rows(c, k, "q", g.q, g.q_row_stride_bytes, g.ns, c->D);
    if (!rc) rc = check_graph_rows(c, k, "factors", g.factors, g.factors_stride_bytes, 1, 1);
    if (rc) return rc;
    GraphMoveBufs b{};
    b.s = static_cast<double*>(g.s);
    b.s_stride = g.s_row_stride_bytes / 8;
    b.c = nc > 0 ? static_cast<double*>(g.c) : nullptr;
    b.c_stride = nc > 0 ? g.c_row_stride_bytes / 8 : 0;
    b.draws = ndraws > 0 ? static_cast<double*>(g.draws) : nullptr;
    b.draws_stride = ndraws > 0 ? g.draws_row_stride_bytes / 8 : 0;
    b.q = static_cast<const double*>(g.q);
    b.q_stride = g.q_row_stride_bytes / 8;
    b.f = static_cast<const double*>(g.factors);
    b.f_stride = g.factors_stride_bytes / 8;
    set.push_back(eb_ctx::ProposalGraph{g.split, g.ns, reinterpret_cast<cudaGraphExec_t>((uintptr_t)g.exec), b});
  }
  CK(c, cudaStreamSynchronize(c->st.get()));
  if (!c->qbuf) CK(c, dev_alloc(c->qbuf, (size_t)c->N * c->D * sizeof(double)));
  if (!c->up_f) CK(c, dev_alloc(c->up_f, (size_t)c->N * sizeof(double)));
  if (!c->gm_ticket) {
    DevPtr<unsigned> t;
    CK(c, dev_alloc(t, sizeof(unsigned)));
    CK(c, cudaMemset(t.get(), 0, sizeof(unsigned)));
    c->gm_ticket = std::move(t);
  }
  const int rc = ensure_graph_err(c);
  if (rc) return rc;
  if ((size_t)slot >= c->props.size()) c->props.resize((size_t)slot + 1);
  if ((size_t)slot >= c->prop_graphs.size()) c->prop_graphs.resize((size_t)slot + 1);
  c->props[(size_t)slot] = eb_ctx::ProposalSlot{nullptr, nullptr, EB_CALLBACK_GRAPH};
  eb_ctx::ProposalGraphs& p = c->prop_graphs[(size_t)slot];
  p.graphs = std::move(set);
  p.draw_kind = draw_kind;
  p.ndraws = ndraws;
  return EB_OK;
}

int eb_proposal_result(eb_ctx* c, const void* q, int64_t q_row_stride_bytes, const void* factors,
                       int64_t f_stride_bytes, int64_t m, uint64_t src_stream) {
  if (!c) return EB_ERR_INVALID;
  if (!c->in_proposal || c->up_where != EB_CALLBACK_DEVICE || c->up_m == 0)
    FAIL(c, EB_ERR_STATE, "eb_proposal_result: only from inside a device-mode user proposal");
  if (m != c->up_m)
    FAIL(c, EB_ERR_INVALID, "the proposal returned %lld rows for %lld walkers", (long long)m, (long long)c->up_m);
  if (!q || !factors) FAIL(c, EB_ERR_INVALID, "eb_proposal_result: null buffer");
  const int64_t row = (int64_t)c->D * (int64_t)sizeof(double);
  if ((m > 1 && q_row_stride_bytes < row) || q_row_stride_bytes <= 0 || q_row_stride_bytes % 8 != 0)
    FAIL(c, EB_ERR_INVALID, "eb_proposal_result: the row stride of q must be a multiple of 8 bytes, at least %lld (got %lld)",
         (long long)row, (long long)q_row_stride_bytes);
  if (f_stride_bytes <= 0 || f_stride_bytes % 8 != 0)
    FAIL(c, EB_ERR_INVALID, "eb_proposal_result: the stride of factors must be a positive multiple of 8 bytes (got %lld)",
         (long long)f_stride_bytes);
  int rc = copy_records(c, c->qbuf.get(), q, (size_t)row, (size_t)q_row_stride_bytes, (size_t)m, src_stream);
  if (rc) return rc;
  // the first copy already waited for src_stream
  return copy_records(c, c->up_f.get(), factors, sizeof(double), (size_t)f_stride_bytes, (size_t)m, 0);
}

int eb_model_set_bounds(eb_ctx* c, const double* lower, const double* upper) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_model_set_bounds: no model set");
  if (c->model.kind == MODEL_EXTERNAL)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_model_set_bounds: a callback model has no box; apply the prior in the function");
  if ((lower == nullptr) != (upper == nullptr))
    FAIL(c, EB_ERR_INVALID, "eb_model_set_bounds: pass both bounds, or NULL for both to clear them");
  const size_t D = (size_t)c->D;
  if (lower) {
    for (size_t k = 0; k < D; ++k) {
      if (isnan(lower[k]) || isnan(upper[k])) FAIL(c, EB_ERR_INVALID, "bounds must not be NaN (parameter %zu)", k);
      if (!(lower[k] < upper[k]))
        FAIL(c, EB_ERR_INVALID, "lower bound must be below the upper bound (parameter %zu: %g >= %g)", k, lower[k],
             upper[k]);
    }
  }
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaStreamSynchronize(c->st.get()));
  DevPtr<double> box;
  if (lower) {
    CK(c, dev_alloc(box, 2 * D * sizeof(double)));
    CK(c, cudaMemcpy(box.get(), lower, D * sizeof(double), cudaMemcpyHostToDevice));
    CK(c, cudaMemcpy(box.get() + D, upper, D * sizeof(double), cudaMemcpyHostToDevice));
  }
  c->model.lo = box.get();
  c->model.hi = lower ? box.get() + D : nullptr;
  c->model_box = std::move(box);
  return EB_OK;
}

}  // extern "C"

// ---- log-prob ----------------------------------------------------------------
// the rows handed to the function for `rows` rows: pinned staging (host mode) or a device copy (device mode)
static int ensure_callback_staging(eb_ctx* c, size_t rows) {
  const bool host = c->cb_where == EB_CALLBACK_HOST;
  if (rows <= c->cb_rows && (host ? c->cb_x != nullptr : c->cb_xdev != nullptr)) return EB_OK;
  rows = std::max(rows, c->cb_rows);
  HostPtr<double> x, lp;
  DevPtr<double> xdev;
  if (host) {
    CK(c, host_alloc(x, rows * (size_t)c->D * sizeof(double)));
    CK(c, host_alloc(lp, rows * sizeof(double)));
  } else {
    CK(c, dev_alloc(xdev, rows * (size_t)c->D * sizeof(double)));
  }
  CK(c, cudaStreamSynchronize(c->st.get()));  // the old buffers may still be in use
  c->cb_x = std::move(x);
  c->cb_lp = std::move(lp);
  c->cb_xdev = std::move(xdev);
  c->cb_rows = rows;
  return EB_OK;
}

// steps 2-7 of a callback half-step (include/emcee_b200.h): the device rows x[m, D] have been enqueued;
// lp[m] (device) gets the callback's values.  scan_x: the rows were not written by a kernel that raises the
// non-finite flags (WalkMove / GaussianMove proposals, the caller's coordinates)
static const eb_ctx::Graph* find_graph(const eb_ctx* c, int64_t m) {
  for (const eb_ctx::Graph& g : c->graphs)
    if (g.m == m) return &g;
  return nullptr;
}

// rows x[rows, D] -> lp[rows] through graph g (g.m >= rows; the rows past `rows` repeat the last one), all enqueued
static int launch_graph_eval(eb_ctx* c, const eb_ctx::Graph& g, const double* x, int64_t rows, double* lp,
                             unsigned long long tag) {
  CK(c, launch_graph_stage(x, rows, g.m, c->D, g.x, g.x_stride, c->status_dev.get(), c->graph_err.get(), tag,
                           c->st.get()));
  CK(c, cudaGraphLaunch(g.exec, c->st.get()));
  CK(c, launch_graph_result(g.lp, g.lp_stride, rows, lp, c->status_dev.get(), c->graph_err.get(), tag, c->st.get()));
  return EB_OK;
}

// run_callback of a graph model (eb_model_set_graphs).  A half-step uses the graph for its m rows and leaves its
// errors on the device; the initial state and compute_log_prob run the nwalkers-row graph in chunks and report
// their errors before returning, as run_callback does.
static int run_graph(eb_ctx* c, const double* x, int64_t m, double* lp, bool scan_x) {
  const size_t D = (size_t)c->D;
  if (scan_x) CK(c, launch_scan_nonfinite(x, (size_t)m * D, 0, c->status_dev.get(), c->st.get()));
  if (c->cb_phase == CB_STEP) {
    const eb_ctx::Graph* g = find_graph(c, m);
    if (!g) FAIL(c, EB_ERR_INVALID, "no captured log-probability graph for %lld rows", (long long)m);
    return launch_graph_eval(c, *g, x, m, lp, graph_err_word(0, (unsigned)c->cb_split, c->step));
  }
  const eb_ctx::Graph* g = find_graph(c, c->N);  // eb_model_set_graphs requires it
  const unsigned long long tag = graph_err_word(0, GRAPH_NO_SPLIT, c->step);
  for (int64_t off = 0; off < m; off += c->N) {
    const int rc = launch_graph_eval(c, *g, x + (size_t)off * D, std::min<int64_t>(c->N, m - off), lp + off, tag);
    if (rc) return rc;
  }
  return fetch_status(c);
}

int run_callback(eb_ctx* c, const double* x, int64_t m, double* lp, bool scan_x) {
  if (c->cb_where == EB_CALLBACK_GRAPH) return run_graph(c, x, m, lp, scan_x);
  const size_t D = (size_t)c->D;
  if (scan_x) CK(c, launch_scan_nonfinite(x, (size_t)m * D, 0, c->status_dev.get(), c->st.get()));
  int rc = fetch_status(c);  // synchronises; ensemble.py:476-479: the function never sees a non-finite row
  if (rc) return rc;
  rc = ensure_callback_staging(c, (size_t)m);
  if (rc) return rc;
  const bool host = c->cb_where == EB_CALLBACK_HOST;
  // the function gets its own copy of the rows: writing to it cannot change the proposals the update reads
  if (host) {
    CK(c, cudaMemcpyAsync(c->cb_x.get(), x, (size_t)m * D * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
    CK(c, cudaStreamSynchronize(c->st.get()));
  } else {
    CK(c, cudaMemcpyAsync(c->cb_xdev.get(), x, (size_t)m * D * sizeof(double), cudaMemcpyDeviceToDevice, c->st.get()));
    // complete before fn runs: a consumer may ignore the stream it is given (torch does) and read x from any
    // stream of its own
    CK(c, cudaStreamSynchronize(c->st.get()));
  }
  c->cb_m = m;
  c->cb_blob_rows = -1;
  c->cb_blob_dst = nullptr;
  c->in_callback = true;
  const int r = host ? c->cb_fn(c->cb_user, c->cb_x.get(), m, (int64_t)D, c->cb_lp.get(), nullptr)
                     : c->cb_fn(c->cb_user, c->cb_xdev.get(), m, (int64_t)D, lp, (void*)c->st.get());
  c->in_callback = false;
  if (r != 0) {
    cudaStreamSynchronize(c->st.get());  // whatever the function enqueued before it failed
    FAIL(c, EB_ERR_CALLBACK, "the log-probability callback failed (returned %d)", r);
  }
  if (c->cb_phase == CB_STEP && c->blobs_live && c->cb_blob_rows < 0)
    FAIL(c, EB_ERR_INVALID, "the log-probability function returned no blobs; the state has blob records of %zu bytes",
         c->blob_bytes);
  if (host) CK(c, cudaMemcpyAsync(lp, c->cb_lp.get(), (size_t)m * sizeof(double), cudaMemcpyHostToDevice, c->st.get()));
  // host-mode blob records ride with the lp copy-back: no synchronisation of their own
  if (c->cb_blob_dst)
    CK(c, cudaMemcpyAsync(c->cb_blob_dst, c->blob_host.get(), (size_t)m * c->cb_blob_bytes, cudaMemcpyHostToDevice,
                          c->st.get()));
  CK(c, launch_scan_nonfinite(lp, (size_t)m, 1, c->status_dev.get(), c->st.get()));
  return fetch_status(c);  // ensemble.py:550-551, before any update
}

// rows of x -> out with the kernel that matches the stepping path of the model
static cudaError_t launch_logprob(eb_ctx* c, const double* x, int64_t rows, double* out) {
  if (c->allow_dmma && c->model.kind == EB_MODEL_GAUSS_DENSE && c->model.chol != nullptr)
    return launch_logprob_dense_dmma(c->model, c->D, x, rows, out, c->status_dev.get(), c->sm_count, c->st.get());
  return launch_logprob_generic(c->model, x, rows, c->D, out, c->status_dev.get(), c->st.get());
}

static int ensure_scratch(eb_ctx* c, size_t rows) {
  if (rows <= c->scratch_rows) return EB_OK;
  DevPtr<double> x, lp;
  CK(c, dev_alloc(x, rows * (size_t)c->D * sizeof(double)));
  CK(c, dev_alloc(lp, rows * sizeof(double)));
  CK(c, cudaStreamSynchronize(c->st.get()));  // the old buffers may still be in use
  c->scratch_x = std::move(x);
  c->scratch_lp = std::move(lp);
  c->scratch_rows = rows;
  return EB_OK;
}

// scratch_lp[m] = the log-probabilities of scratch_x[m] (compute_log_prob): the model's kernel, or the function
static int evaluate_scratch(eb_ctx* c, size_t m) {
  if (c->model.kind == MODEL_EXTERNAL) {
    c->cb_phase = CB_COMPUTE;
    return run_callback(c, c->scratch_x.get(), (int64_t)m, c->scratch_lp.get(), true);
  }
  CK(c, launch_logprob(c, c->scratch_x.get(), (int64_t)m, c->scratch_lp.get()));
  return EB_OK;
}

extern "C" {

int eb_compute_log_prob(eb_ctx* c, const double* coords, size_t m, double* out) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_compute_log_prob: no model set");
  if (m == 0) return EB_OK;
  if (!coords || !out) FAIL(c, EB_ERR_INVALID, "eb_compute_log_prob: null buffer");
  CK(c, cudaSetDevice(c->device));
  int rc = ensure_scratch(c, m);
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(c->scratch_x.get(), coords, m * (size_t)c->D * sizeof(double), cudaMemcpyHostToDevice,
                        c->st.get()));
  rc = evaluate_scratch(c, m);
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(out, c->scratch_lp.get(), m * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
  return fetch_status(c);
}

int eb_compute_log_prob_from(eb_ctx* c, const void* coords, int64_t row_stride_bytes, int64_t m, double* out_dst,
                             uint64_t src_stream) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_compute_log_prob_from");
  NOT_IN_CALLBACK(c);
  if (c->comm.nranks > 1)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_compute_log_prob_from: sharded ensembles take coordinates from host memory");
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_compute_log_prob_from: no model set");
  if (m < 0) FAIL(c, EB_ERR_INVALID, "eb_compute_log_prob_from: negative row count");
  if (m == 0) return EB_OK;
  if (!coords || !out_dst) FAIL(c, EB_ERR_INVALID, "eb_compute_log_prob_from: null buffer");
  const int64_t row = (int64_t)c->D * (int64_t)sizeof(double);
  if (!row_stride_ok(row_stride_bytes, row, m))
    FAIL(c, EB_ERR_INVALID, "eb_compute_log_prob_from: the row stride must be a multiple of 8 bytes, at least %lld (got %lld)",
         (long long)row, (long long)row_stride_bytes);
  CK(c, cudaSetDevice(c->device));
  int rc = check_device_ptr(c, c->device, coords, "eb_compute_log_prob_from", "coords");
  if (!rc) rc = check_device_ptr(c, c->device, out_dst, "eb_compute_log_prob_from", "out_dst");
  if (!rc) rc = ensure_scratch(c, (size_t)m);
  if (!rc) rc = copy_records(c, c->scratch_x.get(), coords, (size_t)row, (size_t)row_stride_bytes, (size_t)m, src_stream);
  if (!rc) rc = evaluate_scratch(c, (size_t)m);
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(out_dst, c->scratch_lp.get(), (size_t)m * sizeof(double), cudaMemcpyDefault, c->st.get()));
  return fetch_status(c);
}

int eb_compute_log_prob_blobs(eb_ctx* c, const double* coords, size_t m, double* out, void** blobs_out,
                              size_t* record_bytes) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_compute_log_prob_blobs");
  NOT_IN_CALLBACK(c);
  if (!blobs_out || !record_bytes) FAIL(c, EB_ERR_INVALID, "eb_compute_log_prob_blobs: null output");
  *blobs_out = nullptr;
  *record_bytes = 0;
  if (c->have_model && c->model.kind != MODEL_EXTERNAL)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_compute_log_prob_blobs: only log-probability callbacks return blobs");
  c->cmp_blobs.reset();
  c->cb_blob_rows = -1;
  const int rc = eb_compute_log_prob(c, coords, m, out);
  if (rc == EB_OK && c->cb_blob_rows >= 0 && c->cmp_blobs) {
    *blobs_out = c->cmp_blobs.release();  // the caller frees them with eb_host_free
    *record_bytes = c->cb_blob_bytes;
  }
  c->cmp_blobs.reset();
  return rc;
}

}  // extern "C"

// ---- state -------------------------------------------------------------------
// rows [r0, r1) this context owns (the whole ensemble on one GPU)
void owned_rows(const eb_ctx* c, int64_t& r0, int64_t& r1) {
  r0 = 0;
  r1 = c->N;
  if (c->comm.nranks > 1) {
    r0 = c->comm.rows_per_rank * c->comm.rank;
    r1 = r0 + c->comm.rows_per_rank;
  }
}

// multi-GPU: make log_prob / accept mask / counters (and coords in P2P mode) of every rank's rows
// valid on this rank.  COLLECTIVE: every rank calls it at the same point (the Python layer does).
int sync_replicas(eb_ctx* c) {
  if (c->comm.nranks == 1 || !c->replicas_dirty) return EB_OK;
  uint64_t launches = 0;
  if (comm_sync_state(c->comm, c->st.get(), c->status_dev.get(), c->logp.get(), c->accepted.get(), c->nacc.get(),
                      launches))
    FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  c->fused_last = false;
  CK(c, cudaStreamSynchronize(c->st.get()));
  c->replicas_dirty = false;
  return EB_OK;
}

// the initial log-probabilities of the uploaded rows [r0, r0 + rows) (ensemble.py:350-358); a user function's
// records of that evaluation become the state's blobs
static int evaluate_initial(eb_ctx* c, int64_t r0, size_t rows) {
  if (c->model.kind != MODEL_EXTERNAL) {
    CK(c, launch_logprob(c, c->coords.get() + (size_t)r0 * c->D, (int64_t)rows, c->logp.get() + r0));
    return EB_OK;
  }
  c->cb_phase = CB_SET_STATE;
  int rc = run_callback(c, c->coords.get(), (int64_t)rows, c->logp.get(), true);  // one GPU: rows == nwalkers
  if (rc) return rc;
  if (c->cb_blob_rows >= 0) {  // the records went to blob_live: they fix the live layout
    c->blob_bytes = c->cb_blob_bytes;
    c->blobs_live = true;
  }
  return EB_OK;
}

extern "C" {

int eb_set_state(eb_ctx* c, const double* coords, const double* log_prob) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!coords) FAIL(c, EB_ERR_INVALID, "eb_set_state: coords is null");
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_set_state: no model set");
  CK(c, cudaSetDevice(c->device));
  const size_t D = (size_t)c->D;
  c->have_state = false;
  c->blobs_live = false;  // a given log_prob comes without blobs (eb_set_state_blobs adds them)
  c->blob_bytes = 0;
  if (log_prob) {
    for (int64_t w = 0; w < c->N; ++w)
      if (isnan(log_prob[w])) FAIL(c, EB_ERR_NAN_INITIAL, "The initial log_prob was NaN");  // ensemble.py:357-358
  }
  // Sharded ensembles: only the rows this rank owns cross PCIe (the host arrays are still indexed by
  // global walker id); non-owned rows are never read by the kernels in P2P mode and are filled by one
  // all-gather in EB_COMM_ALLGATHER mode.
  int64_t r0, r1;
  owned_rows(c, r0, r1);
  const size_t rows = (size_t)(r1 - r0);
  uint64_t launches = 0;
  if (c->comm.nranks > 1 && c->comm.mode == EB_COMM_P2P && c->comm.imported) {
    // no peer may still be pulling the rows that are about to be overwritten
    if (comm_barrier(c->comm, c->st.get(), c->status_dev.get(), launches))
      FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
    c->fused_last = false;
  }
  CK(c, cudaMemcpyAsync(c->coords.get() + (size_t)r0 * D, coords + (size_t)r0 * D, rows * D * sizeof(double),
                        cudaMemcpyHostToDevice, c->st.get()));
  if (log_prob) {
    CK(c, cudaMemcpyAsync(c->logp.get() + r0, log_prob + r0, rows * sizeof(double), cudaMemcpyHostToDevice,
                          c->st.get()));
  } else {
    int rc = evaluate_initial(c, r0, rows);
    if (rc) return rc;
  }
  if (c->comm.nranks > 1) {
    if (c->comm.mode == EB_COMM_ALLGATHER && comm_gather_coords(c->comm, c->st.get(), launches))
      FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
    if (c->comm.mode == EB_COMM_P2P && c->comm.imported &&
        comm_barrier(c->comm, c->st.get(), c->status_dev.get(), launches))  // every rank's block is in place
      FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
    c->replicas_dirty = true;
  }
  int rc = fetch_status(c);
  if (rc) return rc;
  c->have_state = true;
  return EB_OK;
}

int eb_get_state(eb_ctx* c, double* coords, double* log_prob) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->have_state) FAIL(c, EB_ERR_STATE, "eb_get_state: no state set");
  CK(c, cudaSetDevice(c->device));
  int rc = sync_replicas(c);  // multi-GPU: the GLOBAL state (collective)
  if (rc) return rc;
  if (coords)
    CK(c, cudaMemcpyAsync(coords, c->coords.get(), (size_t)c->N * c->D * sizeof(double), cudaMemcpyDeviceToHost,
                          c->st.get()));
  if (log_prob)
    CK(c, cudaMemcpyAsync(log_prob, c->logp.get(), (size_t)c->N * sizeof(double), cudaMemcpyDeviceToHost, c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_set_state_from(eb_ctx* c, const void* coords, int64_t coords_row_stride_bytes, const void* log_prob,
                      int64_t lp_stride_bytes, uint64_t src_stream) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_set_state_from");
  NOT_IN_CALLBACK(c);
  if (c->comm.nranks > 1)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_set_state_from: sharded ensembles take their state from host memory (eb_set_state)");
  if (!coords) FAIL(c, EB_ERR_INVALID, "eb_set_state_from: coords is null");
  if (!c->have_model) FAIL(c, EB_ERR_STATE, "eb_set_state_from: no model set");
  const int64_t row = (int64_t)c->D * (int64_t)sizeof(double);
  if (!row_stride_ok(coords_row_stride_bytes, row, c->N))
    FAIL(c, EB_ERR_INVALID, "eb_set_state_from: the row stride of coords must be a multiple of 8 bytes, at least %lld (got %lld)",
         (long long)row, (long long)coords_row_stride_bytes);
  if (log_prob && !row_stride_ok(lp_stride_bytes, (int64_t)sizeof(double), c->N))
    FAIL(c, EB_ERR_INVALID, "eb_set_state_from: the stride of log_prob must be a positive multiple of 8 bytes (got %lld)",
         (long long)lp_stride_bytes);
  CK(c, cudaSetDevice(c->device));
  int rc = check_device_ptr(c, c->device, coords, "eb_set_state_from", "coords");
  if (!rc && log_prob) rc = check_device_ptr(c, c->device, log_prob, "eb_set_state_from", "log_prob");
  if (rc) return rc;
  const size_t N = (size_t)c->N;
  c->have_state = false;
  c->blobs_live = false;  // as eb_set_state: a given log_prob comes without blobs
  c->blob_bytes = 0;
  rc = copy_records(c, c->coords.get(), coords, (size_t)row, (size_t)coords_row_stride_bytes, N, src_stream);
  if (rc) return rc;
  if (log_prob) {
    // the first copy already waited for src_stream
    rc = copy_records(c, c->logp.get(), log_prob, sizeof(double), (size_t)lp_stride_bytes, N, 0);
    if (rc) return rc;
    CK(c, launch_flag_nan(c->logp.get(), N, FLAG_NAN_INITIAL, c->status_dev.get(), c->st.get()));
  } else {
    rc = evaluate_initial(c, 0, N);
    if (rc) return rc;
  }
  rc = fetch_status(c);
  if (rc) return rc;
  c->have_state = true;
  return EB_OK;
}

int eb_get_state_to(eb_ctx* c, double* coords_dst, double* log_prob_dst) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_get_state_to");
  NOT_IN_CALLBACK(c);
  if (c->comm.nranks > 1)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_get_state_to: sharded ensembles return their state in host memory (eb_get_state)");
  if (!c->have_state) FAIL(c, EB_ERR_STATE, "eb_get_state_to: no state set");
  CK(c, cudaSetDevice(c->device));
  int rc = coords_dst ? check_device_ptr(c, c->device, coords_dst, "eb_get_state_to", "coords_dst") : EB_OK;
  if (!rc && log_prob_dst) rc = check_device_ptr(c, c->device, log_prob_dst, "eb_get_state_to", "log_prob_dst");
  if (rc) return rc;
  if (coords_dst)
    CK(c, cudaMemcpyAsync(coords_dst, c->coords.get(), (size_t)c->N * c->D * sizeof(double), cudaMemcpyDefault,
                          c->st.get()));
  if (log_prob_dst)
    CK(c, cudaMemcpyAsync(log_prob_dst, c->logp.get(), (size_t)c->N * sizeof(double), cudaMemcpyDefault, c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_set_state_blobs(eb_ctx* c, const void* blobs, size_t record_bytes) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_set_state_blobs");
  NOT_IN_CALLBACK(c);
  if (!c->have_state) FAIL(c, EB_ERR_STATE, "eb_set_state_blobs: no state set");
  if ((blobs == nullptr) != (record_bytes == 0))
    FAIL(c, EB_ERR_INVALID, "eb_set_state_blobs: pass records and their size, or NULL, 0 to clear them");
  c->blobs_live = false;
  c->blob_bytes = 0;
  if (!blobs) return EB_OK;
  if (c->model.kind != MODEL_EXTERNAL)
    FAIL(c, EB_ERR_UNSUPPORTED, "eb_set_state_blobs: only log-probability callbacks have blobs");
  CK(c, cudaSetDevice(c->device));
  int rc = ensure_blob_buffers(c, record_bytes);
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(c->blob_live.get(), blobs, (size_t)c->N * record_bytes, cudaMemcpyHostToDevice, c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  c->blob_bytes = record_bytes;
  c->blobs_live = true;
  return EB_OK;
}

int eb_get_blobs(eb_ctx* c, void* out) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->blobs_live) FAIL(c, EB_ERR_STATE, "eb_get_blobs: the state has no blobs");
  if (!out) FAIL(c, EB_ERR_INVALID, "eb_get_blobs: null buffer");
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaMemcpyAsync(out, c->blob_live.get(), (size_t)c->N * c->blob_bytes, cudaMemcpyDeviceToHost, c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_owned_rows(const eb_ctx* c, int64_t* row0, int64_t* nrows) {
  if (!c) return EB_ERR_INVALID;
  int64_t r0, r1;
  owned_rows(c, r0, r1);
  if (row0) *row0 = r0;
  if (nrows) *nrows = r1 - r0;
  return EB_OK;
}

int eb_get_state_rows(eb_ctx* c, int64_t row0, int64_t nrows, double* coords, double* log_prob) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!c->have_state) FAIL(c, EB_ERR_STATE, "eb_get_state_rows: no state set");
  if (row0 < 0 || nrows < 0 || row0 + nrows > c->N) FAIL(c, EB_ERR_INVALID, "eb_get_state_rows: rows out of range");
  int64_t r0, r1;
  owned_rows(c, r0, r1);
  if (c->replicas_dirty && (row0 < r0 || row0 + nrows > r1))
    FAIL(c, EB_ERR_STATE, "eb_get_state_rows: rows [%lld, %lld) are owned by another rank and not replicated here; "
         "read the owned block [%lld, %lld) or call eb_get_state (collective) first",
         (long long)row0, (long long)(row0 + nrows), (long long)r0, (long long)r1);
  CK(c, cudaSetDevice(c->device));
  if (coords && nrows)
    CK(c, cudaMemcpyAsync(coords, c->coords.get() + (size_t)row0 * c->D, (size_t)nrows * c->D * sizeof(double),
                          cudaMemcpyDeviceToHost, c->st.get()));
  if (log_prob && nrows)
    CK(c, cudaMemcpyAsync(log_prob, c->logp.get() + row0, (size_t)nrows * sizeof(double), cudaMemcpyDeviceToHost,
                          c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_set_rng(eb_ctx* c, uint64_t seed, uint64_t step) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_set_rng");
  NOT_IN_CALLBACK(c);
  if (const int rc = running_set_rng(c, seed, step)) return rc;
  c->seed = seed;
  c->step = step;
  return EB_OK;
}

int eb_get_rng(const eb_ctx* c, uint64_t* seed, uint64_t* step) {
  if (!c) return EB_ERR_INVALID;
  if (seed) *seed = c->seed;
  if (step) *step = c->step;
  return EB_OK;
}

}  // extern "C"


namespace {

// rows of `width` bytes at pitches dpitch / spitch: one 2D copy, or one copy per row past the 2D pitch limit
cudaError_t copy_rows(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                      cudaMemcpyKind kind, size_t max_pitch, cudaStream_t st) {
  if (height == 1 || (dpitch <= max_pitch && spitch <= max_pitch))
    return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, kind, st);
  for (size_t r = 0; r < height; ++r) {
    cudaError_t e = cudaMemcpyAsync((char*)dst + r * dpitch, (const char*)src + r * spitch, width, kind, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

int chain_check_slice(eb_chain* ch, const char* who, uint64_t first, uint64_t stride, uint64_t count) {
  if (!for_each_chain_run(ch->start.data(), ch->segs.size(), ch->origin, first, stride, count,
                          [](size_t, uint64_t, uint64_t, uint64_t) {}))
    FAIL(ch, EB_ERR_INVALID, "%s: slots %llu + k * %llu, k < %llu, out of range (capacity %llu slots, stride >= 1)",
         who, (unsigned long long)first, (unsigned long long)stride, (unsigned long long)count,
         (unsigned long long)ch->start.back());
  return EB_OK;
}

// nseg segments (ensembles) of equal size: nseg >= 1 divides the chain's walkers
int chain_check_segments(eb_chain* ch, const char* who, int64_t nseg) {
  if (nseg < 1 || ch->N % nseg != 0)
    FAIL(ch, EB_ERR_INVALID, "%s: nseg = %lld must be >= 1 and divide nwalkers = %lld", who, (long long)nseg,
         (long long)ch->N);
  return EB_OK;
}

// the device part of autocorr.integrated_time over walker slabs of ~1 GiB, for each of nseg segments (ensembles) of
// nw / nseg walkers: acf[nseg][nd][n_t].  fill(xin, w0, wn) enqueues chain[t][w0 .. w0 + wn)[:] -> xin[t][wn * nd]
// for every t on stream st.  A slab holds whole segments, or a part of one segment split as that segment alone
// would be (acf_grid.h), and each segment's walkers are summed in ascending order from zero, so segment k's result
// is bit-identical to the call on segment k alone.  The scratch is one allocation, checked against the free memory.
template <class Obj, class Fill>
int acf_slabs(Obj* c, const char* who, cudaStream_t st, size_t n_t, size_t nw, size_t nd, size_t nseg, double* acf,
              Fill&& fill) {
  if (n_t > ((size_t)1 << 26) || nw * nd > ((size_t)1 << 31))
    FAIL(c, EB_ERR_UNSUPPORTED, "%s: chain too long (n_step <= 2^26)", who);
  const int M = acf_fft_length(n_t);
  const size_t seg_w = nw / nseg;
  const size_t wb = acf_segment_slab_walkers(n_t, nw, nd, nseg);  // slab of walkers sized to ~1 GiB of scratch
  const size_t S = wb * nd, nf = nseg * nd * n_t;
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t b_xin = al(n_t * S * sizeof(double)), b_mean = al(S * sizeof(double)), b_f = al(nf * sizeof(double));
  const size_t b_z = al(S * (size_t)M * sizeof(double2)), b_tw = al((size_t)std::max(1, M / 2) * sizeof(double2));
  DevPtr<char> scratch;
  const int rc = dev_alloc_checked(c, who, "scratch", b_xin + b_mean + b_f + b_z + b_tw, scratch);
  if (rc) return rc;
  double* xin = reinterpret_cast<double*>(scratch.get());
  double* mean = reinterpret_cast<double*>(scratch.get() + b_xin);
  double* f = reinterpret_cast<double*>(scratch.get() + b_xin + b_mean);
  double2* z = reinterpret_cast<double2*>(scratch.get() + b_xin + b_mean + b_f);
  double2* tw = reinterpret_cast<double2*>(scratch.get() + b_xin + b_mean + b_f + b_z);
  CK(c, cudaMemsetAsync(f, 0, nf * sizeof(double), st));
  CK(c, launch_acf_twiddles(tw, M, st));
  for (size_t w0 = 0, wn = 0; w0 < nw; w0 += wn) {
    wn = acf_slab_next(w0, nw, seg_w, wb);
    CK(c, fill(xin, w0, wn));
    CK(c, launch_acf_slab(xin, (int)n_t, (int)wn, (int)nd, M, tw, z, mean, f, (int64_t)seg_w, (int64_t)w0, st));
  }
  CK(c, launch_acf_scale(f, nf, 1.0 / (double)seg_w, st));  // autocorr.py:106  f /= n_w
  CK(c, cudaMemcpyAsync(acf, f, nf * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(c, cudaStreamSynchronize(st));
  return EB_OK;
}

// the base of each stored step of the slice: coords ([N, D] blocks) or log_prob ([N] rows)
std::vector<const double*> chain_slot_table(eb_chain* ch, bool coords, uint64_t first, uint64_t stride,
                                            uint64_t count) {
  std::vector<const double*> t;
  t.reserve(count);
  for_each_chain_run(ch->start.data(), ch->segs.size(), ch->origin, first, stride, count,
                     [&](size_t s, uint64_t off, uint64_t, uint64_t n) {
                       for (uint64_t j = 0; j < n; ++j)
                         t.push_back(coords ? ch->segs[s].x.get() + (off + j * stride) * ch->xs
                                            : ch->segs[s].lp.get() + (off + j * stride) * ch->ls);
                     });
  return t;
}

}  // namespace

// finish_moments and chain_init: context.h
void finish_moments(const double* acc, const double* shift, uint64_t count, size_t D, double* mean, double* cov) {
  if (count == 0) {
    if (mean) std::fill(mean, mean + D, NAN);
    if (cov) std::fill(cov, cov + D * D, NAN);
    return;
  }
  const double m = (double)count;
  if (mean)
    for (size_t d = 0; d < D; ++d) mean[d] = shift[d] + acc[d] / m;
  if (cov)
    for (size_t r = 0; r < D; ++r)
      for (size_t k = 0; k < D; ++k)
        cov[r * D + k] = (acc[D + r * D + k] - acc[r] * acc[k] / m) / (m - 1.0);
}

cudaError_t chain_init(eb_chain* ch, int device, int64_t nwalkers, int ndim) {
  ch->device = device;
  ch->N = nwalkers;
  ch->D = ndim;
  ch->xs = ((size_t)nwalkers * (size_t)ndim + 1) & ~(size_t)1;
  ch->ls = ((size_t)nwalkers + 1) & ~(size_t)1;
  cudaError_t e = cudaSetDevice(device);
  int v = 0;
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device);
  ch->sm_count = v;
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&v, cudaDevAttrMaxPitch, device);
  ch->max_pitch = (size_t)v;
  if (e == cudaSuccess) e = stream_create(ch->st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = dev_alloc(ch->accepted, (size_t)nwalkers * sizeof(double));
  if (e == cudaSuccess) e = dev_alloc(ch->mask, (size_t)nwalkers);
  if (e == cudaSuccess) e = cudaMemsetAsync(ch->accepted.get(), 0, (size_t)nwalkers * sizeof(double), ch->st.get());
  if (e == cudaSuccess) e = cudaStreamSynchronize(ch->st.get());
  return e;
}

extern "C" {


const char* eb_chain_last_error(const eb_chain* ch) { return ch ? ch->err.c_str() : g_create_err.c_str(); }

int eb_chain_create(int device, int64_t nwalkers, int64_t ndim, eb_chain** out) {
  if (!out) return EB_ERR_INVALID;
  *out = nullptr;
  const int rc = check_create_args("eb_chain_create", device, nwalkers, ndim);
  if (rc) return rc;
  std::unique_ptr<eb_chain> ch(new eb_chain());
  CREATE_CK(chain_init(ch.get(), device, nwalkers, (int)ndim));
  *out = ch.release();
  return EB_OK;
}

int eb_chain_destroy(eb_chain* ch) {
  if (!ch) return EB_OK;
  if (ch->ring) FAIL(ch, EB_ERR_INVALID, "eb_chain_destroy: a running window's ring belongs to its engine");
  cudaSetDevice(ch->device);
  cudaStreamSynchronize(ch->st.get());
  delete ch;  // the owners release the segments and buffers, then the stream
  cudaGetLastError();
  return EB_OK;
}

int eb_chain_grow(eb_chain* ch, uint64_t nslots) {
  if (!ch) return EB_ERR_INVALID;
  if (ch->ring) FAIL(ch, EB_ERR_INVALID, "eb_chain_grow: a running window's ring is sized by eb_window_config");
  const uint64_t have = ch->start.back();
  if (nslots <= have) return EB_OK;
  CK(ch, cudaSetDevice(ch->device));
  const uint64_t add = nslots - have;
  const size_t per_slot = (ch->xs + ch->ls) * sizeof(double);
  size_t free_b = 0, total_b = 0;
  CK(ch, cudaMemGetInfo(&free_b, &total_b));
  if (add > total_b / per_slot)  // decided before any allocation
    FAIL(ch, EB_ERR_NOMEM,
         "eb_chain_grow: %llu more slots need %.0f bytes, more than the device's %zu bytes in total (%zu free)",
         (unsigned long long)add, (double)add * (double)per_slot, total_b, free_b);
  ChainSeg seg;
  cudaError_t e = dev_alloc(seg.x, add * ch->xs * sizeof(double));
  if (e == cudaSuccess) e = dev_alloc(seg.lp, add * ch->ls * sizeof(double));
  if (e != cudaSuccess) {  // the chain stays as it was; the free bytes are counted without the half-made segment
    seg = ChainSeg{};
    cudaMemGetInfo(&free_b, &total_b);
  }
  CK_NOMEM(ch, e, "eb_chain_grow: %llu more slots need %zu bytes, %zu bytes free (%s)", (unsigned long long)add,
           (size_t)add * per_slot, free_b, cudaGetErrorString(alloc_err));
  ch->segs.push_back(std::move(seg));
  ch->start.push_back(nslots);
  return EB_OK;
}

int eb_chain_capacity(const eb_chain* ch, uint64_t* nslots, uint64_t* bytes) {
  if (!ch) return EB_ERR_INVALID;
  if (nslots) *nslots = ch->start.back();
  if (bytes)
    *bytes = ch->start.back() * (ch->xs + ch->ls) * sizeof(double) + (uint64_t)ch->N * (sizeof(double) + 1) +
             (ch->ring ? ch->start.back() * (uint64_t)ch->N : 0);
  return EB_OK;
}

int eb_chain_write(eb_chain* ch, uint64_t slot, const double* coords, const double* log_prob,
                   const uint8_t* accepted) {
  if (!ch) return EB_ERR_INVALID;
  if (ch->ring) FAIL(ch, EB_ERR_INVALID, "eb_chain_write: a running window's ring is written by the steps only");
  if (!coords || !log_prob) FAIL(ch, EB_ERR_INVALID, "eb_chain_write: null buffer");
  int rc = chain_check_slice(ch, "eb_chain_write", slot, 1, 1);
  if (rc) return rc;
  CK(ch, cudaSetDevice(ch->device));
  const size_t s = (size_t)(std::upper_bound(ch->start.begin(), ch->start.end(), slot) - ch->start.begin()) - 1;
  const uint64_t off = slot - ch->start[s];
  const size_t N = (size_t)ch->N;
  CK(ch, cudaMemcpyAsync(ch->segs[s].x.get() + off * ch->xs, coords, N * ch->D * sizeof(double), cudaMemcpyHostToDevice,
                         ch->st.get()));
  CK(ch, cudaMemcpyAsync(ch->segs[s].lp.get() + off * ch->ls, log_prob, N * sizeof(double), cudaMemcpyHostToDevice,
                         ch->st.get()));
  if (accepted) {
    CK(ch, cudaMemcpyAsync(ch->mask.get(), accepted, N, cudaMemcpyHostToDevice, ch->st.get()));
    CK(ch, launch_chain_store(nullptr, nullptr, ch->mask.get(), nullptr, nullptr, ch->accepted.get(), 0, 0, ch->N,
                              ch->sm_count, ch->st.get()));
  }
  CK(ch, cudaStreamSynchronize(ch->st.get()));
  return EB_OK;
}

// eb_chain_read (kind = cudaMemcpyDeviceToHost) and eb_chain_read_to (cudaMemcpyDefault, device to device): one copy
// per run of the slice inside a segment
static int chain_read(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* coords, double* log_prob,
                      cudaMemcpyKind kind) {
  const size_t N = (size_t)ch->N, nx = N * ch->D;
  cudaError_t e = cudaSuccess;
  for_each_chain_run(ch->start.data(), ch->segs.size(), ch->origin, first, stride, count,
                     [&](size_t s, uint64_t off, uint64_t k0, uint64_t n) {
                       if (coords && e == cudaSuccess)
                         e = copy_rows(coords + k0 * nx, nx * sizeof(double), ch->segs[s].x.get() + off * ch->xs,
                                       stride * ch->xs * sizeof(double), nx * sizeof(double), n,
                                       kind, ch->max_pitch, ch->st.get());
                       if (log_prob && e == cudaSuccess)
                         e = copy_rows(log_prob + k0 * N, N * sizeof(double), ch->segs[s].lp.get() + off * ch->ls,
                                       stride * ch->ls * sizeof(double), N * sizeof(double), n,
                                       kind, ch->max_pitch, ch->st.get());
                     });
  CK(ch, e);
  CK(ch, cudaStreamSynchronize(ch->st.get()));
  return EB_OK;
}

int eb_chain_read(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* coords, double* log_prob) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_slice(ch, "eb_chain_read", first, stride, count);
  if (rc) return rc;
  CK(ch, cudaSetDevice(ch->device));
  return chain_read(ch, first, stride, count, coords, log_prob, cudaMemcpyDeviceToHost);
}

int eb_chain_read_to(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* coords_dst,
                     double* log_prob_dst) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_slice(ch, "eb_chain_read_to", first, stride, count);
  if (rc || count == 0) return rc;
  CK(ch, cudaSetDevice(ch->device));
  if (coords_dst) rc = check_device_ptr(ch, ch->device, coords_dst, "eb_chain_read_to", "coords_dst");
  if (!rc && log_prob_dst) rc = check_device_ptr(ch, ch->device, log_prob_dst, "eb_chain_read_to", "log_prob_dst");
  if (rc) return rc;
  return chain_read(ch, first, stride, count, coords_dst, log_prob_dst, cudaMemcpyDefault);
}

int eb_chain_read_segments_to(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                              double* coords_dst, double* log_prob_dst) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_read_segments_to", nseg);
  if (!rc) rc = chain_check_slice(ch, "eb_chain_read_segments_to", first, stride, count);
  if (rc || count == 0) return rc;
  CK(ch, cudaSetDevice(ch->device));
  if (coords_dst) rc = check_device_ptr(ch, ch->device, coords_dst, "eb_chain_read_segments_to", "coords_dst");
  if (!rc && log_prob_dst)
    rc = check_device_ptr(ch, ch->device, log_prob_dst, "eb_chain_read_segments_to", "log_prob_dst");
  if (rc) return rc;
  // segment k of stored step t goes to row block t of dst[k]: per run of n slots, one 2D copy per segment (n rows
  // of the run's slots) or per slot (nseg rows of the slot's segments), whichever is fewer
  const size_t K = (size_t)nseg, sn = (size_t)ch->N / K;
  cudaError_t e = cudaSuccess;
  auto part = [&](double* dst, const double* src, size_t w, size_t pitch, uint64_t k0, uint64_t n) {
    // w doubles of a segment; src: the run's first slot, slots pitch doubles apart
    if (n <= K) {
      for (uint64_t j = 0; j < n && e == cudaSuccess; ++j)
        e = copy_rows(dst + (k0 + j) * w, count * w * sizeof(double), src + j * pitch, w * sizeof(double),
                      w * sizeof(double), K, cudaMemcpyDefault, ch->max_pitch, ch->st.get());
    } else {
      for (size_t k = 0; k < K && e == cudaSuccess; ++k)
        e = copy_rows(dst + (k * count + k0) * w, w * sizeof(double), src + k * w, pitch * sizeof(double),
                      w * sizeof(double), n, cudaMemcpyDefault, ch->max_pitch, ch->st.get());
    }
  };
  for_each_chain_run(ch->start.data(), ch->segs.size(), ch->origin, first, stride, count,
                     [&](size_t s, uint64_t off, uint64_t k0, uint64_t n) {
                       if (coords_dst)
                         part(coords_dst, ch->segs[s].x.get() + off * ch->xs, sn * ch->D, stride * ch->xs, k0, n);
                       if (log_prob_dst) part(log_prob_dst, ch->segs[s].lp.get() + off * ch->ls, sn, stride * ch->ls, k0, n);
                     });
  CK(ch, e);
  CK(ch, cudaStreamSynchronize(ch->st.get()));
  return EB_OK;
}

int eb_chain_accepted(eb_chain* ch, double* accepted) {
  if (!ch || !accepted) return EB_ERR_INVALID;
  CK(ch, cudaSetDevice(ch->device));
  if (ch->ring)  // the accepted proposals of the steps still in the window
    CK(ch, launch_mask_sum(ch->slot_mask.get(), ch->filled, ch->N, ch->accepted.get(), ch->st.get()));
  CK(ch, cudaMemcpyAsync(accepted, ch->accepted.get(), (size_t)ch->N * sizeof(double), cudaMemcpyDeviceToHost,
                         ch->st.get()));
  CK(ch, cudaStreamSynchronize(ch->st.get()));
  return EB_OK;
}

int eb_chain_autocorr(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* acf) {
  return eb_chain_autocorr_segments(ch, 1, first, stride, count, acf);
}

int eb_chain_autocorr_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                               double* acf) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_autocorr", nseg);
  if (rc) return rc;
  if (!acf || count == 0) FAIL(ch, EB_ERR_INVALID, "eb_chain_autocorr: empty chain or null buffer");
  rc = chain_check_slice(ch, "eb_chain_autocorr", first, stride, count);
  if (rc) return rc;
  CK(ch, cudaSetDevice(ch->device));
  const size_t nw = (size_t)ch->N, nd = (size_t)ch->D;
  // the slab is filled from the stored slots in place (one strided copy per run of steps inside a segment), so
  // the FFT kernels see the numbers eb_autocorr gets from the host copy of the same slice
  return acf_slabs(ch, "eb_chain_autocorr", ch->st.get(), (size_t)count, nw, nd, (size_t)nseg, acf,
                   [&](double* xin, size_t w0, size_t wn) {
                     cudaError_t e = cudaSuccess;
                     for_each_chain_run(ch->start.data(), ch->segs.size(), ch->origin, first, stride, count,
                                        [&](size_t s, uint64_t off, uint64_t k0, uint64_t n) {
                                          if (e == cudaSuccess)
                                            e = copy_rows(xin + k0 * wn * nd, wn * nd * sizeof(double),
                                                          ch->segs[s].x.get() + off * ch->xs + w0 * nd,
                                                          stride * ch->xs * sizeof(double), wn * nd * sizeof(double),
                                                          n, cudaMemcpyDeviceToDevice, ch->max_pitch, ch->st.get());
                                        });
                     return e;
                   });
}

int eb_chain_select(eb_chain* ch, int what, uint64_t first, uint64_t stride, uint64_t count, const uint64_t* ranks,
                    size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes) {
  return eb_chain_select_segments(ch, 1, what, first, stride, count, ranks, nranks, out, has_nan, passes);
}

int eb_chain_select_segments(eb_chain* ch, int64_t nseg, int what, uint64_t first, uint64_t stride, uint64_t count,
                             const uint64_t* ranks, size_t nranks, double* out, uint8_t* has_nan, uint32_t* passes) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_select", nseg);
  if (rc) return rc;
  if (what != EB_CHAIN_COORDS && what != EB_CHAIN_LOG_PROB)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_select: what must be EB_CHAIN_COORDS or EB_CHAIN_LOG_PROB");
  if (count == 0 || nranks == 0 || !ranks || !out || !has_nan)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_select: empty slice, no rank or null buffer");
  rc = chain_check_slice(ch, "eb_chain_select", first, stride, count);
  if (rc) return rc;
  const uint64_t sn = (uint64_t)ch->N / (uint64_t)nseg;  // rows of a segment in one stored step
  const uint64_t n = count * sn;
  if (n / sn != count) FAIL(ch, EB_ERR_INVALID, "eb_chain_select: slice of more than 2^64 values");
  for (size_t r = 0; r < nranks; ++r)
    if (ranks[r] >= n)
      FAIL(ch, EB_ERR_INVALID, "eb_chain_select: rank %llu of a slice of %llu values per parameter",
           (unsigned long long)ranks[r], (unsigned long long)n);
  CK(ch, cudaSetDevice(ch->device));
  const bool coords = what == EB_CHAIN_COORDS;
  const int D = coords ? ch->D : 1;
  const size_t ncol = (size_t)nseg * D;
  if (ncol > 0x7fffffff) FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_select: more than 2^31 - 1 columns");
  uint32_t np = 0;
  const std::vector<const double*> slots = chain_slot_table(ch, coords, first, stride, count);
  const SelectScratch z = select_scratch(count, (int)ncol, ncol * nranks);
  DevPtr<void> scratch;
  rc = dev_alloc_checked(ch, "eb_chain_select", "scratch", z.bytes, scratch);
  if (rc) return rc;
  const cudaError_t e = select_run(slots.data(), count, (uint32_t)nseg, (uint32_t)sn, D, ranks, nranks, out, has_nan,
                                   &np, z, scratch.get(), ch->sm_count, ch->st.get());
  cudaStreamSynchronize(ch->st.get());
  CK(ch, e);
  if (passes) *passes = np;
  return EB_OK;
}

int eb_chain_moments(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, double* mean, double* cov,
                     uint64_t* n) {
  if (!ch) return EB_ERR_INVALID;
  if (ch->D > 1024) FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_moments is limited to ndim <= 1024");
  int rc = chain_check_slice(ch, "eb_chain_moments", first, stride, count);
  if (rc) return rc;
  const size_t D = (size_t)ch->D, na = D + D * D;
  if (n) *n = count * (uint64_t)ch->N;
  if (count == 0) {
    finish_moments(nullptr, nullptr, 0, D, mean, cov);
    return EB_OK;
  }
  CK(ch, cudaSetDevice(ch->device));
  // [D shift | D + D*D sums | CTA partials of launch_moments]
  const size_t head = ((D + na) * sizeof(double) + 255) & ~(size_t)255;
  DevPtr<void> scratch;
  rc = dev_alloc_checked(ch, "eb_chain_moments", "scratch", head + moments_partial_bytes(ch->D, ch->sm_count), scratch);
  if (rc) return rc;
  double* shift = static_cast<double*>(scratch.get());
  double* acc = shift + D;
  double* partial = reinterpret_cast<double*>(static_cast<char*>(scratch.get()) + head);
  const std::vector<const double*> slots = chain_slot_table(ch, true, first, stride, count);
  // shift = the column mean of the slice's first stored step (as eb_moments takes the first accumulated state's);
  // then every stored step is folded into one accumulator, in slot order
  cudaStream_t st = ch->st.get();
  cudaError_t e = cudaMemsetAsync(acc, 0, na * sizeof(double), st);
  if (e == cudaSuccess) e = launch_colmean(slots[0], ch->N, ch->D, shift, nullptr, st);
  for (size_t k = 0; k < slots.size() && e == cudaSuccess; ++k)
    e = launch_moments(slots[k], ch->N, ch->D, shift, partial, acc, ch->sm_count, st);
  std::vector<double> h(D + na);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h.data(), shift, (D + na) * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  CK(ch, e);
  finish_moments(h.data() + D, h.data(), count * (uint64_t)ch->N, D, mean, cov);
  return EB_OK;
}

int eb_chain_moments_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                              double* mean, double* cov, uint64_t* n) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_moments_segments", nseg);
  if (rc) return rc;
  if (ch->D > 1024) FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_moments_segments is limited to ndim <= 1024");
  rc = chain_check_slice(ch, "eb_chain_moments_segments", first, stride, count);
  if (rc) return rc;
  const size_t D = (size_t)ch->D, na = D + D * D, K = (size_t)nseg;
  const int64_t sn = ch->N / nseg;
  if (n) *n = count * (uint64_t)sn;
  if (count == 0) {
    for (size_t k = 0; k < K; ++k)
      finish_moments(nullptr, nullptr, 0, D, mean ? mean + k * D : nullptr, cov ? cov + k * D * D : nullptr);
    return EB_OK;
  }
  CK(ch, cudaSetDevice(ch->device));
  // [slot table | shift[K, D] | sums[K, D + D*D] | chunk partials[nchunks, K, D + D*D]]
  const uint64_t nchunks = moments_seg_chunks(count, nseg, ch->D);
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t b_tab = al(count * sizeof(double*)), b_head = al((K * D + K * na) * sizeof(double));
  const size_t bytes = b_tab + b_head + nchunks * K * na * sizeof(double);
  DevPtr<void> scratch;
  rc = dev_alloc_checked(ch, "eb_chain_moments_segments", "scratch", bytes, scratch);
  if (rc) return rc;
  char* base = static_cast<char*>(scratch.get());
  const double** tab = reinterpret_cast<const double**>(base);
  double* shift = reinterpret_cast<double*>(base + b_tab);
  double* acc = shift + K * D;
  double* partial = reinterpret_cast<double*>(base + b_tab + b_head);
  const std::vector<const double*> slots = chain_slot_table(ch, true, first, stride, count);
  cudaStream_t st = ch->st.get();
  std::vector<double> h(K * D + K * na);
  cudaError_t e = cudaMemcpyAsync(tab, slots.data(), count * sizeof(double*), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = launch_moments_segments(tab, count, nseg, sn, ch->D, nchunks, shift, partial, acc, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h.data(), shift, h.size() * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  CK(ch, e);
  for (size_t k = 0; k < K; ++k)
    finish_moments(h.data() + K * D + k * na, h.data() + k * D, count * (uint64_t)sn, D,
                   mean ? mean + k * D : nullptr, cov ? cov + k * D * D : nullptr);
  return EB_OK;
}

int eb_chain_histogram(eb_chain* ch, int what, uint64_t first, uint64_t stride, uint64_t count, uint32_t bins,
                       const double* outer, const double* edges, uint64_t* hist) {
  return eb_chain_histogram_segments(ch, 1, what, first, stride, count, bins, outer, edges, hist);
}

int eb_chain_histogram_segments(eb_chain* ch, int64_t nseg, int what, uint64_t first, uint64_t stride, uint64_t count,
                                uint32_t bins, const double* outer, const double* edges, uint64_t* hist) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_histogram", nseg);
  if (rc) return rc;
  if (what != EB_CHAIN_COORDS && what != EB_CHAIN_LOG_PROB)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram: what must be EB_CHAIN_COORDS or EB_CHAIN_LOG_PROB");
  if (bins == 0 || !outer || !edges || !hist) FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram: bins == 0 or null buffer");
  if (bins > (uint32_t)HIST_BINS_MAX)
    FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram is limited to bins <= %d on the device, got %u", HIST_BINS_MAX,
         bins);
  rc = chain_check_slice(ch, "eb_chain_histogram", first, stride, count);
  if (rc) return rc;
  const bool coords = what == EB_CHAIN_COORDS;
  const int D = coords ? ch->D : 1;
  const size_t ncol = (size_t)nseg * D;  // column k * D + d: parameter d of segment k
  if (count == 0) {
    std::fill(hist, hist + ncol * bins, (uint64_t)0);
    return EB_OK;
  }
  const uint64_t sn = (uint64_t)ch->N / (uint64_t)nseg;  // rows of a segment in one stored step
  const uint64_t n = count * sn;
  if (n / sn != count || !hist_rows_fit(n))
    FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram: slice of %llu stored steps is too long",
         (unsigned long long)count);
  if (ncol > 0x7fffffff) FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram: more than 2^31 - 1 columns");
  CK(ch, cudaSetDevice(ch->device));
  const std::vector<const double*> slots = chain_slot_table(ch, coords, first, stride, count);
  DevPtr<void> scratch;
  rc = dev_alloc_checked(ch, "eb_chain_histogram", "scratch", hist1_scratch_bytes(count, ncol, (int)bins), scratch);
  if (rc) return rc;
  bool bad = false;
  const cudaError_t e = hist1_run(slots.data(), count, (uint32_t)nseg, (uint32_t)ch->N, D, (int)bins, outer, edges,
                                  hist, &bad, scratch.get(), ch->sm_count, ch->st.get());
  cudaStreamSynchronize(ch->st.get());
  CK(ch, e);
  if (bad)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram: a value's truncated bin index is above bins (np.histogram raises "
         "IndexError there); the span does not fit the edges");
  return EB_OK;
}

int eb_chain_histogram2d(eb_chain* ch, uint64_t first, uint64_t stride, uint64_t count, const uint32_t* params,
                         size_t nparams, uint32_t bins, const double* edges, uint64_t* hist) {
  return eb_chain_histogram2d_segments(ch, 1, first, stride, count, params, nparams, bins, edges, hist);
}

int eb_chain_histogram2d_segments(eb_chain* ch, int64_t nseg, uint64_t first, uint64_t stride, uint64_t count,
                                  const uint32_t* params, size_t nparams, uint32_t bins, const double* edges,
                                  uint64_t* hist) {
  if (!ch) return EB_ERR_INVALID;
  int rc = chain_check_segments(ch, "eb_chain_histogram2d", nseg);
  if (rc) return rc;
  if (bins == 0 || !params || !edges || !hist)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram2d: bins == 0 or null buffer");
  if (bins > (uint32_t)HIST2_BINS_MAX)
    FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram2d is limited to bins <= %d on the device, got %u",
         HIST2_BINS_MAX, bins);
  if (nparams < 2 || nparams > (size_t)ch->D)
    FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram2d: need 2 <= nparams <= ndim = %d, got %zu", ch->D, nparams);
  std::vector<uint8_t> seen((size_t)ch->D, 0);
  for (size_t k = 0; k < nparams; ++k) {
    if (params[k] >= (uint32_t)ch->D || seen[params[k]])
      FAIL(ch, EB_ERR_INVALID, "eb_chain_histogram2d: params must be distinct and < ndim = %d (params[%zu] = %u)",
           ch->D, k, params[k]);
    seen[params[k]] = 1;
  }
  rc = chain_check_slice(ch, "eb_chain_histogram2d", first, stride, count);
  if (rc) return rc;
  // nseg * npairs * bins^2 can pass 2^64 (2^31 segments, 2^27 pairs, 2^14 cells): refuse it in floating point first
  const double outd = (double)nseg * (double)(nparams * (nparams - 1) / 2) * (double)bins * (double)bins;
  if (outd > (double)((uint64_t)1 << 60))
    FAIL(ch, EB_ERR_NOMEM, "eb_chain_histogram2d: %.0f counts of 8 bytes cannot be held", outd);
  const uint64_t out = (uint64_t)nseg * (nparams * (nparams - 1) / 2) * bins * bins;
  if (count == 0) {
    std::fill(hist, hist + out, (uint64_t)0);
    return EB_OK;
  }
  const uint64_t sn = (uint64_t)ch->N / (uint64_t)nseg;  // rows of a segment in one stored step
  const uint64_t n = count * sn;
  if (n / sn != count || !hist_rows_fit(n))
    FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram2d: slice of %llu stored steps is too long",
         (unsigned long long)count);
  if (hist2_grid_x((uint32_t)nseg, (int)nparams, (int)bins) > 0x7fffffff)
    FAIL(ch, EB_ERR_UNSUPPORTED, "eb_chain_histogram2d: more than 2^31 - 1 (segment, pair tile) blocks");
  CK(ch, cudaSetDevice(ch->device));
  const std::vector<const double*> slots = chain_slot_table(ch, true, first, stride, count);
  DevPtr<void> scratch;
  rc = dev_alloc_checked(ch, "eb_chain_histogram2d", "scratch",
                         hist2_scratch_bytes(count, (uint32_t)nseg, (int)nparams, (int)bins), scratch);
  if (rc) return rc;
  const cudaError_t e = hist2_run(slots.data(), count, (uint32_t)nseg, (uint32_t)ch->N, ch->D, params, (int)nparams,
                                  (int)bins, edges, hist, scratch.get(), ch->sm_count, ch->st.get());
  cudaStreamSynchronize(ch->st.get());
  CK(ch, e);
  return EB_OK;
}

int eb_get_naccepted(eb_ctx* c, uint64_t* naccepted) {
  if (!c || !naccepted) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  int rc = sync_replicas(c);  // multi-GPU: every rank's counters (collective)
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(naccepted, c->nacc.get(), (size_t)c->N * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                        c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_move_picks(const eb_ctx* c, uint64_t* picks, size_t nmoves) {
  if (!c || !picks) return EB_ERR_INVALID;
  for (size_t k = 0; k < nmoves; ++k) picks[k] = k < c->picks.size() ? c->picks[k] : 0;
  return EB_OK;
}

int eb_reset_counters(eb_ctx* c) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  CK(c, cudaMemsetAsync(c->nacc.get(), 0, (size_t)c->N * sizeof(unsigned long long), c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  return EB_OK;
}

int eb_walkers_gram(eb_ctx* c, const double* coords, size_t rows, double* gram, int* flags) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!coords || !gram || rows == 0) FAIL(c, EB_ERR_INVALID, "eb_walkers_gram: null buffer");
  if (c->D > 1024) FAIL(c, EB_ERR_UNSUPPORTED, "eb_walkers_gram is limited to ndim <= 1024");
  CK(c, cudaSetDevice(c->device));
  int rc = ensure_scratch(c, rows);
  if (rc) return rc;
  const size_t D = (size_t)c->D, n = D + D * D;
  DevPtr<double> dwork;  // [D mean | D + D*D accumulators]
  CK(c, dev_alloc(dwork, (D + n) * sizeof(double)));
  if (!c->mom_partial) CK(c, dev_alloc(c->mom_partial, moments_partial_bytes(c->D, c->sm_count)));
  std::vector<double> acc(n);
  int f = 0;
  double* work = dwork.get();
  double* x = c->scratch_x.get();
  cudaStream_t st = c->st.get();
  cudaError_t e = cudaMemcpyAsync(x, coords, rows * D * sizeof(double), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(work, 0, (D + n) * sizeof(double), st);
  if (e == cudaSuccess) e = launch_colmean(x, (int64_t)rows, c->D, work, c->status_dev.get(), st);
  if (e == cudaSuccess)
    e = launch_moments(x, (int64_t)rows, c->D, work, c->mom_partial.get(), work + D, c->sm_count, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(acc.data(), work + D, n * sizeof(double), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(c->status_host.get(), c->status_dev.get(), sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  CK(c, e);
  // the non-finite flags are an ANSWER here (walkers_independent returns False), not an error
  if (*c->status_host & (FLAG_INF_PARAM | FLAG_NAN_PARAM)) f |= 1;
  *c->status_host = 0;
  CK(c, cudaMemsetAsync(c->status_dev.get(), 0, sizeof(int), c->st.get()));
  CK(c, cudaStreamSynchronize(c->st.get()));
  // centred, column-normalised walkers C (ensemble.py:656-661): C^T C = M_jk / (sqrt(M_jj) sqrt(M_kk)); the
  // max-abs scaling of :658-659 cancels, it only matters as the zero-span test.  The square roots are taken
  // before the product, so that the denominator stays normal whenever both sums are.  A sum M_jj that is
  // zero, subnormal or not finite (coordinates near 1e-154 or 1e154 and beyond) has lost its digits: bit 2,
  // and that column's entries are returned as 0 instead of a ratio of rounding noise or a NaN.
  std::vector<double> rt(D);
  for (size_t j = 0; j < D; ++j) {
    const double m = acc[D + j * D + j];
    if (!(m > 0.0)) f |= 2;
    rt[j] = std::isnormal(m) && m > 0.0 ? sqrt(m) : 0.0;
    if (rt[j] == 0.0) f |= 4;
  }
  for (size_t j = 0; j < D; ++j)
    for (size_t k = 0; k < D; ++k) {
      double g = rt[j] > 0.0 && rt[k] > 0.0 ? acc[D + j * D + k] / (rt[j] * rt[k]) : 0.0;
      if (!std::isfinite(g)) {
        g = 0.0;
        f |= 4;
      }
      gram[j * D + k] = g;
    }
  if (flags) *flags = f;
  return EB_OK;
}

int eb_autocorr(eb_ctx* c, const double* chain, size_t n_t, size_t nw, size_t nd, double* acf) {
  if (!c) return EB_ERR_INVALID;
  NOT_IN_CALLBACK(c);
  if (!chain || !acf || n_t == 0 || nw == 0 || nd == 0) FAIL(c, EB_ERR_INVALID, "eb_autocorr: empty chain or null buffer");
  CK(c, cudaSetDevice(c->device));
  return acf_slabs(c, "eb_autocorr", c->st.get(), n_t, nw, nd, 1, acf, [&](double* xin, size_t w0, size_t wn) {
    // chain[t][w0 .. w0 + wn)[:] -> xin[t][wn * nd]: one strided copy (rows of the slab are contiguous in a step)
    return cudaMemcpy2DAsync(xin, wn * nd * sizeof(double), chain + w0 * nd, nw * nd * sizeof(double),
                             wn * nd * sizeof(double), n_t, cudaMemcpyHostToDevice, c->st.get());
  });
}

int eb_last_step_timing(const eb_ctx* c, double* ms, uint64_t* launches) {
  if (!c) return EB_ERR_INVALID;
  if (ms) *ms = c->last_ms;
  if (launches) *launches = c->last_launches;
  return EB_OK;
}

const char* eb_last_kernel_name(const eb_ctx* c) { return c ? c->last_kernel : "none"; }

const char* eb_last_kernel_variant(const eb_ctx* c) { return c ? c->last_variant : "none"; }

int eb_set_option(eb_ctx* c, const char* name, int64_t value) {
  if (!c || !name) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_set_option");
  NOT_IN_CALLBACK(c);
  if (!strcmp(name, "debug_taps")) {
    CK(c, cudaSetDevice(c->device));
    if (value && !c->tap_scalar) {
      const size_t N = (size_t)c->N;
      DevPtr<int64_t> partners, active;
      DevPtr<double> scalar, u;
      CK(c, dev_alloc(partners, 3 * N * sizeof(int64_t)));
      CK(c, dev_alloc(scalar, N * sizeof(double)));
      CK(c, dev_alloc(u, N * sizeof(double)));
      CK(c, dev_alloc(active, N * sizeof(int64_t)));
      c->tap_partners = std::move(partners);
      c->tap_scalar = std::move(scalar);
      c->tap_u = std::move(u);
      c->tap_active = std::move(active);
    }
    c->debug = value != 0;
    return EB_OK;
  }
  if (!strcmp(name, "dmma_timeline")) {
    CK(c, cudaSetDevice(c->device));
    const size_t n = (size_t)c->sm_count * 8 * TL_TILES * TL_EVENTS;
    if (value && !c->timeline) {
      DevPtr<long long> tl;
      CK(c, dev_alloc(tl, n * sizeof(long long)));
      CK(c, cudaMemset(tl.get(), 0, n * sizeof(long long)));
      c->timeline = std::move(tl);
    } else if (!value) {
      c->timeline.reset();
    }
    c->timeline_first_split = value == 2;
    return EB_OK;
  }
  if (!strcmp(name, "l2_flush")) {
    c->l2_flush = value != 0;
    return EB_OK;
  }
  if (!strcmp(name, "dmma_stagger")) {
    c->dmma_stagger = value != 0;
    return EB_OK;
  }
  if (!strcmp(name, "dmma_group")) {
    if (value < 1) FAIL(c, EB_ERR_INVALID, "dmma_group must be >= 1");
    c->dmma_group = (int)std::min<int64_t>(value, 1 << 20);
    return EB_OK;
  }
  if (!strcmp(name, "tma_own_reg")) {
    c->tma_own_reg = value != 0;
    return EB_OK;
  }
  if (!strcmp(name, "dmma_local_first")) {
    c->local_first = (int)std::max<int64_t>(0, std::min<int64_t>(value, 2));
    return EB_OK;
  }
  if (!strcmp(name, "pdl")) {
    c->pdl = (int)std::max<int64_t>(0, std::min<int64_t>(value, 2));
    return EB_OK;
  }
  if (!strcmp(name, "moments_every")) {
    if (value < 0) FAIL(c, EB_ERR_INVALID, "moments_every must be >= 0");
    return moments_config(c, (uint64_t)value);
  }
  if (!strcmp(name, "tma_rows")) {
    c->allow_tma = (int)std::max<int64_t>(0, std::min<int64_t>(value, 2));
    return EB_OK;
  }
  if (!strcmp(name, "dense_dmma")) {
    c->allow_dmma = value != 0;
    return EB_OK;
  }
  FAIL(c, EB_ERR_INVALID, "eb_set_option: unknown option '%s'", name);
}

int eb_debug_timeline(eb_ctx* c, int64_t* out, size_t capacity, size_t* written) {
  if (!c || !out) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_debug_timeline");
  NOT_IN_CALLBACK(c);
  if (!c->timeline) FAIL(c, EB_ERR_STATE, "eb_debug_timeline: enable with eb_set_option(\"dmma_timeline\", 1)");
  CK(c, cudaSetDevice(c->device));
  const size_t n = (size_t)c->sm_count * 8 * TL_TILES * TL_EVENTS;
  if (capacity < n) FAIL(c, EB_ERR_INVALID, "eb_debug_timeline: need room for %zu values", n);
  CK(c, cudaMemcpy(out, c->timeline.get(), n * sizeof(long long), cudaMemcpyDeviceToHost));
  if (written) *written = n;
  return EB_OK;
}

int eb_debug_taps(eb_ctx* c, int64_t* partners, double* scalar, double* u_accept, int64_t* active,
                  int64_t* nactive) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_debug_taps");
  NOT_IN_CALLBACK(c);
  if (!c->debug || !c->tap_scalar) FAIL(c, EB_ERR_STATE, "eb_debug_taps: enable with eb_set_option(\"debug_taps\", 1)");
  CK(c, cudaSetDevice(c->device));
  const size_t N = (size_t)c->N;
  if (partners) CK(c, cudaMemcpy(partners, c->tap_partners.get(), 3 * N * sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (scalar) CK(c, cudaMemcpy(scalar, c->tap_scalar.get(), N * sizeof(double), cudaMemcpyDeviceToHost));
  if (u_accept) CK(c, cudaMemcpy(u_accept, c->tap_u.get(), N * sizeof(double), cudaMemcpyDeviceToHost));
  if (active) CK(c, cudaMemcpy(active, c->tap_active.get(), N * sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (nactive) *nactive = c->tap_count;
  return EB_OK;
}

int eb_host_alloc(size_t bytes, void** out) {
  if (!out || bytes == 0) return EB_ERR_INVALID;
  if (cudaMallocHost(out, bytes) != cudaSuccess) {
    cudaGetLastError();
    *out = nullptr;
    return EB_ERR_CUDA;
  }
  return EB_OK;
}

int eb_host_free(void* ptr) {
  if (ptr && cudaFreeHost(ptr) != cudaSuccess) {
    cudaGetLastError();
    return EB_ERR_CUDA;
  }
  return EB_OK;
}

}  // extern "C"

// the device-memory calls without a context (eb_device_alloc, ...): FAIL / CK write here, and the entry point hands
// the message to eb_last_error(NULL)
struct NoCtx {
  std::string err;
};

static int no_ctx_result(const NoCtx& o, int rc) {
  if (rc) g_create_err = o.err;
  return rc;
}

static int select_device(NoCtx* o, const char* who, int device) {
  int ndev = 0;
  CK(o, cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) FAIL(o, EB_ERR_INVALID, "%s: device index %d out of range", who, device);
  CK(o, cudaSetDevice(device));
  return EB_OK;
}

static int device_alloc(NoCtx* o, int device, size_t bytes, void** out) {
  if (bytes == 0) return EB_OK;  // NULL, as the CUDA Array Interface allows for an empty array
  int rc = select_device(o, "eb_device_alloc", device);
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(o, cudaMemGetInfo(&free_b, &total_b));
  if (bytes > total_b)  // decided before any allocation
    FAIL(o, EB_ERR_NOMEM, "eb_device_alloc: %zu bytes, more than the device's %zu bytes in total (%zu free)", bytes,
         total_b, free_b);
  DevPtr<void> p;
  const cudaError_t e = dev_alloc(p, bytes);
  if (e != cudaSuccess) cudaMemGetInfo(&free_b, &total_b);
  CK_NOMEM(o, e, "eb_device_alloc: %zu bytes, %zu bytes free (%s)", bytes, free_b, cudaGetErrorString(alloc_err));
  *out = p.release();
  return EB_OK;
}

static int device_copy(NoCtx* o, int device, void* dst, const void* src, int64_t width, int64_t src_pitch,
                       int64_t rows, uint64_t src_stream) {
  if (width < 0 || rows < 0) FAIL(o, EB_ERR_INVALID, "eb_device_copy: negative size");
  if (width == 0 || rows == 0) return EB_OK;
  if (!dst || !src) FAIL(o, EB_ERR_INVALID, "eb_device_copy: null buffer");
  if (rows > 1 && src_pitch < width)
    FAIL(o, EB_ERR_INVALID, "eb_device_copy: the source pitch (%lld bytes) is shorter than a row (%lld bytes)",
         (long long)src_pitch, (long long)width);
  int rc = select_device(o, "eb_device_copy", device);
  if (rc) return rc;
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, src) != cudaSuccess) cudaGetLastError();  // not CUDA memory: a host source
  if ((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device != device)
    FAIL(o, EB_ERR_INVALID, "eb_device_copy: src is on device %d, not on device %d", a.device, device);
  StreamPtr st;
  CK(o, stream_create(st, cudaStreamNonBlocking));
  return copy_ordered(o, st.get(), dst, src, (size_t)width, (size_t)src_pitch, (size_t)rows, src_stream);
}

extern "C" {

int eb_device_alloc(int device, size_t bytes, void** out) {
  if (!out) return EB_ERR_INVALID;
  *out = nullptr;
  NoCtx o;
  return no_ctx_result(o, device_alloc(&o, device, bytes, out));
}

int eb_device_free(int device, void* p) {
  if (!p) return EB_OK;
  NoCtx o;
  int rc = select_device(&o, "eb_device_free", device);
  if (!rc) {
    const cudaError_t e = cudaFree(p);
    if (e != cudaSuccess) {
      cudaGetLastError();
      o.err = std::string("eb_device_free: ") + cudaGetErrorString(e);
      rc = EB_ERR_CUDA;
    }
  }
  return no_ctx_result(o, rc);
}

int eb_device_copy(int device, void* dst, const void* src, int64_t width, int64_t src_pitch, int64_t rows,
                   uint64_t src_stream) {
  NoCtx o;
  return no_ctx_result(o, device_copy(&o, device, dst, src, width, src_pitch, rows, src_stream));
}

// ---- multi-GPU ---------------------------------------------------------------
int eb_comm_id(char id[EB_COMM_ID_BYTES]) { return comm_unique_id(id) ? EB_ERR_COMM : EB_OK; }

int eb_comm_init(eb_ctx* c, const char id[EB_COMM_ID_BYTES], int rank, int nranks, int mode) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_comm_init");
  NOT_IN_CALLBACK(c);
  if (c->have_model && c->model.kind == MODEL_EXTERNAL && nranks > 1)
    FAIL(c, EB_ERR_UNSUPPORTED, "log-probability callbacks are not sharded across GPUs");
  if (const int rc = running_check_sharding(c, nranks)) return rc;
  CK(c, cudaSetDevice(c->device));
  c->tbl_n = 0;  // the cached split tables carry the old ownership ranges
  c->have_state = false;  // ownership changes: the state must be set again through the sharded path
  unsigned* flags = reinterpret_cast<unsigned*>(c->coords.get() + (size_t)c->N * c->D);
  if (comm_init(c->comm, id, rank, nranks, mode, c->N, c->D, c->coords.get(), flags, c->table_cap, c->st.get()))
    FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  return EB_OK;
}

int eb_comm_export(eb_ctx* c, char blob[EB_IPC_BLOB_BYTES]) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_comm_export");
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  if (comm_export(c->comm, blob)) FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  return EB_OK;
}

int eb_comm_probe(eb_ctx* c, int peer, int what, double* gbs) {
  if (!c || !gbs) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_comm_probe");
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  if (comm_probe(c->comm, peer, what, c->D, c->st.get(), gbs)) FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  return EB_OK;
}

int eb_comm_import(eb_ctx* c, const char* blobs) {
  if (!c) return EB_ERR_INVALID;
  NOT_BATCH(c, "eb_comm_import");
  NOT_IN_CALLBACK(c);
  CK(c, cudaSetDevice(c->device));
  if (comm_import(c->comm, blobs)) FAIL(c, EB_ERR_COMM, "%s", c->comm.err.c_str());
  return EB_OK;
}

}  // extern "C"
