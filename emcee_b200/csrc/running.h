// The running statistics of an engine (running.cu): moments, histograms, trace, reservoir, autocorrelation and
// window.  Each records the live state after every `every`-th step, for runs that store no chain.  The step driver,
// eb_comm_init and eb_set_rng reach them through the hooks below only; these visit the six in this fixed order.
#pragma once

#include <memory>
#include <vector>

#include "engine.cuh"
#include "hist_bins.h"
#include "owners.h"
#include "reservoir_plan.h"
#include "running_acf.h"
#include "trace_sum.h"

using namespace eb;

// chain moments (eb_moments): sum of (x - shift) and of its outer product over the owned rows of each recorded step
struct RunMoments {
  uint64_t every = 0;
  DevPtr<double> acc;    // [D + D*D] accumulators
  DevPtr<double> shift;  // [D]
  unsigned long long count = 0;
  bool have_shift = false;
};

// histograms (eb_histograms): the rows of each recorded step counted into live.counts
struct RunHistograms {
  uint64_t every = 0;
  bool on = false;  // configured: live holds tables and counts
  LiveHist live;
  DevPtr<void> mem;  // live.mem
  unsigned long long count = 0;  // samples counted
};

// trace (eb_trace_read): one row [2 D + 4] of ensemble statistics per recorded step
struct RunTrace {
  uint64_t every = 0;
  bool on = false;  // configured: live holds its fixed part
  LiveTrace live;
  DevPtr<void> mem;              // live.mem
  DevPtr<double> rows;           // [cap, 2 D + 4], device
  uint64_t cap = 0;
  std::vector<uint64_t> steps;  // the step counter of each recorded row
};

// reservoir (eb_reservoir_read): K of the rows of the recorded steps, in device memory
struct RunReservoir {
  uint64_t every = 0;
  bool on = false;  // configured: live holds its buffers
  LiveReservoir live;
  DevPtr<void> mem;  // live's buffers
  ResSchedule plan;  // rows offered, and the bound of the live entries that decides the compactions
};

// autocorrelation function (eb_running_acf_read): lag sums of every series of the recorded steps
struct RunAutocorr {
  uint64_t every = 0;
  bool on = false;  // configured: live holds its buffers
  uint64_t n = 0;   // steps recorded since the last configuration with every > 0
  LiveRacf live;
  DevPtr<void> mem;  // live's buffers
};

// window (eb_window_config): the last `capacity` of the recorded states, in a ring
struct RunWindow {
  uint64_t every = 0;
  uint64_t n = 0;                    // steps recorded since the last configuration with every > 0
  std::unique_ptr<eb_chain> ring;    // the ring (ring == true), or null before any configuration
  std::vector<uint64_t> steps;       // [capacity] the step counter and the Philox key of each physical slot's step
  std::vector<uint64_t> seeds;
};

struct RunningStats {
  RunMoments moments;
  RunHistograms hist;
  RunTrace trace;
  RunReservoir reservoir;
  RunAutocorr acf;
  RunWindow window;
};

// before the first launch of nsteps steps: room for what they record (the trace's rows)
int running_prepare(eb_ctx* c, uint64_t nsteps);
// a statistic records the state once the step counter reaches n
bool running_due(const eb_ctx* c, uint64_t n);
// record the CURRENT state into every statistic due at the step counter (kernels only, enqueued on the stream)
int running_record(eb_ctx* c, uint64_t& launches);
// eb_comm_init: only the moments can be sharded over nranks > 1
int running_check_sharding(eb_ctx* c, int nranks);
// eb_set_rng: a new seed or an earlier step empties the reservoir
int running_set_rng(eb_ctx* c, uint64_t seed, uint64_t step);
// option "moments_every": allocate and zero the accumulators
int moments_config(eb_ctx* c, uint64_t every);
