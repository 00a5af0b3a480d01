#!/usr/bin/env python
"""Cost of storing a ``BatchSampler``'s chain, and of summarising every ensemble, on the host and on the GPU.

  store      K ensembles of 32 x 5, ``gauss_iso``, StretchMove, one ``run_mcmc`` call of --steps stored steps (after
             --warmup warm-up steps) with ``thin_by`` 1 and 10: ``store=False``, the host ``Backend`` (pinned staging
             and a host copy per stored step) and ``DeviceBackend`` (one copy inside HBM per stored step).  Device
             time is ``eb_last_step_timing`` (CUDA events on the engine's stream, first launch to last); wall time is
             the host clock of the call, which ends in a synchronise.  Both are reported per step.
  summaries  K = 1 024, 2 000 stored steps, ``discard=500``, ``thin=10``: ``get_autocorr_time()``,
             ``get_percentile([16, 50, 84])``, ``get_moments()`` and ``get_chain(flat=True)`` through the device route
             (``DeviceBackend``: segmented kernels, ``cuda=True`` for the chain) against the numpy route (host
             ``Backend``), host wall clock of each call, best of --repeat.

The card name and power limit are read in the same run.

    python scripts/bench_batch_store.py [--steps 200] [--warmup 20] [--repeat 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import emcee_b200  # noqa: E402
from emcee_b200 import DeviceBackend, models  # noqa: E402

N, D = 32, 5


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def p0(K):
    return np.random.default_rng(1).normal(size=(K, N, D))


def sampler(K, store):
    return emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1,
                                   backend=DeviceBackend() if store == "device" else None)


def store_cost(K, store, thin_by, steps, warmup):
    b = sampler(K, store)
    stored = store != "none"
    state = b.run_mcmc(p0(K), warmup, thin_by=thin_by, store=stored, skip_initial_state_check=True)
    if stored:
        b.backend.grow(steps, None)  # growth is not part of a step
    t0 = time.perf_counter()
    b.run_mcmc(state, steps, thin_by=thin_by, store=stored, skip_initial_state_check=True)
    wall = time.perf_counter() - t0
    ms, _ = b._engine.last_step_timing()
    n = steps * thin_by
    return {"K": K, "store": store, "thin_by": thin_by, "device_us_per_step": 1e3 * ms / n,
            "wall_us_per_step": 1e6 * wall / n, "stored_bytes_per_stored_step": K * N * (D + 1) * 8 if stored else 0}


def best_of(fn, repeat):
    best = float("inf")
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def summaries(repeat):
    K, n = 1024, 2000
    out = {"K": K, "stored_steps": n, "discard": 500, "thin": 10}
    runs = {}
    for store in ("device", "host"):
        b = sampler(K, store)
        b.run_mcmc(p0(K), n, skip_initial_state_check=True)
        runs[store] = b
    kw = dict(discard=500, thin=10)
    calls = {
        "get_autocorr_time": lambda b, dev: b.get_autocorr_time(quiet=True, **kw),
        "get_percentile": lambda b, dev: b.get_percentile([16, 50, 84], **kw),
        "get_moments": lambda b, dev: b.get_moments(**kw),
        "get_chain_flat": lambda b, dev: b.get_chain(flat=True, cuda=dev, **kw),
    }
    for name, call in calls.items():
        for store in ("device", "host"):
            call(runs[store], store == "device")  # warm-up: first launches, first allocations
        out[name] = {"device_ms": 1e3 * best_of(lambda: call(runs["device"], True), repeat),
                     "numpy_ms": 1e3 * best_of(lambda: call(runs["host"], False), repeat)}
        print("summary", name, json.dumps(out[name]), flush=True)
    tau_d, tau_h = runs["device"].get_autocorr_time(quiet=True, **kw), runs["host"].get_autocorr_time(quiet=True, **kw)
    out["tau_max_rel_diff"] = float(np.max(np.abs(tau_d - tau_h) / np.abs(tau_h)))
    out["percentile_equal"] = bool(np.array_equal(runs["device"].get_percentile([16, 50, 84], **kw),
                                                  runs["host"].get_percentile([16, 50, 84], **kw)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "shape": [N, D], "steps": a.steps, "store": []}
    for K in (16, 256, 1024, 4096):
        for thin_by in (1, 10):
            for store in ("none", "host", "device"):
                res["store"].append(store_cost(K, store, thin_by, a.steps, a.warmup))
                print("store", json.dumps(res["store"][-1]), flush=True)
    res["summaries"] = summaries(a.repeat)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_batch_store.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
