#!/usr/bin/env python
"""Throughput of ``BatchSampler`` against the same ensembles run one ``EnsembleSampler`` after another.

  batch        K ensembles of 32 x 5, ``gauss_iso``, StretchMove: one ``run_mcmc(store=False)`` call of --steps steps
               after --warmup warm-up steps.  Device time is ``eb_last_step_timing`` (CUDA events on the engine's
               stream, first launch to last); host time is the wall clock of the call, which ends in a synchronise.
  sequential   the same K ensembles as K ``EnsembleSampler`` s, each one ``run_mcmc(store=False)`` call, one after
               another (K <= 256): host wall clock of the whole loop, and the sum of their device times.
  callback     K datasets behind a torch ``CudaArrayFunction`` (lp = -0.5 sum((x - mu_k)^2), mu_k one row of
               data[K, 5]): one batched function called once per half-step, against K samplers each with its own
               function.

Rates are walker-steps per second.  The card name and power limit are read in the same run.

    python scripts/bench_batch.py [--steps 200] [--warmup 20] [--out DIR]
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
from emcee_b200 import models  # noqa: E402

N, D = 32, 5


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def p0(K):
    return np.random.default_rng(1).normal(size=(K, N, D))


def batch_rate(K, model, steps, warmup):
    b = emcee_b200.BatchSampler(K, N, D, model, seeds=1)
    state = b.run_mcmc(p0(K), warmup, store=False, skip_initial_state_check=True)
    t0 = time.perf_counter()
    b.run_mcmc(state, steps, store=False, skip_initial_state_check=True)
    wall = time.perf_counter() - t0
    ms, launches = b._engine.last_step_timing()
    work = K * N * steps
    return {"K": K, "device_rate": work / (ms * 1e-3), "host_rate": work / wall, "launches_per_step": launches / steps}


def sequential_rate(K, make_model, steps, warmup):
    x = p0(K)
    samplers, states = [], []
    for k in range(K):
        s = emcee_b200.EnsembleSampler(N, D, make_model(k), seed=1 + k)
        states.append(s.run_mcmc(x[k], warmup, store=False, skip_initial_state_check=True))
        samplers.append(s)
    dev = 0.0
    t0 = time.perf_counter()
    for s, st in zip(samplers, states):
        s.run_mcmc(st, steps, store=False, skip_initial_state_check=True)
        dev += s._engine.last_step_timing()[0]
    wall = time.perf_counter() - t0
    work = K * N * steps
    return {"K": K, "device_rate": work / (dev * 1e-3), "host_rate": work / wall}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "shape": [N, D], "steps": a.steps, "batch": [], "sequential": [], "callback": []}
    for K in (1, 16, 256, 1024, 4096, 16384):
        res["batch"].append(batch_rate(K, models.GaussianIso(), a.steps, a.warmup))
        print("batch", json.dumps(res["batch"][-1]), flush=True)
    for K in (1, 16, 256):
        res["sequential"].append(sequential_rate(K, lambda k: models.GaussianIso(), a.steps, a.warmup))
        print("sequential", json.dumps(res["sequential"][-1]), flush=True)

    import torch

    steps = max(a.steps // 4, 10)
    for K in (16, 256):
        data = torch.as_tensor(np.random.default_rng(2).normal(size=(K, D)), device="cuda")

        def lp(x, mu):
            return -0.5 * torch.sum((torch.as_tensor(x, device="cuda") - mu) ** 2, dim=-1)

        bfn = models.CudaArrayFunction(lambda x: lp(x, data[:, None, :]))
        row = {"K": K, "batch": batch_rate(K, bfn, steps, 2),
               "sequential": sequential_rate(K, lambda k: models.CudaArrayFunction(lambda x, k=k: lp(x, data[k])),
                                             steps, 2)}
        res["callback"].append(row)
        print("callback", json.dumps(row), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_batch.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
