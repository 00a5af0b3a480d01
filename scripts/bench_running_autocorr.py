#!/usr/bin/env python
"""Cost of the running autocorrelation function (``enable_autocorr``) per step of a ``store=False`` run:

  off        no sums
  every_1    ``enable_autocorr(max_lag, 1)``: the state of every step recorded
  every_10   ``enable_autocorr(max_lag, 10)``: the state of every tenth step recorded

Cases: 65 536 x 128 dense Gaussian (``dense_dmma``) with max_lag 32, 4 096 x 32 and 1 024 x 8 isotropic Gaussian
with max_lag 256 and 1 024.  Each arm is one
``run_mcmc(store=False)`` call of --steps steps (a multiple of 640, so every arm folds whole blocks of 64 recorded
steps); the device time of the call is ``eb_last_step_timing`` (CUDA events on the engine's stream, first launch to
last).  The arms alternate for --rounds rounds after one warm-up call each; the median, minimum and maximum per step
are reported.  ``rec_us`` is the cost of one recorded step: an arm's median per step less the ``off`` median, times
``every``.  ``rec_gbs`` is the bytes one recorded step moves at the least, from shapes: the state read and the ring
written (16 N D), and, over the block of 64, the block and history read once (8 N D (64 + max_lag) / 64) and the
double-double lag sums read and written once (32 N D (max_lag + 1) / 64); ``fma_g`` the lag products, (max_lag + 1)
N D per recorded step, over ``rec_us``.  The HBM copy rate of ``eb_microbench`` (what = 4) and the card name and
power limit are read in the same run; so is one read of rho (``read_ms``).

    python scripts/bench_running_autocorr.py [--rounds 5] [--steps 640] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import time
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import emcee_b200  # noqa: E402
from emcee_b200 import _lib, models  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


ARMS = {"off": 0, "every_1": 1, "every_10": 10}


def case(N, D, dense, max_lag, steps, rounds):
    rng = np.random.default_rng(N + D)
    if dense:
        a = rng.standard_normal((D, D))
        model = models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)))
    else:
        model = models.GaussianIso()
    p0 = rng.standard_normal((N, D))
    samplers, states = {}, {}
    for k, every in ARMS.items():
        s = emcee_b200.EnsembleSampler(N, D, model, seed=7)
        if every:
            s.enable_autocorr(max_lag, every)
        states[k] = s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)  # warm-up
        samplers[k] = s
    per = {k: [] for k in ARMS}
    launches = {}
    for _ in range(rounds):
        for k, s in samplers.items():
            states[k] = s.run_mcmc(states[k], steps, store=False)
            ms, n = s._engine.last_step_timing()
            per[k].append(1e3 * ms / steps)
            launches[k] = n / steps
    kernel = samplers["off"]._engine.last_kernel_name()
    row = dict(N=N, D=D, max_lag=max_lag, kernel=kernel, steps=steps, rounds=rounds)
    off = float(np.median(per["off"]))
    nd = N * D
    rec_bytes = 16 * nd + 8 * nd * (64 + max_lag) / 64 + 32 * nd * (max_lag + 1) / 64
    for k, v in per.items():
        med = float(np.median(v))
        row[k] = dict(step_us=med, min_us=float(np.min(v)), max_us=float(np.max(v)), launches_per_step=launches[k])
        if k != "off":
            us = (med - off) * ARMS[k]
            row[k]["rec_us"] = us
            row[k]["rec_gbs"] = rec_bytes / (us * 1e-6) / 1e9 if us > 0 else None
            row[k]["fma_g_per_s"] = (max_lag + 1) * nd / (us * 1e-6) / 1e9 if us > 0 else None
    s = samplers["every_1"]
    t0 = time.perf_counter()
    s.autocorr_function()
    row["read_ms"] = 1e3 * (time.perf_counter() - t0)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=640)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), hbm_copy_gbs=_lib.microbench(4), rows=[])
    for N, D, dense, max_lag in [(65536, 128, True, 32), (4096, 32, False, 256), (1024, 8, False, 1024)]:
        res["rows"].append(case(N, D, dense, max_lag, a.steps, a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    res["hbm_copy_gbs_after"] = _lib.microbench(4)
    print(res["gpu"], "| HBM copy %.0f / %.0f GB/s (before / after)" % (res["hbm_copy_gbs"], res["hbm_copy_gbs_after"]))
    for r in res["rows"]:
        line = "%6d x %-4d L %-5d %-10s off %7.1f us [%0.1f, %0.1f]" % (
            r["N"], r["D"], r["max_lag"], r["kernel"], r["off"]["step_us"], r["off"]["min_us"], r["off"]["max_us"])
        for k in ("every_1", "every_10"):
            x = r[k]
            line += " | %s %7.1f us [%0.1f, %0.1f] rec %0.1f us" % (k, x["step_us"], x["min_us"], x["max_us"], x["rec_us"])
            if x["rec_gbs"]:
                line += " (%0.0f GB/s, %0.0f G FMA/s)" % (x["rec_gbs"], x["fma_g_per_s"])
        line += " | read %0.1f ms" % r["read_ms"]
        print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_running_autocorr.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
