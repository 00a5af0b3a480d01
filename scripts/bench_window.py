#!/usr/bin/env python
"""Cost of the running window (``enable_window``) per recorded step, against no recording and a ``DeviceBackend``
stored step:

  off      ``run_mcmc(store=False)``, nothing recorded
  window   ``enable_window(size, 1)``, ``run_mcmc(store=False)``: every step recorded into the ring
  device   ``run_mcmc`` storing every step into a ``DeviceBackend``

Cases: 65 536 x 128 dense Gaussian (``dense_dmma``), 4 096 x 32 and 1 024 x 8 isotropic Gaussians.  Each arm is one
``run_mcmc`` call of --steps steps after --warmup warm-up steps; the device time of the call is
``eb_last_step_timing`` (CUDA events on the engine's stream, first launch to last).  The arms alternate for --rounds
rounds; the median, minimum and maximum per step are reported, with the launches per step.  A profiled call of the
window arm (``torch.profiler``, CUDA activity) gives the device time of the copy kernel itself
(``chain_store_kernel``).  Reads of the full window are timed on the host clock, each ending in the library's
synchronisation: ``get_chain(cuda=True)`` and ``get_autocorr_time(quiet=True)``.  The card name and power limit are
read in the same run.

    python scripts/bench_window.py [--rounds 5] [--steps 50] [--warmup 20] [--out DIR]
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


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


ARMS = ("off", "window", "device")


def profiled_store_us(s, state, steps):
    """device time of chain_store_kernel per launch in one profiled call"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        state = s.run_mcmc(state, steps, store=False)
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for e in prof.events():
        if e.device_type.name == "CUDA" and "chain_store_kernel" in e.name:
            tot += e.device_time if hasattr(e, "device_time") else e.cuda_time
            n += 1
    return state, tot / max(n, 1), n


def timed(f, reps=3):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        out.append(1e6 * (time.perf_counter() - t0))
    return float(np.median(out))


def case(N, D, dense, size, steps, warmup, rounds):
    rng = np.random.default_rng(N + D)
    if dense:
        a = rng.standard_normal((D, D))
        model = models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)))
    else:
        model = models.GaussianIso()
    p0 = rng.standard_normal((N, D))
    samplers, states = {}, {}
    for k in ARMS:
        s = emcee_b200.EnsembleSampler(N, D, model, seed=7, backend=DeviceBackend() if k == "device" else None)
        if k == "window":
            s.enable_window(size, 1)
        states[k] = s.run_mcmc(p0, warmup, store=k == "device", skip_initial_state_check=True)
        samplers[k] = s
    per = {k: [] for k in ARMS}
    launches = {}
    for _ in range(rounds):
        for k, s in samplers.items():
            states[k] = s.run_mcmc(states[k], steps, store=k == "device")
            ms, n = s._engine.last_step_timing()
            per[k].append(1e3 * ms / steps)
            launches[k] = n / steps
    row = dict(N=N, D=D, size=size, kernel=samplers["off"]._engine.last_kernel_name(), steps=steps, rounds=rounds)
    off = float(np.median(per["off"]))
    for k, v in per.items():
        med = float(np.median(v))
        row[k] = dict(step_us=med, min_us=float(np.min(v)), max_us=float(np.max(v)), extra_us_per_step=med - off,
                      launches_per_step=launches[k])
    try:
        states["window"], us, n = profiled_store_us(samplers["window"], states["window"], steps)
        row["window"]["store_kernel_us"] = us
        row["window"]["store_kernels"] = n
    except Exception as e:  # the step times above stand without it
        row["profile_error"] = repr(e)
    w = samplers["window"].window()
    row["window"]["filled"] = w.iteration
    row["read_chain_cuda_us"] = timed(lambda: w.get_chain(cuda=True))
    row["read_autocorr_us"] = timed(lambda: w.get_autocorr_time(quiet=True))
    row["window_bytes"] = w.nbytes
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), rows=[])
    for N, D, dense, size in [(65536, 128, True, 16), (4096, 32, False, 256), (1024, 8, False, 1024)]:
        res["rows"].append(case(N, D, dense, size, a.steps, a.warmup, a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    print(res["gpu"])
    for r in res["rows"]:
        print("%6d x %-4d %-10s size %d" % (r["N"], r["D"], r["kernel"], r["size"]))
        for k in ARMS:
            x = r[k]
            print("   %-7s %8.1f us/step [%0.1f, %0.1f] (+%0.1f), %.2f launches/step%s" % (
                k, x["step_us"], x["min_us"], x["max_us"], x["extra_us_per_step"], x["launches_per_step"],
                " | copy kernel %.1f us" % x["store_kernel_us"] if "store_kernel_us" in x else ""))
        print("   full-window get_chain(cuda=True) %.0f us, get_autocorr_time() %.0f us" % (
            r["read_chain_cuda_us"], r["read_autocorr_us"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_window.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
