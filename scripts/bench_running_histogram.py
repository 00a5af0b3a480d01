#!/usr/bin/env python
"""Cost of the running histograms (``enable_histograms``) per step of a ``store=False`` run:

  off      no counting
  1d_20    ``enable_histograms(range, bins=20)``: every parameter, every step
  1d_512   the same with ``bins=512``
  2d_16    ``bins=20`` plus ``params2d=range(16), bins2d=20`` (120 pairs; all 8 parameters, 28 pairs, at ndim 8)

Cases: 65 536 x 128 dense Gaussian (``dense_dmma``) and 1 024 x 8 isotropic Gaussian (``tma_rows``).  Each arm is one
``run_mcmc(store=False)`` call of --steps steps; the device time of the call is ``eb_last_step_timing`` (CUDA events
on the engine's stream, first launch to last).  The arms alternate for --rounds rounds after one warm-up call each;
the median, minimum and maximum per step are reported.  ``count_us`` is an arm's median per step less the ``off``
median, and ``count_gbs`` the bytes one count reads (N * D * 8, the state) over ``count_us``.  The HBM copy rate of
``eb_microbench`` (what = 4) and the card name and power limit are read in the same run.

    python scripts/bench_running_histogram.py [--rounds 5] [--steps 50] [--out DIR]
"""
import argparse
import json
import os
import subprocess
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


ARMS = {
    "off": None,
    "1d_20": dict(bins=20),
    "1d_512": dict(bins=512),
    "2d_16": dict(bins=20, params2d=16, bins2d=20),
}


def case(N, D, dense, steps, rounds):
    rng = np.random.default_rng(N + D)
    if dense:
        a = rng.standard_normal((D, D))
        model = models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)))
    else:
        model = models.GaussianIso()
    p0 = rng.standard_normal((N, D))
    samplers, states = {}, {}
    for k, cfg in ARMS.items():
        s = emcee_b200.EnsembleSampler(N, D, model, seed=7)
        if cfg is not None:
            cfg = dict(cfg)
            if "params2d" in cfg:  # the first 16 parameters, or all of them
                cfg["params2d"] = list(range(min(cfg["params2d"], D)))
            s.enable_histograms([(-4.0, 4.0)] * D, every=1, **cfg)
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
    row = dict(N=N, D=D, kernel=kernel, steps=steps, rounds=rounds)
    off = float(np.median(per["off"]))
    for k, v in per.items():
        med = float(np.median(v))
        row[k] = dict(step_us=med, min_us=float(np.min(v)), max_us=float(np.max(v)), launches_per_step=launches[k])
        if k != "off":
            row[k]["count_us"] = med - off
            row[k]["count_gbs"] = N * D * 8 / ((med - off) * 1e-6) / 1e9 if med > off else None
    # the counts are equal across arms that share bins (same seed, same steps): a cheap consistency check
    row["equal_1d"] = bool(np.array_equal(samplers["1d_20"].histogram()[0], samplers["2d_16"].histogram()[0]))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), hbm_copy_gbs=_lib.microbench(4), rows=[])
    for N, D, dense in [(65536, 128, True), (1024, 8, False)]:
        res["rows"].append(case(N, D, dense, a.steps, a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    res["hbm_copy_gbs_after"] = _lib.microbench(4)
    print(res["gpu"], "| HBM copy %.0f / %.0f GB/s (before / after)" % (res["hbm_copy_gbs"], res["hbm_copy_gbs_after"]))
    for r in res["rows"]:
        line = "%6d x %-4d %-10s off %7.1f us [%0.1f, %0.1f]" % (r["N"], r["D"], r["kernel"], r["off"]["step_us"],
                                                                 r["off"]["min_us"], r["off"]["max_us"])
        for k in ("1d_20", "1d_512", "2d_16"):
            x = r[k]
            line += " | %s %7.1f us [%0.1f, %0.1f] +%0.1f" % (k, x["step_us"], x["min_us"], x["max_us"], x["count_us"])
            if x["count_gbs"]:
                line += " (%0.0f GB/s)" % x["count_gbs"]
        print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_running_histogram.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
