#!/usr/bin/env python
"""Cost of the running trace (``enable_trace``) per step of a ``store=False`` run:

  off        no trace
  every_1    ``enable_trace(1)``: a row after every step
  every_10   ``enable_trace(10)``: a row after every tenth step

Cases: 65 536 x 128 dense Gaussian (``dense_dmma``) and 1 024 x 8 isotropic Gaussian (``tma_rows``).  Each arm is one
``run_mcmc(store=False)`` call of --steps steps; the device time of the call is ``eb_last_step_timing`` (CUDA events
on the engine's stream, first launch to last).  The arms alternate for --rounds rounds after one warm-up call each;
the median, minimum and maximum per step are reported.  ``row_us`` is the cost of one recorded step: an arm's median
per step less the ``off`` median, times ``every``; ``row_gbs`` is the bytes one row reads (N * D * 8, the state) over
``row_us``.  With ``every_1`` on ``dense_dmma`` the difference holds both the two trace kernels and what the step
loses by flushing its grouped launch before every recorded step.  The HBM copy rate of ``eb_microbench`` (what = 4)
and the card name and power limit are read in the same run.

    python scripts/bench_trace.py [--rounds 5] [--steps 50] [--out DIR]
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


ARMS = {"off": 0, "every_1": 1, "every_10": 10}


def case(N, D, dense, steps, rounds):
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
            s.enable_trace(every)
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
            row[k]["row_us"] = (med - off) * ARMS[k]
            row[k]["row_gbs"] = N * D * 8 / (row[k]["row_us"] * 1e-6) / 1e9 if med > off else None
    # the same seed and steps: every tenth row of every_1 is a row of every_10, bit for bit
    one, ten = samplers["every_1"].trace(), samplers["every_10"].trace()
    row["rows_equal"] = bool(all(a[9::10].tobytes() == b.tobytes() for a, b in zip(one, ten)))
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
        for k in ("every_1", "every_10"):
            x = r[k]
            line += " | %s %7.1f us [%0.1f, %0.1f] row %0.1f us" % (k, x["step_us"], x["min_us"], x["max_us"], x["row_us"])
            if x["row_gbs"]:
                line += " (%0.0f GB/s)" % x["row_gbs"]
        line += " | rows equal: %s" % r["rows_equal"]
        print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_trace.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
