#!/usr/bin/env python
"""Cost of the running reservoir (``enable_reservoir``) per step of a ``store=False`` run:

  off             no reservoir
  K{size}_every{e}  ``enable_reservoir(size, e)`` for size 10**4 and 10**6, e = 1 and 10

Cases: 65 536 x 128 dense Gaussian (``dense_dmma``) and 1 024 x 8 isotropic Gaussian (``tma_rows``).  Each arm is one
``run_mcmc(store=False)`` call of --steps steps after --warmup warm-up steps; the device time of the call is
``eb_last_step_timing`` (CUDA events on the engine's stream, first launch to last).  The arms alternate for --rounds
rounds; the median, minimum and maximum per step are reported, with the launches per step.  ``compactions`` is the
number the schedule (``csrc/reservoir_plan.h``, restated below) runs in one timed call.  A separate profiled call per
arm (``torch.profiler``, CUDA activity) sums the device time of the record kernel (``res_filter_kernel``) and of the
compaction kernels (the other ``res_*`` kernels), so that the records alone and the compactions alone are reported
beside the step times.  The card name and power limit are read in the same run.

    python scripts/bench_reservoir.py [--rounds 5] [--steps 50] [--warmup 20] [--out DIR]
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
from emcee_b200 import models  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


ARMS = {"off": None}
for _K in (10**4, 10**6):
    for _e in (1, 10):
        ARMS["K%d_every%d" % (_K, _e)] = (_K, _e)


class Schedule(object):
    """reservoir_plan.h's ResSchedule"""

    def __init__(self, K, N):
        self.K, self.N, self.cap, self.offered, self.bound = K, N, K + max(K, N), 0, 0

    def record(self):
        c = 0
        if self.bound + self.N > self.cap:
            self.bound, c = min(self.K, self.offered), 1
        self.offered += self.N
        self.bound += self.N
        return c


def compactions(K, every, N, step0, steps):
    """compactions in the call that runs steps step0 + 1 .. step0 + steps, the reservoir enabled at step 0"""
    s, c = Schedule(K, N), 0
    for n in range(1, step0 + steps + 1):
        if n % every == 0:
            r = s.record()
            c += r if n > step0 else 0
    return c


COMPACTION_KERNELS = ("res_begin_kernel", "res_hist_kernel", "res_mark_kernel", "res_group_kernel", "res_move_kernel")


def profiled(s, state, steps):
    """(record us, compaction us) of one call, summed over the kernels' device time"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        state = s.run_mcmc(state, steps, store=False)
        torch.cuda.synchronize()
    rec = comp = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        t = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "res_filter_kernel" in name:
            rec += t
        elif any(k in name for k in COMPACTION_KERNELS):
            comp += t
    return state, rec, comp


def case(N, D, dense, steps, warmup, rounds):
    rng = np.random.default_rng(N + D)
    if dense:
        a = rng.standard_normal((D, D))
        model = models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)))
    else:
        model = models.GaussianIso()
    p0 = rng.standard_normal((N, D))
    samplers, states = {}, {}
    for k, arm in ARMS.items():
        s = emcee_b200.EnsembleSampler(N, D, model, seed=7)
        if arm:
            s.enable_reservoir(*arm)
        states[k] = s.run_mcmc(p0, warmup, store=False, skip_initial_state_check=True)
        samplers[k] = s
    per = {k: [] for k in ARMS}
    launches = {}
    done = warmup
    for _ in range(rounds):
        for k, s in samplers.items():
            states[k] = s.run_mcmc(states[k], steps, store=False)
            ms, n = s._engine.last_step_timing()
            per[k].append(1e3 * ms / steps)
            launches[k] = n / steps
        done += steps
    row = dict(N=N, D=D, kernel=samplers["off"]._engine.last_kernel_name(), steps=steps, rounds=rounds)
    off = float(np.median(per["off"]))
    for k, v in per.items():
        med = float(np.median(v))
        row[k] = dict(step_us=med, min_us=float(np.min(v)), max_us=float(np.max(v)), launches_per_step=launches[k])
        if ARMS[k]:
            K, every = ARMS[k]
            row[k]["extra_us_per_step"] = med - off
            row[k]["compactions_per_call"] = compactions(K, every, N, done - steps, steps)
    # the records alone and the compactions alone, in a profiled call of their own
    try:
        for k, arm in ARMS.items():
            if not arm:
                continue
            K, every = arm
            c = compactions(K, every, N, done, steps)
            states[k], rec, comp = profiled(samplers[k], states[k], steps)
            nrec = steps // every
            row[k]["profiled"] = dict(records=nrec, record_us_each=rec / max(nrec, 1), compactions=c,
                                      compaction_us_each=comp / c if c else None)
        done += steps
    except Exception as e:  # the step times above stand without the split
        row["profile_error"] = repr(e)
    # what each arm kept: min(size, offered) rows, all of recorded steps
    for k, arm in ARMS.items():
        if arm:
            r = samplers[k].reservoir()
            row[k]["kept"] = int(r.step.size)
            row[k]["offered"] = samplers[k].reservoir_count()
            row[k]["sorted_steps_ok"] = bool(np.all(r.step % arm[1] == 0))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), rows=[])
    for N, D, dense in [(65536, 128, True), (1024, 8, False)]:
        res["rows"].append(case(N, D, dense, a.steps, a.warmup, a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    print(res["gpu"])
    for r in res["rows"]:
        print("%6d x %-4d %-10s off %7.1f us [%0.1f, %0.1f], %.1f launches/step" % (
            r["N"], r["D"], r["kernel"], r["off"]["step_us"], r["off"]["min_us"], r["off"]["max_us"],
            r["off"]["launches_per_step"]))
        for k, arm in ARMS.items():
            if not arm:
                continue
            x = r[k]
            p = x.get("profiled", {})
            print("   %-16s %7.1f us [%0.1f, %0.1f] (+%0.1f), %.2f launches/step, %d compactions/call | record %s us, "
                  "compaction %s us" % (k, x["step_us"], x["min_us"], x["max_us"], x["extra_us_per_step"],
                                        x["launches_per_step"], x["compactions_per_call"],
                                        "%.1f" % p["record_us_each"] if p else "-",
                                        "%.1f" % p["compaction_us_each"] if p and p["compaction_us_each"] else "-"))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_reservoir.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
