#!/usr/bin/env python
"""Cost of a box prior (models.Bounded) on three workloads, each run unbounded, with a box that never binds
(+-1e300) and with a box that binds, alternated round by round on one engine per arm:

  dense   65 536 x 128 dense Gaussian, stretch (dense_dmma), L2 flushed before every step
  ring    262 144 x 32 ring, stretch (tma_rows register path)
  rosen   16 384 x 256 Rosenbrock, DE 0.8 + snooker 0.2 (tma_rows)

Prints one JSON line per (workload, arm, round) with the device time per step (CUDA events,
eb_last_step_timing) and a summary line per workload: the median of each arm and its ratio to unbounded.

    python scripts/bench_bounds.py [--steps 100] [--rounds 3] [--out DIR]
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
from emcee_b200 import models, moves  # noqa: E402
from oracle import targets as T  # noqa: E402

WORKLOADS = {
    "dense": ("gauss_dense", 65536, 128, [(moves.StretchMove(), 1.0)], True),
    "ring": ("ring", 262144, 32, [(moves.StretchMove(), 1.0)], False),
    "rosen": ("rosenbrock", 16384, 256, [(moves.DEMove(), 0.8), (moves.DESnookerMove(), 0.2)], False),
}


def device_model(kind, t):
    if kind == "gauss_dense":
        return models.GaussianDense(t.icov, t.mean)
    if kind == "ring":
        return models.Ring(t.radius, t.sigma)
    return models.Rosenbrock(t.a, t.b)


def arms(kind, p0):
    """unbounded / never binding / binding: the binding box is 1.5 sd either side of the centre of p0, which
    rejects a good share of the proposals without freezing the ensemble."""
    D = p0.shape[1]
    c, sd = float(np.mean(p0)), float(np.std(p0))
    return {
        "unbounded": None,
        "never_binding": (np.full(D, -1e300), np.full(D, 1e300)),
        "binding": (np.full(D, c - 1.5 * sd), np.full(D, c + 1.5 * sd)),
    }


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default=None, help="comma-separated workloads")
    ap.add_argument("--out", default=None, help="directory for the JSON lines (default: stdout only)")
    args = ap.parse_args()
    card = gpu_name()
    lines = []
    for name, (kind, N, D, mv, flush) in WORKLOADS.items():
        if args.only and name not in args.only.split(","):
            continue
        target, p0 = T.make_config(kind, N, D)
        engines = {}
        for arm, box in arms(kind, p0).items():
            m = device_model(kind, target)
            if box is not None:
                m = models.Bounded(m, *box)
            s = emcee_b200.EnsembleSampler(N, D, m, moves=mv, seed=0xB0B)
            eng = s._engine
            eng.set_option("l2_flush", 1 if flush else 0)
            if box is not None and arm == "binding":
                p = np.clip(p0, box[0], box[1])
            else:
                p = p0
            eng.set_state(p)
            engines[arm] = (eng, s._schedule())
        times = {arm: [] for arm in engines}
        for r in range(args.rounds):
            for arm, (eng, sched) in engines.items():
                eng.step(sched, args.warmup, want_accepted=False)
                eng.step(sched, args.steps, want_accepted=False)
                ms, launches = eng.last_step_timing()
                us = 1e3 * ms / args.steps
                times[arm].append(us)
                rec = {"workload": name, "arm": arm, "round": r, "us_per_step": us, "launches": launches,
                       "variant": eng.last_kernel_variant(), "gpu": card}
                lines.append(rec)
                print(json.dumps(rec), flush=True)
        base = float(np.median(times["unbounded"]))
        summ = {"workload": name, "gpu": card, "N": N, "D": D, "l2_flush": flush, "steps": args.steps,
                "rounds": args.rounds}
        for arm, v in times.items():
            summ[arm + "_us_median"] = float(np.median(v))
            summ[arm + "_us_range"] = [float(min(v)), float(max(v))]
            summ[arm + "_ratio"] = float(np.median(v)) / base
        lines.append(summ)
        print(json.dumps(summ), flush=True)
        for eng, _ in engines.values():
            eng.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_bounds.jsonl"), "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
