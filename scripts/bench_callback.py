#!/usr/bin/env python
"""Throughput of user log-probability functions (models.HostFunction / models.CudaArrayFunction), each row
against its natural baseline:

  iso_map      32 x 5 isotropic Gaussian, HostFunction(vectorize=False) -- the reference with its serial map
  dense_vec    4 096 x 128 dense Gaussian, the numpy target of oracle/targets.py, HostFunction(vectorize=True)
               -- the reference with vectorize=True and the same target
  dense_torch  65 536 x 128 dense Gaussian as a torch CudaArrayFunction -- the fused GaussianDense device model

Stretch move, store=False.  Reported per arm: walker-steps/s from the host clock around run_mcmc (which ends in a
stream synchronisation), and for the callback arms the share of that time spent inside the function (measured
by the wrapper around it).  The card name and power limit are read in the same run.  The reference arms need
oracle/_ref/emcee_reference.zip (built by __graft_entry__.build() when a checkout of the reference exists) and
are skipped without it.

    python scripts/bench_callback.py [--rounds 3] [--out DIR]
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
from oracle import targets as T  # noqa: E402

REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "emcee_reference.zip")
SEED = 0xCB


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def reference():
    if not os.path.exists(REF_ZIP):
        return None
    if REF_ZIP not in sys.path:
        sys.path.insert(0, REF_ZIP)
    import emcee

    assert REF_ZIP in emcee.__file__, emcee.__file__
    return emcee


class Timed(object):
    """fn, with the time spent inside it accumulated."""

    def __init__(self, fn):
        self.fn, self.seconds = fn, 0.0

    def __call__(self, x):
        t0 = time.perf_counter()
        try:
            return self.fn(x)
        finally:
            self.seconds += time.perf_counter() - t0


def torch_dense(t):
    import torch

    icov = torch.as_tensor(t.icov, device="cuda")
    mean = torch.as_tensor(t.mean, device="cuda")

    def f(rows):
        d = torch.as_tensor(rows, device="cuda") - mean
        return -0.5 * ((d @ icov) * d).sum(dim=1)

    return f


def arm_b200(N, D, fn_or_model, p0, steps, rounds):
    timed = None
    if isinstance(fn_or_model, models.CallbackFunction):
        timed = Timed(fn_or_model.fn)
        fn_or_model.fn = timed
    s = emcee_b200.EnsembleSampler(N, D, fn_or_model, seed=SEED)
    s.run_mcmc(p0, 2, store=False, skip_initial_state_check=True)  # warm-up: modules, tables, staging
    out = []
    for _ in range(rounds):
        if timed is not None:
            timed.seconds = 0.0
        t0 = time.perf_counter()
        s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
        wall = time.perf_counter() - t0
        out.append((N * steps / wall, None if timed is None else timed.seconds / wall))
    return out


def arm_reference(emcee, N, D, fn, p0, steps, rounds, vectorize):
    timed = Timed(fn)
    out = []
    for _ in range(rounds):
        np.random.seed(SEED)
        s = emcee.EnsembleSampler(N, D, timed, vectorize=vectorize)
        timed.seconds = 0.0
        t0 = time.perf_counter()
        s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
        wall = time.perf_counter() - t0
        out.append((N * steps / wall, timed.seconds / wall))
    return out


def summary(row, arm, runs, steps, N, D):
    rate = float(np.median([r for r, _ in runs]))
    share = [s for _, s in runs if s is not None]
    return dict(row=row, arm=arm, N=N, D=D, steps=steps, walker_steps_per_s=rate,
                callback_share=float(np.median(share)) if share else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rows", default="iso_map,dense_vec,dense_torch")
    ap.add_argument("--out", default=None, help="directory for bench_callback.json")
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_callback: no CUDA device visible")
    head = dict(gpu=gpu_info())
    print(json.dumps(head), flush=True)
    emcee = reference()
    rows = []
    want = args.rows.split(",")
    if "iso_map" in want:
        N, D, steps = 32, 5, 2000
        t, p0 = T.make_config("gauss_iso", N, D)
        rows.append(summary("iso_map", "HostFunction(map)",
                            arm_b200(N, D, models.HostFunction(t), p0, steps, args.rounds), steps, N, D))
        if emcee is not None:
            rows.append(summary("iso_map", "reference map",
                                arm_reference(emcee, N, D, t, p0, steps, args.rounds, False), steps, N, D))
    if "dense_vec" in want:
        N, D, steps = 4096, 128, 20
        t, p0 = T.make_config("gauss_dense", N, D)
        rows.append(summary("dense_vec", "HostFunction(vectorize)",
                            arm_b200(N, D, models.HostFunction(t, vectorize=True), p0, steps, args.rounds),
                            steps, N, D))
        if emcee is not None:
            rows.append(summary("dense_vec", "reference vectorize",
                                arm_reference(emcee, N, D, t, p0, steps, args.rounds, True), steps, N, D))
    if "dense_torch" in want:
        N, D, steps = 65536, 128, 50
        t, p0 = T.make_config("gauss_dense", N, D)
        try:
            fn = torch_dense(t)
        except Exception as e:  # no torch with CUDA: the device-model arm still runs
            print(json.dumps(dict(row="dense_torch", skipped=str(e))), flush=True)
            fn = None
        if fn is not None:
            rows.append(summary("dense_torch", "CudaArrayFunction(torch)",
                                arm_b200(N, D, models.CudaArrayFunction(fn), p0, steps, args.rounds), steps, N, D))
        rows.append(summary("dense_torch", "GaussianDense device model",
                            arm_b200(N, D, models.GaussianDense(t.icov, t.mean), p0, steps, args.rounds),
                            steps, N, D))
    for r in rows:
        print(json.dumps(r), flush=True)
    print("%-12s %-28s %16s %10s" % ("row", "arm", "walker-steps/s", "callback"))
    for r in rows:
        share = "-" if r["callback_share"] is None else "%.0f%%" % (100 * r["callback_share"])
        print("%-12s %-28s %16.4g %10s" % (r["row"], r["arm"], r["walker_steps_per_s"], share))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_callback.json"), "w") as f:
            json.dump(dict(head, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
