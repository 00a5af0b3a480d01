#!/usr/bin/env python
"""Throughput of KDEMove on the device (kde.cu) and of the route it replaces.

  device     KDEMove on a dense Gaussian model at 4 096 x 16, 16 384 x 32 and 65 536 x 32, store=False: seconds per
             step and walker-steps/s from the engine's device events (eb_last_step_timing), medians of --rounds
             calls of --steps steps after one warm-up call
  lse        the log-density kernel alone (kde_lse_kernel, from a torch.profiler run of its own): its FP64 rate,
             counted from the shapes as one subtract and one fused multiply-add per (point, centre, dimension)
             -- 2 * (2 ns) * nc * D per split -- over its kernel time, and that rate as a share of the card's FP64
             vector peak (SMs x 64 FP64 lanes x the maximum SM clock nvidia-smi reports)
  host       the same sampling through a host user move: a RedBlueMove subclass whose get_proposal is the
             reference's KDEMove.get_proposal (scipy.stats.gaussian_kde on the CPU, the split downloaded and the
             proposals uploaded every half-step), at the two smaller sizes, seconds per step by the host clock

The card name, power limit and maximum SM clock are read in the same run.  The host arm needs
oracle/_ref/emcee_reference.zip (built by __graft_entry__.build()); without it, it reports "not measured".

    python scripts/bench_kde.py [--rounds 3] [--steps 4] [--out DIR]
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
from emcee_b200 import models, moves  # noqa: E402
from oracle import targets as T  # noqa: E402

REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "emcee_reference.zip")
SIZES = [(4096, 16), (16384, 32), (65536, 32)]
HOST_SIZES = [(4096, 16, 3), (16384, 32, 1)]  # N, D, steps
FP64_LANES_PER_SM = 64
SEED = 0xCDE


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [f.strip() for f in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock_mhz=float(clock.split()[0]))
    except Exception as e:
        return dict(name="unknown (%s)" % e, power_limit="unknown", max_sm_clock_mhz=None)


def sampler(N, D, mv):
    target, p0 = T.make_config("gauss_dense", N, D)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(target.icov, target.mean), moves=mv, seed=SEED)
    return s, p0


def device_rows(rounds, steps):
    rows = []
    for N, D in SIZES:
        s, p0 = sampler(N, D, moves.KDEMove())
        state = s.run_mcmc(p0, 1, store=False, skip_initial_state_check=True)
        assert s._engine.last_kernel_name() == "kde"
        t = []
        for _ in range(rounds):
            state = s.run_mcmc(state, steps, store=False, skip_initial_state_check=True)
            ms, _launches = s._engine.last_step_timing()
            t.append(ms * 1e-3 / steps)
        sec = float(np.median(t))
        rows.append(dict(N=N, D=D, s_per_step=sec, walker_steps_per_s=N / sec, rounds=t))
        print("device  %6d x %-3d  %.4e s/step  %.3e walker-steps/s" % (N, D, sec, N / sec), flush=True)
    return rows


def lse_rows(info, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile

    props = torch.cuda.get_device_properties(0)
    peak = None
    if info["max_sm_clock_mhz"]:
        peak = props.multi_processor_count * FP64_LANES_PER_SM * info["max_sm_clock_mhz"] * 1e6
    rows = []
    for N, D in SIZES:
        s, p0 = sampler(N, D, moves.KDEMove())
        state = s.run_mcmc(p0, 1, store=False, skip_initial_state_check=True)
        steps = 2
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.run_mcmc(state, steps, store=False, skip_initial_state_check=True)
        us = sum(e.device_time_total for e in prof.key_averages() if "kde_lse_kernel" in e.key)
        n_a = (N + 1) // 2  # two splits: ceil(N / 2) and floor(N / 2) active walkers
        n_b = N - n_a
        instr = steps * 2 * D * (2 * n_a * n_b + 2 * n_b * n_a)
        rate = instr / (us * 1e-6)
        rows.append(dict(N=N, D=D, kernel_s_per_step=us * 1e-6 / steps, fp64_instr_per_s=rate,
                         share_of_fp64_peak=None if peak is None else rate / peak, fp64_peak_instr_per_s=peak))
        print("lse     %6d x %-3d  %.4e s/step  %.3e FP64 lane-instr/s  %s of peak" % (
            N, D, us * 1e-6 / steps, rate, "n/a" if peak is None else "%.1f%%" % (100 * rate / peak)), flush=True)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "kde_lse.pt.trace.json"))
    return rows


def host_rows():
    if not os.path.exists(REF_ZIP):
        return [dict(N=N, D=D, s_per_step="not measured (no reference package)") for N, D, _ in HOST_SIZES]
    if REF_ZIP not in sys.path:
        sys.path.insert(0, REF_ZIP)
    import emcee

    class HostKDE(moves.RedBlueMove):
        """Today's route: the reference's KDEMove.get_proposal as a host user move."""

        bw_method = None

        def get_proposal(self, s, c, random):
            return emcee.moves.KDEMove.get_proposal(self, s, c, random)

    rows = []
    for N, D, steps in HOST_SIZES:
        s, p0 = sampler(N, D, HostKDE())
        state = s.run_mcmc(p0, 1, store=False, skip_initial_state_check=True)
        t0 = time.perf_counter()
        s.run_mcmc(state, steps, store=False, skip_initial_state_check=True)
        sec = (time.perf_counter() - t0) / steps
        rows.append(dict(N=N, D=D, s_per_step=sec, walker_steps_per_s=N / sec, steps=steps))
        print("host    %6d x %-3d  %.4e s/step  %.3e walker-steps/s" % (N, D, sec, N / sec), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_kde: no CUDA device")
    info = gpu_info()
    print("card: %s, power limit %s, max SM clock %s MHz" % (info["name"], info["power_limit"],
                                                            info["max_sm_clock_mhz"]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    res = dict(gpu=info, device=device_rows(args.rounds, args.steps), lse=lse_rows(info, args.out), host=host_rows())
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(os.path.join(args.out, "bench_kde.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
