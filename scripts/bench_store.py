#!/usr/bin/env python
"""Cost of storing the chain: store=False, the host Backend and DeviceBackend, each at thin_by 1 and 10, on

  dense    65 536 x 128 dense Gaussian, stretch (dense_dmma)
  small     4 096 x 128 dense Gaussian, stretch (dense_dmma)
  ring    262 144 x 32 ring, stretch (tma_rows register path)

Each (mode, thin_by) has its own sampler; every round resets the backends and runs run_mcmc(p0, nstore,
thin_by=...) for every arm in turn, so the arms alternate.  Reported per arm: the device time per step from
eb_last_step_timing (CUDA events on the engine's stream, the stores included) and the wall clock of run_mcmc
(the host Backend's grow, staging and memcpy included), medians over the rounds.  nstore is capped so that the
host chain fits in a quarter of the available host RAM.

Then, on one stored chain of the small workload, the time of get_autocorr_time() and get_chain(discard, thin,
flat=True) through both backends.

    python scripts/bench_store.py [--rounds 3] [--out DIR]
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
from emcee_b200 import Backend, DeviceBackend, models  # noqa: E402
from oracle import targets as T  # noqa: E402

WORKLOADS = {
    "dense": ("gauss_dense", 65536, 128, 64),
    "small": ("gauss_dense", 4096, 128, 512),
    "ring": ("ring", 262144, 32, 64),
}
THINS = (1, 10)


def device_model(kind, t):
    if kind == "gauss_dense":
        return models.GaussianDense(t.icov, t.mean)
    return models.Ring(t.radius, t.sigma)


def host_ram():
    info = {}
    with open("/proc/meminfo") as f:
        for line in f:
            k, v = line.split(":")
            info[k] = int(v.split()[0]) * 1024
    return info["MemTotal"], info["MemAvailable"]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still device measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def make_backend(mode):
    return {"nostore": Backend, "host": Backend, "device": DeviceBackend}[mode]()


def run_arm(s, mode, p0, nstore, thin_by):
    s.reset()
    t0 = time.perf_counter()
    s.run_mcmc(p0, nstore, thin_by=thin_by, store=mode != "nostore", skip_initial_state_check=True)
    wall = time.perf_counter() - t0
    ms, _ = s._engine.last_step_timing()
    return 1e3 * ms / (nstore * thin_by), wall


def bench_workload(name, rounds, out):
    kind, N, D, nstore = WORKLOADS[name]
    step_bytes = 8 * N * (D + 1)
    _, avail = host_ram()
    nstore = int(max(4, min(nstore, avail // 4 // (2 * step_bytes))))  # grow copies: two chains at once
    t, p0 = T.make_config(kind, N, D)
    arms = {}
    for mode in ("nostore", "host", "device"):
        for thin_by in THINS:
            s = emcee_b200.EnsembleSampler(N, D, device_model(kind, t), seed=0xB5, backend=make_backend(mode))
            s.run_mcmc(p0, 4, store=False, skip_initial_state_check=True)  # modules, split tables
            arms[(mode, thin_by)] = s
    res = {k: [] for k in arms}
    for r in range(rounds):
        for (mode, thin_by), s in arms.items():
            us, wall = run_arm(s, mode, p0, nstore, thin_by)
            res[(mode, thin_by)].append((us, wall))
            print(json.dumps(dict(workload=name, mode=mode, thin_by=thin_by, round=r, nstore=nstore,
                                  us_per_step=us, run_mcmc_s=wall)), flush=True)
    summary = []
    for (mode, thin_by), v in res.items():
        us = float(np.median([a for a, _ in v]))
        wall = float(np.median([b for _, b in v]))
        summary.append(dict(workload=name, N=N, D=D, mode=mode, thin_by=thin_by, nstore=nstore,
                            steps=nstore * thin_by, us_per_step=us, run_mcmc_s=wall))
    for s in arms.values():
        if isinstance(s.backend, DeviceBackend):
            s.backend.close()
    del arms
    out.extend(summary)
    return summary


def bench_analysis(rounds, nstore=500):
    kind, N, D, _ = WORKLOADS["small"]
    t, p0 = T.make_config(kind, N, D)
    ss = {}
    for mode in ("host", "device"):
        s = emcee_b200.EnsembleSampler(N, D, device_model(kind, t), seed=0xB6, backend=make_backend(mode))
        s.run_mcmc(p0, nstore, skip_initial_state_check=True)
        ss[mode] = s
    times = {(m, what): [] for m in ss for what in ("autocorr", "get_chain")}
    taus = {}
    for r in range(rounds):
        for m, s in ss.items():
            t0 = time.perf_counter()
            taus[m] = s.get_autocorr_time(quiet=True)
            times[(m, "autocorr")].append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            x = s.get_chain(discard=100, thin=5, flat=True)
            times[(m, "get_chain")].append(time.perf_counter() - t0)
    same = bool(np.array_equal(taus["host"], taus["device"]))
    return [dict(analysis=what, mode=m, N=N, D=D, nstore=nstore, seconds=float(np.median(v)),
                 tau_identical=same, get_chain_shape=list(x.shape))
            for (m, what), v in times.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="dense,small,ring")
    ap.add_argument("--out", default=None, help="directory for bench_store.json")
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_store: no CUDA device visible")
    total, avail = host_ram()
    head = dict(gpu=gpu_info(), host_ram_total=total, host_ram_available=avail)
    print(json.dumps(head), flush=True)
    rows = []
    for name in args.workloads.split(","):
        bench_workload(name, args.rounds, rows)
    rows.extend(bench_analysis(args.rounds))
    print("%-6s %-8s %6s %7s %12s %12s" % ("work", "mode", "thin", "nstore", "us/step", "run_mcmc s"))
    for r in rows:
        if "workload" in r:
            print("%-6s %-8s %6d %7d %12.1f %12.3f" % (r["workload"], r["mode"], r["thin_by"], r["nstore"],
                                                     r["us_per_step"], r["run_mcmc_s"]))
        else:
            print("analysis %-10s %-7s %.4f s (tau identical: %s)" % (r["analysis"], r["mode"], r["seconds"],
                                                                     r["tau_identical"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_store.json"), "w") as f:
            json.dump(dict(head, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
