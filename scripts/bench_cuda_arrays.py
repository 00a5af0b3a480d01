#!/usr/bin/env python
"""What CUDA arrays in and out save, at 65 536 x 128 (dense Gaussian, stretch, dense_dmma):

  read     get_chain(cuda=True) against get_chain() of a DeviceBackend holding 32 stored steps (2 GiB of
           coordinates): wall clock of each call (both are complete when they return), and the rate of the device
           copy counting its read and write bytes, against the data sheet's 3.35 TB/s and the engine's own HBM copy
           micro-benchmark (eb_microbench 4) of the same run.
  run      run_mcmc(p0, k, store=False) for k = 1 and 10 from a DeviceArray p0 with cuda_results=True, against the
           same call from a numpy p0 returning numpy arrays (skip_initial_state_check=True for both: the check
           downloads the coordinates on purpose).

The arms alternate within every round; medians over the rounds.  The card's name and power limit are read in the
same run and printed with the numbers.

    python scripts/bench_cuda_arrays.py [--rounds 7] [--out DIR]
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
from emcee_b200 import DeviceBackend, _lib, models  # noqa: E402
from oracle import targets as T  # noqa: E402

N, D, NSTORE = 65536, 128, 32
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still device measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if _lib.device_count() < 1:
        raise SystemExit("bench_cuda_arrays: no CUDA device visible (the engine has no CPU fallback)")

    target, p0 = T.make_config("gauss_dense", N, D)
    model = models.GaussianDense(target.icov, target.mean)
    results = {"gpu": gpu_info(), "N": N, "D": D, "rounds": args.rounds,
               "hbm_copy_microbench_GBps": _lib.microbench(4)}

    # ---- read: a 2 GiB stored slice, device to device against device to host ----------------------------------
    s = emcee_b200.EnsembleSampler(N, D, model, seed=7, backend=DeviceBackend())
    s.run_mcmc(p0, NSTORE, skip_initial_state_check=True)
    nbytes = NSTORE * N * D * 8
    dev, host = [], []
    for _ in range(args.rounds + 1):  # the first round warms both paths up
        t, a = timed(lambda: s.get_chain(cuda=True))
        dev.append(t)
        del a
        t, a = timed(lambda: s.get_chain())
        host.append(t)
        del a
    dev, host = float(np.median(dev[1:])), float(np.median(host[1:]))
    results["read"] = {"bytes": nbytes, "cuda_s": dev, "host_s": host, "speedup": host / dev,
                       "cuda_GBps_read_plus_write": 2 * nbytes / dev / 1e9,
                       "share_of_3.35TBps": 2 * nbytes / dev / HBM_PEAK,
                       "host_GBps": nbytes / host / 1e9}
    got = s.get_chain(cuda=True)
    assert np.array_equal(got.get()[-1], s.get_chain()[-1]), "the device read differs from the host read"
    del got, s

    # ---- run: CUDA-array p0 and cuda_results against the host form --------------------------------------------
    hs = emcee_b200.EnsembleSampler(N, D, model, seed=11)
    cs = emcee_b200.EnsembleSampler(N, D, model, seed=11, cuda_results=True)
    p0d = _lib._device_array_from_host(p0, 0)
    results["run"] = {}
    for k in (1, 10):  # the two samplers step in lockstep, so their states stay equal
        th, tc = [], []
        for _ in range(args.rounds + 1):
            t, a = timed(lambda: hs.run_mcmc(p0, k, store=False, skip_initial_state_check=True))
            th.append(t)
            t, b = timed(lambda: cs.run_mcmc(p0d, k, store=False, skip_initial_state_check=True))
            tc.append(t)
        assert np.array_equal(a.coords, b.coords.get()), "the CUDA-array run differs from the host run"
        th, tc = float(np.median(th[1:])), float(np.median(tc[1:]))
        ms, _ = cs._engine.last_step_timing()
        results["run"][str(k)] = {"host_ms": 1e3 * th, "cuda_ms": 1e3 * tc, "saved_ms": 1e3 * (th - tc),
                                  "steps_device_ms": ms}

    line = json.dumps(results)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_cuda_arrays.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
