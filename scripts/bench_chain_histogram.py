#!/usr/bin/env python
"""Time of the histograms of a stored device chain against the download-then-numpy route:

  1-D      ``DeviceBackend.get_histogram(bins=20)`` (``eb_chain_select`` for the ranges, then
           ``eb_chain_histogram``) against ``get_chain(flat=True)`` + ``np.histogram`` per column
  2-D      ``get_histogram2d(params=range(16), bins=20)`` (120 pairs) against ``get_chain(flat=True)`` +
           ``np.histogram2d`` per pair
  all      ``get_histogram2d(bins=20)`` of every pair at ndim 128 (8 128 pairs), device only; and the same with
           ``bins=128``, where every pair is a tile of its own that reads its two columns of the whole slice

Cases: 4 096 x 128 with 500 stored steps read with ``discard=100, thin=5``, and 65 536 x 128 with 64 stored steps.
The arms alternate for --rounds rounds; medians of the host clock per call are reported (every call returns host
arrays, so it ends in a stream synchronisation).  ``range_ms`` is the range selection alone (the
``eb_chain_select`` call the device arms make first), so its share of each device call can be read off.  The card
name and power limit are read in the same run.

    python scripts/bench_chain_histogram.py [--rounds 2] [--out DIR]
"""
import argparse
import itertools
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

BINS = 20
PARAMS = list(range(16))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def case(N, D, steps, discard, thin, rounds):
    rng = np.random.default_rng(N)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=5, backend=DeviceBackend())
    s.run_mcmc(rng.standard_normal((N, D)), steps, skip_initial_state_check=True)
    b = s.backend
    kw = dict(discard=discard, thin=thin)
    first, stride, count = emcee_b200.backend.slice_plan(b.iteration, discard, thin)
    ends = np.array([0, count * N - 1], dtype=np.uint64)

    def host_1d():
        flat = b.get_chain(flat=True, **kw)
        out = [np.histogram(flat[:, d], BINS) for d in range(D)]
        return np.array([h for h, _ in out]), np.array([e for _, e in out])

    def host_2d():
        flat = b.get_chain(flat=True, **kw)
        return np.array([np.histogram2d(flat[:, i], flat[:, j], BINS)[0]
                         for i, j in itertools.combinations(PARAMS, 2)])

    arms = {"range": lambda: b._chain.select("chain", first, stride, count, ends),
            "device_1d": lambda: b.get_histogram(BINS, **kw), "host_1d": host_1d,
            "device_2d": lambda: b.get_histogram2d(PARAMS, BINS, **kw), "host_2d": host_2d,
            "device_all_pairs": lambda: b.get_histogram2d(None, BINS, **kw),
            "device_all_pairs_bins128": lambda: b.get_histogram2d(None, 128, **kw)[0].shape}
    for k, fn in arms.items():  # warm every device arm once (the host arms have nothing to warm)
        if not k.startswith("host"):
            fn()
    times = {k: [] for k in arms}
    out = {}
    for _ in range(rounds):
        for k, fn in arms.items():
            t, out[k] = timed(fn)
            times[k].append(t)
    (d1, h1), (d2, h2) = (out["device_1d"], out["host_1d"]), (out["device_2d"][0], out["host_2d"])
    row = dict(N=N, D=D, stored=steps, discard=discard, thin=thin, slice_steps=count,
               slice_mib=count * N * D * 8 / 2.0 ** 20,
               hist_1d_equal=bool(np.array_equal(d1[0], h1[0]) and np.array_equal(d1[1], h1[1])),
               hist_2d_equal=bool(np.array_equal(d2, h2)))
    for k, v in times.items():
        row[k + "_ms"] = 1e3 * float(np.median(v))
    b.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), rounds=a.rounds, rows=[])
    for shape in [(4096, 128, 500, 100, 5), (65536, 128, 64, 0, 1)]:
        res["rows"].append(case(*shape, rounds=a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    print(res["gpu"])
    for r in res["rows"]:
        print("%6d x %d  %3d steps  range %6.2f ms | 1-D: device %7.2f ms  host %9.1f ms | 2-D (16 params): device "
              "%7.2f ms  host %9.1f ms | all pairs: device %8.1f ms, bins=128 %8.1f ms | equal %s %s"
              % (r["N"], r["D"], r["slice_steps"], r["range_ms"], r["device_1d_ms"], r["host_1d_ms"],
                 r["device_2d_ms"], r["host_2d_ms"], r["device_all_pairs_ms"], r["device_all_pairs_bins128_ms"],
                 r["hist_1d_equal"],
                 r["hist_2d_equal"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_chain_histogram.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
