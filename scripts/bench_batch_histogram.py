#!/usr/bin/env python
"""Cost of a ``BatchSampler``'s per-ensemble histograms on the GPU (``DeviceBackend``) and with numpy (host
``Backend``).

K ensembles of 32 x 5, ``gauss_iso``, StretchMove, 2 000 stored steps; every call reads the slice ``discard=500``,
``thin=10`` (150 steps, 4 800 samples per ensemble):

  get_histogram(bins=20)          1-D, every parameter of every ensemble
  get_histogram2d(bins=20)        2-D, all 10 parameter pairs of every ensemble

each with autodetected ranges and with given ones (an array ``[K, 5, 2]``, each ensemble's 0.5 / 99.5 percentiles).
Host wall clock of each call, best of --repeat after one warm-up call; the device route is also split into its three
parts, each timed alone the same way: the range selection (``eb_chain_select_segments`` at ranks 0 and n - 1), the
host edges (``summary.uniform_edges`` / ``searched_edges`` of all columns at once) and the counting
(``eb_chain_histogram[2d]_segments``, which ends in a synchronise).  ``count_1step`` is the counting of a one-step
slice: the part of a count that does not grow with the rows (launch, per-CTA zeroing and flushing of the shared
bins, the memset and copy of the counts).  Every device result is compared with the numpy route's with ``==``.

The card name and power limit are read in the same run.

    python scripts/bench_batch_histogram.py [--K 16 256 1024 4096] [--repeat 3] [--out DIR]
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
from emcee_b200.summary import searched_edges, uniform_edges  # noqa: E402

N, D, STEPS, DISCARD, THIN, BINS = 32, 5, 2000, 500, 10, 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def best_ms(fn, repeat, warm=True):
    if warm:
        fn()
    best = float("inf")
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return 1e3 * best


def same(a, b):
    return all(x == y if isinstance(y, list) else (x.dtype == y.dtype and np.array_equal(x, y)) for x, y in zip(a, b))


def parts(s, given, repeat):
    """the device route's selection, edges and counting, each timed alone"""
    K = s.nbatch
    ch, (first, stride, count) = s.backend._plan(DISCARD, THIN)
    n = count * N
    ranks = np.array([0, n - 1], dtype=np.uint64)
    out = {}
    if given is None:
        out["select_ms"] = best_ms(lambda: ch.select("chain", first, stride, count, ranks, nseg=K), repeat)
        stats, has_nan, _ = ch.select("chain", first, stride, count, ranks, nseg=K)
        lo, hi, nan = stats[:, 0].ravel(), stats[:, 1].ravel(), has_nan.ravel()
        ranges = None
    else:
        out["select_ms"] = 0.0
        lo = hi = np.full(K * D, np.nan)
        nan = np.zeros(K * D, dtype=bool)
        ranges = given.reshape(K * D, 2)
    out["edges_1d_ms"] = best_ms(lambda: uniform_edges(BINS, ranges, lo, hi, nan), repeat)
    out["edges_2d_ms"] = best_ms(lambda: searched_edges(BINS, ranges, lo, hi, nan), repeat)
    outer, edges = uniform_edges(BINS, ranges, lo, hi, nan)
    edges2 = searched_edges(BINS, ranges, lo, hi, nan)
    params = list(range(D))
    out["count_1d_ms"] = best_ms(lambda: ch.histogram("chain", first, stride, count, BINS, outer, edges, nseg=K),
                                 repeat)
    out["count_2d_ms"] = best_ms(lambda: ch.histogram2d(first, stride, count, params, BINS, edges2, nseg=K), repeat)
    out["count_1d_1step_ms"] = best_ms(lambda: ch.histogram("chain", first, stride, 1, BINS, outer, edges, nseg=K),
                                       repeat)
    out["count_2d_1step_ms"] = best_ms(lambda: ch.histogram2d(first, stride, 1, params, BINS, edges2, nseg=K),
                                       repeat)
    return out


def run(K, repeat):
    runs = {}
    p0 = np.random.default_rng(1).normal(size=(K, N, D))
    for store in ("device", "host"):
        s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1,
                                    backend=DeviceBackend() if store == "device" else None)
        s.run_mcmc(p0, STEPS, skip_initial_state_check=True)
        runs[store] = s
    dev, host = runs["device"], runs["host"]
    given = np.moveaxis(host.get_percentile([0.5, 99.5], discard=DISCARD, thin=THIN), 1, 2).copy()
    rows = []
    for rname, rng in (("auto", None), ("given", given)):
        for call in ("get_histogram", "get_histogram2d"):
            fn = lambda s: getattr(s, call)(bins=BINS, range=rng, discard=DISCARD, thin=THIN)
            row = {"K": K, "call": call, "range": rname,
                   "device_ms": best_ms(lambda: fn(dev), repeat),
                   "numpy_ms": best_ms(lambda: fn(host), repeat, warm=False),
                   "equal": bool(same(fn(dev), fn(host)))}
            rows.append(row)
            print("call", json.dumps(row), flush=True)
        row = dict(K=K, range=rname, **parts(dev, None if rng is None else given, repeat))
        rows.append(row)
        print("parts", json.dumps(row), flush=True)
    dev.backend.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, nargs="+", default=[16, 256, 1024, 4096])
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "shape": [N, D], "stored_steps": STEPS, "discard": DISCARD, "thin": THIN, "bins": BINS,
           "rows": []}
    print("gpu", res["gpu"], flush=True)
    for K in a.K:
        res["rows"] += run(K, a.repeat)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_batch_histogram.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
