#!/usr/bin/env python
"""Time of the summaries of a stored device chain against the download-then-numpy route:

  device   ``DeviceBackend.get_percentile([16, 50, 84])`` (``eb_chain_select``) and ``get_moments()``
           (``eb_chain_moments``), each on its own
  host     ``get_chain(flat=True)`` (a pageable download of the slice) followed by ``np.percentile`` /
           ``np.mean`` + ``np.cov``

Cases: 4 096 x 128 with 500 stored steps read with ``discard=100, thin=5``, and 65 536 x 128 with 64 stored steps.
The arms alternate for --rounds rounds; medians of the host clock per call are reported (every call returns host
arrays, so it ends in a stream synchronisation).  ``passes`` is the number of full reads of the slice the
selection made.  The card name and power limit are read in the same run.

    python scripts/bench_chain_summary.py [--rounds 5] [--out DIR]
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
from emcee_b200.summary import percentile_ranks  # noqa: E402

Q = [16, 50, 84]


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

    def host_pct():
        return np.percentile(b.get_chain(flat=True, **kw), Q, axis=0)

    def host_mom():
        flat = b.get_chain(flat=True, **kw)
        return np.mean(flat, axis=0), np.cov(flat, rowvar=False)

    arms = {"device_percentile": lambda: b.get_percentile(Q, **kw), "host_percentile": host_pct,
            "device_moments": lambda: b.get_moments(**kw), "host_moments": host_mom}
    for fn in arms.values():  # warm every arm once
        fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn)[0])
    pd, ph = b.get_percentile(Q, **kw), host_pct()
    (md, cd, _), (mh, ch) = b.get_moments(**kw), host_mom()
    first, stride, count = emcee_b200.backend.slice_plan(b.iteration, discard, thin)
    plan = percentile_ranks(Q, count * N)
    _, _, passes = b._chain.select("chain", first, stride, count, plan.ranks)
    row = dict(N=N, D=D, stored=steps, discard=discard, thin=thin, slice_steps=count,
               slice_mib=count * N * D * 8 / 2.0 ** 20, passes=passes,
               percentile_equal=bool(np.array_equal(pd, ph)),
               moments_max_rel=float(max(np.max(np.abs(md - mh) / np.maximum(np.abs(mh), 1e-300)),
                                         np.max(np.abs(cd - ch)) / np.max(np.abs(ch)))))
    for k, v in times.items():
        row[k + "_ms"] = 1e3 * float(np.median(v))
    b.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=gpu_info(), rounds=a.rounds, rows=[])
    for shape in [(4096, 128, 500, 100, 5), (65536, 128, 64, 0, 1)]:
        res["rows"].append(case(*shape, rounds=a.rounds))
        print(json.dumps(res["rows"][-1]), flush=True)
    print(res["gpu"])
    for r in res["rows"]:
        print("%6d x %d  %3d steps  passes %d  percentile: device %8.2f ms  host %9.1f ms | moments: device %7.2f ms"
              "  host %9.1f ms" % (r["N"], r["D"], r["slice_steps"], r["passes"], r["device_percentile_ms"],
                                    r["host_percentile_ms"], r["device_moments_ms"], r["host_moments_ms"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_chain_summary.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
