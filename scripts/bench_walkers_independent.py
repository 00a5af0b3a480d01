#!/usr/bin/env python
"""Time of the initial-state independence check, ``EnsembleSampler._walkers_independent``, before and after the
host applies the reference's first statements (finite test, numpy's centring, zero-span test, power-of-two column
scaling) ahead of the device Gram matrix.

  before  the raw coordinates straight to ``eb_walkers_gram``, then the D x D eigen-solve (the former path)
  after   ``_walkers_independent`` as it is now
  centring  the host part alone (finite test, mean, span, ldexp)

Well-conditioned 4 096 x 128 and 65 536 x 128 ensembles, where both paths decide on the device.  The arms
alternate for --rounds rounds of --reps calls each; medians of the host clock per call are reported (every call
ends in a stream synchronisation inside ``eb_walkers_gram``).  The card name and power limit are read in the
same run.

    python scripts/bench_walkers_independent.py [--rounds 5] [--reps 20] [--out DIR]
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


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def before(s, x):
    gram, flags = s._engine.walkers_gram(x)
    if flags:
        return False
    ev = np.linalg.eigvalsh(gram)
    return bool(ev[0] > 0 and np.sqrt(ev[-1] / ev[0]) <= 1e6)


def centring(x):
    if not np.all(np.isfinite(x)):
        return None
    c = x - np.mean(x, axis=0)[None, :]
    span = np.amax(np.abs(c), axis=0)
    return np.ldexp(c, -np.frexp(span)[1][None, :])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for bench_walkers_independent.json")
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_walkers_independent: no CUDA device visible")
    head = dict(gpu=gpu_info())
    print(json.dumps(head), flush=True)
    rows = []
    for N, D in ((4096, 128), (65536, 128)):
        x = 3.0 + np.random.default_rng(N).standard_normal((N, D))
        s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=1)
        arms = dict(before=lambda: before(s, x), after=lambda: s._walkers_independent(x),
                    centring=lambda: centring(x))
        assert arms["before"]() and arms["after"]()  # warm-up; both decide True on the device
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    fn()
                times[k].append((time.perf_counter() - t0) / args.reps)
        r = dict(N=N, D=D, **{k + "_ms": 1e3 * float(np.median(v)) for k, v in times.items()})
        rows.append(r)
        print(json.dumps(r), flush=True)
    print("%-12s %12s %12s %12s" % ("N x D", "before ms", "after ms", "centring ms"))
    for r in rows:
        print("%-12s %12.3f %12.3f %12.3f" % ("%dx%d" % (r["N"], r["D"]), r["before_ms"], r["after_ms"],
                                             r["centring_ms"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_walkers_independent.json"), "w") as f:
            json.dump(dict(head, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
