#!/usr/bin/env python
"""Cost of blobs on user log-probability functions: the same function with and without blobs_dtype.

  torch_16     65 536 x 128, torch CudaArrayFunction, 16-byte records (x[0], x[-1])
  torch_1024   65 536 x 128, torch CudaArrayFunction, 1 024-byte records (the whole row)
  host_16      4 096 x 128, HostFunction(vectorize=True) returning an [M, 1 + 2] array, 16-byte records

Each row runs with store=False and into a Backend at thin_by 1 and 10 (reset before every round).  Reported:
walker-steps/s from the host clock around run_mcmc (which ends in a stream synchronisation), the median of
--rounds rounds in which the arms alternate.  The card name and power limit are read in the same run.

    python scripts/bench_blobs.py [--rounds 3] [--out DIR]
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

SEED = 0xB10B


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def torch_fn(blob_cols):
    import torch

    def f(rows):
        x = torch.as_tensor(rows, device="cuda")
        lp = (x * x).sum(1) * -0.5
        if blob_cols is None:
            return lp
        if blob_cols == "row":
            return lp, x.clone()
        return lp, torch.stack([x[:, 0], x[:, -1]], dim=1)

    return f


def host_fn(blobs):
    def f(x):
        lp = -0.5 * np.einsum("ij,ij->i", x, x)
        return np.column_stack([lp, x[:, 0], x[:, -1]]) if blobs else lp

    return f


def arms(row):
    """(name, wrapper) pairs of one row: without and with blobs."""
    if row == "torch_16":
        return [("no blobs", models.CudaArrayFunction(torch_fn(None))),
                ("blobs 16 B", models.CudaArrayFunction(torch_fn("two"), blobs_dtype="f8"))]
    if row == "torch_1024":
        return [("no blobs", models.CudaArrayFunction(torch_fn(None))),
                ("blobs 1024 B", models.CudaArrayFunction(torch_fn("row"), blobs_dtype="f8"))]
    return [("no blobs", models.HostFunction(host_fn(False), vectorize=True)),
            ("blobs 16 B", models.HostFunction(host_fn(True), vectorize=True, blobs_dtype="f8"))]


STORES = [("store=False", dict(store=False)), ("Backend thin_by=1", dict(thin_by=1)),
          ("Backend thin_by=10", dict(thin_by=10))]


def run_row(row, N, D, steps, rounds):
    p0 = np.random.default_rng(1).standard_normal((N, D))
    samplers = [(name, emcee_b200.EnsembleSampler(N, D, fn, seed=SEED)) for name, fn in arms(row)]
    for _, s in samplers:  # warm-up: modules, tables, staging
        s.run_mcmc(p0, 2, store=False, skip_initial_state_check=True)
    out = []
    for store_name, kw in STORES:
        rates = {name: [] for name, _ in samplers}
        for _ in range(rounds):
            for name, s in samplers:  # alternated
                s.reset()
                n = steps // kw.get("thin_by", 1)
                t0 = time.perf_counter()
                s.run_mcmc(p0, n, skip_initial_state_check=True, **kw)
                wall = time.perf_counter() - t0
                rates[name].append(N * n * kw.get("thin_by", 1) / wall)
        for name, _ in samplers:
            r = dict(row=row, arm=name, store=store_name, N=N, D=D, steps=steps,
                     walker_steps_per_s=float(np.median(rates[name])), rounds=rates[name])
            print(json.dumps(r), flush=True)
            out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rows", default="torch_16,torch_1024,host_16")
    ap.add_argument("--out", default=None, help="directory for bench_blobs.json")
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_blobs: no CUDA device visible")
    head = dict(gpu=gpu_info())
    print(json.dumps(head), flush=True)
    rows = []
    for row in args.rows.split(","):
        if row.startswith("torch"):
            rows += run_row(row, 65536, 128, 20, args.rounds)
        else:
            rows += run_row(row, 4096, 128, 20, args.rounds)
    print("%-11s %-13s %-19s %16s" % ("row", "arm", "store", "walker-steps/s"))
    for r in rows:
        print("%-11s %-13s %-19s %16.4g" % (r["row"], r["arm"], r["store"], r["walker_steps_per_s"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_blobs.json"), "w") as f:
            json.dump(dict(head, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
