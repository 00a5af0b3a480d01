#!/usr/bin/env python
"""Throughput of a torch log-probability run as captured CUDA graphs (models.CudaGraphFunction) against the same
function called back per half-step (models.CudaArrayFunction) and, where one exists, the fused registered model:

  iso      32 x 5 isotropic Gaussian       (fused: GaussianIso)
  ring     256 x 32 ring                   (fused: Ring)
  dense4k  4 096 x 128 dense Gaussian      (fused: GaussianDense)
  dense64k 65 536 x 128 dense Gaussian     (fused: GaussianDense)
  iso_devstore  32 x 5 isotropic Gaussian into a DeviceBackend, thin_by=1: every step stored, so the graph arm
                reads the error state once per step

Stretch move.  Walker-steps/s from the host clock around run_mcmc(store=False) (run_mcmc ends in a stream
synchronisation); the median of 3 rounds after a warm-up, the arms of a row alternating within each round.  The card
name and power limit are read in the same run.

    python scripts/bench_graph_function.py [--rounds 3] [--out DIR]
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

import torch  # noqa: E402

import emcee_b200  # noqa: E402
from emcee_b200 import models  # noqa: E402
from oracle import targets as T  # noqa: E402

SEED = 0x6F


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def capture_of(f, ndim):
    """The torch recipe of CudaGraphFunction's docstring."""

    def capture(m):
        x = torch.zeros(m, ndim, dtype=torch.float64, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                f(x)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            lp = f(x)
        return models.CapturedGraph(g.raw_cuda_graph_exec(), x, lp, owner=g)

    return capture


def iso(x):
    return -0.5 * (x * x).sum(-1)


def ring_of(radius, sigma):
    def ring(x):
        d = torch.sqrt((x * x).sum(-1)) - radius
        return -(d * d) / (2.0 * sigma * sigma)

    return ring


def dense_of(t):
    icov = torch.as_tensor(t.icov, device="cuda")
    mean = torch.as_tensor(t.mean, device="cuda")

    def dense(x):
        d = x - mean
        return -0.5 * ((d @ icov) * d).sum(-1)

    return dense


def rows():
    t64 = T.GaussDense(np.linalg.inv(T.random_cov(128, rng=np.random.default_rng(1))))
    yield "iso", 32, 5, iso, models.GaussianIso(), 2000, False
    yield "ring", 256, 32, ring_of(5.0, 0.5), models.Ring(5.0, 0.5), 1000, False
    yield "dense4k", 4096, 128, dense_of(t64), models.GaussianDense(t64.icov), 200, False
    yield "dense64k", 65536, 128, dense_of(t64), models.GaussianDense(t64.icov), 40, False
    yield "iso_devstore", 32, 5, iso, None, 2000, True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for bench_graph_function.json")
    args = ap.parse_args()
    head = dict(bench="graph_function", gpu=gpu_info(), torch=torch.__version__)
    print(json.dumps(head), flush=True)
    results = []
    for name, N, D, f, fused, steps, devstore in rows():
        p0 = np.random.default_rng(2).standard_normal((N, D))
        if name == "ring":
            p0 = p0 / np.linalg.norm(p0, axis=1, keepdims=True) * 5.0 + 0.1 * p0
        arms = {
            "array": models.CudaArrayFunction(lambda r, f=f: f(torch.as_tensor(r, device="cuda"))),
            "graph": models.CudaGraphFunction(capture_of(f, D)),
        }
        if fused is not None:
            arms["fused"] = fused
        samplers = {}
        for arm, fn in arms.items():
            kw = {"backend": emcee_b200.DeviceBackend()} if devstore else {}
            s = emcee_b200.EnsembleSampler(N, D, fn, seed=SEED, **kw)
            s.run_mcmc(p0, 4, store=devstore, skip_initial_state_check=True)  # warm-up
            samplers[arm] = s
        runs = {arm: [] for arm in samplers}
        for _ in range(args.rounds):
            for arm, s in samplers.items():
                if devstore:
                    s.reset()
                t0 = time.perf_counter()
                s.run_mcmc(p0, steps, store=devstore, skip_initial_state_check=True)
                wall = time.perf_counter() - t0
                runs[arm].append(N * steps / wall)
        for arm, r in runs.items():
            row = dict(row=name, arm=arm, N=N, D=D, steps=steps, store=("DeviceBackend" if devstore else False),
                       walker_steps_per_s=float(np.median(r)), rounds=[float(v) for v in r])
            print(json.dumps(row), flush=True)
            results.append(row)
        del samplers
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_graph_function.json"), "w") as fh:
            json.dump(dict(head, rows=results), fh, indent=1)


if __name__ == "__main__":
    main()
