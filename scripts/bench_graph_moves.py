#!/usr/bin/env python
"""Throughput of a torch stretch move run as a captured proposal (moves.CudaGraphRedBlueMove) against the same move
called back per half-step (moves.CudaArrayRedBlueMove) and the built-in StretchMove, on registered device models:

  iso      32 x 5 isotropic Gaussian       (GaussianIso)
  ring     256 x 32 ring                   (Ring)
  dense4k  4 096 x 128 dense Gaussian      (GaussianDense)
  dense64k 65 536 x 128 dense Gaussian     (GaussianDense)

The callback arm draws from a torch generator seeded from its `random`; the captured arm takes two uniform draws per
row from the engine.  Walker-steps/s from the host clock around run_mcmc(store=False) (run_mcmc ends in a stream
synchronisation); the median of 3 rounds after a warm-up, the arms of a row alternating within each round.  The card
name and power limit are read in the same run.

    python scripts/bench_graph_moves.py [--rounds 3] [--out DIR]
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
from emcee_b200 import models, moves  # noqa: E402
from oracle import targets as T  # noqa: E402

SEED = 0x6F


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def stretch(s, c, u, a=2.0):
    """The stretch proposal of stretch.py:30-35 from two uniforms per row."""
    zz = ((a - 1.0) * u[:, 0] + 1.0) ** 2 / a
    idx = torch.clamp((u[:, 1] * c.shape[0]).long(), max=c.shape[0] - 1)
    cr = c[idx]
    return cr - (cr - s) * zz[:, None], (s.shape[1] - 1.0) * torch.log(zz)


class ArrayStretch(moves.CudaArrayRedBlueMove):
    def get_proposal(self, s, c, random):
        S = torch.as_tensor(s, device="cuda")
        C = torch.cat([torch.as_tensor(x, device="cuda") for x in c])
        gen = torch.Generator(device="cuda").manual_seed(int(random.randint(2**62)))
        u = torch.rand((S.shape[0], 2), dtype=torch.float64, device="cuda", generator=gen)
        return stretch(S, C, u)


def capture_of(N, D):
    def capture(ns, counts):
        s = torch.zeros(ns, D, dtype=torch.float64, device="cuda")
        c = torch.zeros(N - ns, D, dtype=torch.float64, device="cuda")
        d = torch.full((ns, 2), 0.5, dtype=torch.float64, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                stretch(s, c, d)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            q, f = stretch(s, c, d)
        return moves.CapturedProposal(g.raw_cuda_graph_exec(), s, c, d, q, f, owner=g)

    return capture


def rows():
    t64 = T.GaussDense(np.linalg.inv(T.random_cov(128, rng=np.random.default_rng(1))))
    yield "iso", 32, 5, models.GaussianIso, 2000
    yield "ring", 256, 32, lambda: models.Ring(5.0, 0.5), 1000
    yield "dense4k", 4096, 128, lambda: models.GaussianDense(t64.icov), 200
    yield "dense64k", 65536, 128, lambda: models.GaussianDense(t64.icov), 40


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for bench_graph_moves.json")
    args = ap.parse_args()
    head = dict(bench="graph_moves", gpu=gpu_info(), torch=torch.__version__)
    print(json.dumps(head), flush=True)
    results = []
    for name, N, D, model, steps in rows():
        p0 = np.random.default_rng(2).standard_normal((N, D))
        if name == "ring":
            p0 = p0 / np.linalg.norm(p0, axis=1, keepdims=True) * 5.0 + 0.1 * p0
        arms = {
            "builtin": lambda: moves.StretchMove(),
            "array": lambda: ArrayStretch(),
            "graph": lambda N=N, D=D: moves.CudaGraphRedBlueMove(capture_of(N, D), ndraws=2),
        }
        samplers = {}
        for arm, mv in arms.items():
            s = emcee_b200.EnsembleSampler(N, D, model(), moves=mv(), seed=SEED)
            s.run_mcmc(p0, 4, store=False, skip_initial_state_check=True)  # warm-up
            samplers[arm] = s
        runs = {arm: [] for arm in samplers}
        for _ in range(args.rounds):
            for arm, s in samplers.items():
                t0 = time.perf_counter()
                s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
                wall = time.perf_counter() - t0
                runs[arm].append(N * steps / wall)
        for arm, r in runs.items():
            row = dict(row=name, arm=arm, N=N, D=D, steps=steps, walker_steps_per_s=float(np.median(r)),
                       rounds=[float(v) for v in r])
            print(json.dumps(row), flush=True)
            results.append(row)
        del samplers
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_graph_moves.json"), "w") as fh:
            json.dump(dict(head, rows=results), fh, indent=1)


if __name__ == "__main__":
    main()
