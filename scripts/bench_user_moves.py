#!/usr/bin/env python
"""Throughput of user-written proposals (RedBlueMove subclasses overriding get_proposal), each row against its
natural baseline:

  iso_numpy    32 x 5 isotropic Gaussian device model, a numpy stretch move -- the reference with the same move
               class and the numpy target (serial map)
  dense_numpy  4 096 x 128 dense Gaussian device model, the same numpy move -- the reference with vectorize=True,
               the same move class and the numpy target of oracle/targets.py
  dense_torch  65 536 x 128 dense Gaussian device model, a torch CudaArrayRedBlueMove -- the built-in StretchMove

store=False.  Each arm runs once to warm up, then the arms of a row alternate for --rounds rounds and the medians
are reported: walker-steps/s from the host clock around run_mcmc (which ends in a stream synchronisation), and
the share of that time spent inside get_proposal.  The card name and power limit are read in the same run.  The
reference arms need oracle/_ref/emcee_reference.zip (built by __graft_entry__.build() when a checkout of the
reference exists) and are skipped without it.

    python scripts/bench_user_moves.py [--rounds 3] [--out DIR]
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
SEED = 0xB7


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers below are still measurements; say what is missing
        return "nvidia-smi unavailable (%s)" % e


def reference():
    if not os.path.exists(REF_ZIP):
        return None
    if REF_ZIP not in sys.path:
        sys.path.insert(0, REF_ZIP)
    import emcee

    assert REF_ZIP in emcee.__file__, emcee.__file__
    return emcee


def stretch_proposal(s, c, random, a=2.0):
    """stretch.py:26-33, written the way a user would."""
    c = np.concatenate(c, axis=0)
    ns, nc = len(s), len(c)
    zz = ((a - 1.0) * random.rand(ns) + 1) ** 2.0 / a
    factors = (s.shape[1] - 1.0) * np.log(zz)
    rint = random.randint(nc, size=(ns,))
    return c[rint] - (c[rint] - s) * zz[:, None], factors


def torch_stretch(s, c, random, a=2.0):
    import torch

    S = torch.as_tensor(s, device="cuda")
    C = torch.cat([torch.as_tensor(x, device="cuda") for x in c])
    gen = torch.Generator(device="cuda").manual_seed(int(random.randint(2**62)))
    u = torch.rand(S.shape[0], device="cuda", dtype=torch.float64, generator=gen)
    zz = ((a - 1.0) * u + 1) ** 2 / a
    rint = torch.randint(C.shape[0], (S.shape[0],), device="cuda", generator=gen)
    cr = C[rint]
    return cr - (cr - S) * zz[:, None], (S.shape[1] - 1.0) * torch.log(zz)


class Clock(object):
    seconds = 0.0


def timed_move(base, fn, clock):
    class Timed(base):
        def get_proposal(self, s, c, random):
            t0 = time.perf_counter()
            try:
                return fn(s, c, random)
            finally:
                clock.seconds += time.perf_counter() - t0

    return Timed()


class Arm(object):
    def __init__(self, name, run, clock=None):
        self.name, self.run, self.clock, self.out = name, run, clock, []

    def once(self, N, steps):
        if self.clock is not None:
            self.clock.seconds = 0.0
        t0 = time.perf_counter()
        self.run(steps)
        wall = time.perf_counter() - t0
        self.out.append((N * steps / wall, None if self.clock is None else self.clock.seconds / wall))


def b200_arm(name, N, D, model, p0, move, clock):
    s = emcee_b200.EnsembleSampler(N, D, model, moves=move, seed=SEED)
    return Arm(name, lambda steps: s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True), clock)


def reference_arm(emcee, name, N, D, target, p0, vectorize):
    clock = Clock()
    move = timed_move(emcee.moves.RedBlueMove, stretch_proposal, clock)
    fn = target if vectorize else (lambda x: float(target(x[None, :])[0]))

    def run(steps):
        np.random.seed(SEED)
        s = emcee.EnsembleSampler(N, D, fn, moves=move, vectorize=vectorize)
        s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)

    return Arm(name, run, clock)


def row(name, arms, N, D, steps, rounds):
    for a in arms:
        a.run(min(steps, 2))  # warm-up: modules, tables, staging
    for _ in range(rounds):
        for a in arms:
            a.once(N, steps)
    out = []
    for a in arms:
        share = [s for _, s in a.out if s is not None]
        out.append(dict(row=name, arm=a.name, N=N, D=D, steps=steps,
                        walker_steps_per_s=float(np.median([r for r, _ in a.out])),
                        proposal_share=float(np.median(share)) if share else None))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rows", default="iso_numpy,dense_numpy,dense_torch")
    ap.add_argument("--out", default=None, help="directory for bench_user_moves.json")
    args = ap.parse_args()
    if emcee_b200._lib.device_count() < 1:
        raise SystemExit("bench_user_moves: no CUDA device visible")
    head = dict(gpu=gpu_info())
    print(json.dumps(head), flush=True)
    emcee = reference()
    want = args.rows.split(",")
    rows = []
    for name, kind, N, D, steps in (("iso_numpy", "gauss_iso", 32, 5, 2000),
                                    ("dense_numpy", "gauss_dense", 4096, 128, 20)):
        if name not in want:
            continue
        t, p0 = T.make_config(kind, N, D)
        model = models.GaussianIso() if kind == "gauss_iso" else models.GaussianDense(t.icov, t.mean)
        clock = Clock()
        arms = [b200_arm("numpy move, device model", N, D, model, p0,
                         timed_move(moves.RedBlueMove, stretch_proposal, clock), clock)]
        if emcee is not None:
            arms.append(reference_arm(emcee, "reference, same move", N, D, t, p0, kind != "gauss_iso"))
        rows += row(name, arms, N, D, steps, args.rounds)
    if "dense_torch" in want:
        N, D, steps = 65536, 128, 50
        t, p0 = T.make_config("gauss_dense", N, D)
        model = models.GaussianDense(t.icov, t.mean)
        clock = Clock()
        arms = [b200_arm("torch move, device model", N, D, model, p0,
                         timed_move(moves.CudaArrayRedBlueMove, torch_stretch, clock), clock),
                b200_arm("built-in StretchMove", N, D, model, p0, moves.StretchMove(), None)]
        rows += row("dense_torch", arms, N, D, steps, args.rounds)
    for r in rows:
        print(json.dumps(r), flush=True)
    print("%-12s %-28s %16s %10s" % ("row", "arm", "walker-steps/s", "proposal"))
    for r in rows:
        share = "-" if r["proposal_share"] is None else "%.0f%%" % (100 * r["proposal_share"])
        print("%-12s %-28s %16.4g %10s" % (r["row"], r["arm"], r["walker_steps_per_s"], share))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_user_moves.json"), "w") as f:
            json.dump(dict(head, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
