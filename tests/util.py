"""Shared helpers: load a golden case and rebuild it on the oracle."""
import glob
import os

import numpy as np

from oracle import redblue as rb
from oracle import targets as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def oracle_target(g):
    kind = str(g["model_kind"])
    d = int(g["ndim"])
    if kind == "gauss_iso":
        return T.GaussIso(d)
    if kind == "gauss_dense":
        return T.GaussDense(g["model_icov"], g["model_mean"])
    if kind == "rosenbrock":
        return T.Rosenbrock(d, *g["model_params"])
    if kind == "ring":
        return T.Ring(d, *g["model_params"])
    raise ValueError(kind)


GAUSS_MODES = ("vector", "random", "sequential")


def oracle_moves(g):
    out = []
    for k, (kind, w, nsplits, rand, p0, p1) in enumerate(g["moves"]):
        kw = dict(nsplits=int(nsplits), randomize_split=bool(rand), live_dangerously=bool(g.get("live_dangerously", False)))
        if kind == 0:
            m = rb.Stretch(a=p0, **kw)
        elif kind == 1:
            m = rb.DE(sigma=p0, gamma0=None if np.isnan(p1) else p1, **kw)
        elif kind == 2:
            m = rb.Snooker(gammas=p0, **kw)
        elif kind == 3:
            m = rb.Walk(s=None if np.isnan(p0) else int(p0), **kw)
        else:
            cov = g["move%d_cov" % k]
            m = rb.Gaussian(cov if cov.ndim else float(cov), GAUSS_MODES[int(p0)], None if np.isnan(p1) else float(p1))
        out.append((m, w))
    return out


def oracle_sampler(g):
    s = rb.OracleSampler(
        int(g["nwalkers"]), int(g["ndim"]), oracle_target(g), oracle_moves(g), seed=int(g["seed"])
    )
    s.set_state(g["p0"])
    return s
