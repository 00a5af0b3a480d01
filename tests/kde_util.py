"""KDEMove golden cases (``oracle/gen_golden_kde.py``): load one, rebuild it on the oracle or on the engine."""
import glob
import os

import numpy as np

from oracle import kde as ok
from oracle import redblue as rb
from oracle.bounded import Bounded
from util import GOLDEN, oracle_target

KDE_GOLDEN = os.path.join(GOLDEN, "kde")


def kde_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(KDE_GOLDEN, "*.npz")))


def load_kde(name):
    return dict(np.load(os.path.join(KDE_GOLDEN, name + ".npz")))


def bw_method(p0, p1):
    """The ``bw_method`` a move row encodes (``include/emcee_b200.h``: p0 NaN Scott, 1 Silverman, 2 scalar p1)."""
    if np.isnan(p0):
        return None
    return "silverman" if p0 == 1.0 else float(p1)


def kde_oracle(g):
    target = oracle_target(g)
    if "model_lower" in g:
        target = Bounded(target, g["model_lower"], g["model_upper"])
    moves = []
    for kind, w, nsplits, rand, p0, p1 in g["moves"]:
        kw = dict(nsplits=int(nsplits), randomize_split=bool(rand))
        moves.append((rb.Stretch(a=p0, **kw) if kind == 0 else ok.KDE(bw_method(p0, p1), **kw), w))
    s = ok.KdeOracleSampler(int(g["nwalkers"]), int(g["ndim"]), target, moves, seed=int(g["seed"]))
    with np.errstate(invalid="ignore"):
        s.set_state(g["p0"])
    return s


def kde_sampler(g, **kw):
    """The engine's sampler of a golden case (needs the built package, not a GPU)."""
    import emcee_b200
    from emcee_b200 import models, moves
    from gpu_util import device_model

    model = device_model(str(g["model_kind"]), g=g)
    if "model_lower" in g:
        model = models.Bounded(model, g["model_lower"], g["model_upper"])
    mv = []
    for kind, w, nsplits, rand, p0, p1 in g["moves"]:
        k = dict(nsplits=int(nsplits), randomize_split=bool(rand))
        mv.append((moves.StretchMove(a=p0, **k) if kind == 0 else moves.KDEMove(bw_method(p0, p1), **k), w))
    return emcee_b200.EnsembleSampler(int(g["nwalkers"]), int(g["ndim"]), model, moves=mv, seed=int(g["seed"]), **kw)
