"""Build the CUDA-side sampler for a golden case / an oracle configuration."""
import numpy as np

import emcee_b200
from emcee_b200 import models, moves


def device_model(kind, g=None, target=None):
    if kind == "gauss_iso":
        return models.GaussianIso()
    if kind == "gauss_dense":
        if g is not None:
            return models.GaussianDense(g["model_icov"], g["model_mean"])
        return models.GaussianDense(target.icov, target.mean)
    if kind == "rosenbrock":
        p = g["model_params"] if g is not None else (target.a, target.b)
        return models.Rosenbrock(*p)
    if kind == "ring":
        p = g["model_params"] if g is not None else (target.radius, target.sigma)
        return models.Ring(*p)
    raise ValueError(kind)


GAUSS_MODES = ("vector", "random", "sequential")


def device_moves(rows, g=None):
    out = []
    for k, (kind, w, nsplits, rand, p0, p1) in enumerate(rows):
        kw = dict(randomize_split=bool(rand))
        if g is not None and g.get("live_dangerously", False):
            kw["live_dangerously"] = True
        if kind == 0:
            m = moves.StretchMove(a=p0, nsplits=int(nsplits), **kw)
        elif kind == 1:
            m = moves.DEMove(sigma=p0, gamma0=None if np.isnan(p1) else p1, nsplits=int(nsplits), **kw)
        elif kind == 2:
            m = moves.DESnookerMove(gammas=p0, **kw)
        elif kind == 3:
            m = moves.WalkMove(s=None if np.isnan(p0) else int(p0), nsplits=int(nsplits), **kw)
        else:
            cov = g["move%d_cov" % k]
            m = moves.GaussianMove(cov if cov.ndim else float(cov), mode=GAUSS_MODES[int(p0)],
                                   factor=None if np.isnan(p1) else float(p1))
        out.append((m, w))
    return out


def single_step_tol(g):
    """Tolerance of one step of a golden case from the reference's previous state.  A whole-complement WalkMove
    whose complement has at most ndim walkers factors a rank-deficient covariance shared by the whole split: the
    trailing pivots of its Cholesky factor are rounding noise of the null space, so its proposals agree to the
    free-running Walk tolerance only."""
    kinds = set(g["moves"][:, 0].astype(int))
    if not kinds & {3, 4}:
        return 1e-12
    N, D = int(g["nwalkers"]), int(g["ndim"])
    for kind, _, P, _, s, _ in g["moves"]:
        if kind == 3 and np.isnan(s) and N - (N + int(P) - 1) // int(P) <= D:
            return 1e-9
    return 1e-11


def golden_sampler(g):
    return emcee_b200.EnsembleSampler(
        int(g["nwalkers"]), int(g["ndim"]), device_model(str(g["model_kind"]), g=g),
        moves=device_moves(g["moves"], g), seed=int(g["seed"]),
    )


def move_rows_from_oracle(oracle_moves):
    rows = []
    for m, w in oracle_moves:
        if m.kind == "stretch":
            rows.append([0, w, m.nsplits, m.randomize_split, m.a, np.nan])
        elif m.kind == "de":
            rows.append([1, w, m.nsplits, m.randomize_split, m.sigma, np.nan if m.gamma0 is None else m.gamma0])
        elif m.kind == "walk":
            rows.append([3, w, m.nsplits, m.randomize_split, np.nan if m.s is None else m.s, np.nan])
        else:
            rows.append([2, w, m.nsplits, m.randomize_split, m.gammas, np.nan])
    return np.array(rows, dtype=np.float64)
