#!/usr/bin/env python
"""Generate ``tests/golden/kde/*.npz`` from the UNMODIFIED reference's ``KDEMove`` (TEST INFRASTRUCTURE).

    python -m oracle.gen_golden_kde          # needs oracle/_ref/emcee_reference.zip (make_ref.py) and scipy

Each case runs the reference's ``EnsembleSampler`` with its own ``moves.KDEMove`` (``kde.py:39-43``: scipy's
``gaussian_kde``, ``resample`` and ``logpdf``).  ``resample`` passes its ``random`` through scipy's
``check_random_state``, which takes only a ``RandomState`` or a ``Generator``; ``oracle.kde.KdePhilox`` is therefore
the shim ``oracle.philox.PhiloxRandom`` with ``resample``'s two draws and a ``RandomState`` at once, and every method
the reference calls is the shim's.
The arrays are those of ``oracle/gen_golden.py`` (``moves`` rows: kind 7 = KDE with ``p0`` / ``p1`` as
``include/emcee_b200.h`` encodes the bandwidth, kind 0 = stretch) plus ``trace_kde_choice`` (the complement rank of
each proposal's kernel centre, first three steps) and, for a bounded model, ``model_lower`` / ``model_upper``."""
import os
import sys

import numpy as np

from . import gen_golden as gg
from . import targets as T
from .bounded import Bounded
from .gen_golden_user_moves import import_reference
from .kde import KdePhilox

OUT = os.path.join(gg.OUT, "kde")
SEED0 = 0x656D636565B2C0  # distinct from the other generators' seeds


def case_list(emcee):
    mv = emcee.moves
    rng = np.random.default_rng(5151)
    d6 = T.make_config("gauss_dense", 64, 6)[0]
    box = Bounded(T.GaussIso(4), -1.5, [1.5, 1.5, 1.5, np.inf])
    p_box = np.clip(rng.standard_normal((64, 4)), -1.4, 1.4)
    return [
        # name, nwalkers, ndim, target, moves, p0, nsteps
        ("kde_scott_iso_64x4", 64, 4, T.GaussIso(4), mv.KDEMove(), rng.standard_normal((64, 4)), 30),
        ("kde_silverman_nsplits3_ring_97x6", 97, 6, T.Ring(6), mv.KDEMove(bw_method="silverman", nsplits=3),
         2.5 * rng.standard_normal((97, 6)), 25),
        ("kde_scalar_rosen_48x4", 48, 4, T.Rosenbrock(4), mv.KDEMove(bw_method=0.3),
         1.0 + 0.1 * rng.standard_normal((48, 4)), 30),
        ("kde_stretch_mix_dense_64x6", 64, 6, d6, [(mv.KDEMove(), 0.5), (mv.StretchMove(), 0.5)],
         rng.standard_normal((64, 6)), 30),
        ("kde_bounded_iso_64x4", 64, 4, box, mv.KDEMove(), p_box, 30),
        ("kde_fixedsplit_iso_40x3", 40, 3, T.GaussIso(3), mv.KDEMove(randomize_split=False),
         rng.standard_normal((40, 3)), 30),
    ]


def describe_moves(moves):
    if not isinstance(moves, list):
        moves = [(moves, 1.0)]
    rows = []
    for m, w in moves:
        if type(m).__name__ == "StretchMove":
            rows.append([0, w, m.nsplits, m.randomize_split, m.a, np.nan])
            continue
        assert type(m).__name__ == "KDEMove"
        bw = m.bw_method
        p0, p1 = (np.nan, np.nan) if bw in (None, "scott") else (1.0, np.nan) if bw == "silverman" else (2.0, bw)
        rows.append([7, w, m.nsplits, m.randomize_split, p0, p1])
    return np.array(rows, dtype=np.float64)


def model_arrays(target):
    if isinstance(target, Bounded):
        out = gg.model_arrays(target.target)
        out["model_lower"] = target.lower
        out["model_upper"] = target.upper
        return out
    return gg.model_arrays(target)


def run_case(emcee, name, nwalkers, ndim, target, moves, p0, nsteps, seed):
    sampler = emcee.EnsembleSampler(nwalkers, ndim, target, moves=moves, vectorize=True)
    shim = KdePhilox(seed)
    shim.trace = []
    sampler._random = shim  # ensemble.py:166
    acc = np.empty((nsteps, nwalkers), dtype=bool)
    prev = np.zeros(nwalkers)
    k = 0
    with np.errstate(invalid="ignore"):
        for _ in sampler.sample(p0, iterations=nsteps, skip_initial_state_check=True):
            now = sampler.backend.accepted.copy()
            acc[k] = (now - prev) > 0.5
            prev = now
            k += 1
        lp0 = np.asarray(target(p0), dtype=np.float64)
    choice = [p for kind, step, _, p in shim.trace if kind == "kde_choice" and step < 3]
    arrays = dict(nwalkers=np.array(nwalkers), ndim=np.array(ndim), seed=np.array(seed, dtype=np.uint64),
                  moves=describe_moves(moves), p0=p0, lp0=lp0, chain=sampler.get_chain(),
                  log_prob=sampler.get_log_prob(), accepted=acc,
                  trace_kde_choice=np.concatenate(choice) if choice else np.zeros(0, np.int64))
    arrays.update(model_arrays(target))
    return arrays


def main():
    os.makedirs(OUT, exist_ok=True)
    emcee = import_reference()
    only = set(sys.argv[1:])
    for idx, case in enumerate(case_list(emcee)):
        if only and case[0] not in only:
            continue
        arrays = run_case(emcee, *case, seed=SEED0 + idx)
        np.savez_compressed(os.path.join(OUT, case[0] + ".npz"), **arrays)
        print("%-36s steps=%3d  acc=%.3f" % (case[0], case[6], arrays["accepted"].mean()))


if __name__ == "__main__":
    main()
