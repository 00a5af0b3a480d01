#!/usr/bin/env python
"""Generate ``tests/golden/bounded/*.npz`` from the UNMODIFIED reference (TEST INFRASTRUCTURE).

    python -m oracle.gen_golden_bounded

The cases of ``oracle/gen_golden.py`` cover the four targets as they are; these
put each one behind a box prior (``oracle.bounded.Bounded``: the target inside
``lower <= x <= upper``, ``-inf`` outside), the ``log_prior + log_like`` form
of an emcee user's log-probability.  Some walkers start outside the box, with
``log_prob = -inf``.  The reference steps them as it steps any target
(``red_blue.py:96-101``, ``mh.py:55-60``): a proposal inside is accepted
(``lnpdiff = +inf``), one outside is rejected (``lnpdiff`` is NaN).

The arrays are those of ``gen_golden.run_case`` plus ``model_lower`` /
``model_upper``.  The cases live in a sub-directory with seeds of their own, so
the 22 existing fixtures and the test modules that glob ``tests/golden/*.npz``
are untouched.
"""

import os
import sys

import numpy as np

from . import gen_golden as gg
from . import targets as T
from .bounded import Bounded

OUT = os.path.join(gg.OUT, "bounded")
SEED0 = 0x656D636565B2B0  # distinct from gen_golden's 0x656D636565B200 + idx


def case_list(emcee):
    mv = emcee.moves
    rng = np.random.default_rng(4242)

    # dense Gaussian with a mean, a box that rejects about a third of the proposals; 4 walkers start outside
    d16 = T.make_config("gauss_dense", 96, 16)[0]
    mean = np.linspace(-1.0, 1.0, 16)
    dense = Bounded(T.GaussDense(d16.icov, mean=mean), mean - 0.9, mean + 1.1)
    p_dense = mean + 0.25 * rng.standard_normal((96, 16))
    p_dense = np.clip(p_dense, dense.lower + 1e-3, dense.upper - 1e-3)
    for k, w in enumerate((3, 17, 50, 95)):
        p_dense[w, 2 * k] = dense.upper[2 * k] + 0.5 if k % 2 else dense.lower[2 * k] - 0.5

    # half-normal: x >= 0 in every parameter (one-sided); 3 walkers start below zero
    half = Bounded(T.GaussIso(5), 0.0, np.inf)
    p_half = np.abs(rng.standard_normal((32, 5)))
    p_half[[1, 9, 30], [0, 2, 4]] *= -1.0

    # Rosenbrock around its mode, a box that binds in every parameter
    rosen = Bounded(T.Rosenbrock(6), 0.85, 1.2)
    p_rosen = np.clip(1.0 + 0.1 * rng.standard_normal((48, 6)), 0.86, 1.19)
    p_rosen[[5, 40], [1, 3]] = 0.5

    # ring: half of it (x0 >= 0), a finite box in the last two parameters, infinite elsewhere
    ring = Bounded(T.Ring(4), [0.0, -np.inf, -np.inf, -4.0], [np.inf, np.inf, 3.0, 4.0])
    p_ring = 2.5 * rng.standard_normal((64, 4))
    p_ring[:, 0] = np.abs(p_ring[:, 0])
    p_ring[:, 2:] = np.clip(p_ring[:, 2:], -3.9, 2.9)
    p_ring[[0, 33], 0] = -1.0

    return [
        # name, nwalkers, ndim, target, moves, p0, nsteps
        ("bounded_stretch_dense_mean_96x16", 96, 16, dense, mv.StretchMove(), p_dense, 40),
        ("bounded_halfnormal_iso_32x5", 32, 5, half, mv.StretchMove(), p_half, 40),
        ("bounded_de_snooker_rosen_48x6", 48, 6, rosen,
         [(mv.DEMove(), 0.8), (mv.DESnookerMove(), 0.2)], p_rosen, 50),
        ("bounded_walk_stretch_gauss_ring_64x4", 64, 4, ring,
         [(mv.WalkMove(s=8), 0.4), (mv.StretchMove(), 0.3), (mv.GaussianMove(0.1), 0.2), (mv.WalkMove(), 0.1)],
         p_ring, 50),
    ]


_base_model_arrays = gg.model_arrays


def model_arrays(target):
    out = _base_model_arrays(target.target)
    out["model_lower"] = target.lower
    out["model_upper"] = target.upper
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    emcee = gg.import_reference()
    gg.OUT = OUT  # run_case writes to the module's OUT
    gg.model_arrays = model_arrays
    only = set(sys.argv[1:])
    for idx, case in enumerate(case_list(emcee)):
        if only and case[0] not in only:
            continue
        with np.errstate(invalid="ignore"):
            gg.run_case(emcee, *case, seed=SEED0 + idx)


if __name__ == "__main__":
    main()
