#!/usr/bin/env python
"""Generate ``tests/golden/user_moves/*.npz`` from the UNMODIFIED reference (TEST INFRASTRUCTURE).

    python -m oracle.gen_golden_user_moves [names]    # needs oracle/_ref/emcee_reference.zip (make_ref.py)

Each case runs the reference's own ``EnsembleSampler`` with ``oracle.philox.PhiloxRandom`` as ``sampler._random``
(``ensemble.py:166``) and user moves written against the reference's plugin boundary: a ``RedBlueMove`` subclass
overriding ``get_proposal`` (``red_blue.py:47,90``) and ``MHMove(proposal_function)`` (``mh.py:31-33,52``).  Their
``random`` argument is rebuilt from the shim's ``(seed, step)`` and a per-step split counter as the draw
specification's purpose 8 (DESIGN.md §2): ``RandomState(Philox(key=seed, counter=(0, step, split, 8)))``.  The
proposal functions and the case table below are plain numpy, shared with ``tests/test_gpu_user_moves.py``, which
runs the same functions on the engine; importing this module does not import the reference."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ZIP = os.path.join(HERE, "_ref", "emcee_reference.zip")
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "user_moves")


def user_random(seed, step, split):
    return np.random.RandomState(np.random.Philox(key=int(seed) & (2**64 - 1), counter=[0, int(step), int(split), 8]))


# ---- the user functions (what an emcee user writes) -----------------------------------------------------------
def stretch_proposal(s, c, random, a=2.0):
    c = np.concatenate(c, axis=0)
    ns, nc = len(s), len(c)
    zz = ((a - 1.0) * random.rand(ns) + 1) ** 2.0 / a
    factors = (s.shape[1] - 1.0) * np.log(zz)
    rint = random.randint(nc, size=(ns,))
    return c[rint] - (c[rint] - s) * zz[:, None], factors


def de_proposal(s, c, random, gamma=0.7, sigma=1e-3):
    c = np.concatenate(c, axis=0)
    ns, nc = len(s), len(c)
    pairs = random.randint(nc, size=(ns, 2))
    g = gamma * (1.0 + sigma * random.randn(ns, 1))
    return s + g * (c[pairs[:, 0]] - c[pairs[:, 1]]), np.zeros(ns)


def mh_proposal(coords, random):
    """A Gaussian random walk with a non-zero log factor: exercises mh.py:57's rounding order."""
    q = coords + 0.3 * random.randn(*coords.shape)
    return q, 0.25 * random.randn(len(coords))


FUNCTIONS = {"stretch": stretch_proposal, "de": de_proposal, "mh": mh_proposal}

# name, nwalkers, ndim, target kind, moves [(kind, function or None, weight, kwargs)], nsteps
CASES = [
    ("stretch_iso_32x5", 32, 5, "gauss_iso", [("user", "stretch", 1.0, {})], 30),
    ("stretch_fixed_nsplits3_ring_45x4", 45, 4, "ring",
     [("user", "stretch", 1.0, dict(nsplits=3, randomize_split=False))], 25),
    ("de_nsplits5_rosen_41x4", 41, 4, "rosenbrock", [("user", "de", 1.0, dict(nsplits=5))], 25),
    ("mh_iso_32x5", 32, 5, "gauss_iso", [("user_mh", "mh", 1.0, {})], 30),
    ("mix_dense_64x6", 64, 6, "gauss_dense",
     [("user", "stretch", 0.3, {}), ("stretch", None, 0.3, {}), ("de", None, 0.2, {}), ("user_mh", "mh", 0.2, {})],
     30),
    ("stretch_nsplits32_ring_70x4", 70, 4, "ring", [("user", "stretch", 1.0, dict(nsplits=32))], 20),
]
SEED = 0x0B200


def case_target(kind, ndim):
    from . import targets as T

    return T.make_config(kind, 8, ndim)[0]


def case_p0(name, nwalkers, ndim, kind):
    rng = np.random.default_rng(sum(map(ord, name)))
    x = rng.standard_normal((nwalkers, ndim))
    return {"ring": 2.5 * x, "rosenbrock": 1.0 + 0.1 * x}.get(kind, x)


# ---- the reference side ---------------------------------------------------------------------------------------
def import_reference():
    if REF_ZIP not in sys.path:
        sys.path.insert(0, REF_ZIP)
    import emcee

    assert REF_ZIP in emcee.__file__, emcee.__file__
    return emcee


def shim_class():
    from .philox import PhiloxRandom

    class UserPhilox(PhiloxRandom):
        """The shim with the accessor a user proposal needs: which call of the step this is."""

        def user_split(self):
            # the first proposal-type call after a step start or an accept phase opens the next split
            self._open_split()
            return self.seed, self._cur, self._split

        def user_mh(self):
            self._phase = "mh"  # mh.py:58's rand(nwalkers) draws the walker-indexed accept uniforms
            return self.seed, self._cur, 0

    return UserPhilox


def reference_moves(emcee, spec):
    class UserRedBlue(emcee.moves.RedBlueMove):
        def __init__(self, fn, **kw):
            self.fn = fn
            super().__init__(**kw)

        def get_proposal(self, s, c, random):
            return self.fn(s, c, user_random(*random.user_split()))

    out = []
    for kind, fname, w, kw in spec:
        if kind == "user":
            m = UserRedBlue(FUNCTIONS[fname], **kw)
        elif kind == "user_mh":
            fn = FUNCTIONS[fname]
            m = emcee.moves.MHMove(lambda x, random, fn=fn: fn(x, user_random(*random.user_mh())))
        elif kind == "stretch":
            m = emcee.moves.StretchMove(**kw)
        else:
            m = emcee.moves.DEMove(**kw)
        out.append((m, w))
    return out


def run_case(emcee, name, nwalkers, ndim, kind, spec, nsteps):
    target = case_target(kind, ndim)
    p0 = case_p0(name, nwalkers, ndim, kind)
    sampler = emcee.EnsembleSampler(nwalkers, ndim, target, moves=reference_moves(emcee, spec), vectorize=True)
    sampler._random = shim_class()(SEED)  # ensemble.py:166
    acc = np.empty((nsteps, nwalkers), dtype=bool)
    prev = np.zeros(nwalkers)
    k = 0
    for _ in sampler.sample(p0, iterations=nsteps, skip_initial_state_check=True):
        now = sampler.backend.accepted.copy()
        acc[k] = (now - prev) > 0.5
        prev = now
        k += 1
    return dict(nwalkers=np.array(nwalkers), ndim=np.array(ndim), seed=np.array(SEED, dtype=np.uint64), p0=p0,
                chain=sampler.get_chain(), log_prob=sampler.get_log_prob(), accepted=acc)


def generate(out_dir=OUT, only=()):
    emcee = import_reference()
    os.makedirs(out_dir, exist_ok=True)
    for name, nwalkers, ndim, kind, spec, nsteps in CASES:
        if only and name not in only:
            continue
        arrays = run_case(emcee, name, nwalkers, ndim, kind, spec, nsteps)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **arrays)
        print("%s: %d steps, acceptance %.3f" % (name, nsteps, arrays["accepted"].mean()))


if __name__ == "__main__":
    generate(only=set(sys.argv[1:]))
