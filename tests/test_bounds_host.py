"""Box priors on the host side: ``models.Bounded`` validation, the oracle's ``Bounded`` against the golden
vectors the unmodified reference produced for bounded targets (``oracle/gen_golden_bounded.py``), and the
bounded cases' own invariants."""
import glob
import os

import numpy as np
import pytest

from oracle import targets as T
from oracle.bounded import Bounded as OracleBounded

from util import GOLDEN, oracle_moves, oracle_target
from oracle import redblue as rb

from emcee_b200 import models

BOUNDED_DIR = os.path.join(GOLDEN, "bounded")


def bounded_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(BOUNDED_DIR, "*.npz")))


def load_bounded(name):
    return dict(np.load(os.path.join(BOUNDED_DIR, name + ".npz")))


def bounded_oracle_sampler(g):
    target = OracleBounded(oracle_target(g), g["model_lower"], g["model_upper"])
    s = rb.OracleSampler(int(g["nwalkers"]), int(g["ndim"]), target, oracle_moves(g), seed=int(g["seed"]))
    s.set_state(g["p0"])
    return s


def test_bounded_cases_exist_and_bind():
    names = bounded_names()
    assert len(names) == 4
    entered = 0
    for name in names:
        g = load_bounded(name)
        # some walkers start outside the box; a walker's log-prob is -inf exactly while it is outside
        assert np.isneginf(g["lp0"]).sum() >= 2, name
        target = OracleBounded(oracle_target(g), g["model_lower"], g["model_upper"])
        assert np.array_equal(np.isneginf(g["log_prob"]), ~target.inbox(g["chain"])), name
        assert not np.isnan(g["log_prob"]).any(), name
        entered += int((np.isneginf(g["lp0"]) & np.isfinite(g["log_prob"][-1])).sum())
    assert entered >= 4


@pytest.mark.parametrize("name", bounded_names())
def test_bounded_restatement_matches_reference(name):
    g = load_bounded(name)
    s = bounded_oracle_sampler(g)
    s.rowwise = True
    assert np.array_equal(s.log_prob, g["lp0"])
    snooker = bool(np.any(g["moves"][:, 0] == 2))
    for k in range(g["chain"].shape[0]):
        acc = s.run(1)
        assert np.array_equal(acc, g["accepted"][k]), (name, k)
        if snooker:  # tolerances of test_oracle_golden.test_restatement_matches_reference
            np.testing.assert_allclose(s.coords, g["chain"][k], rtol=1e-13, atol=1e-15)
            np.testing.assert_allclose(s.log_prob, g["log_prob"][k], rtol=1e-12, atol=1e-14)
        else:
            assert np.array_equal(s.coords, g["chain"][k]), (name, k)
            assert np.array_equal(s.log_prob, g["log_prob"][k]), (name, k)


def test_oracle_bounded_is_closed_box():
    t = OracleBounded(T.GaussIso(3), [-1.0, 0.0, -np.inf], [1.0, np.inf, 2.0])
    x = np.array([[-1.0, 0.0, 2.0], [np.nextafter(-1.0, -2.0), 0.0, 0.0], [0.0, -0.0, -1e100],
                  [0.0, 0.0, np.nextafter(2.0, 3.0)], [0.0, np.nan, 0.0]])
    lp = t(x)
    assert np.array_equal(np.isneginf(lp), [False, True, False, True, True])
    assert lp[0] == T.GaussIso(3)(x[0])


# ---- models.Bounded ------------------------------------------------------------------------------------------
def test_bounded_broadcasts_and_keeps_the_model():
    icov = np.eye(4)
    inner = models.GaussianDense(icov, mean=np.arange(4.0))
    m = models.Bounded(inner, 0.0, [1.0, 2.0, np.inf, 4.0])
    assert m.kind == "gauss_dense"
    assert np.array_equal(m.device_params(4), inner.device_params(4))
    lo, hi = m.bounds(4)
    assert lo.dtype == np.float64 and lo.shape == (4,) and lo.flags.c_contiguous
    assert np.array_equal(lo, np.zeros(4)) and np.array_equal(hi, [1.0, 2.0, np.inf, 4.0])
    assert models.GaussianIso().bounds(3) is None
    with pytest.raises(TypeError):
        m(np.zeros(4))  # still not callable on the host


def test_bounded_accepts_infinite_bounds():
    lo, hi = models.Bounded(models.Ring(), -np.inf, np.inf).bounds(3)
    assert np.isneginf(lo).all() and np.isposinf(hi).all()
    lo, hi = models.Bounded(models.Rosenbrock(), [-np.inf, 0.0], [0.0, np.inf]).bounds(2)
    assert np.array_equal(lo, [-np.inf, 0.0]) and np.array_equal(hi, [0.0, np.inf])


@pytest.mark.parametrize(
    "lower,upper",
    [
        (np.nan, 1.0),
        (0.0, np.nan),
        ([0.0, np.nan], 1.0),
        (1.0, 1.0),  # lower >= upper
        (2.0, 1.0),
        ([0.0, 3.0], [1.0, 2.0]),
        (np.inf, np.inf),
        (-np.inf, -np.inf),
        ([0.0, 1.0], [2.0, 3.0, 4.0]),  # different lengths
        (np.zeros((2, 2)), 1.0),  # not a vector
    ],
)
def test_bounded_refuses_bad_values(lower, upper):
    with pytest.raises(ValueError):
        models.Bounded(models.GaussianIso(), lower, upper)


def test_bounded_refuses_wrong_length_for_ndim():
    m = models.Bounded(models.GaussianIso(), [0.0, 0.0, 0.0], 1.0)
    assert m.bounds(3)[0].shape == (3,)
    with pytest.raises(ValueError):
        m.bounds(4)
    with pytest.raises(ValueError):
        models.Bounded(models.GaussianIso(), 0.0, [1.0, 2.0]).bounds(3)


def test_bounded_wraps_device_models_only():
    with pytest.raises(TypeError):
        models.Bounded(T.GaussIso(3), 0.0, 1.0)
    with pytest.raises(TypeError):
        models.Bounded(models.Bounded(models.GaussianIso(), 0.0, 1.0), 0.0, 1.0)
