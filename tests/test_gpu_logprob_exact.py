"""The log-probability kernels of ``compute_log_prob`` against exact arithmetic.

The reference value of every row is computed exactly with the standard library (Python integers: every double is
an integer times a power of two, so sums of products are exact; the ring's square root with ``decimal`` at 60
digits) and rounded once.  Each device value must lie within a first-order rounding-error bound of the operation
sequence its kernel performs (u = 2**-53, gamma_n = n u / (1 - n u), eta = 2**-1074 for every rounding that can
land in the subnormal range):

* iso, ``-0.5 sum x^2`` (fma chain per lane, then a shuffle tree; every product passes through at most D
  roundings; the factor -0.5 is exact):  gamma_D * 0.5 sum x^2 + (D + 2) eta.
* ring, ``-(sqrt(S) - R)^2 / (2 sigma^2)``: S as iso; sqrt adds u relative, the subtraction u|d|, so
  dd = r (gamma_D / 2 + u) + u |d|; the square, (2 sigma) sigma and the division three more roundings:
  (2 |d| dd + dd^2) / (2 sigma^2) + gamma_3 |lp|.
* Rosenbrock, ``-sum b (x1 - x0^2)^2 + (a - x0)^2`` term by term: dt = 2 u (x0^2 + |x1|),
  d(b t^2) = b (2 |t| dt + 2 u t^2), d(u^2) = 3 u u^2, plus gamma_D times the sum of the terms for the
  accumulation.
* generic dense, ``y_j = sum_k A_kj xc_k`` then ``sum_j y_j xc_j`` with xc = fl(x - mu): every product passes
  through at most 2 D roundings, and xc's own rounding enters twice:  gamma_{2D+2} 0.5 |xc|^T |A| |xc|.
* dense_dmma, ``0.5 |L^T xc|^2`` with the host Cholesky factor L of the symmetric part A_s of A: against the
  exact ``0.5 xc^T A_s xc`` the factorisation contributes its backward error gamma_{D+1} |L| |L^T| (Higham,
  Thm 10.3), each y_n = (L^T xc)_n is off by (gamma_D + u) z_n with z = |L|^T |xc|, the squares and their sum
  add 2 gamma_{D+1} + gamma_D:  gamma_{4D+4} 0.5 |z|^2.

The largest error / bound ratio of each path is printed and must stay below 1.  Overflow of the sum of squares must
give -inf with no error; a walker whose log-probability is -inf must step like the oracle (red_blue.py:96-101:
-inf - -inf is NaN, which is never accepted).
"""
from fractions import Fraction

import numpy as np
import pytest

from logprob_exact import (_ints, _to_float, bound_dense_dmma, bound_dense_generic, bound_iso, bound_ring,
                           bound_rosen, exact_dense, exact_iso, exact_ring, exact_rosen)
from oracle import redblue as rb
from oracle import targets as T

import emcee_b200
from emcee_b200 import models

pytestmark = pytest.mark.gpu


class Tracker(object):
    """Largest |device - exact| / bound of one path."""

    def __init__(self, name):
        self.name, self.worst, self.n = name, 0.0, 0

    def check(self, dev, exact, bound, what):
        """dev: float; exact: Fraction / Decimal / +-inf float."""
        self.n += 1
        if isinstance(exact, float) and np.isinf(exact):
            assert dev == exact, (what, dev, exact)
            return
        assert np.isfinite(dev), (what, dev, exact)
        err = abs(type(exact)(dev) - exact) if not isinstance(exact, Fraction) else abs(Fraction(dev) - exact)
        ratio = float(err) / bound if bound > 0 else (0.0 if err == 0 else np.inf)
        self.worst = max(self.worst, ratio)
        assert ratio < 1.0, (what, dev, float(exact), float(err), bound)

    def report(self):
        print("%s: %d rows, largest error / bound = %.3g" % (self.name, self.n, self.worst))
        assert self.n > 0 and self.worst < 1.0


# ---- inputs -----------------------------------------------------------------------------------------------------
ROWS_SMALL_D = (1, 7, 8, 9, 65, 4097)


def row_counts(D):
    if D <= 9:
        return ROWS_SMALL_D
    if D <= 257:
        return (1, 8, 9, 65)
    return (1, 9)


def _normal(rows, D, seed):
    return np.random.default_rng(seed).standard_normal((rows, D))


def _huge(rows, D, seed, scale):
    z = np.random.default_rng(seed).standard_normal((rows, D))
    return np.sign(z + 0.5) * scale * (1.0 + np.abs(z))


def _engine(D, model):
    return emcee_b200.EnsembleSampler(max(2, 2 * D), D, model, seed=1)._engine


ISO_DIMS = (1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1024, 4096)


def _elementwise(kind, tr, eng, D, x, params):
    dev = eng.compute_log_prob(x)
    for r in range(x.shape[0]):
        row = x[r]
        what = (kind, D, x.shape[0], r)
        if kind == "iso":
            tr.check(float(dev[r]), _to_float_if_inf(exact_iso(row)), bound_iso(row), what)
        elif kind == "ring":
            lp, d = exact_ring(row, *params)
            b = bound_ring(row, params[0], params[1], d, float(lp) if not isinstance(lp, float) else 0.0)
            tr.check(float(dev[r]), lp, b, what)
        else:
            tr.check(float(dev[r]), _to_float_if_inf(exact_rosen(row, *params)), bound_rosen(row, *params), what)
    return dev


def _to_float_if_inf(q):
    f = _to_float(q)
    return f if np.isinf(f) else q


@pytest.mark.parametrize("kind", ["iso", "ring", "rosenbrock"])
def test_generic_models_exact(kind):
    tr = Tracker("generic %s" % kind)
    params = {"iso": (), "ring": (5.0, 0.5), "rosenbrock": (1.0, 100.0)}[kind]
    for D in ISO_DIMS:
        if kind == "rosenbrock" and D < 2:
            continue
        model = {"iso": models.GaussianIso(), "ring": models.Ring(*params), "rosenbrock": models.Rosenbrock(*params)}[kind]
        eng = _engine(D, model)
        for rows in row_counts(D):
            x = _normal(rows, D, seed=D * 7919 + rows)
            if kind == "rosenbrock":
                x = 1.0 + 0.3 * x
            _elementwise(kind, tr, eng, D, x, params)
        # squares in the subnormal range
        _elementwise(kind, tr, eng, D, 1e-160 * _normal(9, D, seed=D + 11), params)
        # overflow of the sum of squares: -inf, and no error
        big = _huge(9, D, seed=D + 13, scale=1e90 if kind == "rosenbrock" else 1e155)
        dev = _elementwise(kind, tr, eng, D, big, params)
        assert np.all(dev == -np.inf)
        if kind == "ring":
            # within 1e-8 of the radius: the cancellation of sqrt(S) - R
            z = _normal(9, D, seed=D + 17)
            z /= np.sqrt(np.sum(z * z, axis=1))[:, None]
            rad = params[0] * (1.0 + np.linspace(-1e-8, 1e-8, 9))[:, None]
            _elementwise(kind, tr, eng, D, z * rad, params)
    tr.report()


def _dense_target(D, kind, seed=29):
    rng = np.random.default_rng(seed + D)
    if kind == "cond1e10":
        q, _ = np.linalg.qr(rng.standard_normal((D, D)))
        A = (q * np.logspace(-5, 5, D)) @ q.T
        return 0.5 * (A + A.T)
    return T.make_config("gauss_dense", 8, D)[0].icov


def _dense_rows(D, rows, mean_kind, seed):
    x = _normal(rows, D, seed)
    if mean_kind == "far":
        mu = np.full(D, 1e4) + np.linspace(0, 1, D)
        return x + mu, mu
    if mean_kind == "mean":
        mu = np.linspace(-0.5, 0.75, D)
        return x + mu, mu
    return x, np.zeros(D)


def _dense_check(tr, eng, D, A, x, mu, L):
    dev = eng.compute_log_prob(x)
    Aint = _ints(A)
    for r in range(x.shape[0]):
        b = bound_dense_dmma(x[r], mu, L) if L is not None else bound_dense_generic(x[r], mu, A)
        tr.check(float(dev[r]), exact_dense(x[r], mu, Aint), b, (D, x.shape[0], r))


def _dense_cases(D, dmma):
    """(A kind, mean kind, rows, scale) of the dense model at one width."""
    rows = (7, 9, 65) if D <= 64 else (9, 17)
    out = [("random", "none", r, 1.0) for r in rows]
    out += [("random", "mean", 9, 1.0), ("random", "none", 9, 1e-160), ("random", "far", 9, 1.0),
            ("cond1e10", "mean", 9, 1.0)]
    return out


@pytest.mark.parametrize("D", list(range(8, 129, 8)))
def test_dense_dmma_exact(D):
    """dense_dmma's stand-alone log-prob kernel at every width, with and without a mean."""
    tr = Tracker("dense_dmma D=%d" % D)
    for akind, mkind, rows, scale in _dense_cases(D, True):
        A = _dense_target(D, akind)
        x, mu = _dense_rows(D, rows, mkind, seed=D * 31 + rows)
        x = x * scale
        mu = mu * scale
        eng = _engine(D, models.GaussianDense(A, mu if mkind != "none" else None))
        L = np.linalg.cholesky(A)
        _dense_check(tr, eng, D, A, x, mu, L)
    tr.report()


@pytest.mark.parametrize("D,dmma", [(1, 1), (3, 1), (20, 1), (37, 1), (129, 1), (136, 1), (264, 1), (64, 0), (128, 0)])
def test_dense_generic_exact(D, dmma):
    """The CUDA-core dense Gaussian: D % 8 != 0, D > 128, and dense_dmma = 0."""
    tr = Tracker("generic dense D=%d dense_dmma=%d" % (D, dmma))
    for akind, mkind, rows, scale in _dense_cases(D, False):
        if D > 200 and rows > 9:
            continue
        A = _dense_target(D, akind)
        x, mu = _dense_rows(D, rows, mkind, seed=D * 37 + rows)
        x = x * scale
        mu = mu * scale
        eng = _engine(D, models.GaussianDense(A, mu if mkind != "none" else None))
        eng.set_option("dense_dmma", dmma)
        _dense_check(tr, eng, D, A, x, mu, None)
    tr.report()


GUARD_PATHS = [
    # id, D, model factory, options
    ("iso-D33", 33, lambda D: models.GaussianIso(), ()),
    ("ring-D64", 64, lambda D: models.Ring(5.0, 0.5), ()),
    ("rosen-D17", 17, lambda D: models.Rosenbrock(), ()),
    ("dense-generic-D37", 37, lambda D: models.GaussianDense(_dense_target(D, "random")), ()),
    ("dense-dmma-off-D64", 64, lambda D: models.GaussianDense(_dense_target(D, "random")), (("dense_dmma", 0),)),
    ("dense-dmma-D24", 24, lambda D: models.GaussianDense(_dense_target(D, "random"), np.ones(D)), ()),
    ("dense-dmma-D128", 128, lambda D: models.GaussianDense(_dense_target(D, "random")), ()),
]


@pytest.mark.parametrize("D,make,options", [c[1:] for c in GUARD_PATHS], ids=[c[0] for c in GUARD_PATHS])
def test_nonfinite_guards_every_path(D, make, options):
    """ensemble.py:476-479: an infinite or NaN coordinate raises ValueError, also when it sits in the last row
    of a partial tile (9 rows: one full 8-row tile and one row of the next)."""
    eng = _engine(D, make(D))
    for k, v in options:
        eng.set_option(k, v)
    x = _normal(9, D, seed=D)
    assert np.all(np.isfinite(eng.compute_log_prob(x)))
    for bad, msg in ((np.inf, "infinite"), (-np.inf, "infinite"), (np.nan, "NaN")):
        y = x.copy()
        y[8, D - 1] = bad
        with pytest.raises(ValueError, match=msg):
            eng.compute_log_prob(y)
        # the engine is usable afterwards
        assert np.all(np.isfinite(eng.compute_log_prob(x)))


STEP_CASES = [
    ("iso-tma-D32", "gauss_iso", 64, 32, lambda t: models.GaussianIso(), "tma_rows"),
    ("ring-tma-D64", "ring", 130, 64, lambda t: models.Ring(t.radius, t.sigma), "tma_rows"),
    ("rosen-generic-D7", "rosenbrock", 40, 7, lambda t: models.Rosenbrock(), "generic"),
]


@pytest.mark.parametrize("name,N,D,make,kernel", [c[1:] for c in STEP_CASES], ids=[c[0] for c in STEP_CASES])
def test_minus_inf_walker_steps_like_the_oracle(name, N, D, make, kernel):
    """One walker at 1e155: its log-prob is -inf; its proposals and every proposal that uses it as the partner
    are rejected (red_blue.py:96-101), everything else steps as in the oracle.  (Not the dense model: there
    numpy's x^T A x of such a row is inf - inf = NaN, an error, while the Cholesky form gives -inf.)"""
    target, p0 = T.make_config(name, N, D)
    p0 = p0.copy()
    p0[5] = 1e155
    with np.errstate(over="ignore", invalid="ignore"):
        o = rb.OracleSampler(N, D, target, [(rb.Stretch(), 1.0)], seed=0x1F)
        o.set_state(p0)
        assert o.log_prob[5] == -np.inf
        o.run(2)
    s = emcee_b200.EnsembleSampler(N, D, make(target), seed=0x1F)
    assert s.compute_log_prob(p0)[0][5] == -np.inf
    last = s.run_mcmc(p0, 2, store=False, skip_initial_state_check=True)
    assert s._engine.last_kernel_name() == kernel
    assert np.array_equal(last.coords, o.coords)
    assert last.log_prob[5] == -np.inf
    np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-11, atol=1e-11)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
