"""Registered device-side log-probability models.

The reference takes an arbitrary Python callable ``log_prob_fn``
(``src/emcee/ensemble.py:79-83``) and evaluates it row by row or through
``pool.map`` (``ensemble.py:486-496``).  A GPU engine cannot call back into
Python per walker, so the drop-in takes a *registered model*: a small object
naming one of the log-probabilities compiled into the CUDA library plus its
parameters.  These classes only carry parameters -- they are deliberately not
callable, so no code path can silently evaluate a model on the host.
"""

import numpy as np

__all__ = ["DeviceModel", "GaussianIso", "GaussianDense", "Rosenbrock", "Ring", "Bounded"]


class DeviceModel(object):
    kind = None

    def device_params(self, ndim):
        """flat float64 parameter vector for ``eb_model_set``"""
        raise NotImplementedError

    def bounds(self, ndim):
        """``(lower, upper)`` of the prior's support for ``eb_model_set_bounds``, or None
        (unbounded)"""
        return None

    def __call__(self, *a, **k):
        raise TypeError(
            "device models are evaluated by the CUDA engine "
            "(EnsembleSampler.compute_log_prob); they cannot be called on the host"
        )


class GaussianIso(DeviceModel):
    """``-0.5 * sum(x**2)`` (the target of the reference's move tests,
    ``tests/integration/test_proposal.py:21-22``)."""

    kind = "gauss_iso"

    def device_params(self, ndim):
        return np.zeros(0)


class GaussianDense(DeviceModel):
    """``-0.5 * (x - mean)^T icov (x - mean)`` with a dense precision matrix
    (``document/plots/oned.py:17-18``)."""

    kind = "gauss_dense"

    def __init__(self, icov, mean=None):
        self.icov = np.ascontiguousarray(icov, dtype=np.float64)
        if self.icov.ndim != 2 or self.icov.shape[0] != self.icov.shape[1]:
            raise ValueError("icov must be a square matrix")
        d = self.icov.shape[0]
        self.mean = np.zeros(d) if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        if self.mean.shape != (d,):
            raise ValueError("mean must have shape (ndim,)")

    def device_params(self, ndim):
        if self.icov.shape[0] != ndim:
            raise ValueError("icov is %dx%d but ndim = %d" % (self.icov.shape + (ndim,)))
        return np.concatenate([self.mean, self.icov.ravel()])


class Rosenbrock(DeviceModel):
    """``-sum_i [ b (x[i+1] - x[i]^2)^2 + (a - x[i])^2 ]``"""

    kind = "rosenbrock"

    def __init__(self, a=1.0, b=100.0):
        self.a, self.b = float(a), float(b)

    def device_params(self, ndim):
        return np.array([self.a, self.b])


class Ring(DeviceModel):
    """``-(|x| - radius)^2 / (2 sigma^2)``"""

    kind = "ring"

    def __init__(self, radius=5.0, sigma=0.5):
        self.radius, self.sigma = float(radius), float(sigma)

    def device_params(self, ndim):
        return np.array([self.radius, self.sigma])


class Bounded(DeviceModel):
    """``model`` restricted to the closed box ``lower <= x <= upper``: the log-probability
    is the model's value inside the box and exactly ``-inf`` outside, which is what the
    usual emcee prior ::

        def log_prior(theta):
            if not ((lower <= theta) & (theta <= upper)).all():
                return -np.inf
            return 0.0

    adds to a log-likelihood.  The bounds are the prior's support, not a
    reparametrisation: walkers move in the same coordinates, proposals outside the
    box are rejected (``red_blue.py:96-101`` with ``lp = -inf``), and walkers that
    start outside have ``log_prob = -inf`` until they accept a proposal inside.

    ``lower`` / ``upper`` are scalars (broadcast to every parameter) or vectors of
    length ``ndim``; ``-inf`` / ``+inf`` give one-sided bounds.  NaN bounds and
    ``lower >= upper`` are refused with ValueError.  Every kernel that evaluates
    the model applies the box, and inside it the values are bit-identical to the
    unbounded model."""

    def __init__(self, model, lower, upper):
        if not isinstance(model, DeviceModel) or isinstance(model, Bounded):
            raise TypeError("Bounded wraps one of the registered device models (not another Bounded)")
        self.model = model
        self.kind = model.kind
        lo = np.array(lower, dtype=np.float64)
        hi = np.array(upper, dtype=np.float64)
        for name, v in (("lower", lo), ("upper", hi)):
            if v.ndim > 1:
                raise ValueError("%s must be a scalar or a vector of length ndim" % name)
            if np.isnan(v).any():
                raise ValueError("%s bound must not be NaN" % name)
        if lo.ndim == 1 and hi.ndim == 1 and lo.shape != hi.shape:
            raise ValueError("lower and upper have different lengths (%d, %d)" % (lo.size, hi.size))
        if not (lo < hi).all():
            raise ValueError("every lower bound must be below its upper bound")
        self.lower, self.upper = lo, hi

    def device_params(self, ndim):
        return self.model.device_params(ndim)

    def bounds(self, ndim):
        out = []
        for name, v in (("lower", self.lower), ("upper", self.upper)):
            if v.ndim == 1 and v.shape != (ndim,):
                raise ValueError("%s bound has length %d but ndim = %d" % (name, v.size, ndim))
            out.append(np.ascontiguousarray(np.broadcast_to(v, (ndim,)), dtype=np.float64))
        return out[0], out[1]
