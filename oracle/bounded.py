"""A target restricted to a box, as numpy (TEST INFRASTRUCTURE ONLY).

``Bounded(target, lower, upper)`` is the usual emcee ``log_prior + log_like``
with a flat prior on the closed box ``lower <= x <= upper``: the target's value
inside, exactly ``-inf`` outside (a NaN coordinate is outside).  It is the
oracle of ``emcee_b200.models.Bounded``.  Vectorised like the targets of
``oracle/targets.py``: ``coords[M, D] -> float64[M]`` or one ``[D]`` row.
"""

import numpy as np

__all__ = ["Bounded"]


class Bounded(object):
    def __init__(self, target, lower, upper):
        self.target = target
        self.kind = target.kind
        self.ndim = target.ndim
        self.lower = np.broadcast_to(np.asarray(lower, dtype=np.float64), (self.ndim,)).copy()
        self.upper = np.broadcast_to(np.asarray(upper, dtype=np.float64), (self.ndim,)).copy()

    def inbox(self, x):
        x = np.asarray(x, dtype=np.float64)
        return np.all((self.lower <= x) & (x <= self.upper), axis=-1)

    def __call__(self, x):
        x = np.asarray(x, dtype=np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            return np.where(self.inbox(x), self.target(x), -np.inf)
