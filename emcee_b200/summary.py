"""``np.percentile`` (default ``linear`` method) split around its order statistics.

``percentile_ranks`` turns ``q`` into the 0-based ranks numpy's ``_quantile`` reads from the partitioned
array (``_get_indexes``: floor / floor + 1 of the virtual index ``(n - 1) q``, clipped to ``[0, n - 1]``),
raising numpy's exceptions for a bad ``q``; ``percentile_finish`` takes the values at those ranks and applies
numpy's ``_lerp`` arithmetic.  Both follow numpy's statements one for one, so that a caller that finds the order
statistics exactly (``DeviceBackend.get_percentile`` does so on the GPU, ``eb_chain_select``) returns what
``np.percentile(x, q, axis=0)`` returns, compared with ``==``."""

import numpy as np

__all__ = ["percentile_ranks", "percentile_finish"]


def _quantile_is_valid(q):
    if q.ndim == 1 and q.size < 10:
        for i in range(q.size):
            if not (0.0 <= q[i] <= 1.0):
                return False
    elif not (q.min() >= 0 and q.max() <= 1):
        return False
    return True


class PercentilePlan(object):
    """Virtual indexes of ``q`` over ``n`` values and the ranks they read: ``ranks`` (sorted, unique) and, for the
    lower and upper neighbours, their positions in ``ranks``."""

    def __init__(self, q, n):
        q = np.asanyarray(np.true_divide(q, np.float64(100)))  # np.percentile: q / 100 in the data's dtype
        if not _quantile_is_valid(q):
            raise ValueError("Percentiles must be in the range [0, 100]")
        if q.ndim > 2:
            raise ValueError("q must be a scalar or 1d")
        n = int(n)
        self.n = n
        self.virtual = np.asanyarray((n - 1) * q)  # the "linear" method's virtual index
        prev = np.asanyarray(np.floor(self.virtual))
        nxt = np.asanyarray(prev + 1)
        above = self.virtual >= n - 1
        if above.any():
            prev[above] = -1
            nxt[above] = -1
        below = self.virtual < 0
        if below.any():
            prev[below] = 0
            nxt[below] = 0
        self.prev = prev.astype(np.intp)
        self.next = nxt.astype(np.intp)
        lo = np.where(self.prev < 0, n - 1, self.prev).astype(np.uint64)
        hi = np.where(self.next < 0, n - 1, self.next).astype(np.uint64)
        self.ranks = np.unique(np.concatenate([lo.ravel(), hi.ravel()]))
        self._lo = np.searchsorted(self.ranks, lo)
        self._hi = np.searchsorted(self.ranks, hi)


def percentile_ranks(q, n):
    """The :class:`PercentilePlan` of ``np.percentile(x, q, axis=0)`` for ``n`` values per column; numpy's
    exceptions for a bad ``q``."""
    return PercentilePlan(q, n)


def percentile_finish(plan, stats, has_nan=None):
    """``np.percentile`` from ``stats[len(plan.ranks), ...]``, the values at ``plan.ranks`` of each column, and
    ``has_nan`` (per column, or None): columns holding a NaN give NaN, as numpy's do."""
    stats = np.asarray(stats, dtype=np.float64)
    previous = stats[plan._lo]
    nxt = stats[plan._hi]
    gamma = np.asanyarray(plan.virtual - plan.prev)
    gamma = np.asanyarray(gamma, dtype=plan.virtual.dtype)
    gamma = gamma.reshape(plan.virtual.shape + (1,) * (stats.ndim - 1))
    # numpy's _lerp
    diff_b_a = np.subtract(nxt, previous)
    result = np.asanyarray(np.add(previous, diff_b_a * gamma))
    np.subtract(nxt, diff_b_a * (1 - gamma), out=result, where=gamma >= 0.5, casting="unsafe")
    if result.ndim == 0:
        result = result[()]
    if has_nan is not None and np.any(has_nan):
        if result.ndim == 0:
            result = np.float64(np.nan)
        else:
            np.copyto(result, np.nan, where=np.asarray(has_nan, dtype=bool).reshape(stats.shape[1:]))
    return result
