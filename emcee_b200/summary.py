"""``np.percentile`` (default ``linear`` method) split around its order statistics.

``percentile_ranks`` turns ``q`` into the 0-based ranks numpy's ``_quantile`` reads from the partitioned
array (``_get_indexes``: floor / floor + 1 of the virtual index ``(n - 1) q``, clipped to ``[0, n - 1]``),
raising numpy's exceptions for a bad ``q``; ``percentile_finish`` takes the values at those ranks and applies
numpy's ``_lerp`` arithmetic.  Both follow numpy's statements one for one, so that a caller that finds the order
statistics exactly (``DeviceBackend.get_percentile`` does so on the GPU, ``eb_chain_select``) returns what
``np.percentile(x, q, axis=0)`` returns, compared with ``==``.

The histogram plan (``histogram_bins``, ``uniform_edges``, ``searched_edges``) gives the edges of
``np.histogram`` / ``np.histogram2d`` of a column from its minimum and maximum alone: numpy depends on the data
only through them (``_get_outer_edges``, ``np.linspace``, the finite-bins check), so numpy's own functions called
on the two-row array ``[min; max]`` return the edges, and raise the exceptions, that they would on the whole
column.  ``DeviceBackend.get_histogram`` / ``get_histogram2d`` then count on the GPU with these edges."""

import itertools
import operator

import numpy as np

try:
    from numpy.lib._histograms_impl import _get_outer_edges, _unsigned_subtract
except ImportError:  # numpy < 2
    from numpy.lib.histograms import _get_outer_edges, _unsigned_subtract

__all__ = ["percentile_ranks", "percentile_finish", "histogram_bins", "uniform_edges", "searched_edges",
           "running_histogram_plan", "HIST_BINS_MAX", "HIST2_BINS_MAX"]

HIST_BINS_MAX = 4096  # eb_chain_histogram (hist_bins.h)
HIST2_BINS_MAX = 128  # eb_chain_histogram2d: a 64 KiB uint32 pair histogram in shared memory


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


def histogram_bins(bins, limit, two_d=False):
    """``bins`` as the device takes it: numpy's own check first (``np.histogram``'s, or ``np.histogram2d``'s when
    ``two_d``: its exception for a bad ``bins``), then an int of at most ``limit`` (``NotImplementedError`` beyond,
    and for the string rules and explicit edge arrays numpy also accepts)."""
    if two_d:
        np.histogramdd(np.empty((0, 2)), bins)
    else:
        np.histogram_bin_edges(np.empty(0), bins)
    if isinstance(bins, str) or np.ndim(bins) != 0:
        raise NotImplementedError("the device histograms take an integer number of bins, not {0!r}".format(bins))
    n = operator.index(bins)
    if n > limit:
        raise NotImplementedError("the device histogram is limited to bins <= {0}, got {1}".format(limit, n))
    return n


def _check_overflow(a2, rng):
    """Refuse a finite range wider than the largest double: ``np.linspace`` overflows there and the edges numpy
    returns are not all finite (numpy then indexes with a NaN-derived integer, or counts nonsense)."""
    lo, hi = (a2[0], a2[1]) if rng is None else rng
    try:
        lo, hi = np.float64(lo), np.float64(hi)
    except (TypeError, ValueError):
        return  # numpy raises its own exception for this range
    with np.errstate(over="ignore", invalid="ignore"):
        if np.isfinite(lo) and np.isfinite(hi) and lo < hi and not np.isfinite(hi - lo):
            raise ValueError("range of [{0}, {1}] is wider than the largest double: its histogram edges would not be "
                             "finite".format(lo, hi))


def _two_rows(lo, hi, has_nan):
    """the ``[min; max]`` stand-in of a column: NaN for a column that holds one (numpy's ``min()`` propagates it)"""
    return np.array([np.nan, np.nan]) if has_nan else np.array([lo, hi], dtype=np.float64)


def _uniform_column(bins, rng, lo, hi, has_nan):
    a2 = _two_rows(lo, hi, has_nan)
    _check_overflow(a2, rng)
    edges = np.histogram_bin_edges(a2, bins, rng)
    first, last = _get_outer_edges(a2, rng)
    span = _unsigned_subtract(last, first)
    if not np.all(np.isfinite(edges)):
        raise ValueError("histogram edges over [{0}, {1}] are not finite".format(first, last))
    return np.array([first, last, span], dtype=np.float64), np.asarray(edges, dtype=np.float64)


def _searched_column(bins, rng, lo, hi, has_nan):
    a2 = _two_rows(lo, hi, has_nan)
    _check_overflow(a2, rng)
    with np.errstate(invalid="ignore"):
        _, (edges,) = np.histogramdd(a2[:, None], bins=bins, range=None if rng is None else [rng])
    if not np.all(np.isfinite(edges)):
        raise ValueError("histogram edges over [{0}, {1}] are not finite".format(edges[0], edges[-1]))
    return np.asarray(edges, dtype=np.float64)


_EXACT_INT = 2**53  # a Python int range bound below this converts to float64 exactly, as numpy converts it


def _range_dtype(r):
    """the dtype numpy forms a given range ``r`` in (its ``linspace`` dtype): float64 for two Python or float64
    numbers, float32 for two float32 scalars; None for anything else (formed one column at a time)"""
    try:
        lo, hi = r
    except (TypeError, ValueError):
        return None
    kinds = set()
    for v in (lo, hi):
        if isinstance(v, float) or (type(v) is int and -_EXACT_INT <= v <= _EXACT_INT):
            kinds.add(np.float64)  # np.float64 is a float
        elif type(v) is np.float32:
            kinds.add(np.float32)
        else:
            return None
    return kinds.pop() if len(kinds) == 1 else None


def _column_plan(rng, lo, hi, has_nan):
    """The columns' ``(first, last)`` before numpy widens an empty range, by linspace dtype: ``groups`` maps float64
    / float32 to ``(columns, first, last, given)``; ``single`` lists the columns whose range has another form.
    ``rng`` is None, a sequence of one entry (None or a pair) per column, or a float array ``[C, 2]``."""
    lo, hi = np.atleast_1d(np.asarray(lo, dtype=np.float64)), np.atleast_1d(np.asarray(hi, dtype=np.float64))
    has_nan = np.atleast_1d(np.asarray(has_nan, dtype=bool))
    C = max(lo.size, hi.size, has_nan.size)
    lo, hi, has_nan = (np.broadcast_to(v, (C,)) for v in (lo, hi, has_nan))
    if rng is None:
        rng = [None] * C
    if isinstance(rng, np.ndarray) and rng.ndim == 2 and rng.dtype.type in (np.float64, np.float32):
        if len(rng) != C:
            raise ValueError("{0} ranges for {1} columns".format(len(rng), C))
        dt = rng.dtype.type
        given = np.ones(C, dtype=bool)
        groups = {dt: (np.arange(C), rng[:, 0].copy(), rng[:, 1].copy(), given)}
        return C, lo, hi, has_nan, groups, np.zeros(0, dtype=np.intp)
    if len(rng) != C:
        raise ValueError("{0} ranges for {1} columns".format(len(rng), C))
    code = np.empty(C, dtype=np.int8)  # 0 autodetected, 1 float64 given, 2 float32 given, 3 single
    glo, ghi = np.empty(C), np.empty(C)
    for c, r in enumerate(rng):
        if r is None:
            code[c] = 0
            continue
        dt = _range_dtype(r)
        if dt is None:
            code[c] = 3
            continue
        code[c] = 1 if dt is np.float64 else 2
        glo[c], ghi[c] = r  # float32 bounds are exact in float64
    auto = code == 0
    with np.errstate(invalid="ignore"):
        first = np.where(has_nan, np.nan, np.minimum(lo, hi))
        last = np.where(has_nan, np.nan, np.maximum(lo, hi))
    f64 = auto | (code == 1)
    first[~auto], last[~auto] = glo[~auto], ghi[~auto]
    groups = {}
    cols = np.flatnonzero(f64)
    if cols.size:
        groups[np.float64] = (cols, first[cols], last[cols], ~auto[cols])
    cols = np.flatnonzero(code == 2)
    if cols.size:
        groups[np.float32] = (cols, first[cols].astype(np.float32), last[cols].astype(np.float32),
                              np.ones(cols.size, dtype=bool))
    return C, lo, hi, has_nan, groups, np.flatnonzero(code == 3)


def _linspace_rows(first, last, bins, dt):
    """``np.linspace(first[c], last[c], bins + 1)`` of every row, computed in ``dt`` as numpy computes one (``y *
    step + start``, the last element set to ``stop``), and the rows whose step is 0: numpy forms those with
    another expression (``y / div * delta``) -- and an array call would switch every row to it -- so the caller
    forms them one at a time."""
    y = np.arange(0, bins + 1, dtype=dt)
    with np.errstate(all="ignore"):  # an overflowing range is refused by the caller
        delta = np.subtract(last, first, dtype=dt)
        step = delta / bins
        edges = y[None, :] * step[:, None] + first[:, None]
    edges[:, -1] = last
    return edges, delta, step == 0


def _edge_columns(bins, rng, lo, hi, has_nan, uniform):
    C, lo, hi, has_nan, groups, single = _column_plan(rng, lo, hi, has_nan)
    outer = np.empty((C, 3)) if uniform else None
    edges = np.empty((C, bins + 1))
    suspect = np.zeros(C, dtype=bool)
    suspect[single] = True
    for dt, (cols, first, last, given) in groups.items():
        with np.errstate(all="ignore"):
            bad = ~(np.isfinite(first) & np.isfinite(last)) | (given & (first > last))
            # _check_overflow: a finite range (the given one, or the column's [lo, hi]) whose float64 width is not
            lo64 = np.where(given, first.astype(np.float64), lo[cols])
            hi64 = np.where(given, last.astype(np.float64), hi[cols])
            bad |= np.isfinite(lo64) & np.isfinite(hi64) & (lo64 < hi64) & ~np.isfinite(hi64 - lo64)
            same = first == last  # _get_outer_edges widens an empty range by 0.5 each way, in the range's dtype
            first = np.where(same, first - dt(0.5), first)
            last = np.where(same, last + dt(0.5), last)
        e, delta, step0 = _linspace_rows(first, last, bins, dt)
        e = e.astype(np.float64)
        bad |= step0 | ~np.all(np.isfinite(e), axis=1)
        if uniform:
            bad |= np.any(e[:, :-1] >= e[:, 1:], axis=1)  # numpy's "Too many bins for data range"
            outer[cols] = np.stack([first, last, delta], axis=1)
        edges[cols] = e
        suspect[cols[bad]] = True
    # every column that may fail, or that numpy forms another way, goes through numpy itself in column order: the
    # first failing one raises what the per-column loop raises
    for c in np.flatnonzero(suspect):
        r = rng[c] if rng is not None else None
        if isinstance(r, np.ndarray):
            r = (r[0], r[1])
        if uniform:
            outer[c], edges[c] = _uniform_column(bins, r, lo[c], hi[c], has_nan[c])
        else:
            edges[c] = _searched_column(bins, r, lo[c], hi[c], has_nan[c])
    return outer, edges


def uniform_edges(bins, rng, lo=np.nan, hi=np.nan, has_nan=False):
    """``(outer[3], edges[bins + 1])`` of ``np.histogram(column, bins, rng)`` for a column with minimum ``lo`` and
    maximum ``hi`` (used only when ``rng`` is None): ``outer`` is numpy's ``(first_edge, last_edge, norm_denom)``
    of its uniform-bin fast path, as float64.  numpy's exceptions for a bad range; ``ValueError`` for an
    overflowing one.

    With arrays ``lo[C]``, ``hi[C]`` and ``has_nan[C]``, the same for ``C`` columns at once: ``rng`` is None, one
    entry (None or a pair) per column or a float array ``[C, 2]``, and the result ``(outer[C, 3], edges[C, bins +
    1])``, each row equal to the one-column call.  The columns are formed together in a few numpy calls; a column
    that may raise, or that numpy forms another way (a step of 0, a range of another type), is formed by numpy
    alone, in column order, so that the exception is the first failing column's."""
    if np.ndim(lo) == 0 and np.ndim(hi) == 0 and np.ndim(has_nan) == 0:
        outer, edges = _edge_columns(bins, [rng], lo, hi, has_nan, uniform=True)
        return outer[0], edges[0]
    return _edge_columns(bins, rng, lo, hi, has_nan, uniform=True)


def searched_edges(bins, rng, lo=np.nan, hi=np.nan, has_nan=False):
    """``edges[bins + 1]`` of one axis of ``np.histogram2d`` / ``np.histogramdd`` for a column with minimum ``lo``
    and maximum ``hi``: ``np.histogramdd`` of the column's ``[min; max]`` alone, which forms each axis's edges
    independently of the others.  numpy's exceptions for a bad range; ``ValueError`` for an overflowing one.  A
    finite range gives non-decreasing edges (``np.linspace`` rounds monotonically), so ``searchsorted`` is the count
    of edges at or below a value.  With arrays ``lo[C]``, ``hi[C]`` and ``has_nan[C]``: ``edges[C, bins + 1]`` of
    ``C`` columns at once, as :func:`uniform_edges` forms them."""
    if np.ndim(lo) == 0 and np.ndim(hi) == 0 and np.ndim(has_nan) == 0:
        return _edge_columns(bins, [rng], lo, hi, has_nan, uniform=False)[1][0]
    return _edge_columns(bins, rng, lo, hi, has_nan, uniform=False)[1]


def running_histogram_plan(ndim, range, bins=10, log_prob_range=None, params2d=None, bins2d=10):
    """The configuration of ``EnsembleSampler.enable_histograms``, formed on the host before anything is counted:
    ``bins``, ``outer[rows, 3]`` / ``edges[rows, bins + 1]`` (``uniform_edges`` of each parameter's range and,
    with ``log_prob_range``, a last row for the log-probabilities), and with ``params2d`` the pair list and
    ``edges2d[len(params2d), bins2d + 1]`` (``searched_edges``).  A streaming count cannot see the data before it
    bins it, so every parameter needs a range (``ValueError``); otherwise numpy's exceptions, the device limits and
    ``params2d``'s checks are those of ``get_histogram`` / ``get_histogram2d``."""
    from .backend import _histogram_params

    if range is None or any(r is None for r in range):
        raise ValueError("running histograms need a (lo, hi) range for every parameter: the edges are fixed "
                         "before the first value is counted, so they cannot be taken from the data")
    ranges = list(range)
    if len(ranges) != ndim:
        raise ValueError("range must hold one (lo, hi) pair per parameter: {0} for ndim = {1}".format(
            len(ranges), ndim))
    n = histogram_bins(bins, HIST_BINS_MAX)
    rows = ranges + ([] if log_prob_range is None else [log_prob_range])
    outer, edges = uniform_edges(n, rows, np.full(len(rows), np.nan), np.full(len(rows), np.nan))
    cfg = dict(bins=n, outer=outer, edges=edges, log_prob=log_prob_range is not None, params2d=None, bins2d=0,
               edges2d=None, pairs=None)
    if params2d is not None:
        params2d = _histogram_params(params2d, ndim)
        n2 = histogram_bins(bins2d, HIST2_BINS_MAX, two_d=True)
        edges2d = searched_edges(n2, [ranges[p] for p in params2d], np.full(len(params2d), np.nan),
                                 np.full(len(params2d), np.nan))
        cfg.update(params2d=params2d, bins2d=n2, edges2d=edges2d, pairs=list(itertools.combinations(params2d, 2)))
    return cfg
