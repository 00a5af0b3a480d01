"""Kernel-density proposals of the complement (reference: ``src/emcee/moves/kde.py:16-43``)."""

import math
import numbers

from .red_blue import RedBlueMove

__all__ = ["KDEMove"]

# include/emcee_b200.h: p0 = the bandwidth rule (NaN: Scott), p1 = a scalar bandwidth
_SILVERMAN = 1.0
_SCALAR = 2.0


class KDEMove(RedBlueMove):
    """A proposal using a KDE of the complementary ensemble (``kde.py:16-28``): each walker's proposal is a draw
    from ``scipy.stats.gaussian_kde`` of the other sets, with the log ratio of the KDE's density at the walker and
    at the proposal as Hastings factor.  Use *a lot* of walkers with this move.

    :param bw_method: ``None`` or ``"scott"`` (Scott's rule), ``"silverman"``, or a positive finite scalar used as
        the bandwidth factor itself, as ``gaussian_kde`` takes it.  A callable receives a scipy ``gaussian_kde`` on
        the host and is refused (``NotImplementedError``).

    The KDE, its draws and its log-density run on the GPU (``kde.cu``): the complement covariance and its Cholesky
    factor once per split, the log-densities from direct differences of whitened rows, O(nwalkers^2 ndim) per step.
    A split whose complement has fewer rows than ``ndim`` raises scipy's ``ValueError`` before any update; a
    singular complement covariance (a Cholesky pivot at or below ``1e-12 * max(diag)``) raises
    ``numpy.linalg.LinAlgError`` at its half-step, where scipy may go on with a factor made of rounding noise.
    ``ndim <= 1024``; sharded ensembles are refused."""

    kind = "kde"

    def __init__(self, bw_method=None, **kwargs):
        if callable(bw_method):
            raise NotImplementedError(
                "KDEMove: a callable bw_method takes a scipy gaussian_kde on the host; the device KDE takes None, "
                "'scott', 'silverman' or a scalar"
            )
        if isinstance(bw_method, str):
            if bw_method not in ("scott", "silverman"):
                raise ValueError("`bw_method` should be 'scott', 'silverman', a scalar or a callable.")
        elif bw_method is not None:
            if isinstance(bw_method, bool) or not isinstance(bw_method, numbers.Real):
                raise ValueError("`bw_method` should be 'scott', 'silverman', a scalar or a callable.")
            if not (math.isfinite(float(bw_method)) and float(bw_method) > 0.0):
                raise ValueError("KDEMove: a scalar bw_method must be finite and > 0 (got %r)" % (bw_method,))
        self.bw_method = bw_method
        super(KDEMove, self).__init__(**kwargs)

    def _params(self):
        if self.bw_method is None or self.bw_method == "scott":
            return float("nan"), float("nan")
        if self.bw_method == "silverman":
            return _SILVERMAN, float("nan")
        return _SCALAR, float(self.bw_method)
