"""Integrated autocorrelation time of a stored chain (reference:
``src/emcee/autocorr.py:20-123``; SURVEY 8f "next").  Post-hoc host analysis of
``Backend.chain``; not part of the walker-update hot path.

Same estimator as the reference -- FFT autocorrelation function per walker and
parameter, averaged over walkers, Sokal's automatic window ``M >= c * tau(M)`` --
evaluated for all walkers and parameters in one batched real FFT instead of a
Python loop over ``(parameter, walker)``."""

import logging

import numpy as np

__all__ = ["function_1d", "integrated_time", "integrated_time_from_acf", "AutocorrError"]

logger = logging.getLogger(__name__)


class AutocorrError(Exception):
    """The chain is too short for a reliable estimate; the current estimate is
    in ``tau`` (``autocorr.py:126-136``)."""

    def __init__(self, tau, *args, **kwargs):
        self.tau = tau
        super(AutocorrError, self).__init__(*args, **kwargs)


def _acf(x):
    """Normalised autocorrelation along axis 0 of ``x[n_t, ...]``."""
    n_t = x.shape[0]
    nfft = 2
    while nfft < 2 * n_t:  # zero-padded to twice the next power of two >= n_t
        nfft <<= 1
    f = np.fft.rfft(x - np.mean(x, axis=0, keepdims=True), n=nfft, axis=0)
    acf = np.fft.irfft(f.real**2 + f.imag**2, n=nfft, axis=0)[:n_t]
    return acf / acf[0]


def function_1d(x):
    x = np.atleast_1d(x)
    if x.ndim != 1:
        raise ValueError("invalid dimensions for 1D autocorrelation function")
    return _acf(np.asarray(x, dtype=np.float64))


def integrated_time(x, c=5, tol=50, quiet=False, has_walkers=True, engine=None):
    """``tau[n_param]`` for ``x[n_step]``, ``x[n_step, n_walker]`` (or
    ``[n_step, n_param]`` with ``has_walkers=False``) or ``x[n_step, n_walker,
    n_param]``; raises :class:`AutocorrError` (or warns when ``quiet``) if the
    chain is shorter than ``tol`` autocorrelation times.

    ``engine`` (an ``_lib.Engine``): evaluate the walker-averaged
    autocorrelation functions on the GPU (``eb_autocorr``: hand-written
    batched FFTs) instead of ``numpy.fft``; the window search below is the same."""
    x = np.atleast_1d(np.asarray(x, dtype=np.float64))
    if x.ndim == 1:
        x = x[:, None, None]
    elif x.ndim == 2:
        x = x[:, None, :] if not has_walkers else x[:, :, None]
    if x.ndim != 3:
        raise ValueError("invalid dimensions")
    if engine is not None:
        rho = engine.autocorr_function(x)  # [n_t, n_d], walker-averaged on the device
    else:
        rho = np.mean(_acf(x), axis=1)  # [n_t, n_d], walker-averaged
    return integrated_time_from_acf(rho, c=c, tol=tol, quiet=quiet)


def integrated_time_from_acf(rho, c=5, tol=50, quiet=False):
    """Sokal's automatic window on the walker-averaged autocorrelation function
    ``rho[n_step, n_param]`` (``autocorr.py:107-123``): ``tau[n_param]``, with the
    :class:`AutocorrError` / warning of :func:`integrated_time`."""
    n_t, n_d = rho.shape
    taus = 2.0 * np.cumsum(rho, axis=0) - 1.0
    lags = np.arange(n_t)[:, None]
    inside = lags < c * taus  # Sokal: smallest M with M >= c * tau(M)
    window = np.where(np.any(inside, axis=0), np.argmin(inside, axis=0), n_t - 1)
    tau_est = taus[window, np.arange(n_d)]
    flag = tol * tau_est > n_t
    if np.any(flag):
        msg = (
            "The chain is shorter than {0} times the integrated "
            "autocorrelation time for {1} parameter(s). Use this estimate "
            "with caution and run a longer chain!\n"
        ).format(tol, np.sum(flag))
        msg += "N/{0} = {1:.0f};\ntau: {2}".format(tol, n_t / tol, tau_est)
        if not quiet:
            raise AutocorrError(tau_est, msg)
        logger.warning(msg)
    return tau_est
