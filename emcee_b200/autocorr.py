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


def integrated_time_from_acf(rho, c=5, tol=50, quiet=False, n_t=None, thin=1):
    """Sokal's automatic window on the walker-averaged autocorrelation function
    ``rho[n_step, n_param]`` (``autocorr.py:107-123``): ``tau[n_param]``, with the
    :class:`AutocorrError` / warning of :func:`integrated_time`.

    ``n_t``: the length of the series when ``rho`` holds only its lags ``0 ..
    max_lag`` (``max_lag = rho.shape[0] - 1 < n_t - 1``, the running
    autocorrelation of ``EnsembleSampler.enable_autocorr``).  A window that
    closes within those lags is the one the whole function gives.  A parameter
    whose window lies beyond them raises :class:`AutocorrError` with ``tau =
    thin * taus[max_lag]`` and a message naming ``max_lag``; with ``quiet`` the
    message is logged as a warning and ``taus[max_lag]`` is the estimate.  The
    length check then uses ``n_t``."""
    L, n_d = rho.shape
    n_t = L if n_t is None else int(n_t)
    taus = 2.0 * np.cumsum(rho, axis=0) - 1.0
    lags = np.arange(L)[:, None]
    inside = lags < c * taus  # Sokal: smallest M with M >= c * tau(M)
    window = np.where(np.any(inside, axis=0), np.argmin(inside, axis=0), L - 1)
    beyond = np.all(inside, axis=0) if n_t > L else np.zeros(n_d, dtype=bool)  # no lag held closes the window
    window[beyond] = L - 1
    tau_est = taus[window, np.arange(n_d)]
    if np.any(beyond):
        msg = (
            "The autocorrelation window of {0} parameter(s) lies beyond max_lag = {1}, the largest lag recorded. "
            "Enable the running autocorrelation with a larger max_lag.\ntau: {2}"
        ).format(np.sum(beyond), L - 1, thin * tau_est)
        if not quiet:
            raise AutocorrError(thin * tau_est, msg)
        logger.warning(msg)
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
