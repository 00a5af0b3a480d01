"""Exact reference and rounding bound for the walker-averaged normalised autocorrelation function that
``eb_autocorr`` / ``eb_chain_autocorr`` compute (``test_gpu_autocorr_exact.py`` holds the derivation of the
bound; ``test_autocorr_exact_host.py`` checks this module against numpy on the CPU)."""
import math

import numpy as np

U = 2.0 ** -53
MU = 4 * U  # |fl(sincospi) - exp(-2 pi i k / M)|: sinpi / cospi are within 2 ulp <= 4 u of |component| <= 1
AMP = 2 ** 12


def gamma(n):
    return n * U / (1.0 - n * U)


def fft_error(M):
    """Higham Thm 24.2: ||fl(F x) - F x||_2 <= E ||F x||_2 for a radix-2 transform of length M = 2^t with twiddle
    error MU:  E = t eta / (1 - t eta), eta = MU + gamma_4 (sqrt 2 + MU)."""
    t = int(M).bit_length() - 1
    eta = MU + gamma(4) * (math.sqrt(2.0) + MU)
    return t * eta / (1.0 - t * eta)


def fft_length(n_t):
    n = 1
    while n < n_t:
        n <<= 1
    return 2 * n


def int_series(rng, n_t, nw, nd, phi=0.9):
    """Integer-valued AR(1) series x[n_t, nw, nd] with |x| <= AMP, each summing to a multiple of n_t, so that the
    device's sequential mean and x - mean are exact.  Returned as float64 (every value is an exact integer)."""
    S = nw * nd
    off = rng.integers(-AMP // 4, AMP // 4 + 1, S)
    x = np.empty((n_t, S), dtype=np.int64)
    v = np.zeros(S)
    for t in range(n_t):
        v = phi * v + rng.normal(0.0, AMP / 8, S)
        x[t] = np.clip(np.rint(v) + off, -AMP + 1, AMP - 1)
    r = x.sum(axis=0) % n_t  # subtract 1 from the last r samples of each series
    x -= (np.arange(n_t)[:, None] >= (n_t - r)[None, :]).astype(np.int64)
    return x.reshape(n_t, nw, nd).astype(np.float64)


def lag_set(n_t, rng):
    """Every lag for n_t <= 4097; else the first 64, the last 64 and 64 random ones."""
    if n_t <= 4097:
        return np.arange(n_t)
    mid = rng.choice(np.arange(64, n_t - 64), 64, replace=False)
    return np.unique(np.concatenate([np.arange(64), np.arange(n_t - 64, n_t), mid]))


def lag_sums(x, lags):
    """a[lag, s] = sum_t d_t d_{t+lag} (int64, exact) of the integer series x[n_t, S] about their exact means, and
    the centred series d."""
    xi = x.astype(np.int64)
    assert np.array_equal(xi, x) and np.abs(xi).max() <= AMP
    n_t = x.shape[0]
    tot = xi.sum(axis=0)
    assert np.all(tot % n_t == 0)
    d = xi - tot // n_t  # |d| <= 2 AMP, so |a| <= n_t 2^26 < 2^63
    a = np.empty((len(lags), x.shape[1]), dtype=np.int64)
    for i, k in enumerate(lags):
        a[i] = np.einsum("ts,ts->s", d[: n_t - k], d[k:])
    return a, d


def exact_acf(x, lags):
    """Exact reference of the walker-averaged ACF of integer series x[n_t, nw, nd] at the given lags.

    Returns (ref[L, nd], r[L, nw, nd], a0[nw, nd]): r = a_k / a_0 per series, each rounded once (NaN where a_0 = 0);
    ref = fsum over walkers of r, divided by nw."""
    n_t, nw, nd = x.shape
    a, _ = lag_sums(x.reshape(n_t, nw * nd), lags)
    a0, _ = lag_sums(x.reshape(n_t, nw * nd), [0])
    with np.errstate(invalid="ignore", divide="ignore"):
        r = (a / a0).reshape(len(lags), nw, nd)  # int64 -> float64 is exact below 2^53; one rounding in the divide
    if nw == 1:
        ref = r[:, 0, :].copy()
    else:
        ref = np.empty((len(lags), nd))
        for i in range(len(lags)):
            for j in range(nd):
                ref[i, j] = math.fsum(r[i, :, j].tolist()) / nw
    return ref, r, a0[0].reshape(nw, nd)


def acf_norm(d, M):
    """||a_full||_2 / a_0 per series of the centred d[n_t, S] (numpy float64: it only scales the bound), where
    a_full is the length-M circular autocorrelation: a_0, a_1 .. a_{n-1}, zeros, a_{n-1} .. a_1."""
    out = np.empty(d.shape[1])
    for c in range(0, d.shape[1], 1 << 15):
        f = np.fft.rfft(d[:, c : c + (1 << 15)], n=M, axis=0)
        a = np.fft.irfft(f.real ** 2 + f.imag ** 2, n=M, axis=0)[: d.shape[0]]
        with np.errstate(invalid="ignore", divide="ignore"):
            out[c : c + (1 << 15)] = np.sqrt(a[0] ** 2 + 2 * np.sum(a[1:] ** 2, axis=0)) / a[0]
    return out


def series_bound(M, norm, extra=0.0):
    """rho per series: |Q_k / M - a_k| <= rho a_0 for the unnormalised inverse transform Q of the power spectrum
    (module docstring of test_gpu_autocorr_exact.py, steps 1-3); extra = 2 nu + nu^2 adds the lag-sum error of a
    rounded mean, and scales the transforms' part by the (1 + nu)^2 it allows in a_0."""
    E = fft_error(M)
    c1 = (1.0 + gamma(2)) * (1.0 + E) ** 2 - 1.0
    return (c1 * (1.0 + E * math.sqrt(M)) + E * norm) * (1.0 + extra) + extra


def walker_mean_bound(rho, r, reference_rounding=True):
    """Bound on |device - reference| of the walker average from the per-series rho[nw, nd] and the per-series
    ratios r[L, nw, nd] (steps 4-5)."""
    nw = r.shape[1]
    ar = np.abs(r)
    beta = (1.0 + U) * rho[None] * (1.0 + ar) / (1.0 - rho[None]) + U * ar
    T = np.abs(r.sum(axis=1)) / nw
    dev = ((beta.sum(axis=1) + gamma(nw) * (ar + beta).sum(axis=1)) * (1.0 + gamma(2))) / nw + gamma(2) * T
    if not reference_rounding:
        return dev
    ref = U * ar.sum(axis=1) / nw
    return dev + ref + gamma(2) * (T + ref)


def mean_rounding(x, a0):
    """extra of series_bound for real-valued series x[n_t, S]: |mean error| <= gamma_n sum |x| / n + u |mean| on
    either route; d_t is then off by e_t with ||e||_2 <= sqrt(n) |eps| (1 + u) + u ||d||_2, and each lag sum by
    at most 2 ||e|| ||d|| + ||e||^2."""
    n_t = x.shape[0]
    eps = gamma(n_t) * np.abs(x).sum(axis=0) / n_t + U * np.abs(x.mean(axis=0))
    nu = (1.0 + U) * math.sqrt(n_t) * eps / np.sqrt(a0) + U
    return 2 * nu + nu ** 2
