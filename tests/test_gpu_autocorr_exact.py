"""The device autocorrelation (``Engine.autocorr_function`` = ``eb_autocorr``, ``Chain.autocorr_function`` =
``eb_chain_autocorr``) against an exact reference, at every FFT geometry and slab shape of ``analysis.cu``.

Exact inputs.  Every series is an integer AR(1) path with |x| <= 2^12 whose sum is a multiple of n_t
(``acf_exact.int_series``).  The device's sequential mean is then exact, d = x - mean is exact, and the lag sums
a_k = sum_t d_t d_{t+k} are exact in int64.  The reference per series is a_k / a_0 rounded once; the walker average
is ``math.fsum`` of those, divided by n_w.  Every lag is checked for n_t <= 4 097; longer series check the first 64,
the last 64 and 64 seeded random lags.  Both device routes must agree bit for bit.

The bound (u = 2^-53, gamma_n = n u / (1 - n u), t = log2 M, ||.|| the 2-norm):

1. Forward transform of the zero-padded d (DIF, twiddles from ``sincospi``, within 2 ulp per component, so
   |w^ - w| <= mu = 4 u).  Higham, *Accuracy and Stability of Numerical Algorithms*, Thm 24.2:
   ||Y^ - Y|| <= E ||Y||, E = t eta / (1 - t eta), eta = mu + gamma_4 (sqrt 2 + mu), and ||Y|| = sqrt(M) ||d||,
   ||d||^2 = a_0.  The theorem is stated for DIT; a DIF butterfly (u + v, (u - v) w^) is off by at most
   eta |u + v|, eta |u - v| per output as well, so the same per-stage argument holds.
2. Power spectrum P^_j = fl(Re^2 + Im^2) = |Y^_j|^2 (1 + theta), |theta| <= gamma_2 (with or without FMA).  In the
   1-norm, sum_j ||Y^_j|^2 - |Y_j|^2| <= 2 ||Y^ - Y|| ||Y|| + ||Y^ - Y||^2 and sum_j |theta| |Y^_j|^2 <=
   gamma_2 ||Y^||^2, so ||P^ - P||_1 <= c1 M a_0 with c1 = (1 + gamma_2)(1 + E)^2 - 1.
3. Inverse transform (DIT, conjugate twiddles, unnormalised): Q^ = F* P^ + e, ||e|| <= E sqrt(M) ||P^||.  The
   exact result is M a_full, where a_full is the length-M circular autocorrelation (a_0 .. a_{n-1}, zeros,
   a_{n-1} .. a_1) and ||P|| = sqrt(M) ||a_full||.  Per lag, |(F* (P^ - P))_k| <= ||P^ - P||_1, so
   |Q^_k / M - a_k| <= rho a_0 with rho = c1 (1 + E sqrt(M)) + E ||a_full|| / a_0.  Only the second term depends on
   the series; its ||a_full|| is taken from numpy's float64 ACF, as it only scales the bound.
4. Division by lag 0 (the device divides Q^_k by Q^_0; M cancels): with r_k = a_k / a_0, |r_k| <= 1,
   |r^_k - r_k| <= beta_k = (1 + u) rho (1 + |r_k|) / (1 - rho) + u |r_k|.
5. Walker average: the slab sums and the sum over slabs are a summation tree of depth <= n_w, then a product by
   fl(1 / n_w): |f^ - T| <= (sum beta + gamma_{n_w} sum (|r| + beta)) (1 + gamma_2) / n_w + gamma_2 |T|, T the
   exact mean.  The reference's own roundings add u sum |r| / n_w + gamma_2 (|T| + u sum |r| / n_w).

Per lag the bound is a constant times t u: about 1e-13 for one walker at M = 2^18 (``acf_exact`` computes it; a
CPU test pins it below 1e-12 there).  With many walkers, gamma_{n_w} of step 5 dominates: it is the worst-case
bound of recursive summation, about n_w u.  The largest error / bound ratio of each geometry class is printed
and must stay below 1.

Real-valued data.  One AR(1) float case per FFT length, against the host ``autocorr._acf`` walker mean.  There the
mean is rounded: on either route |eps| <= gamma_n sum |x| / n + u |mean|, d is off by e with ||e|| <= sqrt(n)
|eps| (1 + u) + u ||d||, and each lag sum by 2 ||e|| ||d|| + ||e||^2 (``acf_exact.mean_rounding``).  The tolerance
is the sum of the two routes' bounds, each steps 1-5 with that term added, taking numpy's FFT to meet the bound of
step 1 as well.

Geometry (S = series per slab = walkers per slab x parameters; B = min(M, 8 192) points per ``fft_local_kernel``
CTA, 128 threads below B = 1 024 and 512 from there; every grid is 1-D since this change, and the grid sizes are
those of ``acf_grid.h``):

=================  =================  ==========  ====================================================================
test id            n_t, nw x nd       M           kernels and grids
=================  =================  ==========  ====================================================================
len-2 / float-2    2, 3 x 2           4           local only, 2 + 2 stages; 128 threads for 2 butterflies; 6 CTAs
len-3 / float-3    3, 3 x 2           8           local only, 3 + 3 stages; n_t = 2^k + 1
len-256            256, 3 x 2         512         local only, 9 + 9 stages, 128 threads
len-257            257, 3 x 2         1 024       local only, 512 threads (the switch at B = 1 024)
len-4096           4 096, 3 x 2       8 192       M = ACF_BLOCK: local stages only, 13 + 13
len-4097           4 097, 3 x 2       16 384      one global stage each way (h = 8 192), 2 local CTAs per series
len-65536          65 536, 3 x 2      131 072     4 global stages each way, 16 local CTAs per series
len-65537          65 537, 3 x 2      262 144     5 global stages each way, 32 local CTAs per series
S65535             100, 4 369 x 15    256         one slab of 65 535 series: 65 535 local CTAs (was grid y's limit)
S65536             100, 8 192 x 8     256         65 536 local CTAs: the first count grid y refused
S65537             100, 65 537 x 1    256         65 537 local CTAs, 2 049 x 8 load tiles, one parameter
S4M                4, 65 536 x 64     8           4 194 304 series, 131 072 series tiles of ``acf_load_kernel``
                                                  (> 2 097 120 series: past grid y there too); every series exact
nd65536            5, 1 x 65 536      16          ``acf_accumulate_kernel`` over 65 536 parameters (1 lag tile each)
slabs3             100, 64 000 x 8    256         3 slabs of 27 413 + 27 413 + 9 174 walkers, each > 65 535 series
monitor            100, 8 192 x 8     256         sampler run (Backend and DeviceBackend), get_autocorr_time(tol=0)
stuck-*            300, 6 x 3 and     512, 256    one series constant (a_0 = 0): NaN for its parameter only
                   100, 8 192 x 8
=================  =================  ==========  ====================================================================

Rows S65535 .. slabs3 (but nd65536: a device chain holds at most 16 384 parameters, so that row runs
``eb_autocorr`` alone) and both stuck rows also write the chain into a ``DeviceBackend`` and require
``get_autocorr_time(tol=0)`` to equal the host-``Backend`` route (``integrated_time(..., engine=)``) bit for bit.
The length rows write it into a ``Chain`` and require its ACF to equal ``eb_autocorr``'s bit for bit.
A constant that is not exactly representable (0.1) gives a tiny a_0 whose value depends on the summation order of
the mean on every route, the reference's included, so it is left out: the stuck series here are integers.
"""
import numpy as np
import pytest

import acf_exact as X
from oracle import targets as T

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, _lib, autocorr, models

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for cls in sorted(WORST):
        print("autocorr %-8s largest error / bound = %.3g" % (cls, WORST[cls]))


@pytest.fixture(scope="module")
def eng():
    return _lib.Engine(8, 2, 1)


def _track(cls, got, want, bound):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.all(np.isfinite(bound[~nan])) and np.all(bound[~nan] > 0)
    ratio = float(np.max(np.abs(got - want)[~nan] / bound[~nan])) if np.any(~nan) else 0.0
    WORST[cls] = max(WORST.get(cls, 0.0), ratio)
    print("autocorr %s: largest error / bound = %.3g" % (cls, ratio))
    assert ratio < 1.0, (cls, ratio)


def _chain_route(x):
    n_t, nw, nd = x.shape
    ch = _lib.Chain(nw, nd)
    try:
        ch.grow(n_t)
        for t in range(n_t):
            ch.write(t, x[t], np.zeros(nw))
        return ch.autocorr_function(0, 1, n_t)
    finally:
        ch.close()


def _backend_route(eng, x):
    """ACF of x stored in a DeviceBackend; its tau must equal the host-Backend route's bit for bit."""
    n_t, nw, nd = x.shape
    b = DeviceBackend()
    try:
        b.reset(nw, nd)
        b.grow(n_t, None)
        for t in range(n_t):
            b.save_step(emcee_b200.State(x[t], log_prob=np.zeros(nw)), np.zeros(nw, dtype=bool))
        tau_d = b.get_autocorr_time(tol=0)
        tau_h = autocorr.integrated_time(x, tol=0, engine=eng)
        assert np.array_equal(tau_d, tau_h, equal_nan=True)
        return b._ch.autocorr_function(0, 1, n_t)
    finally:
        b.close()


def _device(eng, x, route):
    """eb_autocorr's ACF of x, after checking that route ("chain": a Chain, "backend": a DeviceBackend and tau;
    None: eb_autocorr alone) gives the same bits."""
    got = eng.autocorr_function(x)
    assert got.shape == (x.shape[0], x.shape[2])
    if route is not None:
        other = _backend_route(eng, x) if route == "backend" else _chain_route(x)
        assert np.array_equal(got, other, equal_nan=True)
    return got


def _check_exact(cls, got, x, rng):
    n_t, nw, nd = x.shape
    lags = X.lag_set(n_t, rng)
    ref, r, a0 = X.exact_acf(x, lags)
    M = X.fft_length(n_t)
    norm = X.acf_norm((x - x.mean(axis=0)).reshape(n_t, nw * nd), M).reshape(nw, nd)
    _track(cls, got[lags], ref, X.walker_mean_bound(X.series_bound(M, norm), r))
    return ref


LENGTHS = [2, 3, 256, 257, 4096, 4097, 65536, 65537]


@pytest.mark.parametrize("n_t", LENGTHS, ids=["len-%d" % n for n in LENGTHS])
def test_lengths_exact(eng, n_t):
    rng = np.random.default_rng(n_t)
    x = X.int_series(rng, n_t, 3, 2)
    got = _device(eng, x, "chain")
    _check_exact("M=%d" % X.fft_length(n_t), got, x, rng)


@pytest.mark.parametrize("n_t", LENGTHS, ids=["float-%d" % n for n in LENGTHS])
def test_lengths_real_valued(eng, n_t):
    rng = np.random.default_rng(100 + n_t)
    nw, nd = 3, 2
    x = np.empty((n_t, nw, nd))
    x[0] = rng.normal(size=(nw, nd))
    for t in range(1, n_t):
        x[t] = 0.9 * x[t - 1] + rng.normal(size=(nw, nd))
    x += np.array([3.7, -120.25])  # a mean for the subtraction to round
    got = _device(eng, x, "chain")
    r = autocorr._acf(x)
    want = r.mean(axis=1)
    M = X.fft_length(n_t)
    d = (x - x.mean(axis=0)).reshape(n_t, nw * nd)
    a0 = np.sum(d * d, axis=0)
    rho = X.series_bound(M, X.acf_norm(d, M), X.mean_rounding(x.reshape(n_t, -1), a0)).reshape(nw, nd)
    _track("float", got, want, 2 * X.walker_mean_bound(rho, r, reference_rounding=False))


SLAB_SHAPES = {
    "S65535": (100, 4369, 15),
    "S65536": (100, 8192, 8),
    "S65537": (100, 65537, 1),
    "S4M": (4, 65536, 64),
    "nd65536": (5, 1, 65536),
    "slabs3": (100, 64000, 8),
}


@pytest.mark.parametrize("name", list(SLAB_SHAPES))
def test_slab_shapes_exact_on_both_routes(eng, name):
    n_t, nw, nd = SLAB_SHAPES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x = X.int_series(rng, n_t, nw, nd)
    got = _device(eng, x, "backend" if nd <= 16384 else None)  # a device chain holds at most 16 384 parameters
    _check_exact(name, got, x, rng)


def test_monitor_pattern_on_both_backends():
    """The convergence-monitor loop of the reference's tutorial: get_autocorr_time(tol=0) after 100 stored steps
    of 8 192 x 8 walkers, the first shape past 65 535 series per slab."""
    N, D, steps = 8192, 8, 100
    target, p0 = T.make_config("gauss_iso", N, D)
    taus, chains = [], []
    for b in (Backend(), DeviceBackend()):
        s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=0x91, backend=b)
        s.run_mcmc(p0, steps, skip_initial_state_check=True)
        taus.append(s.get_autocorr_time(tol=0))
        chains.append(s.get_chain())
    assert np.array_equal(chains[0], chains[1])
    assert np.all(np.isfinite(taus[0])) and np.array_equal(taus[0], taus[1])
    # and the ACF behind it, against numpy under the real-valued tolerance
    x = chains[0]
    got = s._engine.autocorr_function(x)
    r = autocorr._acf(x)
    M = X.fft_length(steps)
    d = (x - x.mean(axis=0)).reshape(steps, N * D)
    rho = X.series_bound(M, X.acf_norm(d, M), X.mean_rounding(x.reshape(steps, -1), np.sum(d * d, axis=0)))
    _track("monitor", got, r.mean(axis=1), 2 * X.walker_mean_bound(rho.reshape(N, D), r, reference_rounding=False))


@pytest.mark.parametrize("shape", [(300, 6, 3), (100, 8192, 8)], ids=["stuck-small", "stuck-S65536"])
def test_stuck_walker(eng, shape):
    n_t, nw, nd = shape
    rng = np.random.default_rng(n_t + nw)
    x = X.int_series(rng, n_t, nw, nd)
    clean = eng.autocorr_function(x)
    w, p = nw // 2, 1
    x[:, w, p] = 7.0  # never moves in the window: a_0 = 0 for this series
    got = _device(eng, x, "backend")  # equal NaN tau on both routes
    ref = _check_exact("stuck", got, x, rng)
    assert np.all(np.isnan(got[:, p])) and np.all(np.isnan(ref[:, p]))
    others = [j for j in range(nd) if j != p]
    assert np.array_equal(got[:, others], clean[:, others])
    # a NaN tau for that parameter, and no AutocorrError from it at the default tol
    tau = autocorr.integrated_time_from_acf(got[:, [p]])
    assert np.isnan(tau[0])
    tau = autocorr.integrated_time(x, tol=0, engine=eng)
    assert np.isnan(tau[p]) and np.all(np.isfinite(tau[others]))
