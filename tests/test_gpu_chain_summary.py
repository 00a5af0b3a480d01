"""Summaries of a stored device chain (``DeviceBackend.get_percentile`` / ``get_moments``; ``eb_chain_select``,
``eb_chain_moments``) against the host ``Backend``'s numpy expressions.

* Twin runs into ``Backend()`` and ``DeviceBackend()``: ``get_percentile`` equal to ``np.percentile`` of the host
  slice (``np.array_equal``) for ``"chain"`` and ``"log_prob"`` over a ``discard`` / ``thin`` grid, resumed runs
  (several segments), odd ``nwalkers``, ndim 1, 7, 128, 257 and 1024, and a bounded model that stores ``-inf``.
  The device moments of the whole chain equal, bit for bit, the running moments (``enable_moments(1)``) of the
  same run: both fold the same rows in the same order about the first stored step's column mean.
* Crafted chains uploaded with ``save_step``: constants, two values, integer ties, +-0.0, subnormals, +-1e308,
  +-inf, a NaN in one parameter only, values that share their top 48 bits; ``passes`` shows that the short path
  (one read and a compaction) and the long path (a histogram pass per byte) both ran.
* 65 536 x 128 with 32 stored steps over two segments.
* ``get_moments`` against a two-pass long-double reference under the bound of ``test_moments_exact``
  (``test_gpu_proposals_exact``), at ndim 1, 129 and 1024 and on a chain drifting far from the first slot's mean.
* Error contracts.
"""
import math

import numpy as np
import pytest

import proposals_exact as PX
from oracle import targets as T
from test_gpu_bounds import _box_and_p0
from test_gpu_proposals_exact import Tracker, sm_count

from gpu_util import device_model

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, models

pytestmark = pytest.mark.gpu

QS = [[16, 50, 84], 0, 100, 50, 1e-12, 100 - 1e-12, [[5, 50], [95, 99.5]], np.linspace(0, 100, 41)]


def _same(got, want):
    assert np.shape(got) == np.shape(want)
    assert np.array_equal(got, want, equal_nan=True)


def _percentiles_equal(h, d, grid):
    for discard, thin in grid:
        for q in QS:
            for name in ("chain", "log_prob"):
                want = h.get_percentile(q, discard=discard, thin=thin, name=name)
                got = d.get_percentile(q, discard=discard, thin=thin, name=name)
                _same(got, want)


def _twin(N, D, model, p0, seed, calls):
    """the same run into Backend() and DeviceBackend(), resumed len(calls) times (one segment per call)"""
    out = []
    for backend in (Backend(), DeviceBackend()):
        s = emcee_b200.EnsembleSampler(N, D, model, seed=seed, backend=backend)
        s.enable_moments(1)
        st = p0
        for n in calls:
            st = s.run_mcmc(st, n, skip_initial_state_check=True)
        out.append(s)
    h, d = out
    assert np.array_equal(h.get_chain(), d.get_chain())
    return h, d


def _grid(it):
    """(discard, thin) pairs of non-empty slices (np.percentile of an empty slice raises IndexError)"""
    pairs = {(0, 1), (1, 1), (3, 2), (it // 2, 3), (it - 1, 1), (0, it), (2, 7)}
    return sorted((d, t) for d, t in pairs if d + t - 1 < it)


@pytest.mark.parametrize("N,D,calls", [(33, 1, (6, 5, 4)), (63, 7, (10, 9)), (513, 128, (5, 4)), (515, 257, (3, 3)),
                                       (2049, 1024, (2, 2))],
                         ids=["N33-D1", "N63-D7", "N513-D128", "N515-D257", "N2049-D1024"])
def test_twin_percentiles_and_moments(N, D, calls):
    rng = np.random.default_rng(N + D)
    p0 = rng.standard_normal((N, D))
    h, d = _twin(N, D, models.GaussianIso(), p0, 0x5E + D, calls)
    _percentiles_equal(h, d, _grid(h.iteration))
    mean, cov, n = d.get_moments()
    mr, cr, nr = d.moments()
    assert n == nr == h.iteration * N
    assert np.array_equal(mean, mr) and np.array_equal(cov, cr)
    hm, hc, hn = h.get_moments(discard=1, thin=2)
    dm, dc, dn = d.get_moments(discard=1, thin=2)
    assert hn == dn
    np.testing.assert_allclose(dm, hm, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dc, hc, rtol=1e-8, atol=1e-12)


def test_twin_bounded_stores_minus_inf():
    N, D = 2 * (8 * 20 + 1), 32
    target, p0 = T.make_config("ring", N, D)
    lo, hi, pb = _box_and_p0(target, p0, 0)
    model = models.Bounded(device_model("ring", target=target), lo, hi)
    h, d = _twin(N, D, model, pb, 0x57, (6, 5))
    assert np.isneginf(d.get_log_prob()[0]).any()
    _percentiles_equal(h, d, _grid(h.iteration))
    # the smallest stored log-probability is -inf; np.percentile(q=0) interpolates -inf + (-inf - -inf) * 0 = NaN
    v, _, _ = d.backend._chain.select("log_prob", 0, 1, d.iteration, np.array([0], dtype=np.uint64))
    assert np.isneginf(v[0, 0]) and np.isnan(d.get_percentile(0, name="log_prob"))


# ---- crafted chains ------------------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072009e-308, 1e308, -1e308,
                    np.inf, -np.inf, 1.0, -1.0, 3.0, -7.5])


def _upload(x, lp):
    """the same steps x[steps, N, D], lp[steps, N] into both backends through save_step"""
    steps, N, D = x.shape
    out = []
    for b in (Backend(), DeviceBackend()):
        b.reset(N, D)
        b.grow(steps, None)
        for k in range(steps):
            b.save_step(emcee_b200.State(x[k], log_prob=lp[k]), np.zeros(N, dtype=bool))
        out.append(b)
    return out


def _crafted(steps, N, seed):
    rng = np.random.default_rng(seed)
    n = (steps, N)
    x = np.empty(n + (8,))
    x[..., 0] = 2.0                                                   # constant: all 64 bits by histogram
    x[..., 1] = rng.choice([-1.5, 4.0], n)                            # two distinct values
    x[..., 2] = rng.integers(-3, 4, n)                                # integers with heavy ties
    x[..., 3] = rng.choice(SPECIAL, n)                                # +-0, subnormals, +-1e308, +-inf
    x[..., 4] = rng.standard_normal(n)
    x[..., 5] = rng.standard_normal(n)
    x[steps // 2, N // 3, 5] = np.nan                                 # NaN in one parameter only
    base = np.float64(-1.2345).view(np.uint64) & ~np.uint64(0xFFFF)
    x[..., 6] = (base | rng.integers(0, 1 << 16, n).astype(np.uint64)).view(np.float64)  # top 48 bits shared
    x[..., 7] = rng.standard_normal(n) * 1e-310                       # subnormal spread
    lp = rng.standard_normal(n)
    lp[0, ::5] = -np.inf
    return x, lp


def _exact_stats(flat, ranks):
    srt = np.sort(flat, axis=0)
    v = srt[np.asarray(ranks, dtype=np.intp)]
    return np.where(v == 0, 0.0, v)


def test_crafted_chain_long_and_short_paths():
    steps, N = 200, 64  # 12 800 values per parameter
    x, lp = _crafted(steps, N, 11)
    h, d = _upload(x, lp)
    _percentiles_equal(h, d, [(0, 1), (7, 3), (150, 1), (190, 1)])
    flat = h.get_chain(flat=True)
    nan = np.isnan(flat).any(axis=0)
    assert nan.tolist() == [False] * 5 + [True] + [False] * 2
    assert np.all(np.isnan(d.get_percentile([10, 90])[:, 5]))
    ranks = np.array([0, 1, 6399, 12798, 12799], dtype=np.uint64)
    # long path: every column in one call; the constant column resolves all 64 bits, one histogram pass per byte
    v, has_nan, passes = d._chain.select("chain", 0, 1, steps, ranks)
    assert has_nan.tolist() == nan.tolist() and passes == 8
    want = _exact_stats(flat, ranks)
    ok = ~nan
    assert np.array_equal(v[:, ok].view(np.uint64), want[:, ok].view(np.uint64))
    # values sharing their top 48 bits: six histogram passes resolve them, a seventh splits the rest, then a
    # compaction
    h1, d1 = _upload(x[..., 6:7].copy(), lp)
    v, _, passes = d1._chain.select("chain", 0, 1, steps, ranks)
    assert passes == 8 and np.array_equal(v, _exact_stats(h1.get_chain(flat=True), ranks))
    # short path: at most 4 096 values per parameter are compacted by the first read
    v, _, passes = d._chain.select("chain", 150, 1, 50, np.array([0, 1600, 3199], dtype=np.uint64))
    assert passes == 1
    sub = h.get_chain(flat=True, discard=150)
    assert np.array_equal(v[:, ok], _exact_stats(sub, [0, 1600, 3199])[:, ok])
    # typical data: a few histogram passes, then a compaction
    h2, d2 = _upload(x[..., 4:5].copy(), lp)
    _, _, passes = d2._chain.select("chain", 0, 1, steps, ranks)
    assert 2 <= passes <= 4
    v, has_nan, _ = d._chain.select("log_prob", 0, 1, steps, ranks)
    assert v.shape == (5, 1) and not has_nan[0]
    assert np.array_equal(v[:, 0], _exact_stats(h.get_log_prob(flat=True), ranks))


def test_many_ranks_and_repeated_ranks():
    steps, N = 40, 257
    x, lp = _crafted(steps, N, 12)
    h, d = _upload(x, lp)
    q = np.linspace(0, 100, 997)  # ~2 000 ranks: more histogram groups than one CTA holds
    _same(d.get_percentile(q), h.get_percentile(q))
    ranks = np.array([5, 5, 10279, 0, 5], dtype=np.uint64)  # any order, repeats
    v, nan, _ = d._chain.select("chain", 0, 1, steps, ranks)
    want = _exact_stats(h.get_chain(flat=True), ranks)
    assert np.array_equal(v[:, ~nan], want[:, ~nan])


def test_scale_65536x128_two_segments():
    N, D = 65536, 128
    rng = np.random.default_rng(3)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=9, backend=DeviceBackend())
    st = s.run_mcmc(rng.standard_normal((N, D)), 16, skip_initial_state_check=True)
    s.run_mcmc(st, 16)
    flat = s.get_chain(flat=True, discard=2)
    q = [16, 50, 84]
    _same(s.get_percentile(q, discard=2), np.percentile(flat, q, axis=0))
    lp = s.get_log_prob(flat=True, discard=2)
    _same(s.get_percentile(q, discard=2, name="log_prob"), np.percentile(lp, q, axis=0))
    _, _, passes = s.backend._chain.select("chain", 2, 1, 30, np.array([0, 10 ** 6], dtype=np.uint64))
    print("65536 x 128, 30 stored steps: %d passes" % passes)
    mean, cov, n = s.get_moments(discard=2)
    assert n == flat.shape[0]
    np.testing.assert_allclose(mean, flat.mean(axis=0), rtol=1e-9, atol=1e-12)


# ---- moments against a long-double reference ---------------------------------------------------------------------
@pytest.mark.parametrize("N,D,calls,start,discard,thin",
                         [(301, 1, (12,), "near", 0, 1), (300, 129, (6, 5), "near", 1, 2),
                          (2048, 1024, (3,), "near", 0, 1), (300, 129, (40,), "far", 0, 1)],
                         ids=["D1", "D129-two-segments-thinned", "D1024", "D129-drift-1e4-sigma"])
def test_moments_exact(N, D, calls, start, discard, thin):
    """``get_moments`` against a two-pass reference of the stored slice, under the bound of
    ``test_gpu_proposals_exact.test_moments_exact`` with one accumulation per stored step (depth = rows one CTA
    stages + CTA partials + stored steps) and the shift = the column mean of the slice's first stored step."""
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here")
    rng = np.random.default_rng(N + D)
    X0 = rng.standard_normal((N, D))
    if start == "far":
        X0 += 1.0e4
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=0x40 + D, backend=DeviceBackend())
    st = X0
    for n in calls:
        st = s.run_mcmc(st, n, skip_initial_state_check=True)
    rows = s.get_chain(discard=discard, thin=thin)
    mean_d, cov_d, m = s.get_moments(discard=discard, thin=thin)
    assert m == rows.shape[0] * N
    X = rows.reshape(-1, D)
    shift = PX.colmean_device_order(rows[0])
    Y = X - shift
    depth, _, _ = PX.moments_depth(N, D, sm_count(), rows.shape[0])
    hi = np.array([math.fsum(X[:, k]) for k in range(D)])
    lo = np.array([math.fsum(np.r_[X[:, k], -hi[k]]) for k in range(D)])
    mean_ref = (hi.astype(np.longdouble) + lo.astype(np.longdouble)) / np.longdouble(m)
    aY = np.abs(Y)
    S1 = Y.sum(axis=0)
    U = PX.U
    b_mean = (U + PX.gamma(depth)) * aY.sum(axis=0) / m + 2 * U * np.abs(S1) / m + (U + PX.ULD) * np.abs(mean_d)
    tm = Tracker("slice moments mean N=%d D=%d %s" % (N, D, start))
    tm.check(np.abs(mean_d.astype(np.longdouble) - mean_ref).astype(np.float64), b_mean, "mean")
    i = np.r_[np.arange(D), np.zeros(D, np.int64), rng.integers(0, D, 1024)]
    j = np.r_[np.arange(D), np.arange(D), rng.integers(0, D, 1024)]
    Xc = X.astype(np.longdouble) - mean_ref
    ref = np.empty(len(i), dtype=np.longdouble)
    P = np.empty(len(i))
    for a in range(0, len(i), 256):
        sl = slice(a, a + 256)
        ref[sl] = np.sum(Xc[:, i[sl]] * Xc[:, j[sl]], axis=0) / np.longdouble(m - 1)
        P[sl] = np.sum(aY[:, i[sl]] * aY[:, j[sl]], axis=0)
    aS1 = np.abs(S1)
    dS1 = (U + PX.gamma(depth)) * aY.sum(axis=0)
    cov_ref = ref.astype(np.float64)
    b_cov = ((2 * U + PX.gamma(depth)) * P + (dS1[i] * aS1[j] + aS1[i] * dS1[j]) / m
             + 2 * U * aS1[i] * aS1[j] / m) / (m - 1) + 2 * U * np.abs(cov_ref)
    b_cov += PX.gamma(m + 2, PX.ULD) * P / (m - 1)
    tc = Tracker("slice moments cov N=%d D=%d %s" % (N, D, start))
    tc.check(np.abs(cov_d[i, j].astype(np.longdouble) - ref).astype(np.float64), b_cov, "cov")
    tm.report()
    tc.report()


# ---- error contracts -----------------------------------------------------------------------------------------------
def test_error_contracts():
    d = DeviceBackend()
    d.reset(8, 3)
    for fn in (lambda: d.get_percentile(50), lambda: d.get_moments()):
        with pytest.raises(AttributeError, match="store == True"):
            fn()
    h = Backend()
    h.reset(8, 3)
    rng = np.random.default_rng(0)
    for b in (h, d):
        b.grow(4, None)
        for _ in range(4):
            b.save_step(emcee_b200.State(rng.standard_normal((8, 3)), log_prob=np.zeros(8)), np.ones(8, dtype=bool))
        rng = np.random.default_rng(0)
    for q in (-1, 101, np.nan, [[[50]]], "a"):
        with pytest.raises(Exception) as want:
            h.get_percentile(q)
        with pytest.raises(type(want.value)) as got:
            d.get_percentile(q)
        assert str(got.value) == str(want.value)
    with pytest.raises(IndexError):  # an empty slice fails as np.percentile does
        d.get_percentile(50, discard=4)
    mean, cov, n = d.get_moments(discard=4)
    assert n == 0 and np.all(np.isnan(mean)) and np.all(np.isnan(cov))
    _same(d.get_percentile([]), h.get_percentile([]))
    with pytest.raises(ValueError):
        d.get_percentile(50, name="blobs")
    d.close()
    for fn in (lambda: d.get_percentile(50), lambda: d.get_moments()):
        with pytest.raises(ValueError, match="closed"):
            fn()
    wide = DeviceBackend()
    wide.reset(4, 1025)
    wide.grow(1, None)
    wide.save_step(emcee_b200.State(np.ones((4, 1025)), log_prob=np.zeros(4)), np.ones(4, dtype=bool))
    with pytest.raises(NotImplementedError):
        wide.get_moments()
    _same(wide.get_percentile(50), np.ones(1025))
    wide.close()
