"""Histograms of a stored device chain (``DeviceBackend.get_histogram`` / ``get_histogram2d``;
``eb_chain_histogram``, ``eb_chain_histogram2d``) against the host ``Backend``'s numpy expressions, with
``np.array_equal`` and equal dtypes for counts and edges.

* Twin runs into ``Backend()`` and ``DeviceBackend()``: a ``discard`` / ``thin`` grid, resumed runs (several
  segments), odd ``nwalkers``, ndim 1, 7, 128 and 257, ``"chain"`` and ``"log_prob"``, ``range=None`` and ranges that
  cut the data, ``bins`` 1 / 10 / 20 / 4096 (1-D) and 1 / 20 / 128 (2-D), ``params`` subsets out of order; and a
  bounded model that stores ``-inf`` log-probabilities.
* Crafted chains uploaded with ``save_step``: values on the edges and one ulp either side, NaN (numpy's
  ``ValueError`` when the range is autodetected, dropped under a given range), +-inf, constant columns.
* Limits: ``bins`` 4097 / 129 raise ``NotImplementedError``; a column holding +-1.5e308 raises the overflow
  ``ValueError``.
* 65 536 x 128 over two segments: 1-D of every parameter and 2-D of ``params=range(16)`` against numpy, and all
  8 128 pairs on the device, spot-checked.
"""
import itertools

import numpy as np
import pytest

from oracle import targets as T
from test_gpu_bounds import _box_and_p0

from gpu_util import device_model

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, models

pytestmark = pytest.mark.gpu


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, list):
            assert g == w
            continue
        assert g.dtype == w.dtype and g.shape == w.shape
        assert np.array_equal(g, w)


def _both(h, d, fn):
    """fn(backend) on both backends: equal results, or the same exception type and message"""
    try:
        want = fn(h)
    except Exception as e:  # noqa: B902
        with pytest.raises(type(e)) as got:
            fn(d)
        assert str(got.value) == str(e)
        return
    _same(fn(d), want)


def _twin(N, D, model, p0, seed, calls):
    out = []
    for backend in (Backend(), DeviceBackend()):
        s = emcee_b200.EnsembleSampler(N, D, model, seed=seed, backend=backend)
        st = p0
        for n in calls:
            st = s.run_mcmc(st, n, skip_initial_state_check=True)
        out.append(s)
    h, d = out
    assert np.array_equal(h.get_chain(), d.get_chain())
    return h, d


def _grid(it):
    pairs = {(0, 1), (1, 1), (3, 2), (it // 2, 3), (it - 1, 1), (0, it), (2, 7), (it, 1)}  # (it, 1): empty slice
    return sorted((d, t) for d, t in pairs if d + t - 1 <= it)


def _cutting_ranges(h, D, dtype=float):
    """ranges that cut the data: the middle of each column's spread (as float, or as numpy float32 scalars, which
    numpy subtracts in float32)"""
    flat = h.get_chain(flat=True)
    lo, hi = np.percentile(flat, [20, 70], axis=0)
    return [(dtype(lo[d]), dtype(hi[d])) for d in range(D)]


@pytest.mark.parametrize("N,D,calls", [(33, 1, (6, 5, 4)), (63, 7, (10, 9)), (513, 128, (5, 4)), (515, 257, (3, 3))],
                         ids=["N33-D1", "N63-D7", "N513-D128", "N515-D257"])
def test_twin_histograms(N, D, calls):
    rng = np.random.default_rng(N + D)
    h, d = _twin(N, D, models.GaussianIso(), rng.standard_normal((N, D)), 0x4A + D, calls)
    cut, cut32 = _cutting_ranges(h, D), _cutting_ranges(h, D, np.float32)
    lp = h.get_log_prob(flat=True)
    lp_cut = (float(np.percentile(lp, 10)), float(np.percentile(lp, 60)))
    lp_cut32 = tuple(np.float32(v) for v in lp_cut)
    for discard, thin in _grid(h.iteration):
        kw = dict(discard=discard, thin=thin)
        for bins in (1, 10, 20, 4096):
            for rng_ in (None, cut, cut32):
                _both(h, d, lambda b: b.get_histogram(bins, rng_, **kw))
            for rng_ in (None, lp_cut, lp_cut32):
                _both(h, d, lambda b: b.get_histogram(bins, rng_, name="log_prob", **kw))
        if D < 2:
            continue
        subsets = [None] if D <= 7 else [[5, 0, 3], list(range(0, D, D // 9))[::-1]]
        for params in subsets + [[D - 1, 0]]:
            for bins in (1, 20, 128):
                for rng_ in (None, cut, cut32):
                    _both(h, d, lambda b: b.get_histogram2d(params, bins, rng_, **kw))


def test_float32_range_top_edge():
    """numpy's float32-scalar range: its norm_denom is the float32 difference, so values at the top edge give
    f > bins, which numpy truncates and counts in the last bin"""
    steps, N = 6, 40
    rng = np.random.default_rng(32)
    lo, hi = np.float32(-0.3), np.float32(0.1)
    x = rng.uniform(-0.4, 0.2, (steps, N, 2))
    x[0, :3, 0] = (float(hi), 0.0, float(lo))
    x[1, :10, 1] = float(hi)
    x[2, :10, 1] = np.nextafter(float(hi), -1.0)
    h, d = _upload(x, rng.standard_normal((steps, N)))
    for bins in (1, 10, 20, 4096):
        _both(h, d, lambda b: b.get_histogram(bins, [(lo, hi), (lo, hi)]))
        _both(h, d, lambda b: b.get_histogram(bins, [(lo, hi), (lo, hi)], discard=1, thin=2))
        _both(h, d, lambda b: b.get_histogram(bins, (lo, hi), name="log_prob"))
    for bins in (1, 10, 128):
        _both(h, d, lambda b: b.get_histogram2d(None, bins, [(lo, hi), (lo, hi)]))
    want = np.histogram(h.get_chain(flat=True)[:, 0], 1, range=(lo, hi))[0]
    assert want[0] > 0 and np.array_equal(d.get_histogram(1, [(lo, hi), (lo, hi)])[0][0], want)


def test_twin_bounded_stores_minus_inf():
    N, D = 2 * (8 * 20 + 1), 32
    target, p0 = T.make_config("ring", N, D)
    lo, hi, pb = _box_and_p0(target, p0, 0)
    model = models.Bounded(device_model("ring", target=target), lo, hi)
    h, d = _twin(N, D, model, pb, 0x57, (6, 5))
    assert np.isneginf(d.get_log_prob()[0]).any()
    # autodetected: numpy's "autodetected range of [-inf, ...] is not finite"; a given range drops -inf
    with pytest.raises(ValueError, match="autodetected range of \\[-inf"):
        d.get_histogram(name="log_prob")
    for kw in (dict(), dict(discard=3, thin=2)):
        _both(h, d, lambda b: b.get_histogram(name="log_prob", **kw))
        _both(h, d, lambda b: b.get_histogram(20, (-50.0, 0.0), name="log_prob", **kw))
        _both(h, d, lambda b: b.get_histogram(20, **kw))
        _both(h, d, lambda b: b.get_histogram2d([4, 1, 30], 20, **kw))


# ---- crafted chains ------------------------------------------------------------------------------------------------
def _upload(x, lp):
    steps, N, D = x.shape
    out = []
    for b in (Backend(), DeviceBackend()):
        b.reset(N, D)
        b.grow(steps, None)
        for k in range(steps):
            b.save_step(emcee_b200.State(x[k], log_prob=lp[k]), np.zeros(N, dtype=bool))
        out.append(b)
    return out


def _on_edges(rng, n, lo, hi, bins):
    e = np.linspace(lo, hi, bins + 1)
    v = np.r_[e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf)]
    return rng.choice(v, n)


def test_crafted_edges_nan_inf_constant():
    steps, N = 40, 65
    rng = np.random.default_rng(21)
    n = (steps, N)
    x = np.empty(n + (7,))
    x[..., 0] = _on_edges(rng, n, -1.0, 1.0, 10)          # on numpy's edges for bins=10 over [-1, 1], and +-1 ulp
    x[..., 1] = _on_edges(rng, n, 0.1, 0.7, 20)
    x[..., 2] = 2.5                                       # constant: widened by 0.5
    x[..., 3] = rng.standard_normal(n)
    x[7, 3, 3] = np.nan                                   # NaN: numpy's ValueError autodetected, dropped in a range
    x[..., 4] = rng.standard_normal(n)
    x[0, 1, 4] = np.inf                                   # +inf
    x[..., 5] = rng.choice([0.0, -0.0, 5e-324, -5e-324, 1e-310], n)  # zeros and subnormals
    x[..., 6] = rng.integers(-3, 4, n)                    # integer ties on the edges of [-3, 3]
    lp = rng.standard_normal(n)
    h, d = _upload(x, lp)
    given = [(-1.0, 1.0), (0.1, 0.7), (2.0, 3.0), (-1.0, 1.0), (-2.0, 2.0), (-1e-310, 1e-310), (-3, 3)]
    ok = [0, 1, 2, 5, 6]
    with pytest.raises(ValueError, match="autodetected range of \\[nan, nan\\]"):
        d.get_histogram()
    for kw in (dict(), dict(discard=4, thin=3), dict(discard=39)):
        for bins in (1, 3, 10, 20, 4096):
            _both(h, d, lambda b: b.get_histogram(bins, given, **kw))
            _both(h, d, lambda b: b.get_histogram(bins, **kw))  # numpy's NaN error, except in the last step alone
        for bins in (1, 10, 20, 128):
            _both(h, d, lambda b: b.get_histogram2d(None, bins, given, **kw))
            _both(h, d, lambda b: b.get_histogram2d(ok[::-1], bins, None, **kw))
            _both(h, d, lambda b: b.get_histogram2d([0, 3], bins, None, **kw))  # NaN column: numpy's ValueError
            _both(h, d, lambda b: b.get_histogram2d([4, 0], bins, None, **kw))  # +inf column
    # each parameter alone with an autodetected range, where numpy can form one
    for p in ok:
        h1, d1 = _upload(x[..., p:p + 1].copy(), lp)
        for bins in (1, 10, 4096):
            _both(h1, d1, lambda b: b.get_histogram(bins))
            _both(h1, d1, lambda b: b.get_histogram(bins, name="log_prob"))


def test_limits_and_overflow():
    steps, N, D = 3, 16, 3
    rng = np.random.default_rng(5)
    x = rng.standard_normal((steps, N, D))
    x[1, 2, 1], x[2, 5, 1] = -1.5e308, 1.5e308
    h, d = _upload(x, rng.standard_normal((steps, N)))
    with pytest.raises(NotImplementedError, match="4096"):
        d.get_histogram(4097, [(-1, 1)] * D)
    with pytest.raises(NotImplementedError, match="128"):
        d.get_histogram2d(bins=129)
    for fn in (lambda: d.get_histogram(), lambda: d.get_histogram(1), lambda: d.get_histogram2d(),
               lambda: d.get_histogram2d([1, 0], bins=1)):
        with pytest.raises(ValueError, match="wider than the largest double"):
            fn()
    # the other columns are fine, and so is a given range for the wide one
    _both(h, d, lambda b: b.get_histogram(10, [(-1, 1), (-8e307, 8e307), (-3, 3)]))
    _both(h, d, lambda b: b.get_histogram2d([2, 0], 20))
    _both(h, d, lambda b: b.get_histogram2d(None, 20, [(-1, 1), (-8e307, 8e307), (-3, 3)]))
    for fn in (lambda b: b.get_histogram(0), lambda b: b.get_histogram2d(bins=0), lambda b: b.get_histogram(2.5),
               lambda b: b.get_histogram(10, [(1, 0)] * D), lambda b: b.get_histogram(10, [(0, np.inf)] * D)):
        _both(h, d, fn)
    with pytest.raises(ValueError):
        d.get_histogram2d([0, 0])
    with pytest.raises(ValueError):
        d.get_histogram(range=[(0, 1)])


# ---- scale -------------------------------------------------------------------------------------------------------
def test_scale_65536x128_two_segments():
    N, D = 65536, 128
    rng = np.random.default_rng(3)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=9, backend=DeviceBackend())
    st = s.run_mcmc(rng.standard_normal((N, D)), 8, skip_initial_state_check=True)
    s.run_mcmc(st, 8)
    flat = s.get_chain(flat=True, discard=2)
    h, e = s.get_histogram(20, discard=2)
    for k in range(D):
        wh, we = np.histogram(flat[:, k], 20)
        assert np.array_equal(h[k], wh) and np.array_equal(e[k], we)
    params = list(range(16))
    h2, e2, pairs = s.get_histogram2d(params, 20, discard=2)
    assert pairs == list(itertools.combinations(params, 2))
    for p, (i, j) in enumerate(pairs):
        wh, wx, wy = np.histogram2d(flat[:, i], flat[:, j], 20)
        assert np.array_equal(h2[p], wh) and np.array_equal(e2[i], wx) and np.array_equal(e2[j], wy)
    ha, ea, pa = s.get_histogram2d(None, 20, discard=2)
    assert ha.shape == (8128, 20, 20) and len(pa) == 8128
    assert np.all(ha.sum(axis=(1, 2)) == flat.shape[0])  # autodetected ranges hold every value
    for p in (0, 1, 127, 4000, 8127):
        i, j = pa[p]
        wh, _, _ = np.histogram2d(flat[:, i], flat[:, j], 20)
        assert np.array_equal(ha[p], wh)
