"""``BatchSampler.get_histogram`` / ``get_histogram2d`` counted on the GPU (``eb_chain_histogram_segments``,
``eb_chain_histogram2d_segments``) against the host ``Backend``'s per-ensemble numpy route.

* The same batch stored into ``DeviceBackend()`` and into ``Backend()`` gives equal histograms (``==``, same dtypes)
  and edges, or the same exception, across K in {1, 3, 64, 1 024}, shapes 32 x 5, 37 x 3 and 64 x 8, the three
  moves, slices inside and across the two storage blocks of a backend grown by two calls, an empty slice, bins
  {1, 20, 4 096} (1-D) and {1, 20, 128} (2-D), the three ``range`` forms (one per-ensemble range excluding every value
  of its ensemble) and ``name="log_prob"``.
* K = 1 equals the twin ``EnsembleSampler``'s own ``DeviceBackend.get_histogram*``.
* A NaN in one ensemble raises that ensemble's exception; with explicit ranges its NaN values are dropped.
* K = 8 192 at 32 x 5, and 2-D counts that cannot fit: ``MemoryError``, after which the sampler still works.
"""
import numpy as np
import pytest

from test_gpu_batch import _p0, _seeds

import emcee_b200
from emcee_b200 import DeviceBackend, State, models, moves

pytestmark = pytest.mark.gpu

MOVES = {"stretch": moves.StretchMove, "de": moves.DEMove, "snooker": moves.DESnookerMove}


def _grown(K, N, D, move, seed=3):
    """A batch storing on the device and its host-stored twin, each grown by two ``run_mcmc`` calls (30 + 25
    steps): the device chain holds two storage blocks."""
    out = []
    for backend in (DeviceBackend(), None):
        s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), moves=MOVES[move](), seeds=_seeds(K, seed),
                                    backend=backend)
        s.run_mcmc(_p0(K, N, D, seed), 30, skip_initial_state_check=True)
        s.run_mcmc(None, 25, skip_initial_state_check=True)
        out.append(s)
    return out


def _outcome(fn):
    try:
        return True, fn()
    except Exception as e:  # noqa: B902 -- the exception itself is compared
        return False, (type(e), str(e))


def _assert_same(dev_fn, host_fn):
    ok_d, got = _outcome(dev_fn)
    ok_h, want = _outcome(host_fn)
    assert ok_d == ok_h, (got, want)
    if not ok_h:
        assert got == want
        return want
    for g, w in zip(got, want):
        if isinstance(w, list):
            assert g == w
            continue
        assert g.dtype == w.dtype and g.shape == w.shape
        assert np.array_equal(g, w)
    return want


def _ranges(host, K, D, name="chain"):
    """the three ``range`` forms: None, shared (some parameters autodetected), per ensemble from get_percentile
    (the last ensemble's excludes every value)"""
    if name == "log_prob":
        p = host.get_percentile([0.5, 99.5], name="log_prob")  # [K, 2]
        p[-1] = (1e6, 2e6)
        return [None, (float(p[:, 0].min()), float(p[:, 1].max())), p]
    p = np.moveaxis(host.get_percentile([0.5, 99.5]), 1, 2).copy()  # [K, D, 2]
    p[-1] = (50.0, 60.0)
    shared = [None if d % 2 else (-1.0 + 0.1 * d, 1.0) for d in range(D)]
    return [None, shared, p]


CASES = [(1, 32, 5, "stretch"), (3, 37, 3, "de"), (3, 32, 5, "snooker"), (64, 64, 8, "snooker"),
         (64, 32, 5, "de"), (1024, 32, 5, "stretch")]
SLICES = [(0, 1), (10, 3), (33, 2), (55, 1)]  # whole, across the two blocks, second block only, empty


@pytest.mark.parametrize("K,N,D,move", CASES)
def test_histogram_equals_host(K, N, D, move):
    dev, host = _grown(K, N, D, move)
    big = K >= 1024
    for discard, thin in SLICES[1:2] if big else SLICES:
        for bins in (1, 20, 4096):
            kw = dict(bins=bins, discard=discard, thin=thin)
            _assert_same(lambda: dev.get_histogram(**kw), lambda: host.get_histogram(**kw))
        for bins in (1, 20) if big else (1, 20, 128):
            kw = dict(bins=bins, discard=discard, thin=thin)
            _assert_same(lambda: dev.get_histogram2d(**kw), lambda: host.get_histogram2d(**kw))
    for name in ("chain", "log_prob"):
        for rng in _ranges(host, K, D, name):
            for discard, thin in ((10, 3), (55, 1)):
                kw = dict(bins=20, range=rng, discard=discard, thin=thin, name=name)
                h, e = _assert_same(lambda: dev.get_histogram(**kw), lambda: host.get_histogram(**kw))
                assert h.shape[0] == K and e.shape[0] == K
    params = [D - 1, 0, 1] if D > 2 else None
    for rng in _ranges(host, K, D):
        kw = dict(params=params, bins=20, range=rng, discard=10, thin=3)
        _assert_same(lambda: dev.get_histogram2d(**kw), lambda: host.get_histogram2d(**kw))


def test_excluded_ensemble_counts_nothing():
    K, N, D = 3, 32, 5
    dev, host = _grown(K, N, D, "stretch")
    rng = np.moveaxis(host.get_percentile([0, 100]), 1, 2).copy()
    rng[1] = (50.0, 60.0)
    h, e = _assert_same(lambda: dev.get_histogram(bins=7, range=rng), lambda: host.get_histogram(bins=7, range=rng))
    assert h[1].sum() == 0 and np.all(h[[0, 2]].sum(axis=2) == 55 * N)
    h2, _, _ = _assert_same(lambda: dev.get_histogram2d(bins=7, range=rng),
                            lambda: host.get_histogram2d(bins=7, range=rng))
    assert h2[1].sum() == 0 and np.all(h2[[0, 2]].sum(axis=(2, 3)) == 55 * N)


@pytest.mark.parametrize("move", ["stretch", "de", "snooker"])
def test_one_ensemble_equals_twin(move):
    N, D = 32, 5
    seed = _seeds(1, 8)[0]
    b = emcee_b200.BatchSampler(1, N, D, models.GaussianIso(), moves=MOVES[move](), seeds=[seed],
                                backend=DeviceBackend())
    t = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=MOVES[move](), seed=seed,
                                   backend=DeviceBackend())
    p0 = _p0(1, N, D, 8)
    b.run_mcmc(p0, 40, skip_initial_state_check=True)
    t.run_mcmc(p0[0], 40, skip_initial_state_check=True)
    assert np.array_equal(b.get_chain()[:, 0], t.get_chain())
    for kw in (dict(bins=20), dict(bins=4096, discard=5, thin=2), dict(bins=20, name="log_prob"),
               dict(bins=3, range=[(-1.0, 1.0)] * D)):
        h, e = b.get_histogram(**kw)
        th, te = t.backend.get_histogram(**kw)
        assert np.array_equal(h[0], th) and np.array_equal(e[0], te) and h.dtype == th.dtype
    for kw in (dict(bins=20), dict(params=[3, 1], bins=128, discard=5, thin=2)):
        h, e, pairs = b.get_histogram2d(**kw)
        th, te, tpairs = t.backend.get_histogram2d(**kw)
        assert np.array_equal(h[0], th) and np.array_equal(e[0], te) and pairs == tpairs


def _nan_batch(backend_cls, K, N, D, n, j, d):
    """A batch over a chain written directly, with ensemble ``j``'s parameter ``d`` NaN at one stored value."""
    rng = np.random.default_rng(5)
    x = rng.normal(size=(n, K, N, D))
    x[3, j, 4, d] = np.nan
    lp = rng.normal(size=(n, K, N))
    b = backend_cls()
    b.reset(K * N, D)
    b.grow(n, None)
    for s in range(n):
        b.save_step(State(x[s].reshape(K * N, D), log_prob=lp[s].reshape(K * N), random_state=None),
                    np.zeros(K * N, dtype=bool))
    return emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, backend=b)


def test_nan_in_one_ensemble():
    K, N, D, n = 4, 8, 3, 6
    dev = _nan_batch(DeviceBackend, K, N, D, n, 2, 1)
    host = _nan_batch(emcee_b200.Backend, K, N, D, n, 2, 1)
    for call in (lambda s: s.get_histogram(), lambda s: s.get_histogram2d()):
        ok, err = _outcome(lambda: call(host))
        assert not ok and "autodetected range of [nan, nan]" in err[1]
        _assert_same(lambda: call(dev), lambda: call(host))
    rng = np.tile([-1.5, 1.5], (K, D, 1))
    h, _ = _assert_same(lambda: dev.get_histogram(bins=9, range=rng), lambda: host.get_histogram(bins=9, range=rng))
    assert h[2, 1].sum() <= n * N - 1  # the NaN is dropped
    h2, _, _ = _assert_same(lambda: dev.get_histogram2d(bins=9, range=rng),
                            lambda: host.get_histogram2d(bins=9, range=rng))
    assert h2.shape == (K, 3, 9, 9) and h2[2, 0].sum() <= n * N - 1


def test_scale_8192():
    K, N, D = 8192, 32, 5
    out = []
    for backend in (DeviceBackend(), None):
        s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=_seeds(K, 4), backend=backend)
        s.run_mcmc(_p0(K, N, D, 4), 12, skip_initial_state_check=True)
        out.append(s)
    dev, host = out
    _assert_same(lambda: dev.get_histogram(bins=20), lambda: host.get_histogram(bins=20))
    _assert_same(lambda: dev.get_histogram(bins=20, name="log_prob"),
                 lambda: host.get_histogram(bins=20, name="log_prob"))
    _assert_same(lambda: dev.get_histogram2d(params=[0, 3, 4], bins=20),
                 lambda: host.get_histogram2d(params=[0, 3, 4], bins=20))


def test_counts_that_cannot_fit():
    K, N, D = 512, 128, 64  # 2-D counts at bins 128: 512 * 2016 pairs * 128^2 * 8 bytes = 135 GB
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, backend=DeviceBackend())
    p0 = _p0(K, N, D)
    s.run_mcmc(p0, 2, skip_initial_state_check=True)
    with pytest.raises(MemoryError):
        s.get_histogram2d(bins=128)
    s.run_mcmc(None, 2, skip_initial_state_check=True)
    assert s.iteration == 4
    h, e, pairs = s.get_histogram2d(params=[0, 1], bins=20)
    assert h.shape == (K, 1, 20, 20) and np.all(h.sum(axis=(1, 2, 3)) == 4 * N)


def test_nseg_must_divide_walkers():
    s = emcee_b200.BatchSampler(4, 8, 2, models.GaussianIso(), seeds=1, backend=DeviceBackend())
    s.run_mcmc(_p0(4, 8, 2), 5, skip_initial_state_check=True)
    ch = s.backend._ch  # 32 walkers
    for nseg in (0, 3, 33):
        with pytest.raises(ValueError, match="nseg"):
            ch.histogram("chain", 0, 1, 5, 4, np.zeros((nseg * 2, 3)), np.zeros((nseg * 2, 5)), nseg=nseg)
        with pytest.raises(ValueError, match="nseg"):
            ch.histogram2d(0, 1, 5, [0, 1], 4, np.zeros((nseg * 2, 5)), nseg=nseg)
