"""Host side of ``BatchSampler.get_histogram`` / ``get_histogram2d``.

* ``summary.uniform_edges`` / ``searched_edges`` over arrays of columns equal the one-column numpy calls bit for bit
  (``outer`` and ``edges`` compared as int64 views), including constant huge columns (``np.linspace``'s step-0
  branch) beside ordinary ones, subnormal spans, infinities, NaN flags, float32 ranges and ranges of other types, at
  bins 1, 20 and 4 096; a failing column raises what the first failing column raises under the per-column loop.
* The host ``Backend`` route: row ``k`` is numpy on ensemble ``k``'s flat slice, for 1-D, ``log_prob`` and 2-D, in
  the three ``range`` forms; other shapes raise ``ValueError``.
* The ``DeviceBackend`` route over a stand-in chain: the ``nseg`` passed down, the column layout of the edge tables,
  the reshapes, the error precedence (lowest ensemble, then parameter) and no device call for an empty slice.
"""
import itertools

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import DeviceBackend, _lib, models
from emcee_b200 import summary as S

from test_batch_device_backend_host import _Chain, _StoreEngine
from test_batch_host import _Engine, _p0


def _outcome(fn):
    try:
        return True, fn()
    except Exception as e:  # noqa: B902 -- the exception itself is compared
        return False, (type(e), str(e))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


# ---- 1. edges of many columns ----------------------------------------------------------------------------------------
def _random_columns(rng, C):
    lo = rng.standard_normal(C) * 10.0 ** rng.integers(-300, 300, C)
    hi = lo + np.abs(rng.standard_normal(C)) * 10.0 ** rng.integers(-300, 300, C)
    hi[::7] = lo[::7]  # equal min / max: widened by 0.5
    lo[::11] = hi[::11] = 1e17  # constant and huge: the widening is lost, np.linspace's step is 0
    lo[5], hi[5] = 5e-324, 1e-323  # a subnormal span
    lo[13], hi[13] = -3.0, -3.0
    nan = np.zeros(C, dtype=bool)
    nan[17::97] = True
    ranges = [None] * C
    for c in range(0, C, 3):
        ranges[c] = (float(lo[c]) - 1.0, float(hi[c]) + 1.0)
    for c in range(1, C, 13):
        ranges[c] = (np.float32(-0.3), np.float32(0.1))  # float32 arithmetic, float32 norm_denom
    for c in range(2, C, 17):
        ranges[c] = (0, 0)  # Python ints, an empty range
    for c in range(4, C, 19):
        ranges[c] = (np.int64(-2), np.int64(3))  # formed by numpy alone
    for c in range(8, C, 23):
        ranges[c] = (np.float32(1.0), 2.5)  # mixed types: formed by numpy alone
    return lo, hi, nan, ranges


def _check_columns(bins, ranges, lo, hi, nan):
    """the column form against the one-column form, which is numpy on the [min; max] stand-in"""
    C = len(lo)
    for vec, two_d in ((S.uniform_edges, False), (S.searched_edges, True)):
        if two_d and bins > S.HIST2_BINS_MAX:
            continue
        per = [_outcome(lambda: vec(bins, ranges[c], lo[c], hi[c], nan[c])) for c in range(C)]
        good = [c for c in range(C) if per[c][0]]
        got = vec(bins, [ranges[c] for c in good], lo[good], hi[good], nan[good])
        for i, c in enumerate(good):
            want = per[c][1]
            if two_d:
                assert got.dtype == np.float64 and np.array_equal(_bits(got[i]), _bits(want)), c
            else:
                assert np.array_equal(_bits(got[0][i]), _bits(want[0])), c
                assert np.array_equal(_bits(got[1][i]), _bits(want[1])), c
        bad = [c for c in range(C) if not per[c][0]]
        if bad:
            assert _outcome(lambda: vec(bins, ranges, lo, hi, nan)) == per[bad[0]]


@pytest.mark.parametrize("bins", [1, 20, 4096])
def test_column_edges_equal_one_column_calls(bins):
    rng = np.random.default_rng(bins)
    lo, hi, nan, ranges = _random_columns(rng, 300)
    _check_columns(bins, ranges, lo, hi, nan)
    # infinities, the step-0 columns and the failing ones dropped: the rest in one call
    with np.errstate(invalid="ignore"):
        keep = [c for c in range(300) if _outcome(lambda: S.uniform_edges(bins, ranges[c], lo[c], hi[c], nan[c]))[0]]
    _check_columns(bins, [ranges[c] for c in keep], lo[keep], hi[keep], nan[keep])


def test_one_column_equals_numpy():
    """the one-column form is still numpy's np.histogram / np.histogram2d edges of a whole column"""
    rng = np.random.default_rng(4)
    cols = [rng.standard_normal(200), np.full(200, 1e17), np.r_[rng.standard_normal(199), np.inf],
            np.full(200, 2.5), rng.standard_normal(200) * 1e-310]
    for c in cols:
        for given in (None, (-1.0, 1.0), (np.float32(-0.3), np.float32(0.1))):
            for bins in (1, 20, 4096):
                args = (bins, given, np.min(c), np.max(c), False)
                ok, got = _outcome(lambda: S.uniform_edges(*args))
                okw, want = _outcome(lambda: np.histogram(c, bins, range=given)[1])
                assert ok == okw and (np.array_equal(_bits(got[1]), _bits(want)) if ok else got == want)
                if bins <= 128:
                    ok, got = _outcome(lambda: S.searched_edges(*args))
                    okw, want = _outcome(lambda: np.histogram2d(c, c, bins, range=None if given is None
                                                                else [given, given])[1])
                    assert ok == okw and (np.array_equal(_bits(got), _bits(want)) if ok else got == want)


def test_step_zero_columns_beside_others():
    """np.linspace of array endpoints switches every row to ``y / div * delta`` when one row's step is 0; the
    constant huge columns are formed apart, so the others keep numpy's one-column edges"""
    lo = np.array([0.1, 1e17, -3.7, 1e17, 2.0])
    hi = np.array([0.7, 1e17, 5.1, 1e17, 2.0])
    nan = np.zeros(5, dtype=bool)
    e = S.searched_edges(20, None, lo, hi, nan)
    for c in range(5):
        assert np.array_equal(_bits(e[c]), _bits(S.searched_edges(20, None, lo[c], hi[c], False)))
    assert np.all(e[1] == 1e17)
    with pytest.raises(ValueError, match="Too many bins"):
        S.uniform_edges(20, None, lo, hi, nan)
    ok = [0, 2, 4]
    o, e = S.uniform_edges(20, None, lo[ok], hi[ok], nan[ok])
    for i, c in enumerate(ok):
        w = S.uniform_edges(20, None, lo[c], hi[c], False)
        assert np.array_equal(_bits(o[i]), _bits(w[0])) and np.array_equal(_bits(e[i]), _bits(w[1]))


def test_float32_range_array():
    rng = np.random.default_rng(9)
    r = np.sort(rng.standard_normal((50, 2)), axis=1)
    for a in (r, r.astype(np.float32)):
        for bins in (1, 20, 4096):
            o, e = S.uniform_edges(bins, a, np.full(50, np.nan), np.full(50, np.nan), np.zeros(50, dtype=bool))
            for c in range(50):
                w = np.histogram(np.empty(0), bins, range=a[c])[1]
                assert np.array_equal(_bits(e[c]), _bits(w))
                assert o[c, 2] == np.subtract(a[c, 1], a[c, 0])  # numpy's norm_denom, in the range's dtype


@pytest.mark.parametrize("pos", [0, 3, 9])
def test_first_failing_column_raises(pos):
    C = 10
    lo, hi, nan = np.zeros(C), np.ones(C), np.zeros(C, dtype=bool)
    for kind in ("nan", "inf", "reversed", "overflow"):
        ranges = [None] * C
        if pos + 1 < C:  # a later column fails differently: it must not be the one reported
            ranges[pos + 1] = (2.0, 1.0)
        n2 = nan.copy()
        lo2 = lo.copy()
        if kind == "nan":
            n2[pos] = True
        elif kind == "inf":
            lo2[pos] = -np.inf
        elif kind == "reversed":
            ranges[pos] = (1.0, 0.0)
        else:
            ranges[pos] = (-1.7e308, 1.7e308)
        for fn in (S.uniform_edges, S.searched_edges):
            got = _outcome(lambda: fn(10, ranges, lo2, hi, n2))
            want = _outcome(lambda: fn(10, ranges[pos], lo2[pos], hi[pos], n2[pos]))
            assert not got[0] and got == want, (kind, pos, got, want)


def test_running_plan_uses_the_column_form():
    cfg = S.running_histogram_plan(3, [(-1.0, 1.0), (0.0, 0.0), (np.float32(0.1), np.float32(0.7))], bins=20,
                                   log_prob_range=(-5, 0), params2d=[2, 0], bins2d=8)
    rows = [(-1.0, 1.0), (0.0, 0.0), (np.float32(0.1), np.float32(0.7)), (-5, 0)]
    for d, r in enumerate(rows):
        assert np.array_equal(cfg["edges"][d], np.histogram(np.empty(0), 20, range=r)[1])
    for k, p in enumerate([2, 0]):
        want = np.histogram2d(np.empty(0), np.empty(0), 8, range=[rows[p], rows[p]])[1]
        assert np.array_equal(cfg["edges2d"][k], want)


# ---- 2. host Backend route -------------------------------------------------------------------------------------------
class _Random(_Engine):
    def _advance(self):
        self.step_count += 1
        rng = np.random.default_rng(self.step_count)
        self.x = rng.normal(size=(self.nwalkers, self.ndim))
        self.lp = rng.normal(size=self.nwalkers)


class _RandomStore(_StoreEngine, _Random):
    pass


def _batch(K, N, D, **kw):
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, **kw)
    s.run_mcmc(_p0(K, N, D), 12, skip_initial_state_check=True)
    return s


def _range_forms(K, D, log_prob=False):
    rng = np.random.default_rng(2)
    if log_prob:
        per = np.sort(rng.normal(size=(K, 2)), axis=1)
        return [None, (-1.0, 1.0), per, (-1, 1)]
    per = np.sort(rng.normal(size=(K, D, 2)), axis=2)
    per[0, 0] = (50.0, 60.0)  # excludes every value
    return [None, [(-1.0, 1.0)] * D, [None if d % 2 else (-0.5, 0.5 + d) for d in range(D)], per, per.tolist()]


def _per_ensemble(rng):
    """the per-ensemble form: an array, or nested lists of one"""
    return isinstance(rng, np.ndarray) or (isinstance(rng, list) and isinstance(rng[0], list))


def _numpy_1d(flat, k, d, bins, r):
    return np.histogram(flat[k][:, d] if d is not None else flat[k], bins=bins, range=r)


@pytest.mark.parametrize("discard,thin", [(0, 1), (3, 2)])
def test_host_route_is_numpy_per_ensemble(monkeypatch, discard, thin):
    monkeypatch.setattr(_lib, "BatchEngine", _Random)
    K, N, D = 4, 6, 3
    s = _batch(K, N, D)
    flat = s.get_chain(flat=True, discard=discard, thin=thin)
    flat_lp = s.get_log_prob(flat=True, discard=discard, thin=thin)
    for rng in _range_forms(K, D):
        h, e = s.get_histogram(bins=5, range=rng, discard=discard, thin=thin)
        assert h.shape == (K, D, 5) and e.shape == (K, D, 6) and h.dtype == np.int64 and e.dtype == np.float64
        for k in range(K):
            for d in range(D):
                r = None if rng is None else (rng[k][d] if _per_ensemble(rng) else rng[d])
                wh, we = _numpy_1d(flat, k, d, 5, r)
                assert np.array_equal(h[k, d], wh) and np.array_equal(e[k, d], we)
        for params in (None, [2, 0], [1, 2, 0]):
            h2, e2, pairs = s.get_histogram2d(params=params, bins=4, range=rng, discard=discard, thin=thin)
            P = list(range(D)) if params is None else params
            assert pairs == list(itertools.combinations(P, 2)) and h2.dtype == np.float64
            for k in range(K):
                rr = None if rng is None else (rng[k] if _per_ensemble(rng) else rng)
                for p, (i, j) in enumerate(pairs):
                    wh, wi, wj = np.histogram2d(flat[k][:, i], flat[k][:, j], bins=4,
                                                range=None if rr is None else [rr[i], rr[j]])
                    assert np.array_equal(h2[k, p], wh)
                    assert np.array_equal(e2[k, P.index(i)], wi) and np.array_equal(e2[k, P.index(j)], wj)
    for rng in _range_forms(K, D, log_prob=True):
        h, e = s.get_histogram(bins=5, range=rng, discard=discard, thin=thin, name="log_prob")
        assert h.shape == (K, 5) and e.shape == (K, 6)
        for k in range(K):
            r = None if rng is None else (rng[k] if _per_ensemble(rng) else rng)
            wh, we = _numpy_1d(flat_lp, k, None, 5, r)
            assert np.array_equal(h[k], wh) and np.array_equal(e[k], we)


@pytest.mark.parametrize("device", [False, True])
def test_bad_range_shapes(monkeypatch, device):
    monkeypatch.setattr(_lib, "BatchEngine", _RandomStore)
    monkeypatch.setattr(_lib, "Chain", _CountingChain)
    K, N, D = 3, 6, 2
    s = _batch(K, N, D, backend=DeviceBackend() if device else None)
    _CountingChain.calls = []
    for rng in ([(-1, 1)] * (D + 1), np.zeros((K, D, 3)), np.zeros((K + 1, D, 2)), np.zeros((D, 3)),
                [(-1, 1, 2), None], np.zeros((K, 2))):
        with pytest.raises(ValueError, match="range"):
            s.get_histogram(range=rng)
        with pytest.raises(ValueError, match="range"):
            s.get_histogram2d(range=rng)
    for rng in ((-1, 1, 2), np.zeros((K, 3)), np.zeros((K, D, 2)), [(0, 1)]):
        with pytest.raises(ValueError, match="range"):
            s.get_histogram(range=rng, name="log_prob")
    with pytest.raises(ValueError, match="histograms are taken of"):
        s.get_histogram(name="blobs")
    assert _CountingChain.calls == []


# ---- 3. DeviceBackend route over a stand-in chain --------------------------------------------------------------------
class _CountingChain(_Chain):
    """``_Chain`` with the summaries ``BatchSampler`` reaches: the selection and the two counts, in numpy, each
    recorded with the ``nseg`` and table shapes it was given."""

    calls = []

    def _flat(self, what, first, stride, count, nseg):
        x, lp = self.read(first, stride, count)
        v = x if what == "chain" else lp[..., None]
        n, W = v.shape[:2]
        return np.swapaxes(v.reshape(n, nseg, W // nseg, -1), 0, 1).reshape(nseg, n * (W // nseg), -1)

    def select(self, what, first, stride, count, ranks, nseg=1):
        _CountingChain.calls.append(("select", nseg, tuple(int(r) for r in ranks)))
        flat = self._flat(what, first, stride, count, nseg)
        out = np.sort(flat, axis=1)[:, np.asarray(ranks, dtype=np.intp)]
        has_nan = np.isnan(flat).any(axis=1)
        return (out[0], has_nan[0], 1) if nseg == 1 else (out, has_nan, 1)

    def histogram(self, what, first, stride, count, bins, outer, edges, nseg=1):
        _CountingChain.calls.append(("histogram", nseg, outer.shape, edges.shape))
        flat = self._flat(what, first, stride, count, nseg)
        D = flat.shape[2]
        hist = np.empty((nseg * D, bins), dtype=np.int64)
        for c in range(nseg * D):  # numpy's uniform-bin rule over the given outer edges
            hist[c] = np.histogram(flat[c // D][:, c % D], bins, range=(outer[c, 0], outer[c, 1]))[0]
            assert np.array_equal(np.histogram_bin_edges([], bins, range=(outer[c, 0], outer[c, 1])), edges[c])
        return hist

    def histogram2d(self, first, stride, count, params, bins, edges, nseg=1):
        _CountingChain.calls.append(("histogram2d", nseg, tuple(params), edges.shape))
        flat = self._flat("chain", first, stride, count, nseg)
        m = len(params)
        out = np.empty((nseg, m * (m - 1) // 2, bins, bins), dtype=np.uint64)
        for k in range(nseg):
            for p, (a, b) in enumerate(itertools.combinations(range(m), 2)):
                out[k, p] = np.histogram2d(flat[k][:, params[a]], flat[k][:, params[b]],
                                           bins=[edges[k * m + a], edges[k * m + b]])[0]
        return out if nseg > 1 else out[0]


@pytest.fixture
def stand_in(monkeypatch):
    _CountingChain.calls = []
    monkeypatch.setattr(_lib, "BatchEngine", _RandomStore)
    monkeypatch.setattr(_lib, "Chain", _CountingChain)


@pytest.mark.parametrize("K", [1, 3])
def test_device_route_layout_and_reshapes(stand_in, K):
    N, D = 6, 3
    dev = _batch(K, N, D, backend=DeviceBackend())
    host = _batch(K, N, D)
    for rng in _range_forms(K, D):
        _CountingChain.calls = []
        h, e = dev.get_histogram(bins=5, range=rng, discard=2, thin=3)
        wh, we = host.get_histogram(bins=5, range=rng, discard=2, thin=3)
        assert h.dtype == wh.dtype and np.array_equal(h, wh) and np.array_equal(e, we)
        sel = [("select", K, (0, 3 * N - 1))] if rng is None or (not _per_ensemble(rng) and None in rng) else []
        assert _CountingChain.calls == sel + [("histogram", K, (K * D, 3), (K * D, 6))]
        _CountingChain.calls = []
        h2, e2, pairs = dev.get_histogram2d(params=[2, 0], bins=4, range=rng, discard=2, thin=3)
        wh2, we2, wpairs = host.get_histogram2d(params=[2, 0], bins=4, range=rng, discard=2, thin=3)
        assert h2.dtype == wh2.dtype and np.array_equal(h2, wh2) and np.array_equal(e2, we2) and pairs == wpairs
        assert _CountingChain.calls[-1] == ("histogram2d", K, (2, 0), (K * 2, 5))
    for rng in _range_forms(K, D, log_prob=True):
        h, e = dev.get_histogram(bins=5, range=rng, name="log_prob")
        wh, we = host.get_histogram(bins=5, range=rng, name="log_prob")
        assert h.shape == (K, 5) and np.array_equal(h, wh) and np.array_equal(e, we)


def test_device_route_error_precedence(stand_in):
    """the first failing (ensemble, parameter) in the host route's loop order raises, before any count"""
    K, N, D = 4, 6, 3
    dev = _batch(K, N, D, backend=DeviceBackend())
    host = _batch(K, N, D)
    for b in (dev, host):  # ensemble 2's parameter 1, and ensemble 3's parameter 0, hold a NaN
        x = b.backend._ch.x if b is dev else b.backend.chain
        x[5, 2 * N + 1, 1] = np.nan
        x[6, 3 * N + 4, 0] = np.nan
    per = np.tile([-1.0, 1.0], (K, D, 1))
    per[3, 2] = (1.0, 0.0)
    per[2, 2] = (0.0, np.inf)
    for kw in (dict(), dict(range=per), dict(range=[None, (-1.0, 1.0), (2.0, 1.0)])):
        for call in (lambda s: s.get_histogram(**kw), lambda s: s.get_histogram2d(**kw),
                     lambda s: s.get_histogram2d(params=[2, 1], **kw)):
            _CountingChain.calls = []
            want = _outcome(lambda: call(host))
            assert not want[0]
            assert _outcome(lambda: call(dev)) == want
            assert all(c[0] == "select" for c in _CountingChain.calls)


def test_device_route_empty_slice_and_bins(stand_in):
    K, N, D = 3, 6, 2
    dev = _batch(K, N, D, backend=DeviceBackend())
    host = _batch(K, N, D)
    _CountingChain.calls = []
    for rng in _range_forms(K, D):
        h, e = dev.get_histogram(bins=4, range=rng, discard=12)
        wh, we = host.get_histogram(bins=4, range=rng, discard=12)
        assert h.dtype == wh.dtype and np.array_equal(h, wh) and np.array_equal(e, we)
        h2, e2, _ = dev.get_histogram2d(bins=4, range=rng, discard=12)
        wh2, we2, _ = host.get_histogram2d(bins=4, range=rng, discard=12)
        assert h2.dtype == wh2.dtype and np.array_equal(h2, wh2) and np.array_equal(e2, we2)
    h, e = dev.get_histogram(bins=4, discard=12, name="log_prob")
    assert h.shape == (K, 4) and np.array_equal(e, host.get_histogram(bins=4, discard=12, name="log_prob")[1])
    assert _CountingChain.calls == []
    for bins, two_d in ((4097, False), (129, True), (2.5, False)):
        with pytest.raises((NotImplementedError, TypeError)):
            (dev.get_histogram2d if two_d else dev.get_histogram)(bins=bins)
    with pytest.raises(NotImplementedError):
        dev.get_histogram(bins="auto")
    assert _CountingChain.calls == []
