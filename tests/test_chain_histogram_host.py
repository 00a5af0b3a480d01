"""Host-side parts of the stored-chain histograms (``get_histogram`` / ``get_histogram2d``), no GPU needed:

1. the bin rules of ``eb_chain_histogram`` / ``eb_chain_histogram2d`` (``emcee_b200/csrc/hist_bins.h``, compiled for
   the host) against ``np.histogram`` / ``np.histogram2d`` on adversarial values: every edge and one ulp either side,
   +-0, subnormals, NaN, +-inf, ranges from 1e-300 to 1e300 wide, ``bins`` 1, 2, 3, 10 and 4096; and the pair tiles
   of the 2-D kernel, run on the CPU, against ``np.histogram2d`` of every pair;
2. the host plan (``emcee_b200.summary``): numpy on ``[min; max]`` gives the edges, or the exception, that numpy
   gives on the whole column; an overflowing range raises the documented ``ValueError``;
3. argument checks, and ``Backend.get_histogram*`` against the plain numpy expressions."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import backend as B
from emcee_b200 import summary as S

HERE = os.path.dirname(os.path.abspath(__file__))
DROP, BAD = -1, -2

SPECIAL = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072009e-308, 1e-300, -1e-300,
                    1e300, -1e300, 1.7976931348623157e308, -1.7976931348623157e308, np.inf, -np.inf, np.nan, -np.nan,
                    1.0, -1.0, 0.5, 3.0])


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("histogram") / "libhistogram_probe.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(HERE, "helpers", "histogram_host.cpp")], check=True)
    lib = C.CDLL(out)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    lib.probe_uniform.argtypes = [dp, C.c_size_t, C.c_double, C.c_double, C.c_double, C.c_int, dp, ip]
    lib.probe_searched.argtypes = [dp, C.c_size_t, dp, C.c_int, ip]
    lib.probe_ntiles.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.probe_hist2.restype = C.c_int
    lib.probe_hist2.argtypes = [dp, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.c_int, C.c_int, dp, C.c_size_t,
                                C.c_int, C.POINTER(C.c_uint64)]
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _uniform(probe, x, bins, rng):
    """per-value bins of the header's uniform rule, with the plan's edges for column x"""
    outer, edges = S.uniform_edges(bins, rng, np.min(x), np.max(x), bool(np.isnan(x).any()))
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty(x.size, dtype=np.intc)
    probe.probe_uniform(_dp(x), x.size, outer[0], outer[1], outer[2], bins, _dp(edges),
                        out.ctypes.data_as(C.POINTER(C.c_int)))
    return out, edges


def _searched(probe, x, edges):
    x = np.ascontiguousarray(x, dtype=np.float64)
    edges = np.ascontiguousarray(edges, dtype=np.float64)
    out = np.empty(x.size, dtype=np.intc)
    probe.probe_searched(_dp(x), x.size, _dp(edges), edges.size - 1, out.ctypes.data_as(C.POINTER(C.c_int)))
    return out


def _counts(idx, bins):
    assert not np.any(idx == BAD)
    return np.bincount(idx[idx >= 0], minlength=bins)


def _probes(edges, lo, hi):
    """every edge, one ulp either side of it, and the special values: the values to bin"""
    e = np.asarray(edges)
    return np.r_[e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf), SPECIAL, lo, hi]


# (lo, hi) ranges from 1e-300 to 1e300 wide, around 0 and off it
RANGES = [(0.0, 1.0), (-1.0, 1.0), (-1e-300, 1e-300), (1.0, 1.0 + 1e-12), (-3e300, 2e300), (1e300, 1.5e300),
          (-5e-324, 5e-324), (0.1, 0.7), (-7.25, -7.0), (1e-310, 3e-310), (-1e300, -1e-300)]


@pytest.mark.parametrize("bins", [1, 2, 3, 10, 4096])
def test_uniform_rule_matches_np_histogram(probe, bins):
    rng = np.random.default_rng(bins)
    for lo, hi in RANGES:
        try:
            np.histogram_bin_edges([lo, hi], bins)
        except ValueError:
            continue  # too many bins for this range: numpy raises, and so does the plan (test_plan_*)
        _, edges = np.histogram([lo, hi], bins)
        x = _probes(edges, lo, hi)
        x = np.r_[x, rng.uniform(lo, hi, 500) if np.isfinite(hi - lo) else []]
        # the autodetected range of x itself (NaN / inf inside it make numpy raise), and the given range (lo, hi)
        for given in (None, (lo, hi)):
            xx = x[(x >= lo) & (x <= hi)] if given is None else x  # autodetected: min lo, max hi
            idx, ed = _uniform(probe, xx, bins, given)
            h, e = np.histogram(xx, bins, range=given)
            assert np.array_equal(ed, e)
            assert np.array_equal(_counts(idx, bins), h), (lo, hi, bins, given)
        # one value at a time on the edges: the exact bin, not only the totals
        sub = np.r_[edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf)]
        idx, _ = _uniform(probe, np.r_[sub, lo, hi], bins, (lo, hi))
        for v, i in zip(sub, idx):
            h, _ = np.histogram([v], bins, range=(lo, hi))
            assert (i == DROP and h.sum() == 0) or (i >= 0 and h[i] == 1), (v, i, lo, hi, bins)


def test_uniform_rule_float32_range(probe):
    """A range of float32 scalars: numpy subtracts it in float32, so its norm_denom is below the float64 difference
    and f can exceed bins; numpy truncates, moves bins to bins - 1 and counts."""
    lo, hi = np.float32(-0.3), np.float32(0.1)
    x = np.array([float(hi), 0.0, float(lo)])
    for bins in (1, 10):
        idx, e = _uniform(probe, x, bins, (lo, hi))
        h, we = np.histogram(x, bins, range=(lo, hi))
        assert np.array_equal(e, we) and np.array_equal(_counts(idx, bins), h)
    rng = np.random.default_rng(32)
    for _ in range(300):
        a, b = np.sort(rng.standard_normal(2) * 10.0 ** rng.integers(-3, 4, 2)).astype(np.float32)
        if not a < b:
            continue
        bins = int(rng.choice([1, 2, 3, 10, 20, 4096]))
        try:
            edges = np.histogram_bin_edges([], bins, range=(a, b))
        except ValueError:
            continue
        v = np.r_[edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf), float(a), float(b),
                  rng.uniform(float(a), float(b), 200)]
        idx, e = _uniform(probe, v, bins, (a, b))
        h, we = np.histogram(v, bins, range=(a, b))
        assert np.array_equal(e, we) and np.array_equal(_counts(idx, bins), h), (a, b, bins)
        for val, i in zip(v[-210:], idx[-210:]):  # the top edge and its neighbours one at a time
            h1, _ = np.histogram([val], bins, range=(a, b))
            assert (i == DROP and h1.sum() == 0) or (i >= 0 and h1[i] == 1), (val, i, a, b, bins)


def test_pair_tile_count_closed_form(probe):
    listed, closed = C.c_uint64(), C.c_uint64()
    for m in list(range(2, 40)) + [127, 128, 257, 1024]:
        for b in range(1, 34):
            probe.probe_ntiles(m, b, C.byref(listed), C.byref(closed))
            assert listed.value == closed.value, (m, b)


@pytest.mark.parametrize("bins", [1, 2, 3, 10, 128])
def test_searched_rule_matches_np_histogram2d(probe, bins):
    rng = np.random.default_rng(100 + bins)
    for lo, hi in RANGES:
        edges = np.linspace(lo, hi, bins + 1)
        x = _probes(edges, lo, hi)
        y = rng.permutation(x)
        for given in (None, (lo, hi)):
            inside = (x >= lo) & (x <= hi) & (y >= lo) & (y <= hi)
            xx, yy = (x, y) if given is not None else (x[inside], y[inside])
            rr = None if given is None else [given, given]
            try:
                want, ex, ey = np.histogram2d(xx, yy, bins, range=rr)
            except ValueError:
                continue  # linspace overflow (numpy's own failure; the plan refuses such a range)
            ix, iy = _searched(probe, xx, ex), _searched(probe, yy, ey)
            ok = (ix >= 0) & (iy >= 0)
            got = np.zeros((bins, bins))
            np.add.at(got, (ix[ok], iy[ok]), 1)
            assert np.array_equal(got, want), (lo, hi, bins, given)
    # NaN is an outlier, whatever the edges
    assert np.all(_searched(probe, np.array([np.nan, -np.nan]), np.linspace(0, 1, 11)) == DROP)


def test_duplicate_edges_of_a_narrow_range(probe):
    """np.histogram2d does not refuse too many bins: linspace repeats edges, and searchsorted still counts them"""
    lo = 1.0
    hi = np.nextafter(np.nextafter(lo, 2), 2)
    x = np.array([lo, np.nextafter(lo, 2), hi, hi, lo])
    want, ex, ey = np.histogram2d(x, x[::-1], 10, range=[(lo, hi), (lo, hi)])
    assert np.any(ex[:-1] == ex[1:])
    ix, iy = _searched(probe, x, ex), _searched(probe, x[::-1], ey)
    got = np.zeros((10, 10))
    np.add.at(got, (ix, iy), 1)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("m,bins,hist_bytes,block_max",
                         [(2, 3, 1 << 20, 32), (7, 4, 3 * 3 * 16 * 4, 32), (9, 5, 1, 32), (13, 2, 1 << 20, 4),
                          (40, 20, 160 * 1024, 32)])
def test_pair_tiles_cover_every_pair_once(probe, m, bins, hist_bytes, block_max):
    rng = np.random.default_rng(m)
    D = m + 3
    x = rng.standard_normal((300, D))
    x[::7, 1] = np.nan
    x[5, 2] = np.inf
    params = rng.permutation(D)[:m].astype(np.uint32)
    rngs = [(-2.0, 2.0)] * D
    edges = np.array([S.searched_edges(bins, rngs[p]) for p in params])
    npairs = m * (m - 1) // 2
    hist = np.empty((npairs, bins, bins), dtype=np.uint64)
    ntiles = probe.probe_hist2(_dp(np.ascontiguousarray(x)), x.shape[0], D,
                               params.ctypes.data_as(C.POINTER(C.c_uint32)), m, bins, _dp(edges), hist_bytes,
                               block_max, hist.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert ntiles >= 1
    for p, (i, j) in enumerate(itertools.combinations(params.tolist(), 2)):
        want, _, _ = np.histogram2d(x[:, i], x[:, j], bins, range=[rngs[i], rngs[j]])
        assert np.array_equal(hist[p], want), (p, i, j)


# ---- 2. host plan ---------------------------------------------------------------------------------------------------
def _columns(rng, n=500):
    cols = [rng.standard_normal(n), rng.standard_normal(n) * 1e-300, rng.standard_normal(n) * 1e300,
            np.full(n, 2.5), np.full(n, 0.0), np.full(n, 1e300), np.full(n, -7.0), np.full(n, 5e-324),
            np.r_[rng.standard_normal(n - 1), np.nan], np.r_[rng.standard_normal(n - 1), np.inf],
            np.r_[rng.standard_normal(n - 1), -np.inf], np.array([1.0, np.nextafter(1.0, 2)] * (n // 2)),
            rng.integers(-3, 4, n).astype(float), np.r_[np.full(n - 1, 3.0), np.nextafter(3.0, 4)]]
    return cols


def _same_outcome(got_fn, want_fn):
    try:
        want = want_fn()
    except Exception as e:  # noqa: B902
        with pytest.raises(type(e)) as got:
            got_fn()
        assert str(got.value) == str(e)
        return None
    got = got_fn()
    assert np.array_equal(got, want) and got.dtype == np.float64
    return got


@pytest.mark.parametrize("bins", [1, 3, 10, 20, 4096])
def test_plan_edges_equal_numpy_on_the_whole_column(bins):
    rng = np.random.default_rng(bins)
    for c in _columns(rng):
        lo, hi, nan = np.nanmin(c) if not np.isnan(c).all() else np.nan, np.nanmax(c), bool(np.isnan(c).any())
        for given in (None, (-1.0, 1.0), (0.0, 0.0), (2.5, 2.5)):
            _same_outcome(lambda: S.uniform_edges(bins, given, lo, hi, nan)[1],
                          lambda: np.histogram(c, bins, range=given)[1])
            if bins <= 128:
                other = rng.standard_normal(c.size)
                _same_outcome(lambda: S.searched_edges(bins, given, lo, hi, nan),
                              lambda: np.histogram2d(c, other, bins, range=None if given is None
                                                     else [given, (-1, 1)])[1])
        # the outer edges and the span are numpy's: (first, last) widen a constant column by 0.5
        try:
            outer, edges = S.uniform_edges(bins, None, lo, hi, nan)
        except ValueError:
            continue
        assert outer[0] == edges[0] and outer[1] == edges[-1] and outer[2] == outer[1] - outer[0]


def test_plan_bad_ranges_raise_numpys_exception():
    c = np.linspace(-1, 1, 50)
    for given in [(1.0, 0.0), (0.0, np.inf), (np.nan, 1.0), (-np.inf, np.inf)]:
        _same_outcome(lambda: S.uniform_edges(10, given, -1.0, 1.0), lambda: np.histogram(c, 10, range=given)[1])
        _same_outcome(lambda: S.searched_edges(10, given, -1.0, 1.0),
                      lambda: np.histogram2d(c, c, 10, range=[given, (0, 1)])[1])
    # a NaN anywhere in an autodetected column: "autodetected range of [nan, nan] is not finite"
    with pytest.raises(ValueError, match=r"autodetected range of \[nan, nan\] is not finite"):
        S.uniform_edges(10, None, 0.0, 1.0, has_nan=True)
    with pytest.raises(ValueError, match=r"autodetected range of \[nan, nan\] is not finite"):
        S.searched_edges(10, None, 0.0, 1.0, has_nan=True)


@pytest.mark.parametrize("bins", [1, 2, 10])
def test_plan_overflowing_range_raises_its_value_error(bins):
    for lo, hi, given in [(-1.5e308, 1.5e308, None), (0.0, 1.0, (-1.7e308, 1.7e308)), (-1e308, 1e308, None)]:
        with pytest.raises(ValueError, match="wider than the largest double"):
            S.uniform_edges(bins, given, lo, hi)
        with pytest.raises(ValueError, match="wider than the largest double"):
            S.searched_edges(bins, given, lo, hi)
    # just inside: the edges are finite and numpy's
    e = S.uniform_edges(4, None, -8e307, 8e307)[1]
    assert np.array_equal(e, np.histogram_bin_edges([-8e307, 8e307], 4))


def test_plan_bins_checks():
    for bins in (0, -3):
        with pytest.raises(ValueError, match="`bins` must be positive"):
            S.histogram_bins(bins, S.HIST_BINS_MAX)
        with pytest.raises(ValueError, match=r"`bins\[0\]` must be positive"):
            S.histogram_bins(bins, S.HIST2_BINS_MAX, two_d=True)
    with pytest.raises(TypeError):
        S.histogram_bins(2.5, S.HIST_BINS_MAX)
    with pytest.raises(NotImplementedError, match="4096"):
        S.histogram_bins(4097, S.HIST_BINS_MAX)
    with pytest.raises(NotImplementedError, match="128"):
        S.histogram_bins(129, S.HIST2_BINS_MAX, two_d=True)
    with pytest.raises(NotImplementedError):
        S.histogram_bins("auto", S.HIST_BINS_MAX)
    assert S.histogram_bins(np.int64(4096), S.HIST_BINS_MAX) == 4096


# ---- 3. arguments and Backend ---------------------------------------------------------------------------------------
def _host_backend(nsteps=30, nwalkers=9, ndim=4, seed=7):
    rng = np.random.default_rng(seed)
    b = emcee_b200.Backend()
    b.reset(nwalkers, ndim)
    b.grow(nsteps, None)
    for _ in range(nsteps):
        st = emcee_b200.State(rng.standard_normal((nwalkers, ndim)), log_prob=rng.standard_normal(nwalkers))
        b.save_step(st, np.ones(nwalkers, dtype=bool))
    return b


def test_params_and_range_checks():
    assert B._histogram_params(None, 3) == [0, 1, 2]
    assert B._histogram_params([5, 0, 3], 6) == [5, 0, 3]
    for bad in ([1, 1], [0], [], [0, 6], [-1, 2]):
        with pytest.raises(ValueError):
            B._histogram_params(bad, 6)
    with pytest.raises(TypeError):
        B._histogram_params([0, 1.5], 6)
    with pytest.raises(ValueError, match="one \\(lo, hi\\) pair per parameter"):
        B._histogram_ranges([(0, 1)] * 3, 4)
    b = _host_backend()
    with pytest.raises(ValueError):
        b.get_histogram2d(params=[2, 2])
    with pytest.raises(ValueError):
        b.get_histogram(range=[(0, 1)])
    with pytest.raises(ValueError):
        b.get_histogram(name="blobs")
    d = emcee_b200.DeviceBackend(device=3)  # nothing stored: AttributeError, as Backend
    for fn in (lambda: d.get_histogram(), lambda: d.get_histogram2d()):
        with pytest.raises(AttributeError):
            fn()
    d.close()
    for fn in (lambda: d.get_histogram(), lambda: d.get_histogram2d()):
        with pytest.raises(ValueError, match="closed"):
            fn()


def test_backend_methods_are_the_numpy_expressions():
    b = _host_backend()
    rngs = [(-1, 1), (0, 2), (-3, 0.5), (-0.1, 0.1)]
    for discard, thin in [(0, 1), (5, 3), (29, 1), (30, 1)]:
        flat = b.get_chain(flat=True, discard=discard, thin=thin)
        lp = b.get_log_prob(flat=True, discard=discard, thin=thin)
        for bins, rng in [(10, None), (7, rngs)]:
            h, e = b.get_histogram(bins, rng, discard=discard, thin=thin)
            assert h.dtype == np.int64 and e.dtype == np.float64 and h.shape == (4, bins) and e.shape == (4, bins + 1)
            for d in range(4):
                wh, we = np.histogram(flat[:, d], bins, range=None if rng is None else rng[d])
                assert np.array_equal(h[d], wh) and np.array_equal(e[d], we)
            h, e = b.get_histogram(bins, None if rng is None else rng[1], discard=discard, thin=thin, name="log_prob")
            wh, we = np.histogram(lp, bins, range=None if rng is None else rng[1])
            assert np.array_equal(h, wh) and np.array_equal(e, we)
            for params in (None, [3, 0, 2]):
                h, e, pairs = b.get_histogram2d(params, bins, rng, discard=discard, thin=thin)
                ps = list(range(4)) if params is None else params
                assert pairs == list(itertools.combinations(ps, 2))
                assert h.dtype == np.float64 and h.shape == (len(pairs), bins, bins) and e.shape == (len(ps), bins + 1)
                for p, (i, j) in enumerate(pairs):
                    wh, wx, wy = np.histogram2d(flat[:, i], flat[:, j], bins,
                                                range=None if rng is None else [rng[i], rng[j]])
                    assert np.array_equal(h[p], wh)
                    assert np.array_equal(e[ps.index(i)], wx) and np.array_equal(e[ps.index(j)], wy)
