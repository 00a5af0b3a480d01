"""The host plan of ``EnsembleSampler.enable_histograms`` (``summary.running_histogram_plan``): the refusal of a
missing range, numpy's exceptions for a bad ``bins`` or range, the device limits, the ``params2d`` checks, and the
edges handed to the engine against ``np.histogram_bin_edges`` / ``np.histogramdd``."""
import itertools

import numpy as np
import pytest

from emcee_b200.summary import running_histogram_plan

try:
    from numpy.lib._histograms_impl import _get_outer_edges
except ImportError:  # numpy < 2
    from numpy.lib.histograms import _get_outer_edges

R3 = [(-1.0, 1.0), (0.0, 5.0), (-3.5, 2.25)]


def _numpy_error(fn):
    try:
        fn()
    except Exception as e:  # noqa: B902
        return type(e), str(e)
    return None


@pytest.mark.parametrize("rng", [None, [None, (0, 1), (0, 1)], [(0, 1), None, (0, 1)], ((0, 1), (0, 1), None)])
def test_missing_range_refused(rng):
    with pytest.raises(ValueError, match="need a \\(lo, hi\\) range for every parameter"):
        running_histogram_plan(3, rng)


def test_range_count():
    with pytest.raises(ValueError, match="one \\(lo, hi\\) pair per parameter"):
        running_histogram_plan(3, R3[:2])


@pytest.mark.parametrize("bins", [0, -3, 2.5, "x", [1, 2, 3], np.float64(4.0)])
def test_bad_bins_numpy_exception(bins):
    want = _numpy_error(lambda: np.histogram_bin_edges(np.empty(0), bins))
    if want is None:  # numpy accepts it (a string rule or explicit edges): the device does not
        with pytest.raises(NotImplementedError):
            running_histogram_plan(3, R3, bins)
        return
    with pytest.raises(want[0]) as got:
        running_histogram_plan(3, R3, bins)
    assert str(got.value) == want[1]


@pytest.mark.parametrize("bad", [(1.0, 0.0), (0.0, np.inf), (np.nan, 1.0), (-np.inf, 0.0)])
def test_bad_range_numpy_exception(bad):
    rng = [R3[0], bad, R3[2]]
    want = _numpy_error(lambda: np.histogram(np.zeros(3), 10, bad))
    assert want is not None
    with pytest.raises(want[0]) as got:
        running_histogram_plan(3, rng)
    assert str(got.value) == want[1]
    want2 = _numpy_error(lambda: np.histogram2d(np.zeros(3), np.zeros(3), 10, [R3[0], bad]))
    with pytest.raises(want2[0]):
        running_histogram_plan(3, [R3[0], R3[0], R3[2]], log_prob_range=bad)
    with pytest.raises(want2[0]):
        running_histogram_plan(3, [R3[0], bad, R3[2]], bins=10, params2d=[0, 1])


def test_overflowing_range():
    with pytest.raises(ValueError, match="wider than the largest double"):
        running_histogram_plan(2, [(-1.5e308, 1.5e308), (0, 1)])


def test_bins_limits():
    running_histogram_plan(2, R3[:2], 4096)
    with pytest.raises(NotImplementedError, match="bins <= 4096"):
        running_histogram_plan(2, R3[:2], 4097)
    running_histogram_plan(2, R3[:2], 10, params2d=[0, 1], bins2d=128)
    with pytest.raises(NotImplementedError, match="bins <= 128"):
        running_histogram_plan(2, R3[:2], 10, params2d=[0, 1], bins2d=129)
    with pytest.raises(ValueError):  # numpy's histogramdd check
        running_histogram_plan(2, R3[:2], 10, params2d=[0, 1], bins2d=0)


@pytest.mark.parametrize("params", [[0], [], [1, 1], [0, 3], [-1, 0], [0, 1.5]])
def test_params2d_checks(params):
    with pytest.raises((ValueError, TypeError)):
        running_histogram_plan(3, R3, params2d=params)


def test_no_2d_or_log_prob_by_default():
    cfg = running_histogram_plan(3, R3)
    assert cfg["params2d"] is None and cfg["edges2d"] is None and not cfg["log_prob"]
    assert cfg["edges"].shape == (3, 11) and cfg["outer"].shape == (3, 3)


@pytest.mark.parametrize("bins", [1, 7, 20, 4096])
@pytest.mark.parametrize("f32", [False, True])
def test_edges_are_numpys(bins, f32):
    cast = np.float32 if f32 else float
    rng = [(cast(lo), cast(hi)) for lo, hi in R3]
    lp = (cast(-40.0), cast(-1.0))
    cfg = running_histogram_plan(3, rng, bins, log_prob_range=lp, params2d=[2, 0, 1], bins2d=min(bins, 128))
    assert cfg["bins"] == bins and cfg["log_prob"]
    assert cfg["edges"].dtype == np.float64 and cfg["edges"].shape == (4, bins + 1)
    for d, r in enumerate(rng + [lp]):
        want = np.histogram(np.zeros(0), bins, r)[1]
        assert want.dtype == np.float64
        assert np.array_equal(cfg["edges"][d], want)
        assert np.array_equal(cfg["edges"][d], np.histogram_bin_edges(np.zeros(0), bins, r))
        first, last = _get_outer_edges(np.zeros(0), r)
        assert cfg["outer"][d, 0] == first and cfg["outer"][d, 1] == last
        assert cfg["outer"][d, 2] == np.float64(last - first)  # numpy's norm_denom, in the range's own type
    b2 = min(bins, 128)
    assert cfg["pairs"] == list(itertools.combinations([2, 0, 1], 2))
    assert cfg["edges2d"].shape == (3, b2 + 1)
    for k, p in enumerate([2, 0, 1]):
        _, e = np.histogramdd(np.zeros((0, 1)), bins=b2, range=[rng[p]])
        assert np.array_equal(cfg["edges2d"][k], e[0])
    for (i, j) in cfg["pairs"]:
        _, ei, ej = np.histogram2d(np.zeros(0), np.zeros(0), b2, [rng[i], rng[j]])
        assert np.array_equal(cfg["edges2d"][[2, 0, 1].index(i)], ei)
        assert np.array_equal(cfg["edges2d"][[2, 0, 1].index(j)], ej)
