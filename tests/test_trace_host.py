"""Host side of the running trace (``EnsembleSampler.enable_trace`` / ``trace`` / ``best_sample``), no GPU needed:

1. the summation order of ``emcee_b200/csrc/trace_sum.h``, restated for the host in
   ``tests/helpers/trace_sum_host.cpp``, against a long-double two-pass reference (and ``math.fsum`` / ``fractions``
   on small ensembles).  The bounds are first-order rounding bounds of the header's tree, ``depth =
   trace_depth(N)`` additions on the longest path and ``u = 2**-53``, with ``d = x - x[0]`` the shifted terms:

   * ``|mean - exact| <= (depth + 2) u sum|d| / N + 2 u |exact|``;
   * ``|var - exact| <= (3 depth + 12) u sum(d**2) / (N - 1) + 4 u exact`` (``S2`` carries ``depth + 3`` roundings
     per term, ``S1**2 / N`` twice ``depth + 3`` and ``(sum|d|)**2 / N <= sum d**2``);
   * ``|log_prob_mean - exact| <= (depth + 1) u sum|log_prob| / N + u |exact|``;

   that is a few ulp times the condition of each sum, at N = 65 536 about 40 u.
2. argument checks and the lifecycle of the Python methods over a stand-in engine."""
import ctypes as C
import math
import os
import pickle
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import emcee_b200
from emcee_b200.ensemble import Trace

HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -53


def build_probe(directory):
    out = os.path.join(str(directory), "libtrace_sum_probe.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out,
                    os.path.join(HERE, "helpers", "trace_sum_host.cpp")], check=True)
    lib = C.CDLL(out)
    dp = C.POINTER(C.c_double)
    lib.probe_trace_depth.restype = C.c_int
    lib.probe_trace_depth.argtypes = [C.c_uint64]
    lib.probe_trace_columns.restype = None
    lib.probe_trace_columns.argtypes = [dp, C.c_uint64, C.c_int, dp, dp]
    lib.probe_trace_log_prob.restype = None
    lib.probe_trace_log_prob.argtypes = [dp, C.POINTER(C.c_uint8), C.c_uint64, dp]
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def host_columns(lib, x):
    """(mean[D], var[D]) of x[N, D] in the header's order"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    N, D = x.shape
    mean, var = np.empty(D), np.empty(D)
    lib.probe_trace_columns(_dp(x), N, D, _dp(mean), _dp(var))
    return mean, var


def host_log_prob(lib, lp, acc=None):
    """(log_prob_mean, log_prob_max, accepted, argmax walker) of lp[N] in the header's order"""
    lp = np.ascontiguousarray(lp, dtype=np.float64)
    acc = np.zeros(lp.size, dtype=np.uint8) if acc is None else np.ascontiguousarray(acc, dtype=np.uint8)
    out = np.empty(4)
    lib.probe_trace_log_prob(_dp(lp), acc.ctypes.data_as(C.POINTER(C.c_uint8)), lp.size, _dp(out))
    return out[0], out[1], int(out[2]), int(out[3])


def column_bounds(lib, x):
    """(exact mean, exact var, mean bound, var bound) of x[N, D], the exact values in long double, two passes"""
    N = x.shape[0]
    depth = lib.probe_trace_depth(N)
    xl = x.astype(np.longdouble)
    d = xl - xl[0]  # the reference is shifted too, so that its own rounding (2**-64) stays relative to the spread
    dm = d.mean(axis=0)
    mean = xl[0] + dm
    with np.errstate(invalid="ignore", divide="ignore"):
        var = np.square(d - dm).sum(axis=0) / np.longdouble(N - 1)
        tol_mean = (depth + 2) * U * np.abs(d).sum(axis=0) / N + 2 * U * np.abs(mean)
        tol_var = (3 * depth + 12) * U * np.square(d).sum(axis=0) / np.longdouble(N - 1) + 4 * U * var
    return mean, var, tol_mean, tol_var


def check_columns(lib, x, mean, var):
    em, ev, tm, tv = column_bounds(lib, x)
    assert np.all(np.abs(mean - em) <= tm)
    if x.shape[0] == 1:
        assert np.all(np.isnan(var))
    else:
        assert np.all(var >= 0) and np.all(np.abs(var - ev) <= tv)


def agree_with_numpy(lib, x, mean, var):
    """numpy's own sums are not exact: np.mean / np.var along axis 0 add the rows one after the other, so they may be
    off by e = N u sum|x| / N and by (N + 3) u var + e**2 N / (N - 1) (its variance is taken about its own mean, and
    is not 0 for a constant column); the two results differ by at most both bounds"""
    N = x.shape[0]
    _, ev, tm, tv = column_bounds(lib, x)
    slack_mean = N * U * np.abs(x).sum(axis=0) / N
    slack_var = (N + 3) * U * ev.astype(float) + np.square(slack_mean) * N / (N - 1)
    assert np.all(np.abs(mean - np.mean(x, axis=0)) <= tm.astype(float) + slack_mean)
    assert np.all(np.abs(var - np.var(x, axis=0, ddof=1)) <= tv.astype(float) + slack_var)


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    return build_probe(tmp_path_factory.mktemp("trace_sum"))


# ---- the summation order ------------------------------------------------------------------------------------------
def test_depth(probe):
    # 15 additions in a leaf, 15 over the leaves of a chunk, one per level of the tree over the chunks
    assert probe.probe_trace_depth(1) == 30
    assert probe.probe_trace_depth(256) == 30
    assert probe.probe_trace_depth(257) == 31
    assert probe.probe_trace_depth(4096) == 34
    assert probe.probe_trace_depth(65536) == 38
    assert probe.probe_trace_depth(65536 + 1) == 39
    assert probe.probe_trace_depth(262144) == 40


SHAPES = [(1, 1), (1, 7), (2, 1), (2, 7), (3, 7), (3, 128), (15, 7), (17, 257), (255, 7), (257, 7), (273, 128),
          (4095, 7), (4096, 1), (4096, 7), (4096, 128), (4096, 257), (4097, 7), (65536, 7), (65536, 128), (65537, 1)]


@pytest.mark.parametrize("N,D", SHAPES)
@pytest.mark.parametrize("kind", ["normal", "far", "constant"])
def test_columns_against_long_double(probe, N, D, kind):
    rng = np.random.default_rng(N * 1000 + D)
    if kind == "normal":
        x = rng.standard_normal((N, D)) * np.logspace(-3, 3, D) + np.linspace(-2, 2, D)
    elif kind == "far":  # the ensemble sits 1e4 sigma from the origin: the shift keeps the second moments small
        x = 1e4 + rng.standard_normal((N, D))
    else:
        x = np.tile(rng.standard_normal(D) * 1e3, (N, 1))
    mean, var = host_columns(probe, x)
    check_columns(probe, x, mean, var)
    if kind == "constant":
        assert np.array_equal(mean, x[0])
        if N > 1:
            assert np.all(var == 0.0) and not np.any(np.signbit(var))
    if kind == "far" and N >= 255:
        # raw second moments would lose (1e4)**2 / u of the variance; the shifted sums keep it to about 1e-13
        assert np.all(np.abs(var - np.var(x, axis=0, ddof=1)) <= 1e-12 * var)
    if N > 1:
        agree_with_numpy(probe, x, mean, var)


def test_n1_is_numpys_nan(probe):
    x = np.array([[1.5, -2.0, 0.0]])
    mean, var = host_columns(probe, x)
    assert np.array_equal(mean, x[0]) and np.all(np.isnan(var))
    with np.errstate(invalid="ignore", divide="ignore"), pytest.warns(RuntimeWarning):
        assert np.all(np.isnan(np.var(x, axis=0, ddof=1)))


@pytest.mark.parametrize("N", [2, 3, 37, 300])
def test_columns_against_fractions(probe, N):
    x = np.random.default_rng(N).standard_normal((N, 2)) * [1.0, 1e-6] + [0.0, 3e5]
    mean, var = host_columns(probe, x)
    depth = probe.probe_trace_depth(N)
    for j in range(2):
        col = [Fraction(v) for v in x[:, j]]
        m = sum(col) / N
        v = sum((c - m) ** 2 for c in col) / (N - 1)
        d = [c - col[0] for c in col]
        assert abs(Fraction(mean[j]) - m) <= Fraction((depth + 2) * U) * sum(abs(t) for t in d) / N + 2 * U * abs(m)
        assert abs(Fraction(var[j]) - v) <= Fraction((3 * depth + 12) * U) * sum(t * t for t in d) / (N - 1) + 4 * U * v
        assert abs(mean[j] - math.fsum(x[:, j]) / N) <= 40 * U * max(abs(mean[j]), np.abs(x[:, j] - x[0, j]).max())


@pytest.mark.parametrize("N", [1, 2, 3, 16, 17, 255, 256, 257, 4096, 4099, 65536, 65537])
def test_log_prob_side(probe, N):
    rng = np.random.default_rng(N)
    lp = -0.5 * rng.chisquare(5, N) - 100.0
    acc = (rng.random(N) < 0.4).astype(np.uint8)
    mean, mx, nacc, arg = host_log_prob(probe, lp, acc)
    depth = probe.probe_trace_depth(N)
    exact = lp.astype(np.longdouble).mean()
    assert abs(mean - exact) <= (depth + 1) * U * np.abs(lp).sum() / N + U * abs(exact)
    assert abs(mean - math.fsum(lp) / N) <= (depth + 2) * U * np.abs(lp).sum() / N
    assert mx == lp.max() and arg == int(np.argmax(lp)) and nacc == int(acc.sum())


@pytest.mark.parametrize("N", [5, 300, 4097])
def test_log_prob_infinities_and_ties(probe, N):
    lp = np.linspace(-3.0, -1.0, N)
    lp[::3] = -np.inf
    mean, mx, _, arg = host_log_prob(probe, lp)
    assert mean == -np.inf == np.mean(lp) and mx == lp.max() and arg == int(np.argmax(lp))
    # all at -inf: numpy's argmax is walker 0
    assert host_log_prob(probe, np.full(N, -np.inf))[1:] == (-np.inf, 0, 0)
    # a tie: the lowest walker, wherever the tree joins its chunk
    for first in (0, 1, N // 2, N - 2):
        lp = np.full(N, -7.0)
        lp[[first, N - 1]] = -2.5
        assert host_log_prob(probe, lp)[3] == first == int(np.argmax(lp))
    lp = np.full(N, 1.25)
    assert host_log_prob(probe, lp)[:2] == (1.25, 1.25) and host_log_prob(probe, lp)[3] == 0


# ---- the Python methods over a stand-in engine ---------------------------------------------------------------------
class _Engine(object):
    """records what EnsembleSampler asks of the engine's trace functions"""

    def __init__(self, ndim):
        self.ndim, self.calls, self.rows = ndim, [], 0

    def trace_config(self, every):
        self.calls.append(every)
        if every > 0:
            self.rows = 0

    def trace_count(self):
        return self.rows

    def trace_read(self, first=0):
        n = max(self.rows - first, 0)
        rows = np.arange(n * (2 * self.ndim + 4), dtype=np.float64).reshape(n, 2 * self.ndim + 4)
        return np.arange(first + 1, first + 1 + n, dtype=np.uint64), rows

    def trace_best(self):
        return np.zeros(self.ndim), -1.0, 3, 2

    def get_rng(self):
        return 1, 0


def _sampler(ndim=3):
    s = object.__new__(emcee_b200.EnsembleSampler)
    s.ndim, s.nwalkers, s._rdv, s._hist, s._trace_every = ndim, 8, None, None, None
    s._engine, s._pinned = _Engine(ndim), None
    return s


def test_reading_before_enabling():
    s = _sampler()
    for read in (s.trace, s.best_sample, s.trace_autocorr_time):
        with pytest.raises(RuntimeError, match="not enabled"):
            read()


@pytest.mark.parametrize("every", [1.0, "2", None, 2.5])
def test_every_must_be_an_index(every):
    s = _sampler()
    with pytest.raises(TypeError):
        s.enable_trace(every)
    assert s._engine.calls == [] and s._trace_every is None


def test_every_negative():
    s = _sampler()
    with pytest.raises(ValueError, match="every must be >= 0"):
        s.enable_trace(-1)
    s.enable_trace(np.int64(4))  # anything with __index__
    assert s._engine.calls == [4] and s._trace_every == 4


def test_every_zero_keeps_the_cadence_of_the_rows():
    s = _sampler()
    s.enable_trace(3)
    s._engine.rows = 5
    s.enable_trace(0)
    assert s._engine.calls == [3, 0] and s._trace_every == 3 and s._engine.rows == 5
    assert s.trace().step.size == 5
    s.enable_trace(2)
    assert s._trace_every == 2 and s.trace().step.size == 0


def test_trace_shapes_and_dtypes():
    s = _sampler(ndim=3)
    s.enable_trace()
    with pytest.raises(RuntimeError, match="no step yet"):
        s.best_sample()
    s._engine.rows = 4
    t = s.trace()
    assert isinstance(t, Trace) and t._fields == ("step", "mean", "var", "log_prob_mean", "log_prob_max", "accepted")
    assert t.step.dtype == np.uint64 and t.accepted.dtype == np.int64
    assert t.mean.shape == t.var.shape == (4, 3) and t.log_prob_mean.shape == t.log_prob_max.shape == (4,)
    assert np.array_equal(t.mean[1], [10, 11, 12]) and np.array_equal(t.var[1], [13, 14, 15])
    assert t.log_prob_mean[1] == 16 and t.log_prob_max[1] == 17 and t.accepted[1] == 18
    for discard in (4, 9):  # at and beyond the rows: empty, of the right shape and dtype
        e = s.trace(discard=discard)
        assert e.step.shape == (0,) and e.step.dtype == np.uint64 and e.mean.shape == e.var.shape == (0, 3)
        assert e.accepted.shape == (0,) and e.accepted.dtype == np.int64 and e.log_prob_max.dtype == np.float64
    assert np.array_equal(s.trace(discard=1).step, [2, 3, 4])
    with pytest.raises(ValueError, match="discard must be >= 0"):
        s.trace(discard=-1)
    with pytest.raises(TypeError):
        s.trace(discard=1.5)
    assert s.best_sample()[1:] == (-1.0, 3, 2)


def test_sharded_refused():
    s = _sampler()
    s._rdv = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.enable_trace()
    s = _sampler()
    s.backend = emcee_b200.Backend()
    s.enable_trace()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(object())


def test_rows_are_not_pickled():
    s = _sampler()
    s.enable_trace(2)
    state = s.__getstate__()
    assert state["_trace_every"] is None and "_engine" not in state
    pickle.dumps(state)
