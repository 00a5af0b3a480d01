"""Host-side parts of the stored-chain summaries (``get_percentile`` / ``get_moments``), no GPU needed:

1. the host finisher (``emcee_b200.summary``): fed the exact order statistics from ``np.partition``, it must give
   ``np.percentile`` bit for bit, and raise numpy's exceptions for a bad ``q``; its ranks at ``n`` near 2^40 must
   be numpy's ``_get_indexes``;
2. the key transform and the selection plan of ``eb_chain_select`` (``emcee_b200/csrc/select_keys.h``, compiled
   for the host, the whole selection run on the CPU) against ``np.sort``;
3. ``Backend.get_percentile`` / ``get_moments`` against the plain numpy expressions."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200.summary import percentile_finish, percentile_ranks

HERE = os.path.dirname(os.path.abspath(__file__))

QS = [0, 100, 50, [16, 50, 84], 1e-12, 100 - 1e-12, [[5, 50], [95, 99.5]], 37.5, np.float32(33.3), 7,
      np.linspace(0, 100, 101), []]


def _finish_from_partition(x, q):
    plan = percentile_ranks(q, x.shape[0])
    if plan.ranks.size == 0:
        return percentile_finish(plan, np.empty((0,) + x.shape[1:]))
    idx = plan.ranks.astype(np.intp)
    stats = np.partition(x, idx, axis=0)[idx]
    return percentile_finish(plan, stats, np.isnan(x).any(axis=0))


def _same(got, want):
    assert np.shape(got) == np.shape(want)
    assert type(got) is type(want) or (isinstance(got, np.ndarray) and isinstance(want, np.ndarray))
    assert np.array_equal(got, want, equal_nan=True)


# ---- 1. host finisher --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 3, 10 ** 6])
def test_finisher_matches_numpy(n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 5))
    x[:, 1] = np.round(x[:, 1] * 2)  # heavy ties
    x[:, 2] = 1.5  # constant
    x[:, 3] = np.where(x[:, 3] > 0, np.inf, -np.inf) if n > 2 else [np.inf, -np.inf][:n]
    x[:, 4] *= 1e300
    for q in QS:
        _same(_finish_from_partition(x, q), np.percentile(x, q, axis=0))
        _same(_finish_from_partition(x[:, 0], q), np.percentile(x[:, 0], q))


def test_finisher_nan_columns():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((1000, 3))
    x[17, 1] = np.nan
    for q in QS:
        _same(_finish_from_partition(x, q), np.percentile(x, q, axis=0))
    y = x[:, 1].copy()
    for q in (50, [16, 84]):
        _same(_finish_from_partition(y, q), np.percentile(y, q))


@pytest.mark.parametrize("q", [-1, 101, np.nan, [50, 200], [[[50]]], "a", [-1e-300]])
def test_finisher_bad_q_raises_numpys_exception(q):
    with pytest.raises(Exception) as want:
        np.percentile(np.zeros((4, 2)), q, axis=0)
    with pytest.raises(type(want.value)) as got:
        percentile_ranks(q, 4)
    assert str(got.value) == str(want.value)


def test_ranks_near_2_40():
    """The virtual indexes and neighbours at n near 2^40: numpy's own _get_indexes on the same virtual indexes."""
    from numpy.lib import _function_base_impl as fb

    for n in (2 ** 40 - 1, 2 ** 40, 2 ** 40 + 3, 3 * 2 ** 38 + 1):
        q = np.array([0, 1e-12, 16, 50, 84, 99.999999, 100 - 1e-12, 100])
        plan = percentile_ranks(q, n)
        vi = (n - 1) * np.true_divide(q, np.float64(100))
        prev, nxt = fb._get_indexes(np.empty(0), vi, n)
        assert np.array_equal(plan.prev, prev) and np.array_equal(plan.next, nxt)
        assert np.array_equal(plan.virtual, vi)
        assert plan.ranks.max() <= n - 1 and plan.ranks[-1] == n - 1
        lo = np.where(prev < 0, n - 1, prev)
        assert np.array_equal(plan.ranks[plan._lo], lo)


# ---- 2. key transform and selection plan -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("select") / "libselect_probe.so")
    subprocess.run(
        ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", "select_host.cpp")],
        check=True,
    )
    lib = C.CDLL(out)
    u64 = C.POINTER(C.c_uint64)
    dp = C.POINTER(C.c_double)
    lib.probe_keys.argtypes = [dp, C.c_size_t, u64, dp]
    lib.probe_select.restype = C.c_int
    lib.probe_select.argtypes = [dp, C.c_uint64, C.c_int, u64, C.c_size_t, C.c_uint64, dp, C.POINTER(C.c_uint8)]
    return lib


SPECIAL = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072009e-308, 1e308, -1e308,
                    np.inf, -np.inf, 1.0, -1.0, np.nextafter(1.0, 2), np.nextafter(-1.0, -2), 3.0, 3.0, -7.5])


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _u64(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def test_keys_preserve_order(probe):
    rng = np.random.default_rng(3)
    x = np.r_[SPECIAL, rng.standard_normal(2000) * 10.0 ** rng.integers(-300, 300, 2000)]
    keys = np.empty(x.size, dtype=np.uint64)
    back = np.empty(x.size)
    probe.probe_keys(_dp(x), x.size, _u64(keys), _dp(back))
    assert np.array_equal(back, x) and not np.any(np.signbit(back[x == 0]))  # -0.0 -> +0.0, all else round-trips
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(x[order], np.sort(x))
    # NaN keys fall outside [-inf, +inf]: a parameter that holds one is answered with NaN, never selected
    nan = np.array([np.nan, -np.nan])
    nk = np.empty(2, dtype=np.uint64)
    probe.probe_keys(_dp(nan), 2, _u64(nk), _dp(np.empty(2)))
    kinf = np.empty(2, dtype=np.uint64)
    probe.probe_keys(_dp(np.array([-np.inf, np.inf])), 2, _u64(kinf), _dp(np.empty(2)))
    assert all(k > kinf[1] or k < kinf[0] for k in nk)


def _select(probe, x, ranks, budget=1 << 23):
    rows, D = x.shape
    ranks = np.ascontiguousarray(ranks, dtype=np.uint64)
    out = np.empty((ranks.size, D))
    has_nan = np.zeros(D, dtype=np.uint8)
    passes = probe.probe_select(_dp(np.ascontiguousarray(x)), rows, D, _u64(ranks), ranks.size, budget, _dp(out),
                                has_nan.ctypes.data_as(C.POINTER(C.c_uint8)))
    assert passes > 0
    return out, has_nan.astype(bool), passes


def _check(probe, x, ranks, **kw):
    out, has_nan, passes = _select(probe, x, ranks, **kw)
    assert np.array_equal(has_nan, np.isnan(x).any(axis=0))
    srt = np.sort(x, axis=0)
    want = srt[np.asarray(ranks, dtype=np.intp)]
    want[:, has_nan] = np.nan
    want = np.where(want == 0, 0.0, want)  # +0.0 for either zero
    assert np.array_equal(out.view(np.uint64)[:, ~has_nan], want.view(np.uint64)[:, ~has_nan])
    assert np.all(np.isnan(out[:, has_nan]))
    return passes


def test_select_special_values(probe):
    rng = np.random.default_rng(4)
    n = 6000
    x = np.empty((n, 7))
    x[:, 0] = rng.choice(SPECIAL, n)                        # ties, +-0, subnormals, +-inf, +-1e308
    x[:, 1] = np.round(rng.standard_normal(n) * 3)          # integers with heavy ties
    x[:, 2] = 2.0                                           # constant: every one of the 64 bits by histogram
    x[:, 3] = rng.standard_normal(n)
    x[:, 4] = rng.standard_normal(n)
    x[100, 4] = np.nan                                      # NaN in one parameter only
    base = np.float64(1.2345).view(np.uint64) & ~np.uint64(0xFFFF)
    x[:, 5] = (base | rng.integers(0, 1 << 16, n).astype(np.uint64)).view(np.float64)  # top 48 bits shared
    x[:, 6] = rng.choice([-1.0, 1.0], n)                    # two distinct values
    ranks = np.unique(np.r_[0, 1, n // 2, n - 2, n - 1, rng.integers(0, n, 20)])
    passes = _check(probe, x, ranks)
    assert passes == 8  # the constant column resolves all 64 bits


def test_select_short_and_long_paths(probe):
    rng = np.random.default_rng(5)
    small = rng.standard_normal((3000, 3))
    assert _check(probe, small, [0, 1500, 2999]) == 1  # at most SEL_CAP values: compacted in the first pass
    big = rng.standard_normal((200000, 2))
    assert _check(probe, big, [0, 31999, 100000, 199999]) <= 4
    shared = np.empty((200000, 1))
    base = np.float64(-3.5).view(np.uint64) & ~np.uint64(0xFFFF)
    shared[:, 0] = (base | rng.integers(0, 1 << 16, 200000).astype(np.uint64)).view(np.float64)
    assert _check(probe, shared, [0, 100000, 199999]) >= 7


def test_select_many_ranks_split_columns(probe):
    """More histogram groups than one CTA holds: a parameter's groups split over several one-column tasks; and
    a candidate budget too small to compact every group at once."""
    rng = np.random.default_rng(6)
    x = rng.standard_normal((100000, 3))
    x[:, 1] = rng.integers(0, 5000, 100000)
    ranks = np.linspace(0, 99999, 300).astype(np.uint64)
    _check(probe, x, ranks)
    _check(probe, x, ranks, budget=5000)
    _check(probe, x, np.sort(np.r_[ranks, ranks[::7]]))  # repeated ranks (the probe takes them sorted)


# ---- 3. Backend ------------------------------------------------------------------------------------------------
def _host_backend(nsteps=40, nwalkers=9, ndim=3, seed=7):
    rng = np.random.default_rng(seed)
    b = emcee_b200.Backend()
    b.reset(nwalkers, ndim)
    b.grow(nsteps, None)
    for _ in range(nsteps):
        st = emcee_b200.State(rng.standard_normal((nwalkers, ndim)), log_prob=rng.standard_normal(nwalkers))
        b.save_step(st, np.ones(nwalkers, dtype=bool))
    return b


def test_backend_methods_are_the_numpy_expressions():
    b = _host_backend()
    for discard, thin in [(0, 1), (5, 3), (39, 1), (0, 40)]:
        flat = b.get_chain(flat=True, discard=discard, thin=thin)
        for q in QS:
            _same(b.get_percentile(q, discard=discard, thin=thin), np.percentile(flat, q, axis=0))
            lp = b.get_log_prob(flat=True, discard=discard, thin=thin)
            _same(b.get_percentile(q, discard=discard, thin=thin, name="log_prob"), np.percentile(lp, q, axis=0))
        mean, cov, n = b.get_moments(discard=discard, thin=thin)
        assert n == len(flat)
        assert np.array_equal(mean, np.mean(flat, axis=0))
        assert np.array_equal(cov, np.cov(flat, rowvar=False))
    mean, cov, n = b.get_moments(discard=40)
    assert n == 0 and np.all(np.isnan(mean)) and np.all(np.isnan(cov)) and cov.shape == (3, 3)
    one = _host_backend(ndim=1)
    assert one.get_moments()[1].shape == (1, 1)
    with pytest.raises(ValueError):
        b.get_percentile(50, name="blobs")


def test_readers_before_anything_was_stored():
    b = emcee_b200.Backend()
    b.reset(4, 2)
    for fn in (lambda: b.get_percentile(50), lambda: b.get_moments()):
        with pytest.raises(AttributeError):
            fn()
    d = emcee_b200.DeviceBackend(device=3)
    for fn in (lambda: d.get_percentile(50), lambda: d.get_moments()):
        with pytest.raises(AttributeError):
            fn()
    d.close()
    for fn in (lambda: d.get_percentile(50), lambda: d.get_moments()):
        with pytest.raises(ValueError):
            fn()
