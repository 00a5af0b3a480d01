"""Host side of the running autocorrelation function (``EnsembleSampler.enable_autocorr`` / ``autocorr_function`` /
``autocorr_time``), no GPU needed:

1. the numpy statement of the blocked sums (``tests/running_acf_ref.py``) against ``autocorr._acf`` and a long-double
   reference on random series, and against exact integer lag sums, within the bound DESIGN §5.7 derives;
2. its results bit-identical at every cut of the recorded steps into reads, mid-block included;
3. the g++ probe of ``emcee_b200/csrc/running_acf.h`` (``tests/helpers/running_acf_host.cpp``) equal to it with ``==``;
4. the window rules of ``autocorr.integrated_time_from_acf`` for a function held up to ``max_lag``;
5. argument checks and the lifecycle of the Python methods over a stand-in engine."""
import ctypes as C
import logging
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import autocorr

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import acf_exact  # noqa: E402
import running_acf_ref as ref  # noqa: E402


def build_probe(directory):
    out = os.path.join(str(directory), "librunning_acf_probe.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out,
                    os.path.join(HERE, "helpers", "running_acf_host.cpp")], check=True)
    lib = C.CDLL(out)
    dp = C.POINTER(C.c_double)
    lib.probe_running_acf.restype = None
    lib.probe_running_acf.argtypes = [dp, C.c_uint64, C.c_uint64, C.c_int, C.c_uint64, C.POINTER(C.c_uint64),
                                      C.c_uint64, dp]
    lib.probe_fma.restype = None
    lib.probe_fma.argtypes = [dp, dp, dp, C.c_uint64, dp]
    return lib


def probe_rho(lib, x, max_lag, reads=()):
    x = np.ascontiguousarray(x, dtype=np.float64)
    n, N, D = x.shape
    rho = np.zeros((min(n, max_lag + 1), D))
    r = np.ascontiguousarray(sorted(reads), dtype=np.uint64)
    dp = C.POINTER(C.c_double)
    lib.probe_running_acf(x.ctypes.data_as(dp), n, N, D, max_lag, r.ctypes.data_as(C.POINTER(C.c_uint64)), r.size,
                          rho.ctypes.data_as(dp))
    return rho


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    return build_probe(tmp_path_factory.mktemp("running_acf_probe"))


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def ar1(rng, n, N, D, phi=0.9, drift=0.0, offset=0.0):
    x = np.empty((n, N, D))
    v = rng.normal(size=(N, D))
    for t in range(n):
        v = phi * v + rng.normal(size=(N, D))
        x[t] = v + offset + drift * np.exp(-t / 20.0)
    return x


# ---- 1. the statement against the estimator -------------------------------------------------------------------------
def test_fma_emulation(probe):
    rng = np.random.default_rng(1)
    a = rng.normal(size=20000) * 10.0 ** rng.integers(-8, 8, 20000)
    b = rng.normal(size=20000) * 10.0 ** rng.integers(-8, 8, 20000)
    c = -a * b * (1 + rng.normal(size=20000) * 1e-14)  # heavy cancellation: the single rounding shows
    c[::3] = rng.normal(size=c[::3].size)
    c[::7] = 0.0
    out = np.empty_like(a)
    dp = C.POINTER(C.c_double)
    probe.probe_fma(a.ctypes.data_as(dp), b.ctypes.data_as(dp), c.ctypes.data_as(dp), a.size, out.ctypes.data_as(dp))
    assert same(ref.fma(a, b, c), out)


@pytest.mark.parametrize("n,N,D,max_lag,drift,offset", [
    (150, 5, 3, 20, 0.0, 0.0),
    (200, 3, 2, 300, 0.0, 0.0),  # n - 1 <= max_lag: every lag
    (300, 4, 2, 40, 30.0, 0.0),  # burn-in kept in the window
    (257, 70, 1, 16, 0.0, 1e4),  # two walker chunks, a mean far from the fluctuations
])
def test_statement_against_acf(n, N, D, max_lag, drift, offset):
    rng = np.random.default_rng(n + N)
    x = ar1(rng, n, N, D, drift=drift, offset=offset)
    rho = ref.running_acf(x, max_lag)
    L = min(n, max_lag + 1)
    assert rho.shape == (L, D)
    bound = ref.rounding_bound(x, max_lag)
    r, _ = ref.exact_parts(x, max_lag)
    assert np.all(np.abs(rho - r.mean(axis=1)) <= bound + 2.0 ** -60 * np.abs(r).mean(axis=1))
    want = np.mean(autocorr._acf(x), axis=1)[:L]
    fft = ref.fft_bound(x)[:L]
    assert np.all(np.abs(rho - want) <= bound + fft)


@pytest.mark.parametrize("n,N,D,max_lag", [(130, 3, 2, 12), (64, 2, 3, 80), (200, 66, 1, 8)])
def test_statement_against_exact_lag_sums(n, N, D, max_lag):
    rng = np.random.default_rng(7 * n)
    x = acf_exact.int_series(rng, n, N, D)
    rho = ref.running_acf(x, max_lag)
    L = min(n, max_lag + 1)
    exact, r, _ = acf_exact.exact_acf(x, np.arange(L))
    bound = ref.rounding_bound(x, max_lag)
    # integer values: y and every lag product are exact, so only the double-double combination and the final
    # roundings remain; the bound covers them
    assert np.all(np.abs(rho - exact) <= bound + acf_exact.U * np.abs(exact))


def test_constant_walker_is_nan(probe):
    rng = np.random.default_rng(3)
    x = ar1(rng, 80, 4, 2)
    x[:, 2, 1] = 1.5
    rho = ref.running_acf(x, 10)
    assert np.all(np.isnan(rho[:, 1])) and np.all(np.isfinite(rho[:, 0]))
    with np.errstate(invalid="ignore"):
        assert np.all(np.isnan(np.mean(autocorr._acf(x), axis=1)[:11, 1]))
    assert same(probe_rho(probe, x, 10), rho)


# ---- 2. cuts --------------------------------------------------------------------------------------------------------
def test_reads_change_nothing():
    rng = np.random.default_rng(11)
    x = ar1(rng, 200, 3, 2, drift=5.0)
    whole = ref.running_acf(x, 24)
    for cuts in ([0], [62, 63, 64], list(range(0, 200, 17)), [127, 128, 129, 190], list(range(200))):
        assert same(ref.running_acf(x, 24, cuts=cuts), whole)
    # a read after each prefix is the whole statement of that prefix
    acc = ref.RunningAcf(24, 3, 2)
    for t in range(150):
        acc.record(x[t])
        if t in (0, 1, 63, 64, 100, 149):
            assert same(acc.read(), ref.running_acf(x[: t + 1], 24))


# ---- 3. the header against the statement ----------------------------------------------------------------------------
@pytest.mark.parametrize("n,N,D,max_lag", [
    (1, 2, 2, 5), (2, 3, 1, 1), (63, 2, 3, 7), (64, 2, 3, 7), (65, 2, 3, 70), (200, 5, 2, 33), (300, 130, 1, 9),
])
def test_probe_equals_statement(probe, n, N, D, max_lag):
    rng = np.random.default_rng(n * 31 + max_lag)
    x = ar1(rng, n, N, D, drift=10.0)
    want = ref.running_acf(x, max_lag)
    assert same(probe_rho(probe, x, max_lag), want)
    assert same(probe_rho(probe, x, max_lag, reads=range(0, n, 5)), want)


# ---- 4. the window rules --------------------------------------------------------------------------------------------
def _acf_of(tau_true, n, D=3, seed=0):
    rng = np.random.default_rng(seed)
    phi = (tau_true - 1.0) / (tau_true + 1.0)
    x = ar1(rng, n, 8, D, phi=phi)
    return np.mean(autocorr._acf(x), axis=1)


def test_window_within_max_lag_is_the_whole_functions():
    rho = _acf_of(4.0, 4000)
    whole = autocorr.integrated_time_from_acf(rho, quiet=True)
    for max_lag in (60, 200, 3999):
        got = autocorr.integrated_time_from_acf(rho[: max_lag + 1], n_t=4000, thin=3)
        assert np.array_equal(got, whole)


def test_all_lags_held_is_integrated_time_from_acf():
    rho = _acf_of(3.0, 500, seed=2)
    for c, tol in ((5, 50), (2, 10), (8, 1000)):
        try:
            want = autocorr.integrated_time_from_acf(rho, c=c, tol=tol)
        except autocorr.AutocorrError as e:
            with pytest.raises(autocorr.AutocorrError) as got:
                autocorr.integrated_time_from_acf(rho, c=c, tol=tol, n_t=500)
            assert np.array_equal(got.value.tau, e.tau) and str(got.value) == str(e)
        else:
            assert np.array_equal(autocorr.integrated_time_from_acf(rho, c=c, tol=tol, n_t=500), want)


def test_window_beyond_max_lag(caplog):
    rho = _acf_of(20.0, 5000, seed=4)
    taus = 2.0 * np.cumsum(rho[:31], axis=0) - 1.0
    with pytest.raises(autocorr.AutocorrError, match="max_lag = 30") as e:
        autocorr.integrated_time_from_acf(rho[:31], n_t=5000, thin=3)
    assert "larger max_lag" in str(e.value)
    assert np.array_equal(e.value.tau, 3 * taus[30])
    with caplog.at_level(logging.WARNING, logger="emcee_b200.autocorr"):
        got = autocorr.integrated_time_from_acf(rho[:31], n_t=5000, thin=3, quiet=True)
    assert np.array_equal(got, taus[30]) and "max_lag = 30" in caplog.text


# ---- 5. the Python methods over a stand-in engine -------------------------------------------------------------------
class _Engine(object):
    def __init__(self, ndim):
        self.ndim, self.calls, self.n, self.rho = ndim, [], 0, None

    def running_acf_config(self, max_lag, every):
        self.calls.append((max_lag, every))
        if every > 0 or not self.calls[:-1]:
            self.n = 0

    def running_acf_count(self):
        return self.n

    def running_acf_read(self, max_lag):
        return self.rho[: min(self.n, max_lag + 1)]

    def get_rng(self):
        return 1, 0


def _sampler(ndim=3):
    s = object.__new__(emcee_b200.EnsembleSampler)
    s.ndim, s.nwalkers, s._rdv, s._hist, s._trace_every, s._reservoir_every = ndim, 8, None, None, None, None
    s._autocorr = None
    s._engine, s._pinned = _Engine(ndim), None
    return s


def test_reading_before_enabling():
    s = _sampler()
    for read in (s.autocorr_count, s.autocorr_function, s.autocorr_time):
        with pytest.raises(RuntimeError, match="not enabled"):
            read()


@pytest.mark.parametrize("max_lag,every,err", [(0, 1, ValueError), (-3, 1, ValueError), (4, -1, ValueError),
                                               (4.0, 1, TypeError), ("4", 1, TypeError), (4, 1.5, TypeError),
                                               (None, 1, TypeError)])
def test_arguments(max_lag, every, err):
    s = _sampler()
    with pytest.raises(err):
        s.enable_autocorr(max_lag, every)
    assert s._engine.calls == [] and s._autocorr is None


def test_lifecycle():
    s = _sampler(ndim=2)
    s.enable_autocorr(np.int64(40), np.int64(3))
    assert s._engine.calls == [(40, 3)] and s._autocorr == (40, 3)
    rho = _acf_of(2.0, 3000, D=2, seed=5)
    s._engine.rho, s._engine.n = rho, 3000
    assert s.autocorr_count() == 3000 and s.autocorr_function().shape == (41, 2)
    want = 3 * autocorr.integrated_time_from_acf(rho[:41], n_t=3000, thin=3)
    assert np.array_equal(s.autocorr_time(), want)
    s.enable_autocorr(7, 0)  # every=0: keeps the lags, the cadence and the sums
    assert s._autocorr == (40, 3) and s.autocorr_count() == 3000 and s.autocorr_function().shape == (41, 2)
    s.enable_autocorr(10, 2)  # every > 0: drops what was recorded
    assert s._autocorr == (10, 2) and s.autocorr_count() == 0 and s.autocorr_function().shape == (0, 2)
    with pytest.raises(RuntimeError, match="no step"):
        s.autocorr_time()


def test_autocorr_time_window_beyond_max_lag():
    s = _sampler(ndim=3)
    s.enable_autocorr(30, 2)
    s._engine.rho, s._engine.n = _acf_of(20.0, 5000, seed=4), 5000
    with pytest.raises(autocorr.AutocorrError, match="max_lag = 30") as e:
        s.autocorr_time()
    taus = 2.0 * np.cumsum(s._engine.rho[:31], axis=0) - 1.0
    assert np.array_equal(e.value.tau, 2 * taus[30])
    assert np.array_equal(s.autocorr_time(quiet=True), 2 * taus[30])


def test_sharded_refused():
    s = _sampler()
    s._rdv = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.enable_autocorr(4)
    s = _sampler()
    s.backend = emcee_b200.Backend()
    s.enable_autocorr(4)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(object())


def test_sums_are_not_pickled():
    s = _sampler()
    s.enable_autocorr(4, 2)
    state = s.__getstate__()
    assert state["_autocorr"] is None and "_engine" not in state
    pickle.dumps(state)
