"""The running autocorrelation function (``EnsembleSampler.enable_autocorr`` / ``autocorr_function`` /
``autocorr_time``; ``eb_running_acf_config``, ``eb_running_acf_read``) against the chain the same run stores.

* Twins: a ``store=False`` run with the sums enabled and a stored run of the same seed (host ``Backend`` and
  ``DeviceBackend``).  The device's rho equals the g++ probe of ``running_acf.h`` run on the stored chain with ``==``,
  ``np.mean(_acf(chain), axis=1)[:max_lag + 1]`` within the derived bound, and ``autocorr_time()`` equals
  ``get_autocorr_time(thin=every)`` with the same windows.  Every kernel path and move kind.
* Exactness: ``MHMove(HostProposal)`` walking through an integer series under a constant model records it exactly;
  rho is within the bound of exact integer lag sums.
* Invariance: one call, many short calls, ``sample()`` and ``iterations=None`` give the same bytes, reads mid-block
  included.
* Nothing else moves: chain, log-probabilities, accept counts, trace and reservoir are the same bytes with the sums
  on.
* Lifecycle: ``every=0``, re-enable, ``MemoryError`` with nothing changed, a stuck walker's NaN, a window beyond
  ``max_lag``, the state error before configuration.
"""
import numpy as np
import pytest

import acf_exact
import running_acf_ref as ref
from test_running_acf_host import build_probe, probe_rho, same

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, autocorr, models, moves

pytestmark = pytest.mark.gpu

SEED = 0xAC0F


def _dense(D):
    rng = np.random.default_rng(D)
    a = rng.standard_normal((D, D))
    return models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)), np.linspace(-1, 1, D))


def _graph_iso(D):
    from test_gpu_graph_function import Capture, iso_columns

    return models.CudaGraphFunction(Capture(iso_columns, D))


def _gauss_mh(coords, random):
    return coords + 0.3 * random.standard_normal(coords.shape), np.zeros(coords.shape[0])


CASES = {
    # name: (N, D, model, moves)
    "dense_dmma": (4096, 128, lambda: _dense(128), None),
    "tma_rows": (64, 8, lambda: models.GaussianIso(), None),
    "generic_odd": (37, 3, lambda: models.GaussianIso(), None),
    "walk_gaussian": (41, 4, lambda: models.GaussianIso(),
                      lambda: [(moves.WalkMove(s=5), 0.5), (moves.GaussianMove(0.3), 0.5)]),
    "kde": (64, 4, lambda: models.GaussianIso(), lambda: moves.KDEMove()),
    "graph_fn": (33, 5, lambda: _graph_iso(5), None),
    "user_move": (32, 4, lambda: models.GaussianIso(), lambda: moves.MHMove(moves.HostProposal(_gauss_mh))),
}


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    return build_probe(tmp_path_factory.mktemp("running_acf_probe_gpu"))


def _make(case, backend=None):
    N, D, model, mv = CASES[case]
    return emcee_b200.EnsembleSampler(N, D, model(), moves=None if mv is None else mv(), seed=SEED, backend=backend)


def _p0(case):
    N, D = CASES[case][:2]
    return np.random.default_rng(N * D).standard_normal((N, D)) * 0.5 + 3.0  # starts off the mode: burn-in


TWINS = [
    # case, every, max_lag, steps
    ("dense_dmma", 1, 32, 150),
    ("tma_rows", 3, 20, 600),
    ("tma_rows", 1, 400, 100),  # n below max_lag: every lag
    ("generic_odd", 1, 24, 700),
    ("walk_gaussian", 3, 16, 330),
    ("kde", 1, 30, 200),
    ("graph_fn", 1, 12, 140),
    ("user_move", 3, 10, 250),
]


@pytest.mark.parametrize("case,every,max_lag,steps", TWINS)
def test_twins(probe, case, every, max_lag, steps):
    s = _make(case)
    s.enable_autocorr(max_lag, every)
    s.run_mcmc(_p0(case), steps, store=False)
    rho = s.autocorr_function()
    n = steps // every
    assert s.autocorr_count() == n and rho.shape == (min(n, max_lag + 1), CASES[case][1])
    for backend in (Backend(), DeviceBackend()):
        t = _make(case, backend)
        t.run_mcmc(_p0(case), steps // every, thin_by=every)  # steps // every stored, every `every`-th
        x = t.get_chain()
        assert x.shape[0] == n
        assert same(probe_rho(probe, x, max_lag), rho)  # the device's arithmetic, operation for operation
        if x.size <= 4e6:
            want = np.mean(autocorr._acf(x), axis=1)[: max_lag + 1]
            assert np.all(np.abs(rho - want) <= ref.rounding_bound(x, max_lag) + ref.fft_bound(x)[: max_lag + 1])
        _same_time(s, t, every)


def _same_time(s, t, every):
    """autocorr_time() against get_autocorr_time of the twin (stored thinned by `every`, so times `every`): the same
    windows where they close within max_lag, else the error naming max_lag"""
    max_lag = s._autocorr[0]
    x = t.get_chain()
    rho = np.mean(autocorr._acf(x), axis=1)
    taus = 2.0 * np.cumsum(rho, axis=0) - 1.0
    inside = np.arange(x.shape[0])[:, None] < 5 * taus
    beyond = x.shape[0] - 1 > max_lag and np.any(np.all(inside[: max_lag + 1], axis=0))
    if beyond:
        with pytest.raises(autocorr.AutocorrError, match="max_lag"):
            s.autocorr_time()
        return
    for kw in ({"quiet": True}, {"tol": 0, "quiet": True}):
        np.testing.assert_allclose(s.autocorr_time(**kw), every * t.get_autocorr_time(**kw), rtol=1e-9)


def test_after_burn_in(probe):
    s, t = _make("tma_rows"), _make("tma_rows", Backend())
    st = s.run_mcmc(_p0("tma_rows"), 200, store=False)
    s.enable_autocorr(299, 1)  # every lag of the 300 recorded steps: the windows are the stored chain's
    s.run_mcmc(st, 300, store=False)
    t.run_mcmc(_p0("tma_rows"), 500)
    x = t.get_chain(discard=200)
    assert same(probe_rho(probe, x, 299), s.autocorr_function())
    np.testing.assert_allclose(s.autocorr_time(quiet=True), t.get_autocorr_time(discard=200, quiet=True), rtol=1e-9)


def test_exact_integer_series():
    """MHMove(HostProposal) that proposes the next row of an integer-valued series; a constant model accepts every
    proposal, so the recorded states are that series exactly"""
    n, N, D, max_lag = 300, 16, 3, 40
    rng = np.random.default_rng(5)
    series = np.concatenate([np.zeros((1, N, D)), acf_exact.int_series(rng, n, N, D)])  # start, then the n recorded
    at = {"t": 0}

    def next_row(coords, random):
        at["t"] += 1
        return series[at["t"]].copy(), np.zeros(N)

    s = emcee_b200.EnsembleSampler(N, D, models.HostFunction(lambda x: np.zeros(x.shape[0]), vectorize=True),
                                   moves=moves.MHMove(moves.HostProposal(next_row)), seed=SEED)
    s.enable_autocorr(max_lag)
    s.run_mcmc(series[0], n, store=False, skip_initial_state_check=True)
    x = series[1:]
    exact, _, _ = acf_exact.exact_acf(x, np.arange(max_lag + 1))
    rho = s.autocorr_function()
    assert np.all(np.abs(rho - exact) <= ref.rounding_bound(x, max_lag) + acf_exact.U * np.abs(exact))


def _rho_after(case, cut, max_lag=20, every=1, total=300):
    s = _make(case)
    s.enable_autocorr(max_lag, every)
    st = _p0(case)
    reads = []
    if cut == "one":
        s.run_mcmc(st, total, store=False)
    elif cut == "many":
        done = 0
        for k in [1, 62, 1, 1, 63, 7, 50]:
            st = s.run_mcmc(st, k, store=False)
            reads.append(s.autocorr_function())  # mid-block reads
            done += k
        s.run_mcmc(st, total - done, store=False)
    elif cut == "sample":
        for k, _ in enumerate(s.sample(st, iterations=total, store=False)):
            if k in (0, 63, 64, 100):
                reads.append(s.autocorr_function())
    elif cut == "unbounded":
        for k, _ in enumerate(s.sample(st, iterations=None, store=False)):
            if k + 1 == total:
                break
    return s.autocorr_function(), reads


@pytest.mark.parametrize("case", ["tma_rows", "generic_odd", "dense_dmma"])
def test_invariance(case):
    want, _ = _rho_after(case, "one")
    for cut in ("many", "sample", "unbounded"):
        got, reads = _rho_after(case, cut)
        assert same(got, want), cut


def test_nothing_else_moves():
    out = []
    for on in (False, True):
        s = _make("dense_dmma", DeviceBackend())
        s.enable_trace(1)
        s.enable_reservoir(100, 2)
        if on:
            s.enable_autocorr(16, 1)
        s.run_mcmc(_p0("dense_dmma"), 70)
        out.append((s.get_chain(), s.get_log_prob(), s.acceptance_fraction, s.trace().mean,
                    s.reservoir().coords))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_lifecycle():
    s = _make("tma_rows")
    with pytest.raises(RuntimeError, match="not enabled"):
        s.autocorr_function()
    with pytest.raises(RuntimeError):  # the library's EB_ERR_STATE through the engine
        s._engine.running_acf_read(4)
    s.enable_autocorr(8, 1)
    st = s.run_mcmc(_p0("tma_rows"), 90, store=False)
    first = s.autocorr_function()
    s.enable_autocorr(8, 0)  # freezes
    st = s.run_mcmc(st, 20, store=False)
    assert s.autocorr_count() == 90 and same(s.autocorr_function(), first)
    s.enable_autocorr(5, 2)  # re-enable: new lags, recorded from scratch
    s.run_mcmc(st, 40, store=False)
    assert s.autocorr_count() == 20 and s.autocorr_function().shape == (6, 8)
    with pytest.raises(MemoryError):
        s.enable_autocorr(2 ** 40, 1)
    assert s.autocorr_count() == 20 and s.autocorr_function().shape == (6, 8)  # nothing changed


def test_stuck_walker_is_nan():
    """a walker the model never lets move keeps a constant series: 0 / 0, NaN in every lag of its parameters"""
    N, D = 32, 4

    def lp(x):
        out = -0.5 * np.sum(np.square(x), axis=1)
        out[np.all(x == 7.0, axis=1)] = 1e300  # walker 5 sits at a point no proposal beats
        return out

    p0 = np.random.default_rng(1).standard_normal((N, D))
    p0[5] = 7.0
    s = emcee_b200.EnsembleSampler(N, D, models.HostFunction(lp, vectorize=True), seed=SEED)
    s.enable_autocorr(10)
    s.run_mcmc(p0, 100, store=False, skip_initial_state_check=True)
    assert np.all(np.isnan(s.autocorr_function()))


def test_window_beyond_max_lag():
    s = _make("tma_rows")
    s.enable_autocorr(3, 1)
    s.run_mcmc(_p0("tma_rows"), 400, store=False)
    with pytest.raises(autocorr.AutocorrError, match="max_lag = 3"):
        s.autocorr_time()
    rho = s.autocorr_function()
    taus = 2.0 * np.cumsum(rho, axis=0) - 1.0
    assert np.array_equal(s.autocorr_time(quiet=True), taus[3])
