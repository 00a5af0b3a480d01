"""``BatchSampler`` storing into a ``DeviceBackend``, and the per-ensemble summaries read where the chain is.

* Store: the same batch stored into ``DeviceBackend()`` and into the host ``Backend()`` gives byte-equal chains,
  log-probabilities, accept counts, final states and last samples, across moves x models x shapes x K x ``thin_by``,
  split ``run_mcmc`` calls, ``sample()``, a torch ``CudaArrayFunction`` over per-ensemble data (also returning NaN in
  the middle of a run: ``iteration`` is the number of steps stored) and K = 8 192.
* ``cuda=True`` reads equal the host reads, flat (``[K, n N, D]``, ``eb_chain_read_segments_to``) and not flat.
* ``get_autocorr_time``: row ``k`` equals, with ``==``, the twin ``EnsembleSampler`` storing into its own
  ``DeviceBackend`` (``eb_chain_autocorr_segments`` against ``eb_chain_autocorr``), agrees with the host route's
  numpy FFTs within DESIGN 5.6's ``rtol = 1e-8``, and names the same failing ensembles.
* ``get_percentile`` equals ``np.percentile`` of each ensemble's flat slice with ``==``, including a NaN in one
  ensemble's parameter; ``get_moments`` meets a long-double bound, agrees with the host route and repeats bit for bit.
* Refusals: ``nseg`` that does not divide the walkers, and a ``grow`` that cannot fit.
"""
import numpy as np
import pytest

import proposals_exact as PX
from test_gpu_batch import MODELS, MOVES, _cases, _lp, _p0, _seeds

import emcee_b200
from emcee_b200 import DeviceBackend, State, autocorr, models, moves

pytestmark = pytest.mark.gpu

STEPS = 40


def _pair(K, N, D, model, move, seeds):
    """A batch storing on the device and its host-stored twin batch."""
    dev = emcee_b200.BatchSampler(K, N, D, model(), moves=move(), seeds=seeds, backend=DeviceBackend())
    host = emcee_b200.BatchSampler(K, N, D, model(), moves=move(), seeds=seeds)
    return dev, host


def _assert_same_store(dev, host, last_d=None, last_h=None):
    assert dev.iteration == host.iteration
    assert np.array_equal(dev.get_chain(), host.get_chain())
    assert np.array_equal(dev.get_log_prob(), host.get_log_prob())
    assert np.array_equal(dev.backend.accepted, host.backend.accepted)
    assert np.array_equal(dev.acceptance_fraction, host.acceptance_fraction)
    ld, lh = dev.get_last_sample(), host.get_last_sample()
    assert np.array_equal(ld.coords, lh.coords) and np.array_equal(ld.log_prob, lh.log_prob)
    assert ld.random_state[2] == lh.random_state[2]
    assert np.array_equal(ld.random_state[1], lh.random_state[1])
    if last_d is not None:
        assert np.array_equal(last_d.coords, last_h.coords)
        assert np.array_equal(last_d.log_prob, last_h.log_prob)


# ---- store ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mv,model,K,N,D,P,rand,thin_by", _cases())
def test_store_equals_host(mv, model, K, N, D, P, rand, thin_by):
    dev, host = _pair(K, N, D, lambda: MODELS[model](D), lambda: MOVES[mv](P, rand), _seeds(K))
    p0 = _p0(K, N, D)
    ld = dev.run_mcmc(p0, STEPS, thin_by=thin_by, skip_initial_state_check=True)
    lh = host.run_mcmc(p0, STEPS, thin_by=thin_by, skip_initial_state_check=True)
    _assert_same_store(dev, host, ld, lh)


def test_split_calls_sample_and_resume():
    K, N, D = 6, 32, 5
    p0 = _p0(K, N, D)
    one = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40)
    one.run_mcmc(p0, 60, thin_by=3, skip_initial_state_check=True)
    two = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40,
                                  backend=DeviceBackend())
    two.run_mcmc(p0, 25, thin_by=3, skip_initial_state_check=True)
    two.run_mcmc(None, 20, thin_by=3)
    # a sampler built on the initialised backend resumes from its last sample and random state
    three = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=1,
                                    backend=two.backend)
    assert three.iteration == 45 and three.random_state[2] == 135
    three.run_mcmc(None, 15, thin_by=3)
    _assert_same_store(three, one)
    four = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40,
                                   backend=DeviceBackend())
    for _ in four.sample(p0, iterations=60, thin_by=3, skip_initial_state_check=True):
        pass
    _assert_same_store(four, one)


@pytest.mark.parametrize("nan_at", [None, 31])
def test_torch_function_and_nan(nan_at):
    """A torch ``CudaArrayFunction`` over ``data[K, D]``; with ``nan_at``, ensemble 1's rows turn NaN at that call,
    and both stores stop with the same steps stored."""
    torch = pytest.importorskip("torch")
    K, N, D = 3, 32, 4
    data = torch.as_tensor(np.random.default_rng(2).normal(size=(K, D)), device="cuda")

    def make():
        calls = [0]

        def fn(x):
            calls[0] += 1
            lp = _lp(torch.as_tensor(x, device="cuda"), data)
            if nan_at is not None and calls[0] == nan_at:
                lp[1] = float("nan")
            return lp

        return models.CudaArrayFunction(fn)

    dev, host = _pair(K, N, D, make, moves.StretchMove, _seeds(K, 5))
    p0 = _p0(K, N, D, 4)
    if nan_at is None:
        ld = dev.run_mcmc(p0, STEPS, skip_initial_state_check=True)
        lh = host.run_mcmc(p0, STEPS, skip_initial_state_check=True)
        _assert_same_store(dev, host, ld, lh)
        return
    for s in (dev, host):
        with pytest.raises(ValueError, match="returned NaN"):
            s.run_mcmc(p0, STEPS, skip_initial_state_check=True)
    assert dev.iteration == host.iteration == 14
    assert dev.backend.random_state[2] == host.backend.random_state[2] == 14
    assert np.array_equal(dev.get_chain(), host.get_chain())
    assert np.array_equal(dev.get_log_prob(), host.get_log_prob())


def test_store_8192():
    K, N, D = 8192, 32, 5
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, _seeds(K, 3))
    p0 = _p0(K, N, D, 21)
    ld = dev.run_mcmc(p0, 20, skip_initial_state_check=True)
    lh = host.run_mcmc(p0, 20, skip_initial_state_check=True)
    _assert_same_store(dev, host, ld, lh)


# ---- reads ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("discard,thin", [(0, 1), (3, 2), (10, 7), (39, 1)])
def test_cuda_reads(discard, thin):
    K, N, D = 5, 12, 3
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, _seeds(K, 8))
    p0 = _p0(K, N, D, 6)
    dev.run_mcmc(p0, 20, skip_initial_state_check=True)
    dev.backend.grow(20, None)  # a second device segment: the slices cross it
    dev.run_mcmc(None, 20)
    host.run_mcmc(p0, 20, skip_initial_state_check=True)
    host.run_mcmc(None, 20)
    for name in ("chain", "log_prob"):
        for flat in (False, True):
            want = host.get_value(name, flat=flat, discard=discard, thin=thin)
            got = dev.get_value(name, flat=flat, discard=discard, thin=thin, cuda=True)
            assert got.shape == want.shape
            assert np.array_equal(got.get(), want)
            assert np.array_equal(dev.get_value(name, flat=flat, discard=discard, thin=thin), want)


# ---- autocorrelation ----------------------------------------------------------------------------------------------
def test_autocorr_equals_twins_and_host():
    K, N, D, n = 6, 32, 3, 400
    seeds = _seeds(K, 17)
    p0 = _p0(K, N, D, 12)
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, seeds)
    dev.run_mcmc(p0, n, skip_initial_state_check=True)
    host.run_mcmc(p0, n, skip_initial_state_check=True)
    for discard, thin in ((0, 1), (100, 3)):
        tau_d = dev.get_autocorr_time(discard=discard, thin=thin, quiet=True)
        tau_h = host.get_autocorr_time(discard=discard, thin=thin, quiet=True)
        np.testing.assert_allclose(tau_d, tau_h, rtol=1e-8)
        for k in range(K):
            t = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.StretchMove(), seed=seeds[k],
                                           backend=DeviceBackend())
            t._engine.set_option("tma_rows", 0)
            t._engine.set_option("dense_dmma", 0)
            t.run_mcmc(p0[k], n, skip_initial_state_check=True)
            assert np.array_equal(tau_d[k], t.get_autocorr_time(discard=discard, thin=thin, quiet=True))
    # a tol in the widest gap between the ensembles' estimates: some fail, and both routes name the same ones
    tau_all = dev.get_autocorr_time(quiet=True)
    tau = np.sort(tau_all.max(axis=1))
    g = int(np.argmax(np.diff(tau)))
    tol = n / (0.5 * (tau[g] + tau[g + 1]))
    failing = np.flatnonzero(tau_all.max(axis=1) * tol > n).tolist()
    errs = []
    for s in (dev, host):
        with pytest.raises(autocorr.AutocorrError) as e:
            s.get_autocorr_time(tol=tol)
        errs.append(str(e.value).split("\n")[0])
        np.testing.assert_allclose(e.value.tau, tau_all, rtol=1e-8)
    assert errs[0] == errs[1], errs
    assert "ensemble(s) {0}".format(failing) in errs[0], (errs, failing)


# ---- percentiles ----------------------------------------------------------------------------------------------------
QS = [[16, 50, 84], 0, 100, 50, [[5, 50], [95, 99.5]], np.linspace(0, 100, 21)]


@pytest.mark.parametrize("discard,thin", [(0, 1), (5, 3)])
@pytest.mark.parametrize("name", ["chain", "log_prob"])
def test_percentile_equals_numpy(name, discard, thin):
    K, N, D = 7, 16, 3
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, _seeds(K, 23))
    p0 = _p0(K, N, D, 13)
    dev.run_mcmc(p0, 30, skip_initial_state_check=True)
    host.run_mcmc(p0, 30, skip_initial_state_check=True)
    flat = host.get_value(name, flat=True, discard=discard, thin=thin)
    for q in QS:
        want = np.array([np.percentile(flat[k], q, axis=0) for k in range(K)])
        got = dev.get_percentile(q, discard=discard, thin=thin, name=name)
        assert got.shape == want.shape
        assert np.array_equal(got, want)
        assert np.array_equal(host.get_percentile(q, discard=discard, thin=thin, name=name), want)


def test_percentile_nan_in_one_ensemble():
    K, N, D, n, j, d = 4, 8, 3, 6, 2, 1
    rng = np.random.default_rng(3)
    x = rng.normal(size=(n, K, N, D))
    x[4, j, 5, d] = np.nan
    lp = rng.normal(size=(n, K, N))
    b = DeviceBackend()
    b.reset(K * N, D)
    b.grow(n, None)
    for s in range(n):
        b.save_step(State(x[s].reshape(K * N, D), log_prob=lp[s].reshape(K * N), random_state=None),
                    np.zeros(K * N, dtype=bool))
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, backend=b)
    flat = np.swapaxes(x, 0, 1).reshape(K, n * N, D)
    for q in ([16, 50, 84], 0, 100):
        want = np.array([np.percentile(flat[k], q, axis=0) for k in range(K)])
        got = s.get_percentile(q)
        assert np.array_equal(got, want, equal_nan=True)
        only = np.zeros((K, D), dtype=bool)
        only[j, d] = True
        assert np.array_equal(np.isnan(got), np.broadcast_to(only.reshape((K,) + (1,) * (got.ndim - 2) + (D,)),
                                                             got.shape))


# ---- moments ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,N,D,start", [(9, 32, 5, "near"), (3, 96, 40, "near"), (5, 32, 5, "far")])
def test_moments_exact(K, N, D, start):
    """``get_moments`` of each ensemble against a two-pass long-double reference, under the bound of
    ``test_gpu_chain_summary.test_moments_exact`` with the segmented kernel's accumulation depth: each sum of
    ``eb_chain_moments_segments`` is one chain of FMAs (S2) or additions (S1) over the ``cs * N`` rows of a chunk of
    ``cs`` stored steps, then a chain of additions over the chunks, so at most ``count * N + count`` operations deep.
    The shift is the sequential column mean of the ensemble's first stored step."""
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here")
    rng = np.random.default_rng(K + D)
    p0 = rng.standard_normal((K, N, D)) + (1.0e4 if start == "far" else 0.0)
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, _seeds(K, 31))
    dev.run_mcmc(p0, 50, skip_initial_state_check=True)
    host.run_mcmc(p0, 50, skip_initial_state_check=True)
    mean_d, cov_d, m = dev.get_moments(discard=4, thin=2)
    mean_h, cov_h, m_h = host.get_moments(discard=4, thin=2)
    rows = dev.get_chain(discard=4, thin=2)
    assert m == m_h == rows.shape[0] * N
    again = dev.get_moments(discard=4, thin=2)
    assert np.array_equal(again[0], mean_d) and np.array_equal(again[1], cov_d)
    # within rtol = 1e-10 of the numpy route, measured against each ensemble's spread where an entry is near zero
    scale = np.sqrt(np.einsum("kii->ki", np.abs(cov_h)))
    assert np.all(np.abs(mean_d - mean_h) <= 1e-10 * (np.abs(mean_h) + scale))
    assert np.all(np.abs(cov_d - cov_h) <= 1e-10 * (np.abs(cov_h) + scale[:, :, None] * scale[:, None, :]))
    depth = rows.shape[0] * N + rows.shape[0]
    for k in range(K):
        X = rows[:, k].reshape(-1, D)
        shift = np.cumsum(rows[0, k], axis=0)[-1] / N  # the device's order: walkers ascending
        r_mean, r_cov = PX.segment_moments_ratios(X, shift, mean_d[k], cov_d[k], depth)
        assert r_mean <= 1.0 and r_cov <= 1.0, (k, r_mean, r_cov)


def test_empty_slices_and_bad_q():
    K, N, D = 3, 16, 2
    dev, host = _pair(K, N, D, models.GaussianIso, moves.StretchMove, _seeds(K, 2))
    p0 = _p0(K, N, D)
    dev.run_mcmc(p0, 5, skip_initial_state_check=True)
    host.run_mcmc(p0, 5, skip_initial_state_check=True)
    for s in (dev, host):
        with pytest.raises(ValueError, match="Percentiles must be in the range"):
            s.get_percentile(101)
        with pytest.raises(IndexError):
            s.get_percentile(50, discard=5)
        mean, cov, n = s.get_moments(discard=5)
        assert n == 0 and mean.shape == (K, D) and cov.shape == (K, D, D)
        assert np.isnan(mean).all() and np.isnan(cov).all()


# ---- refusals -----------------------------------------------------------------------------------------------------
def test_nseg_must_divide_walkers():
    s = emcee_b200.BatchSampler(4, 8, 2, models.GaussianIso(), seeds=1, backend=DeviceBackend())
    s.run_mcmc(_p0(4, 8, 2), 5, skip_initial_state_check=True)
    ch = s.backend._ch  # 32 walkers
    calls = [lambda g: ch.autocorr_function(0, 1, 5, nseg=g),
             lambda g: ch.select("chain", 0, 1, 5, np.array([0], dtype=np.uint64), nseg=g),
             lambda g: ch.moments(0, 1, 5, nseg=g)]
    for nseg in (3, 5, 33):
        for call in calls + [lambda g: ch.read_segments_to(g, 0, 1, 5)]:
            with pytest.raises(ValueError, match="nseg"):
                call(nseg)
    for call in calls[:2]:
        with pytest.raises(ValueError, match="nseg"):
            call(0)


def test_grow_that_cannot_fit():
    K, N, D = 4, 32, 5
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, backend=DeviceBackend())
    p0 = _p0(K, N, D)
    with pytest.raises(MemoryError):
        s.run_mcmc(p0, 10**9, skip_initial_state_check=True)
    assert s.iteration == 0
    s.run_mcmc(p0, 5, skip_initial_state_check=True)
    assert s.iteration == 5 and s.get_chain().shape == (5, K, N, D)
    assert s.get_percentile(50).shape == (K, D)
