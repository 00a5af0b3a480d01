"""Device-side chain analysis through the C ABI: running moments (eb_moments), the
independence check (eb_walkers_gram), sharded state read-back on one GPU, and that the
programmatic-dependent-launch chain does not change results.

Tolerances: moments vs numpy on the reference-generated golden chains rtol 1e-12 (fp64
summation order); at 4096 x 128 vs the oracle rtol 1e-6 (north_star's chain mean / cov bar)."""
import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T

from gpu_util import golden_sampler
from util import golden_names, load_golden

import emcee_b200
from emcee_b200 import ensemble as ens
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["stretch_iso_32x5", "stretch_dense_mean_96x16", "de_rosen_40x4", "stretch_iso_odd_37x3"])
def test_moments_match_numpy_on_golden_chains(name):
    g = load_golden(name)
    s = golden_sampler(g)
    s.enable_moments(1)
    nsteps = g["chain"].shape[0]
    s.run_mcmc(g["p0"], nsteps, store=False, skip_initial_state_check=True)
    mean, cov, n = s.moments()
    flat = g["chain"].reshape(-1, g["chain"].shape[-1])
    assert n == flat.shape[0]
    exact = set(g["moves"][:, 0].astype(int)) == {0}
    tol = 1e-12 if exact else 1e-9  # DE chains agree with the reference to 1e-12 per step, not bit for bit
    np.testing.assert_allclose(mean, flat.mean(0), rtol=tol, atol=tol)
    np.testing.assert_allclose(cov, np.atleast_2d(np.cov(flat, rowvar=False)), rtol=max(tol, 1e-11), atol=tol)
    # accept total = sum of the reference's accept masks
    _, _, _, nacc = s._engine.moments()
    assert nacc == int(g["accepted"].sum())


def test_moments_thinned_and_reset():
    g = load_golden("stretch_ring_80x6")
    s = golden_sampler(g)
    s.enable_moments(3)
    s.run_mcmc(g["p0"], 30, store=False, skip_initial_state_check=True)
    mean, cov, n = s.moments()
    flat = g["chain"][2:30:3].reshape(-1, 6)
    assert n == flat.shape[0]
    np.testing.assert_allclose(mean, flat.mean(0), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(cov, np.cov(flat, rowvar=False), rtol=1e-11, atol=1e-13)
    s.enable_moments(1)  # resets
    assert s.moments()[2] == 0


def test_moments_at_scale_vs_oracle():
    """4096 x 128 dense Gaussian (BASELINE config 2): chain mean / covariance within 1e-6 of the CPU
    oracle's chain (north_star's bar); the states themselves agree bit for bit."""
    N, D, steps, seed = 4096, 128, 12, 0xC0FFEE
    target, p0 = T.make_config("gauss_dense", N, D)
    o = rb.OracleSampler(N, D, target, [(rb.Stretch(), 1.0)], seed=seed)
    o.set_state(p0)
    s1 = np.zeros(D)
    flat = []
    for _ in range(steps):
        o.run(1)
        flat.append(o.coords.copy())
    flat = np.concatenate(flat)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(target.icov), seed=seed)
    s.enable_moments(1)
    last = s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
    assert np.array_equal(last.coords, o.coords)
    mean, cov, n = s.moments()
    assert n == N * steps
    np.testing.assert_allclose(mean, flat.mean(0), rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(cov, np.cov(flat, rowvar=False), rtol=1e-6, atol=1e-9)
    assert s._engine.last_kernel_name() == "dense_dmma"


@pytest.mark.parametrize(
    "shape",
    [(64, 5), (300, 17), (4096, 128), (2048, 256),
     # above 128 columns the moment sums take several passes (MOM_MAXB); odd row counts leave partial CTAs
     (301, 129), (517, 255), (1041, 520), (2053, 1023), (2049, 1024)],
)
def test_walkers_gram_matches_host(shape):
    rng = np.random.default_rng(5)
    N, D = shape
    x = rng.standard_normal((N, D)) @ rng.standard_normal((D, D)) + 3.0
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=1)
    gram, flags = s._engine.walkers_gram(x)
    assert flags == 0
    c = x - x.mean(0)
    c /= np.abs(c).max(0)
    c /= np.sqrt((c ** 2).sum(0))
    np.testing.assert_allclose(gram, c.T @ c, rtol=1e-10, atol=1e-12)
    assert s._walkers_independent(x) == bool(ens.walkers_independent(x))


def test_walkers_independent_decisions():
    """The cases the reference's own tests pin (tests/unit/test_sampler.py:212-222, test_ensemble.py):
    dependent, degenerate and non-finite ensembles are refused, a healthy one is accepted."""
    rng = np.random.default_rng(11)
    N, D = 32, 4
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=1)
    good = rng.standard_normal((N, D))
    assert s._walkers_independent(good)
    line = np.outer(rng.standard_normal(N), np.ones(D))  # rank 1
    assert not s._walkers_independent(line)
    const = good.copy()
    const[:, 2] = 1.5  # zero span
    assert not s._walkers_independent(const)
    bad = good.copy()
    bad[3, 1] = np.inf
    assert not s._walkers_independent(bad)
    nearly = good.copy()
    nearly[:, 3] = nearly[:, 0] + 1e-9 * rng.standard_normal(N)  # cond ~ 1e9: the host SVD decides
    assert s._walkers_independent(nearly) == bool(ens.walkers_independent(nearly))
    with pytest.raises(ValueError, match="large condition number"):
        s.run_mcmc(line, 1)
    # small offsets around a large mean stay independent (ensemble.py:656 centres first)
    assert s._walkers_independent(1e6 + 1e-3 * good)


def test_owned_rows_and_row_reads_on_one_gpu():
    g = load_golden("stretch_dense_64x8")
    s = golden_sampler(g)
    last = s.run_mcmc(g["p0"], 5, store=False, skip_initial_state_check=True)
    assert s.owned_rows == slice(0, 64)
    c = np.zeros((64, 8))
    lp = np.zeros(64)
    s._engine.get_state_rows(10, 20, c, lp)
    assert np.array_equal(c[10:30], last.coords[10:30]) and np.all(c[:10] == 0) and np.all(c[30:] == 0)
    assert np.array_equal(lp[10:30], last.log_prob[10:30])
    with pytest.raises(ValueError):
        s._engine.get_state_rows(60, 10, c, lp)


def test_pdl_chain_does_not_change_results():
    N, D, steps = 2048, 64, 20
    target, p0 = T.make_config("gauss_dense", N, D)
    out = []
    for pdl in (1, 0):
        s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(target.icov), seed=9)
        s._engine.set_option("pdl", pdl)
        last = s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
        assert s._engine.last_kernel_name() == "dense_dmma"
        out.append((last.coords.copy(), last.log_prob.copy(), s._engine.naccepted()))
    for a, b in zip(out[0], out[1]):
        assert np.array_equal(a, b)


def test_host_moves_are_rejected_up_front():
    class HostMove(object):
        def propose(self, model, state):
            return state, None

    with pytest.raises(TypeError, match="device moves"):
        emcee_b200.EnsembleSampler(8, 2, models.GaussianIso(), moves=HostMove())
    with pytest.raises(TypeError, match="device moves"):
        emcee_b200.EnsembleSampler(8, 2, models.GaussianIso(), moves=[(moves.StretchMove(), 0.5), (HostMove(), 0.5)])


# ---- autocorrelation on the device (autocorr.py:49-123) ---------------------------------------------
import os  # noqa: E402

from emcee_b200 import autocorr  # noqa: E402

_FIX = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "fixtures", "autocorr_reference.npz"))


def _ar1_chain(seed, n, w, d):
    rng = np.random.default_rng(seed)
    x = np.empty((n, w, d))
    x[0] = 0
    e = rng.random((n, w, d))
    for i in range(1, n):
        x[i] = x[i - 1] * 0.9 + e[i]
    return x


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_device_autocorr_matches_reference_fixture(name):
    """tau from the GPU FFTs vs the values the UNMODIFIED reference computed for the same seeded AR(1)
    chains (tests/fixtures/autocorr_reference.npz, oracle/gen_autocorr_fixture.py).  FFT lengths
    16 384 .. 131 072: shared-memory stages plus the global-memory large-span passes."""
    seed, n, w, d = (int(v) for v in _FIX["cfg_" + name])
    s = emcee_b200.EnsembleSampler(8, 2, models.GaussianIso(), seed=1)
    x = _ar1_chain(seed, n, w, d)
    tau = autocorr.integrated_time(x, quiet=True, engine=s._engine)
    np.testing.assert_allclose(tau, _FIX["tau_" + name], rtol=1e-8)
    rho_dev = s._engine.autocorr_function(x)
    rho_host = np.mean(autocorr._acf(x), axis=1)
    np.testing.assert_allclose(rho_dev, rho_host, rtol=0, atol=2e-10)


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 3, 2), (37, 5, 3), (1000, 64, 5), (3000, 2, 2), (4096, 3, 1), (4097, 2, 2)])
def test_device_autocorr_function_small_and_odd_lengths(shape):
    n, w, d = shape
    s = emcee_b200.EnsembleSampler(8, 2, models.GaussianIso(), seed=1)
    x = _ar1_chain(7, n, w, d) if n > 1 else np.ones((1, 1, 1))
    got = s._engine.autocorr_function(x)
    want = np.mean(autocorr._acf(x), axis=1)
    assert got.shape == (n, d)
    if n == 1:
        assert np.all(np.isnan(got)) and np.all(np.isnan(want))  # 0 / 0, as numpy gives
        return
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    if shape == (3000, 2, 2):  # the reference's function_1d on the fixture's own series (seed 5)
        x5 = _ar1_chain(5, 3000, 2, 2)
        np.testing.assert_allclose(s._engine.autocorr_function(x5[:, :1, :1])[:16, 0], _FIX["acf_head"], rtol=1e-9, atol=1e-12)


def test_sampler_get_autocorr_time_uses_the_device():
    g = load_golden("stretch_iso_32x5")
    s = golden_sampler(g)
    s.run_mcmc(g["p0"], 60, skip_initial_state_check=True)
    tau_dev = s.get_autocorr_time(quiet=True)
    tau_host = autocorr.integrated_time(s.get_chain(), quiet=True)
    np.testing.assert_allclose(tau_dev, tau_host, rtol=1e-9)
    with pytest.raises(autocorr.AutocorrError):
        s.get_autocorr_time()
