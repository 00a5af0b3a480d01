"""WalkMove / MHMove / GaussianMove on the device vs the oracle at sizes beyond the golden cases, and their
host-side contracts (reference: moves/walk.py, moves/mh.py, moves/gaussian.py).  Golden-vector parity of the
same moves is in tests/test_gpu_parity.py (test_golden_chain / _single_steps / _run_mcmc_bulk pick the new
fixtures up by name).  Tolerance 1e-9: normals go through device log / sincos, WalkMove through a Cholesky
factor; accept masks and counts must still agree exactly."""
import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T

from gpu_util import device_model

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu


def _run_pair(name, N, D, omoves, dmoves, nsteps, seed=0x3A7):
    target, p0 = T.make_config(name, N, D)
    o = rb.OracleSampler(N, D, target, omoves, seed=seed)
    o.set_state(p0)
    s = emcee_b200.EnsembleSampler(N, D, device_model(name, target=target), moves=dmoves, seed=seed)
    k = 0
    for state in s.sample(p0, iterations=nsteps, skip_initial_state_check=True, store=False):
        o.run(1)
        k += 1
        np.testing.assert_allclose(state.coords, o.coords, rtol=1e-9, atol=1e-10, err_msg="step %d" % k)
        np.testing.assert_allclose(state.log_prob, o.log_prob, rtol=1e-8, atol=1e-8)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    return s, o


def test_walk_whole_complement_at_scale():
    s, o = _run_pair("gauss_dense", 4096, 32, [(rb.Walk(), 1.0)], moves.WalkMove(), 6)
    assert s._engine.last_kernel_name() == "walk"
    assert 0.05 < o.naccepted.mean() / 6 < 0.95


def test_walk_whole_complement_odd_sizes_three_splits():
    _run_pair("ring", 1003, 7, [(rb.Walk(nsplits=3), 1.0)], moves.WalkMove(nsplits=3), 6)


@pytest.mark.parametrize("name,D", [("gauss_iso", 136), ("ring", 260)])
def test_walk_whole_complement_above_128_dims(name, D):
    """The moment sums of the complement take several passes above 128 columns (analysis.cu MOM_MAXB), and
    cov_chol factors a matrix larger than 128 x 128."""
    s, _ = _run_pair(name, 4 * D + 3, D, [(rb.Walk(), 1.0)], moves.WalkMove(), 4)
    assert s._engine.last_kernel_variant() == "walk"


def test_walk_helper_subsets():
    _run_pair("rosenbrock", 512, 16, [(rb.Walk(s=40), 1.0)], moves.WalkMove(s=40), 6)
    # rank-deficient covariances (s <= ndim): the walk stays in the helpers' span
    _run_pair("gauss_iso", 256, 12, [(rb.Walk(s=5), 1.0)], moves.WalkMove(s=5), 6)


@pytest.mark.parametrize("mode,factor", [("vector", None), ("random", 1.7), ("sequential", None)])
def test_gaussian_scalar_and_diagonal(mode, factor):
    D = 24
    _run_pair("gauss_iso", 2048, D, [(rb.Gaussian(0.04, mode, factor), 1.0)], moves.GaussianMove(0.04, mode=mode, factor=factor), 7)
    var = np.linspace(0.01, 0.09, D)
    _run_pair("ring", 1024, D, [(rb.Gaussian(var, mode, factor), 1.0)], moves.GaussianMove(var, mode=mode, factor=factor), 7)


def test_gaussian_full_covariance():
    D = 64
    target, _ = T.make_config("gauss_dense", 8, D)
    cov = 0.02 * np.linalg.inv(target.icov)
    s, o = _run_pair("gauss_dense", 4096, D, [(rb.Gaussian(cov, factor=1.3), 1.0)], moves.GaussianMove(cov, factor=1.3), 6)
    assert s._engine.last_kernel_name() == "gaussian"


def test_mixture_with_sequential_index_across_calls():
    """A stateful move inside a mixture: its dimension index advances only on the steps it is picked, across
    run_mcmc calls and the step-by-step generator alike (gaussian.py:102-103)."""
    N, D, seed = 256, 5, 77
    target, p0 = T.make_config("gauss_iso", N, D)
    om = [(rb.Gaussian(np.full(D, 0.1), "sequential"), 0.6), (rb.Stretch(), 0.4)]
    o = rb.OracleSampler(N, D, target, om, seed=seed)
    o.set_state(p0)
    dm = [(moves.GaussianMove(np.full(D, 0.1), mode="sequential"), 0.6), (moves.StretchMove(), 0.4)]
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=dm, seed=seed)
    st = s.run_mcmc(p0, 7, store=False, skip_initial_state_check=True)
    o.run(7)
    np.testing.assert_allclose(st.coords, o.coords, rtol=1e-9, atol=1e-10)
    assert dm[0][0].index == om[0][0].index
    for st in s.sample(st, iterations=6, store=False, skip_initial_state_check=True):
        o.run(1)
        np.testing.assert_allclose(st.coords, o.coords, rtol=1e-9, atol=1e-10)
    st = s.run_mcmc(st, 5, skip_initial_state_check=True)
    o.run(5)
    np.testing.assert_allclose(st.coords, o.coords, rtol=1e-9, atol=1e-10)
    assert dm[0][0].index == om[0][0].index
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))


def test_mh_propose_through_the_plugin_boundary():
    """MHMove.propose(model, state) as the reference's sampler calls it (ensemble.py:409)."""
    N, D, seed = 128, 3, 5
    target, p0 = T.make_config("gauss_iso", N, D)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=seed)
    mv = moves.GaussianMove(0.2)
    state = emcee_b200.State(p0, log_prob=s.compute_log_prob(p0)[0])
    state, acc = mv.propose(s.model, state)
    o = rb.OracleSampler(N, D, target, [(rb.Gaussian(0.2), 1.0)], seed=seed)
    o.set_state(p0)
    acc_o = o.run(1)
    assert np.array_equal(acc, acc_o)
    np.testing.assert_allclose(state.coords, o.coords, rtol=1e-12, atol=1e-13)
    with pytest.raises(ValueError, match="Dimension mismatch"):
        moves.GaussianMove(np.ones(4)).propose(s.model, state)


def test_errors():
    s = emcee_b200.EnsembleSampler(64, 4, models.GaussianIso(), moves=moves.WalkMove(s=40), seed=1)
    with pytest.raises(ValueError, match="WalkMove needs"):
        s.run_mcmc(np.random.default_rng(0).standard_normal((64, 4)), 1, skip_initial_state_check=True)
    s = emcee_b200.EnsembleSampler(64, 4, models.GaussianIso(), moves=moves.GaussianMove(np.ones(3)), seed=1)
    with pytest.raises(ValueError, match="Invalid proposal scale dimensions"):
        s.run_mcmc(np.random.default_rng(0).standard_normal((64, 4)), 1, skip_initial_state_check=True)
    # a red-blue move still refuses nwalkers < 2 ndim (red_blue.py:64-70); the Metropolis family does not
    s = emcee_b200.EnsembleSampler(6, 4, models.GaussianIso(), moves=moves.WalkMove(), seed=1)
    with pytest.raises(RuntimeError):
        s.run_mcmc(np.random.default_rng(0).standard_normal((6, 4)), 1, skip_initial_state_check=True)
    s = emcee_b200.EnsembleSampler(6, 4, models.GaussianIso(), moves=moves.GaussianMove(0.1), seed=1)
    s.run_mcmc(np.random.default_rng(0).standard_normal((6, 4)), 3, skip_initial_state_check=True)
