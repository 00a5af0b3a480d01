"""Parity of the CUDA path (through the C ABI) with the golden vectors of the
unmodified reference and with the oracle at larger sizes.

Tolerances (fp64):
  * complement indices, accept masks, accept counts ........ bit-exact
  * stretch-move coordinates (sub, mul, sub, no FMA) ....... bit-exact
  * log-probabilities ....................................... rtol 1e-12 (summation order differs)
  * DE / snooker coordinates ................................ rtol 1e-12 (cos/log of Box-Muller,
    BLAS dot order in the reference's per-walker snooker loop)
"""
import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T

from gpu_util import device_model, device_moves, golden_sampler, move_rows_from_oracle, single_step_tol
from util import golden_names, load_golden, oracle_sampler

import emcee_b200

pytestmark = pytest.mark.gpu

LP_RTOL, LP_ATOL = 1e-12, 1e-12


def _tols(g):
    """(exact, rtol, atol) for free-running chains.  The snooker update divides by
    |s - z| (de_snooker.py:42-43): last-bit differences in the dot products grow
    by ~1.6x per step (the numpy oracle with einsum instead of per-row np.dot
    drifts to 1e-8 after 40 steps against the reference itself), so free-running
    snooker chains are compared loosely and every single step tightly
    (test_golden_single_steps)."""
    kinds = set(g["moves"][:, 0].astype(int))
    if kinds == {0}:
        return True, 0.0, 0.0
    if 2 in kinds:
        return False, 1e-5, 1e-6
    if kinds & {3, 4}:
        # WalkMove / GaussianMove: normals through device log / sincos (last-ulp differences from numpy's),
        # WalkMove also through a Cholesky factor whose rounding scales with cond(cov)
        return False, 1e-9, 1e-11
    return False, 1e-12, 1e-12


@pytest.mark.parametrize("name", golden_names())
def test_golden_chain(name):
    g = load_golden(name)
    s = golden_sampler(g)
    nsteps = g["chain"].shape[0]
    exact, rtol, atol = _tols(g)
    k = 0
    for state in s.sample(g["p0"], iterations=nsteps, skip_initial_state_check=True):
        if exact:
            assert np.array_equal(state.coords, g["chain"][k]), (name, k)
        else:
            np.testing.assert_allclose(state.coords, g["chain"][k], rtol=rtol, atol=atol, err_msg="%s step %d" % (name, k))
        np.testing.assert_allclose(state.log_prob, g["log_prob"][k], rtol=max(rtol, LP_RTOL), atol=max(10 * atol, LP_ATOL))
        k += 1
    assert k == nsteps
    assert np.array_equal(s.backend.accepted, g["accepted"].sum(axis=0))
    assert s.random_state == ("philox4x32-10", int(g["seed"]), nsteps)


@pytest.mark.parametrize("name", golden_names())
def test_golden_single_steps(name):
    """Every step on its own: start from the reference's state k-1, run step k,
    compare with the reference's state k -- no error compounding, so the
    tolerance is tight for every move (and exact for the stretch move)."""
    g = load_golden(name)
    s = golden_sampler(g)
    eng = s._engine
    exact = _tols(g)[0]
    step_tol = single_step_tol(g)
    lp_tol = step_tol if step_tol > 1e-11 else LP_RTOL  # a rank-deficient Walk: its log-probs follow its coordinates
    prev_c, prev_lp = g["p0"], g["lp0"]
    for k in range(g["chain"].shape[0]):
        for m in s._moves:  # GaussianMove "sequential" (single-move schedules here): k earlier picks
            if hasattr(m, "index"):
                m.index = k % int(g["ndim"])
        sched = s._schedule()
        eng.set_state(prev_c, prev_lp)
        eng.set_rng(int(g["seed"]), k)
        acc = eng.step(sched, 1)
        coords, lp = eng.get_state()
        assert np.array_equal(acc, g["accepted"][k]), (name, k)
        if exact:
            assert np.array_equal(coords, g["chain"][k]), (name, k)
        else:
            np.testing.assert_allclose(coords, g["chain"][k], rtol=step_tol, atol=step_tol, err_msg="%s step %d" % (name, k))
        np.testing.assert_allclose(lp, g["log_prob"][k], rtol=lp_tol, atol=max(lp_tol, LP_ATOL))
        prev_c, prev_lp = g["chain"][k], g["log_prob"][k]


@pytest.mark.parametrize("name", golden_names())
def test_golden_run_mcmc_bulk(name):
    """run_mcmc = one C-ABI call for the whole run; must equal the stepwise chain."""
    g = load_golden(name)
    s = golden_sampler(g)
    nsteps = g["chain"].shape[0]
    exact, rtol, atol = _tols(g)
    last = s.run_mcmc(g["p0"], nsteps, skip_initial_state_check=True)
    np.testing.assert_allclose(s.get_chain(), g["chain"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(s.get_log_prob(), g["log_prob"], rtol=max(rtol, LP_RTOL), atol=max(10 * atol, LP_ATOL))
    assert np.array_equal(s.backend.accepted, g["accepted"].sum(axis=0))
    assert np.array_equal(last.coords, s.get_chain()[-1])
    # store=False path gives the same final state
    s2 = golden_sampler(g)
    last2 = s2.run_mcmc(g["p0"], nsteps, skip_initial_state_check=True, store=False)
    assert np.array_equal(last2.coords, last.coords) and np.array_equal(last2.log_prob, last.log_prob)
    assert np.array_equal(s2._engine.naccepted(), g["accepted"].sum(axis=0).astype(np.uint64))


def test_initial_log_prob_matches():
    for name in golden_names():
        g = load_golden(name)
        s = golden_sampler(g)
        lp, blobs = s.compute_log_prob(g["p0"])
        assert blobs is None and lp.dtype == np.float64
        np.testing.assert_allclose(lp, g["lp0"], rtol=LP_RTOL, atol=LP_ATOL)


def test_draw_taps_bit_exact():
    """rint / zz / accept uniforms of a half-step, against the oracle's taps."""
    g = load_golden("stretch_dense_64x8")
    o = oracle_sampler(g)
    s = golden_sampler(g)
    eng = s._engine
    eng.set_option("debug_taps", 1)
    eng.set_state(g["p0"])
    sched = s._schedule()
    for _ in range(5):
        o.run(1)
        eng.step(sched, 1)
        taps = eng.debug_taps()  # last half-step = split 1
        assert np.array_equal(taps["active"], o.taps["active"])
        assert np.array_equal(taps["partners"][0], o.taps["partner"])
        assert np.array_equal(taps["scalar"], o.taps["zz"])
        assert np.array_equal(taps["u_accept"], o.taps["u_accept"])


CASES = [
    # name, N, D, moves, nsteps
    ("gauss_dense", 4096, 128, [(rb.Stretch(), 1.0)], 12),
    ("gauss_dense", 2048, 64, [(rb.Stretch(a=2.5, nsplits=3), 1.0)], 8),
    ("gauss_dense", 1000, 24, [(rb.Stretch(randomize_split=False), 1.0)], 8),
    # dense_dmma with partial tiles (active counts not multiples of 8), three splits, fewer tiles than SMs
    ("gauss_dense", 1004, 32, [(rb.Stretch(), 1.0)], 10),
    ("gauss_dense", 301, 48, [(rb.Stretch(nsplits=3), 1.0)], 10),
    ("gauss_dense", 100, 16, [(rb.Stretch(a=1.5), 1.0)], 10),
    ("gauss_dense", 20000, 96, [(rb.Stretch(), 1.0)], 6),
    ("gauss_iso", 512, 37, [(rb.Stretch(), 1.0)], 10),
    ("ring", 16384, 32, [(rb.Stretch(), 1.0)], 8),
    ("rosenbrock", 2048, 256, [(rb.DE(), 0.8), (rb.Snooker(), 0.2)], 12),
    ("rosenbrock", 1024, 16, [(rb.DE(sigma=1e-3, gamma0=0.7), 1.0)], 8),
    ("gauss_iso", 640, 5, [(rb.Snooker(gammas=1.2), 1.0)], 8),
]


@pytest.mark.parametrize("D", [8, 24, 40, 56, 72, 80, 88, 104, 112, 120])
def test_dense_dmma_every_width(D):
    """the tensor-core kernel is instantiated for every ndim = 8k <= 128 (with and without a mean)"""
    N = 2 * D + 8 * (D % 5) + 42  # active counts that are not multiples of 8
    target, p0 = T.make_config("gauss_dense", N, D)
    mean = np.linspace(-0.5, 0.5, D) if D % 16 == 8 else None
    tgt = T.GaussDense(target.icov, mean)
    o = rb.OracleSampler(N, D, tgt, [(rb.Stretch(), 1.0)], seed=D)
    o.set_state(p0)
    s = emcee_b200.EnsembleSampler(N, D, emcee_b200.models.GaussianDense(target.icov, mean), seed=D)
    last = s.run_mcmc(p0, 6, store=False, skip_initial_state_check=True)
    o.run(6)
    assert s._engine.last_kernel_name() == "dense_dmma"
    assert np.array_equal(last.coords, o.coords)
    np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-11, atol=1e-11)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))


@pytest.mark.parametrize("name,N,D,omoves,nsteps", CASES)
def test_against_oracle(name, N, D, omoves, nsteps):
    target, p0 = T.make_config(name, N, D)
    seed = 0xB200 + N + D
    o = rb.OracleSampler(N, D, target, omoves, seed=seed)
    o.set_state(p0)
    s = emcee_b200.EnsembleSampler(
        N, D, device_model(name, target=target), moves=device_moves(move_rows_from_oracle(omoves)), seed=seed
    )
    stretch_only = all(m.kind == "stretch" for m, _ in omoves)
    snooker = any(m.kind == "snooker" for m, _ in omoves)
    tol = 1e-6 if snooker else 1e-11  # free-running snooker chains amplify last-bit differences (see _tols)
    k = 0
    for state in s.sample(p0, iterations=nsteps, skip_initial_state_check=True, store=False):
        acc_o = o.run(1)
        k += 1
        if stretch_only:
            assert np.array_equal(state.coords, o.coords), k
        else:
            np.testing.assert_allclose(state.coords, o.coords, rtol=tol, atol=tol)
        np.testing.assert_allclose(state.log_prob, o.log_prob, rtol=max(tol, 1e-11), atol=max(100 * tol, 1e-11))
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    # chain moments within 1e-6 relative (north_star): trivially true when the states agree
    np.testing.assert_allclose(state.coords.mean(0), o.coords.mean(0), rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(np.cov(state.coords.T), np.cov(o.coords.T), rtol=1e-6, atol=1e-9)
