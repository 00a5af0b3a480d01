"""KDEMove on the device (``kde.cu``) against the unmodified reference's golden runs, the oracle, and an exact
log-sum-exp; the reference's statistical gates; errors, resume and storage paths."""
import numpy as np
import pytest

import emcee_b200
from emcee_b200 import models, moves
from emcee_b200.backend import DeviceBackend
from gpu_util import device_model
from kde_util import kde_names, kde_oracle, kde_sampler, load_kde
from oracle import kde as ok
from oracle import redblue as rb
from oracle import targets as T

pytestmark = pytest.mark.gpu

# Hastings factors of the golden cases: the device's log-sum-exp and its Cholesky factor (moment sums on the tensor
# pipe) against the oracle's (scipy's solve_triangular and numpy's LAPACK factor of np.cov): agree to this bound,
# relative to 1 + |factor|, well inside the accuracy test's derived bound for these shapes
FACTOR_TOL = 1e-10


def _schedule(s):
    return s._schedule()


@pytest.mark.parametrize("name", kde_names())
def test_golden_single_steps(name):
    """Each step from the reference's previous state: accept masks and centres bit for bit, coordinates 1e-11."""
    g = load_kde(name)
    s = kde_sampler(g)
    eng = s._engine
    eng.set_option("debug_taps", 1)
    o = kde_oracle(g)
    x, lp = g["p0"], g["lp0"]
    sched = _schedule(s)
    for k in range(g["chain"].shape[0]):
        eng.set_state(x, lp)
        o.coords, o.log_prob = x.copy(), lp.copy()
        o.taps = {}
        acc = eng.step(sched, 1)
        with np.errstate(invalid="ignore"):
            o.run(1)
        np.testing.assert_array_equal(acc, g["accepted"][k], err_msg="%s step %d" % (name, k))
        xs, lps = eng.get_state()
        np.testing.assert_allclose(xs, g["chain"][k], rtol=1e-11, atol=1e-11, err_msg="step %d" % k)
        np.testing.assert_allclose(lps, g["log_prob"][k], rtol=1e-11, atol=1e-11)
        if "rank" in o.taps:  # a KDE step: the last split's centres and factors
            taps = eng.debug_taps()
            np.testing.assert_array_equal(taps["active"], o.taps["active"])
            np.testing.assert_array_equal(taps["partners"][0], o.taps["partner"])
            np.testing.assert_array_equal(taps["u_accept"], o.taps["u_accept"])
            err = np.abs(taps["scalar"] - o.taps["factors"]) / (1.0 + np.abs(o.taps["factors"]))
            assert err.max() <= FACTOR_TOL, (k, err.max())
        x, lp = g["chain"][k], g["log_prob"][k]
    assert eng.last_kernel_name() in ("kde", "generic", "tma_rows", "dense_dmma")


@pytest.mark.parametrize("name", kde_names())
def test_golden_free_running(name):
    g = load_kde(name)
    s = kde_sampler(g)
    with np.errstate(invalid="ignore"):
        s.run_mcmc(g["p0"], g["chain"].shape[0], skip_initial_state_check=True)
    np.testing.assert_allclose(s.get_chain(), g["chain"], rtol=1e-9, atol=1e-9)
    acc = np.diff(np.concatenate([np.zeros((1, g["accepted"].shape[1])), np.cumsum(g["accepted"], 0)]), axis=0)
    assert np.array_equal(s.backend.accepted, acc.sum(0))


def _torch_logpdf(c, L, x):
    """The oracle's ``kde_logpdf`` with the log-sum-exps on the GPU through torch (direct differences, FP64)."""
    import torch
    from scipy.linalg import solve_triangular

    yc = torch.as_tensor(solve_triangular(L, c.T, lower=True).T, device="cuda")
    yx = torch.as_tensor(solve_triangular(L, x.T, lower=True).T, device="cuda")
    out = []
    for b in range(0, len(x), 2048):
        d = torch.cdist(yx[b:b + 2048], yc, compute_mode="donot_use_mm_for_euclid_dist")
        out.append(torch.logsumexp(-0.5 * d * d, dim=1))
    return torch.cat(out).cpu().numpy()


@pytest.mark.parametrize("N", [16384, 65536])
def test_one_step_at_scale(N, monkeypatch):
    D = 32
    monkeypatch.setattr(ok.KdeOracleSampler, "logpdf", staticmethod(_torch_logpdf))
    target, p0 = T.make_config("gauss_dense", N, D)
    o = ok.KdeOracleSampler(N, D, target, [(ok.KDE(), 1.0)], seed=0xC0DE)
    o.set_state(p0)
    s = emcee_b200.EnsembleSampler(N, D, device_model("gauss_dense", target=target), moves=moves.KDEMove(),
                                   seed=0xC0DE)
    last = s.run_mcmc(p0, 1, store=False, skip_initial_state_check=True)
    o.run(1)
    assert s._engine.last_kernel_name() == "kde"
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    np.testing.assert_allclose(last.coords, o.coords, rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-10, atol=1e-10)


def _exact_factors(c, s, q, bw):
    """LSE_c(-|y_s - y_c|^2 / 2) - LSE_c(-|y_q - y_c|^2 / 2) with y = (bw L)^-1 x, L L^T = np.cov(c), in mpmath at
    40 digits from the rows as stored (doubles are exact inputs)."""
    import mpmath as mp

    mp.mp.dps = 40
    nc, D = c.shape
    C = [[mp.mpf(float(v)) for v in row] for row in c]
    mean = [mp.fsum(C[r][d] for r in range(nc)) / nc for d in range(D)]
    cov = mp.matrix(D, D)
    for a in range(D):
        for b in range(D):
            cov[a, b] = mp.fsum((C[r][a] - mean[a]) * (C[r][b] - mean[b]) for r in range(nc)) / (nc - 1)
    P = mp.inverse(cov) / (mp.mpf(float(bw)) ** 2)

    def lse(x):
        X = [mp.mpf(float(v)) for v in x]
        ts = []
        for r in range(nc):
            v = mp.matrix([X[d] - C[r][d] for d in range(D)])
            ts.append(-(v.T * P * v)[0] / 2)
        m = max(ts)
        return m + mp.log(mp.fsum(mp.exp(t - m) for t in ts)), m

    out, tmax = [], []
    for i in range(len(s)):
        ls, ms = lse(s[i])
        lq, mq = lse(q[i])
        out.append(float(ls - lq))
        tmax.append(float(-ms - mq))
    return np.array(out), np.array(tmax)


@pytest.mark.parametrize("case", [
    # name, nwalkers, ndim, centre, scale, bw_method
    ("unit", 40, 3, 0.0, 1.0, None),
    ("far", 48, 4, 1e4, 1.0, None),
    ("narrow", 40, 3, 0.0, 1.0, 0.05),
    ("far_narrow_silverman", 64, 5, -1e4, 2.0, "silverman"),
    ("anisotropic", 64, 4, 3.0, np.array([1e-3, 1.0, 30.0, 1.0]), 0.05),
])
def test_factors_against_exact_log_sum_exp(case):
    r"""Every factor of the last split against an exact (40-digit) log-sum-exp of the same rows.

    Bound.  With u = 2^-53, the device computes t_c = -|y_p - y_c|^2 / 2 with y = M^-1 (x - m), M = bw L:
      * x - m is exact where x and m agree to a factor of two (Sterbenz) and within u |x - m| otherwise; m's own
        error is a shift common to every row and cancels in y_p - y_c;
      * L comes from moment sums of nc rows about the ensemble mean and a Cholesky factorisation: a relative
        perturbation of M of at most eta = (nc + D) u cond(L), which changes every t by at most 2 eta |t|;
      * y = M^-1 v (D fused products) and |y_p - y_c|^2 (D direct differences and fused products) each add a
        relative error of at most (D + 2) u, i.e. 2 (D + 2) u |t| with the whitening's cond(L) amplification;
      * the online log-sum-exp adds at most (nc + 2) u to each sum, i.e. to each log.
    The terms within a few units of the largest dominate each sum, so with T_i = |t*_s| + |t*_q| (the largest terms
    of the two sums) |f_i - f_exact| <= 2 (nc + 3 D + 4) u cond(L) (1 + T_i) + 2 (nc + 2) u.  The assertion uses
    four times that."""
    name, N, D, centre, scale, bw = case
    rng = np.random.default_rng(sum(map(ord, name)))
    p0 = centre + scale * rng.standard_normal((N, D))
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.KDEMove(bw, live_dangerously=True), seed=9)
    eng = s._engine
    eng.set_option("debug_taps", 1)
    # log_prob = -inf: every proposal is accepted, so the new state holds every proposal
    eng.set_state(p0, np.full(N, -np.inf))
    eng.step(_schedule(s), 1)
    taps = eng.debug_taps()
    x1, _ = eng.get_state()
    act = taps["active"]
    comp = np.setdiff1d(np.arange(N), act)  # the complement of the last split, already moved by the first
    c, s_rows, q = x1[comp], p0[act], x1[act]
    n = len(comp)
    bwv = n ** (-1.0 / (D + 4)) if bw is None else (n * (D + 2) / 4.0) ** (-1.0 / (D + 4)) if bw == "silverman" else bw
    f_exact, T_i = _exact_factors(c, s_rows, q, bwv)
    L = np.linalg.cholesky(np.cov(c, rowvar=0))
    cond = np.linalg.cond(L)
    u = 2.0 ** -53
    bound = 4 * (2 * (n + 3 * D + 4) * u * cond * (1 + T_i) + 2 * (n + 2) * u)
    err = np.abs(taps["scalar"] - f_exact)
    assert np.all(err <= bound), (name, float(np.max(err / bound)), float(err.max()))


# ---- the reference's statistical gates (tests/integration/test_kde.py) ------------------------------------------
def test_normal_kde():
    from test_gpu_api import _stat_check

    _stat_check(moves.KDEMove())


def test_uniform_kde():
    from test_gpu_api import _stat_check

    _stat_check(moves.KDEMove(), start="uniform")


def test_nsplits_kde():
    from test_gpu_api import _stat_check

    _stat_check(moves.KDEMove(nsplits=5))


# ---- refusals, errors, resume, storage ---------------------------------------------------------------------------
def test_too_few_complement_rows_is_refused_before_any_update():
    # nsplits=3 over 20 walkers: the first split's complement has 13 rows, fewer than ndim = 14
    p0 = np.random.default_rng(1).standard_normal((20, 14))
    s = emcee_b200.EnsembleSampler(20, 14, models.GaussianIso(), moves=moves.KDEMove(nsplits=3, live_dangerously=True),
                                   seed=1)
    with pytest.raises(ValueError, match="Number of dimensions is greater than number of samples"):
        s.run_mcmc(p0, 3, skip_initial_state_check=True)
    assert s.iteration == 0 and s._engine.get_rng()[1] == 0


def _singular_case():
    """Even walkers lie in the plane x2 = 0 inside a box prior that admits only that plane's neighbourhood; odd
    walkers start outside it (log_prob -inf).  Stretch steps move nobody; the first KDE step's first split (the odd
    complement) runs, its second (the even, flat complement) is singular."""
    N, D = 40, 3
    rng = np.random.default_rng(77)
    p0 = rng.standard_normal((N, D))
    p0[0::2, 2] = 0.0
    model = models.Bounded(models.GaussianIso(), [-np.inf, -np.inf, -1e-300], [np.inf, np.inf, 1e-300])
    sched = [(moves.StretchMove(randomize_split=False), 0.7), (moves.KDEMove(randomize_split=False), 0.3)]
    return N, D, p0, model, sched


@pytest.mark.parametrize("backend", ["host", "device"])
def test_singular_complement_raises_at_its_half_step(backend):
    N, D, p0, model, sched = _singular_case()
    seed = 3
    from oracle import philox as px

    k = next(i for i in range(100) if px.move_choice(seed, i, [0.7, 0.3]) == 1)  # the first KDE step
    assert k > 0
    kw = dict(backend=DeviceBackend()) if backend == "device" else {}
    s = emcee_b200.EnsembleSampler(N, D, model, moves=sched, seed=seed, **kw)
    with pytest.raises(np.linalg.LinAlgError, match="lower-dimensional subspace"):
        s.run_mcmc(p0, k + 5, skip_initial_state_check=True)
    assert s.iteration == k and s._engine.get_rng()[1] == k
    ref = emcee_b200.EnsembleSampler(N, D, model, moves=sched, seed=seed)
    ref.run_mcmc(p0, k, skip_initial_state_check=True)
    np.testing.assert_array_equal(s.get_chain(), ref.get_chain())
    np.testing.assert_array_equal(s.get_log_prob(), ref.get_log_prob())
    # the state after the error holds the first split of step k (it moved nobody: no in-box proposal)
    np.testing.assert_array_equal(s.get_last_sample().coords, ref.get_last_sample().coords)
    # resuming runs into the same half-step again: the error is a property of the state, not of the call
    with pytest.raises(np.linalg.LinAlgError):
        s.run_mcmc(s.get_last_sample(), 3, skip_initial_state_check=True)
    assert s.iteration == k


def test_resume_continues_the_uninterrupted_chain():
    target, p0 = T.make_config("ring", 256, 4)
    mv = [(moves.KDEMove(), 0.6), (moves.StretchMove(), 0.4)]
    ref = emcee_b200.EnsembleSampler(256, 4, models.Ring(), moves=mv, seed=11)
    ref.run_mcmc(p0, 12, skip_initial_state_check=True)
    s = emcee_b200.EnsembleSampler(256, 4, models.Ring(), moves=mv, seed=11)
    s.run_mcmc(p0, 5, skip_initial_state_check=True)
    s.run_mcmc(s.get_last_sample(), 7, skip_initial_state_check=True)
    np.testing.assert_array_equal(s.get_chain(), ref.get_chain())


@pytest.mark.parametrize("nsplits", [2, 7, 32])
def test_nsplits_and_bounds_against_the_oracle(nsplits):
    N, D = 515, 4
    target, p0 = T.make_config("rosenbrock", N, D)
    lo, hi = np.full(D, 0.7), np.full(D, 1.3)
    from oracle.bounded import Bounded

    o = ok.KdeOracleSampler(N, D, Bounded(target, lo, hi), [(ok.KDE("silverman", nsplits=nsplits), 1.0)], seed=5)
    p0 = np.clip(p0, 0.71, 1.29)
    o.set_state(p0)
    s = emcee_b200.EnsembleSampler(N, D, models.Bounded(device_model("rosenbrock", target=target), lo, hi),
                                   moves=moves.KDEMove("silverman", nsplits=nsplits), seed=5)
    for k, state in enumerate(s.sample(p0, iterations=4, store=False, skip_initial_state_check=True)):
        o.run(1)
        np.testing.assert_allclose(state.coords, o.coords, rtol=1e-9, atol=1e-10, err_msg="step %d" % k)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))


@pytest.mark.parametrize("where", ["host", "device"])
def test_user_log_probability_function(where):
    N, D = 256, 5
    target, p0 = T.make_config("gauss_iso", N, D)
    if where == "host":
        model = models.HostFunction(lambda x: -0.5 * np.sum(x * x, axis=1), vectorize=True)
    else:
        import torch

        model = models.CudaArrayFunction(lambda x: -0.5 * torch.sum(torch.as_tensor(x, device="cuda") ** 2, dim=1))
    mv = [(moves.KDEMove(0.4), 0.5), (moves.StretchMove(), 0.5)]
    s = emcee_b200.EnsembleSampler(N, D, model, moves=mv, seed=21)
    o = ok.KdeOracleSampler(N, D, target, [(ok.KDE(0.4), 0.5), (rb.Stretch(), 0.5)], seed=21)
    o.set_state(p0)
    s.run_mcmc(p0, 6, skip_initial_state_check=True)
    o.run(6)
    np.testing.assert_allclose(s.get_last_sample().coords, o.coords, rtol=1e-9, atol=1e-10)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))


def test_host_and_device_backends_store_the_same_bytes():
    target, p0 = T.make_config("gauss_dense", 300, 6)
    mv = [(moves.KDEMove(), 0.5), (moves.StretchMove(), 0.3), (moves.WalkMove(), 0.2)]
    a = emcee_b200.EnsembleSampler(300, 6, device_model("gauss_dense", target=target), moves=mv, seed=4)
    b = emcee_b200.EnsembleSampler(300, 6, device_model("gauss_dense", target=target), moves=mv, seed=4,
                                   backend=DeviceBackend())
    a.run_mcmc(p0, 20, thin_by=2, skip_initial_state_check=True)
    b.run_mcmc(p0, 20, thin_by=2, skip_initial_state_check=True)
    assert a.get_chain().tobytes() == b.get_chain().tobytes()
    assert a.get_log_prob().tobytes() == b.get_log_prob().tobytes()
    assert np.array_equal(a.backend.accepted, b.backend.accepted)
    c = emcee_b200.EnsembleSampler(300, 6, device_model("gauss_dense", target=target), moves=mv, seed=4)
    last = c.run_mcmc(p0, 40, store=False, skip_initial_state_check=True)  # thin_by=2: 20 iterations of 2 steps
    assert last.coords.tobytes() == a.get_chain()[-1].tobytes()
