"""The running trace (``EnsembleSampler.enable_trace`` / ``trace`` / ``best_sample`` / ``trace_autocorr_time``;
``eb_trace_config``, ``eb_trace_read``, ``eb_trace_best``) against stored twins of the same seed.

* ``mean``, ``var`` and ``log_prob_mean`` equal, with ``==``, the host restatement of ``csrc/trace_sum.h``
  (``tests/helpers/trace_sum_host.cpp``) applied to the twin's ``get_chain(thin=every)`` / ``get_log_prob``, and
  agree with numpy within the bounds ``test_trace_host.py`` states; ``log_prob_max``, ``step``, ``accepted`` and the
  best sample are exact.
* The rows do not depend on how the steps were run: ``every``, split calls, ``sample(thin_by=...)``, storing or not,
  either backend, every kernel path and move kind, user functions and a user move.
* ``trace_autocorr_time`` against ``autocorr.integrated_time`` of the downloaded means, and against the stored
  twin's ``get_autocorr_time`` on a target with independent walkers.
* Lifecycle, refusals, ``MemoryError`` before any launch, and 65 536 x 128 / 262 144 x 32.
"""
import pickle

import numpy as np
import pytest

from test_trace_host import agree_with_numpy, build_probe, host_columns, host_log_prob
from user_moves_ref import NumpyStretch, gauss_mh

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, autocorr, models, moves
from emcee_b200.dist import Rendezvous

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    return build_probe(tmp_path_factory.mktemp("trace_sum_gpu"))


def _cb_iso(x):
    return -0.5 * np.sum(np.square(x), axis=1)


def _cb_flat(x):
    return np.full(x.shape[0], -1.5)


def _torch_iso(rows):
    import torch

    x = torch.as_tensor(rows, device="cuda")
    return (x * x).sum(dim=1) * -0.5


def _dense(D):
    rng = np.random.default_rng(D)
    a = rng.standard_normal((D, D))
    return models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)), np.linspace(-1, 1, D))


CASES = {
    # name: (N, D, model, moves, expected kernel name)
    "tma_rows": (64, 8, lambda: models.GaussianIso(), None, "tma_rows"),
    "generic_odd": (37, 3, lambda: models.GaussianIso(), None, "generic"),
    "dense_dmma": (96, 16, lambda: _dense(16), None, "dense_dmma"),
    "dense_dmma_chunks": (528, 16, lambda: _dense(16), None, "dense_dmma"),  # three chunks of rows, the last short
    "walk": (48, 4, lambda: models.GaussianIso(), lambda: moves.WalkMove(s=5), "walk"),
    "gaussian": (40, 4, lambda: models.GaussianIso(), lambda: moves.GaussianMove(0.3), "gaussian"),
    "de_snooker": (48, 6, lambda: models.Rosenbrock(),
                   lambda: [(moves.DEMove(), 0.7), (moves.DESnookerMove(), 0.3)], "tma_rows"),
    "bounded": (64, 5, lambda: models.Bounded(models.GaussianIso(), [-0.4] * 5, [np.inf] * 5), None, None),
    "host_fn": (32, 5, lambda: models.HostFunction(_cb_iso, vectorize=True), None, "callback"),
    "cuda_array_fn": (32, 5, lambda: models.CudaArrayFunction(_torch_iso), None, "callback"),
    "user_move": (32, 5, lambda: models.GaussianIso(),
                  lambda: [(NumpyStretch(), 0.5), (moves.MHMove(moves.HostProposal(gauss_mh)), 0.5)], None),
    "tie": (33, 3, lambda: models.HostFunction(_cb_flat, vectorize=True), None, "callback"),
}


def _make(case, backend=None, seed=0x7ACE):
    N, D, model, mv, _ = CASES[case]
    return emcee_b200.EnsembleSampler(N, D, model(), moves=None if mv is None else mv(), seed=seed, backend=backend)


def _p0(case):
    N, D = CASES[case][:2]
    return np.random.default_rng(N * D).standard_normal((N, D)) * 0.5 + 0.1


def _same_trace(a, b):
    assert a._fields == b._fields
    for u, v in zip(a, b):
        assert u.dtype == v.dtype and u.shape == v.shape and u.tobytes() == v.tobytes()


def _check_against_twin(probe, s, t, every, numpy_too=True):
    """s traced every `every`-th step from step 0; t stored every step of the same run"""
    tr = s.trace()
    chain, lp = t.get_chain(thin=every), t.get_log_prob(thin=every)
    n = chain.shape[0]
    assert tr.step.dtype == np.uint64 and np.array_equal(tr.step, every * np.arange(1, n + 1, dtype=np.uint64))
    assert tr.mean.shape == tr.var.shape == (n, s.ndim) and tr.accepted.dtype == np.int64
    for k in range(n):
        mean, var = host_columns(probe, chain[k])
        assert np.array_equal(tr.mean[k], mean) and np.array_equal(tr.var[k], var)
        lpm, lpx, _, walker = host_log_prob(probe, lp[k])
        assert tr.log_prob_mean[k] == lpm and tr.log_prob_max[k] == lpx == lp[k].max()
        assert walker == int(np.argmax(lp[k]))
        if numpy_too:
            agree_with_numpy(probe, chain[k], tr.mean[k], tr.var[k])
            assert tr.log_prob_mean[k] == np.mean(lp[k]) or abs(tr.log_prob_mean[k] - np.mean(lp[k])) <= (
                2 * s.nwalkers * 2.0 ** -53 * np.abs(lp[k]).mean())
    # a walker that accepted moved: the accept count of a step is the number of rows that changed in it
    full = np.concatenate([t._trace_p0[None], t.get_chain()])
    moved = (full[1:] != full[:-1]).any(axis=2).sum(axis=1)
    assert np.array_equal(tr.accepted, moved[every - 1 :: every])
    # the best sample is numpy's argmax of the flat log-probabilities of the recorded steps
    coords, best_lp, step, walker = s.best_sample()
    flat = int(np.argmax(lp.reshape(-1)))
    k, w = divmod(flat, s.nwalkers)
    assert (step, walker) == (every * (k + 1), w) and best_lp == lp[k, w]
    assert coords.dtype == np.float64 and np.array_equal(coords, chain[k, w])


def _twin(case, total, backend):
    t = _make(case, backend)
    t._trace_p0 = _p0(case)
    t.run_mcmc(t._trace_p0, total, skip_initial_state_check=True)
    return t


@pytest.mark.parametrize("case", list(CASES))
def test_twins(probe, case):
    calls = (7, 5)  # two calls; the second starts off the cadence of every = 3
    runs = {}
    for every in (1, 3):
        s = _make(case)
        s.enable_trace(every)
        st = _p0(case)
        for n in calls:
            st = s.run_mcmc(st, n, store=False, skip_initial_state_check=True)
        want = CASES[case][4]
        if want is not None:
            assert s._engine.last_kernel_name() == want
        runs[every] = s
    twins = [_twin(case, sum(calls), b) for b in (Backend(), DeviceBackend())]
    assert np.array_equal(twins[0].get_chain(), twins[1].get_chain())
    for every, s in runs.items():
        for t in twins:
            _check_against_twin(probe, s, t, every)
    assert runs[1].trace().accepted.sum() == twins[0].backend.accepted.sum() == twins[1].backend.accepted.sum()
    # every = 3 recorded the same bytes as the matching rows of every = 1
    one, three = runs[1].trace(), runs[3].trace()
    _same_trace(three, type(one)(*(f[2::3] for f in one)))
    if case == "bounded":
        assert np.isinf(one.log_prob_mean).any() and np.isfinite(one.log_prob_max).all()
    if case == "tie":  # a constant log-probability: the first recorded step, walker 0
        assert runs[1].best_sample()[1:] == (-1.5, 1, 0) and runs[3].best_sample()[1:] == (-1.5, 3, 0)


@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma", "host_fn", "gaussian"])
def test_independent_of_how_the_steps_run(probe, case):
    total = 12
    ref = _make(case)
    ref.enable_trace(3)
    ref.run_mcmc(_p0(case), total, store=False, skip_initial_state_check=True)
    want = ref.trace()
    assert want.step.tolist() == [3, 6, 9, 12]
    # the same run again: the same bytes
    again = _make(case)
    again.enable_trace(3)
    again.run_mcmc(_p0(case), total, store=False, skip_initial_state_check=True)
    _same_trace(again.trace(), want)
    assert again.best_sample()[1:] == ref.best_sample()[1:]
    assert np.array_equal(again.best_sample()[0], ref.best_sample()[0])
    # one step per call, resumed
    s = _make(case)
    s.enable_trace(3)
    st = _p0(case)
    for _ in range(total):
        st = s.run_mcmc(st, 1, store=False, skip_initial_state_check=True)
    _same_trace(s.trace(), want)
    # sample(thin_by=3) as a generator, storing into either backend while recording
    for backend in (Backend(), DeviceBackend()):
        s = _make(case, backend)
        s.enable_trace(3)
        assert sum(1 for _ in s.sample(_p0(case), iterations=4, thin_by=3, skip_initial_state_check=True)) == 4
        _same_trace(s.trace(), want)
        chain, lp = s.get_chain(), s.get_log_prob()
        for k in range(4):  # its own stored steps are what it recorded
            mean, var = host_columns(probe, chain[k])
            assert np.array_equal(want.mean[k], mean) and np.array_equal(want.var[k], var)
            assert want.log_prob_max[k] == lp[k].max()
        assert want.accepted.sum() == s.backend.accepted.sum()  # a thinned store counts its stored steps only
        # run_mcmc storing with thin_by
        s = _make(case, type(backend)())
        s.enable_trace(3)
        s.run_mcmc(_p0(case), 4, thin_by=3, skip_initial_state_check=True)
        _same_trace(s.trace(), want)
    assert list(s.sample(s.get_last_sample(), iterations=0, skip_initial_state_check=True)) == []
    _same_trace(s.trace(), want)


def test_recording_leaves_the_chain_alone():
    out = []
    for on in (False, True):
        s = _make("dense_dmma", Backend())
        if on:
            s.enable_trace(2)
        s.run_mcmc(_p0("dense_dmma"), 10, skip_initial_state_check=True)
        out.append(s)
    assert np.array_equal(out[0].get_chain(), out[1].get_chain())
    assert np.array_equal(out[0].get_log_prob(), out[1].get_log_prob())
    assert np.array_equal(out[0].backend.accepted, out[1].backend.accepted)


# ---- autocorrelation time of the ensemble mean ---------------------------------------------------------------------
def test_autocorr_time_is_integrated_time_of_the_means():
    s = _make("tma_rows")
    s.enable_trace(2)
    s.run_mcmc(_p0("tma_rows"), 400, store=False, skip_initial_state_check=True)
    mean = s.trace().mean
    with pytest.raises(autocorr.AutocorrError) as short:  # 200 rows are fewer than 50 autocorrelation times
        s.trace_autocorr_time()
    with pytest.raises(autocorr.AutocorrError) as want:
        autocorr.integrated_time(mean[:, None, :])
    assert np.array_equal(short.value.tau, want.value.tau) and str(short.value) == str(want.value)
    tau = s.trace_autocorr_time(quiet=True)
    assert tau.shape == (8,) and np.array_equal(tau, 2 * autocorr.integrated_time(mean[:, None, :], quiet=True))
    tau = s.trace_autocorr_time(discard=50, c=4, tol=0)
    assert np.array_equal(tau, 2 * autocorr.integrated_time(mean[50:, None, :], c=4, tol=0))


def test_autocorr_time_against_the_stored_chain():
    """GaussianMove on the isotropic Gaussian: the walkers are independent chains with one autocorrelation function,
    which their mean shares.  The stored twin averages 32 walkers' functions, the trace has the one series of the
    mean, so its estimate is the noisier one: with n = 60 000 steps and a window of about 5 tau = 50 lags its
    standard error is about sqrt(2 (2 * 50 + 1) / n) = 6 %, inside the 20 % the reference's test_autocorr.py allows."""
    N, D, n = 32, 2, 60000
    p0 = np.random.default_rng(3).standard_normal((N, D))
    mk = lambda b: emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.GaussianMove(1.5), seed=11,  # noqa: E731
                                              backend=b)
    s = mk(None)
    s.enable_trace()
    s.run_mcmc(p0, n, store=False, skip_initial_state_check=True)
    t = mk(Backend())
    t.run_mcmc(p0, n, skip_initial_state_check=True)
    tau, want = s.trace_autocorr_time(), t.get_autocorr_time()
    assert np.all(want > 2) and np.all(np.abs(tau - want) <= 0.2 * want), (tau, want)


# ---- lifecycle and refusals ------------------------------------------------------------------------------------------
def test_lifecycle():
    case = "tma_rows"
    N, D = CASES[case][:2]
    s = _make(case)
    for read in (s.trace, s.best_sample, s.trace_autocorr_time):
        with pytest.raises(RuntimeError, match="not enabled"):
            read()
    s.enable_trace()
    assert s.trace().step.size == 0
    with pytest.raises(RuntimeError, match="no step yet"):
        s.best_sample()
    st = s.run_mcmc(_p0(case), 5, store=False, skip_initial_state_check=True)
    first = s.trace()
    assert first.step.tolist() == [1, 2, 3, 4, 5]
    assert s.trace(discard=2).step.tolist() == [3, 4, 5] and np.array_equal(s.trace(discard=2).mean, first.mean[2:])
    for discard in (5, 6, 10 ** 9):
        e = s.trace(discard=discard)
        assert e.step.shape == (0,) and e.step.dtype == np.uint64 and e.mean.shape == e.var.shape == (0, D)
        assert e.log_prob_mean.shape == e.log_prob_max.shape == e.accepted.shape == (0,)
        assert e.mean.dtype == np.float64 and e.accepted.dtype == np.int64
    best = s.best_sample()
    # every = 0 freezes the rows and the best sample
    s.enable_trace(0)
    st = s.run_mcmc(st, 4, store=False)
    _same_trace(s.trace(), first)
    assert s.best_sample()[1:] == best[1:] and np.array_equal(s.best_sample()[0], best[0])
    # re-enabling drops both; the rows grow across calls and keep what they held
    s.enable_trace(2)
    assert s.trace().step.size == 0
    with pytest.raises(RuntimeError, match="no step yet"):
        s.best_sample()
    st = s.run_mcmc(st, 1, store=False)  # step 10
    head = s.trace()
    assert head.step.tolist() == [10]
    for n in (1, 2, 40):
        st = s.run_mcmc(st, n, store=False)
    tr = s.trace()
    assert tr.step.tolist() == list(range(10, 54, 2)) and tr.mean[0].tobytes() == head.mean[0].tobytes()
    assert s.best_sample()[2] in tr.step and s.best_sample()[1] == tr.log_prob_max.max()
    # pickling drops the rows
    s2 = pickle.loads(pickle.dumps(s))
    with pytest.raises(RuntimeError, match="not enabled"):
        s2.trace()
    s2.run_mcmc(st, 2, store=False)
    with pytest.raises(RuntimeError, match="not enabled"):
        s2.best_sample()
    with pytest.raises(ValueError, match="every must be >= 0"):
        s.enable_trace(-2)
    assert s.trace().step.size == tr.step.size


def test_sharded_refused_both_ways():
    s = _make("tma_rows")
    s.enable_trace()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(Rendezvous())
    s = _make("tma_rows")
    s.attach(Rendezvous())
    with pytest.raises(NotImplementedError, match="sharded"):
        s.enable_trace()


def test_rows_beyond_the_device_memory_error():
    """10**12 recorded steps of a 2 048-parameter ensemble are 33 PB of rows: refused from the count, before any
    allocation or launch, and the rows recorded so far stay"""
    D = 2048
    s = emcee_b200.EnsembleSampler(2 * D + 2, D, models.GaussianIso(), seed=3)
    p0 = np.random.default_rng(1).standard_normal((2 * D + 2, D))
    s.enable_trace()
    st = s.run_mcmc(p0, 2, store=False, skip_initial_state_check=True)
    with pytest.raises(MemoryError, match="bytes free"):
        s.run_mcmc(st, 10 ** 12, store=False)
    assert s.random_state[2] == 2 and s.trace().step.tolist() == [1, 2]
    s.run_mcmc(st, 1, store=False)
    assert s.trace().step.tolist() == [1, 2, 3]


# ---- at scale ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,D,kernel", [(65536, 128, "dense_dmma"), (262144, 32, None)])
def test_scale(probe, N, D, kernel):
    steps, every = 6, 2
    rng = np.random.default_rng(5)
    if kernel == "dense_dmma":
        a = rng.standard_normal((D, D))
        model = lambda: models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)))  # noqa: E731
    else:
        model = lambda: models.GaussianIso()  # noqa: E731
    p0 = rng.standard_normal((N, D))
    s = emcee_b200.EnsembleSampler(N, D, model(), seed=9)
    s.enable_trace(every)
    s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
    if kernel is not None:
        assert s._engine.last_kernel_name() == kernel
    t = emcee_b200.EnsembleSampler(N, D, model(), seed=9, backend=DeviceBackend())
    t._trace_p0 = p0
    t.run_mcmc(p0, steps, skip_initial_state_check=True)
    _check_against_twin(probe, s, t, every, numpy_too=False)
    tr = s.trace()
    np.testing.assert_allclose(tr.mean, t.get_chain(thin=every).mean(axis=1), rtol=0, atol=1e-13)
    np.testing.assert_allclose(tr.var, t.get_chain(thin=every).var(axis=1, ddof=1), rtol=1e-12)
