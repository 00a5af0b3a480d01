"""Host side of ``BatchSampler``: argument checks and refusals (raised before any device work), seed derivation, the
``[n, K, N, D]`` / flat ``[K, n N, D]`` slicing, per-ensemble autocorrelation times, the batched initial-state check
and the batched callback's reshape, over a stand-in engine."""

import ctypes as C
import logging

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, autocorr, models, moves
from emcee_b200.batch import _batch_seeds, _walkers_independent


class _Engine(object):
    """The calls ``BatchSampler`` makes on ``_lib.BatchEngine``.  A stored step ``s`` (1-based) of row ``r`` holds
    ``coords = s * 1000 + r + [0, 0.1, 0.2, ...]`` and ``log_prob = -(s * 1000 + r)``."""

    created = []

    def __init__(self, nbatch, nwalkers, ndim, seeds, device=0):
        self.nbatch, self.ens_walkers, self.ndim = nbatch, nwalkers, ndim
        self.nwalkers = nbatch * nwalkers
        self.seeds, self.step_count = np.array(seeds, dtype=np.uint64), 0
        self.calls = []
        _Engine.created.append(self)

    def set_model(self, kind, params):
        self.calls.append(("model", kind))

    def set_bounds(self, lo, hi):
        self.calls.append(("bounds",))

    def set_callback(self, fn, where):
        self.calls.append(("callback", where))

    def set_state(self, coords, log_prob):
        assert coords.shape == (self.nwalkers, self.ndim)
        self.calls.append(("state",))
        self.x = coords.copy()
        self.lp = np.zeros(self.nwalkers) if log_prob is None else log_prob.copy()

    def get_state(self):
        return self.x.copy(), self.lp.copy()

    def get_rng(self):
        return self.seeds.copy(), self.step_count

    def set_rng(self, seeds, step):
        self.seeds, self.step_count = np.array(seeds, dtype=np.uint64), step

    def _advance(self):
        self.step_count += 1
        s = self.step_count
        rows = np.arange(self.nwalkers)
        self.x = (s * 1000.0 + rows)[:, None] + 0.1 * np.arange(self.ndim)[None, :]
        self.lp = -(s * 1000.0 + rows)

    def step(self, sched, nsteps, want_accepted=True):
        for _ in range(nsteps):
            self._advance()

    def step_store(self, sched, nsteps, thin_by, chain, log_prob, accepted):
        k = 0
        for j in range(nsteps):
            self._advance()
            accepted += (np.arange(self.nwalkers) % 2 == 0)
            if (j + 1) % thin_by == 0:
                chain[k], log_prob[k] = self.x, self.lp
                k += 1

    def compute_log_prob(self, x):
        return -np.sum(x**2, axis=1)


@pytest.fixture
def stand_in(monkeypatch):
    _Engine.created = []
    monkeypatch.setattr(_lib, "BatchEngine", _Engine)
    return _Engine


def _p0(K, N, D, seed=1):
    return np.random.default_rng(seed).normal(size=(K, N, D))


# ---- refusals ---------------------------------------------------------------------------------------------------
def _graph_fn():
    return models.CudaGraphFunction(lambda m: None)


@pytest.mark.parametrize("make,err,match", [
    (lambda: dict(log_prob_fn=_graph_fn()), NotImplementedError, "CudaGraphFunction"),
    (lambda: dict(log_prob_fn=models.HostFunction(np.sum, vectorize=False)), NotImplementedError, "vectorize=False"),
    (lambda: dict(log_prob_fn=models.HostFunction(np.sum, vectorize=True, blobs_dtype=float)), NotImplementedError,
     "blobs_dtype"),
    (lambda: dict(log_prob_fn=models.CudaArrayFunction(np.sum, blobs_dtype=float)), NotImplementedError, "blobs_dtype"),
    (lambda: dict(log_prob_fn=np.sum), TypeError, "registered device model"),
    (lambda: dict(moves=[(moves.StretchMove(), 0.5), (moves.DEMove(), 0.5)]), NotImplementedError, "exactly one"),
    (lambda: dict(moves=moves.WalkMove()), NotImplementedError, "exactly one"),
    (lambda: dict(moves=moves.KDEMove()), NotImplementedError, "exactly one"),
    (lambda: dict(moves=moves.GaussianMove(1.0)), NotImplementedError, "exactly one"),
    (lambda: dict(nbatch=0), ValueError, "nbatch"),
    (lambda: dict(nbatch=2**26, nwalkers=32), ValueError, "2\\*\\*31"),
    (lambda: dict(seeds=[1, 2]), ValueError, "one integer per ensemble"),
])
def test_refusals_before_device_work(stand_in, make, err, match):
    kw = dict(nbatch=3, nwalkers=8, ndim=2, log_prob_fn=models.GaussianIso())
    kw.update(make())
    with pytest.raises(err, match=match):
        emcee_b200.BatchSampler(kw.pop("nbatch"), kw.pop("nwalkers"), kw.pop("ndim"), kw.pop("log_prob_fn"), **kw)
    assert stand_in.created == []


def test_accepted_models_and_moves(stand_in):
    for fn, call in [(models.GaussianIso(), ("model", "gauss_iso")),
                     (models.CudaArrayFunction(np.sum), ("callback", "device")),
                     (models.HostFunction(np.sum, vectorize=True), ("callback", "host"))]:
        s = emcee_b200.BatchSampler(2, 8, 2, fn, moves=[moves.DEMove()])
        assert s._engine.calls == [call]
        assert isinstance(s.move, moves.DEMove)
    s = emcee_b200.BatchSampler(2, 8, 2, models.Bounded(models.GaussianIso(), -1, 1),
                                moves=[(moves.DESnookerMove(), 1.0)])
    assert s._engine.calls == [("model", "gauss_iso"), ("bounds",)]


def test_few_walkers_and_shapes(stand_in):
    s = emcee_b200.BatchSampler(2, 6, 4, models.GaussianIso(), seeds=1)
    with pytest.raises(RuntimeError, match="fewer walkers than twice"):
        s.run_mcmc(_p0(2, 6, 4), 3)
    s = emcee_b200.BatchSampler(2, 8, 2, models.GaussianIso(), seeds=1)
    with pytest.raises(ValueError, match="incompatible input dimensions"):
        s.run_mcmc(_p0(3, 8, 2), 3)
    with pytest.raises(ValueError, match="incompatible input dimensions"):
        s.run_mcmc(emcee_b200.State(_p0(2, 8, 2), log_prob=np.zeros((2, 7))), 3)
    with pytest.raises(ValueError, match="never been called"):
        s.run_mcmc(None, 3)
    with pytest.raises(ValueError, match="Invalid thinning"):
        s.run_mcmc(_p0(2, 8, 2), 3, thin_by=0)
    assert ("state",) not in s._engine.calls


# ---- seeds ------------------------------------------------------------------------------------------------------
def test_seeds():
    assert _batch_seeds(5, 3).tolist() == [5, 6, 7]
    assert _batch_seeds(2**64 - 2, 3).tolist() == [2**64 - 2, 2**64 - 1, 0]
    assert _batch_seeds([9, 2**64 + 3, np.uint64(4)], 3).tolist() == [9, 3, 4]
    np.random.seed(17)
    before = np.random.get_state()
    want = emcee_b200.ensemble._seed_from_numpy()
    got = _batch_seeds(None, 4)
    after = np.random.get_state()
    assert got.tolist() == [(want + k) % 2**64 for k in range(4)]
    assert all(np.array_equal(a, b) for a, b in zip(before[1:3], after[1:3]))  # numpy's state is not consumed
    with pytest.raises(TypeError):
        _batch_seeds(1.5, 2)


def test_random_state_round_trip(stand_in):
    s = emcee_b200.BatchSampler(3, 8, 2, models.GaussianIso(), seeds=[4, 5, 6])
    name, seeds, step = s.random_state
    assert name == "philox4x32-10" and seeds.dtype == np.uint64 and seeds.tolist() == [4, 5, 6] and step == 0
    s.random_state = ("philox4x32-10", [7, 8, 9], 11)
    assert s.random_state[1].tolist() == [7, 8, 9] and s.random_state[2] == 11
    s.random_state = "garbage"  # ignored, as EnsembleSampler ignores it
    assert s.random_state[2] == 11


# ---- slicing ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("thin_by", [1, 3])
@pytest.mark.parametrize("discard,thin", [(0, 1), (2, 1), (0, 3), (1, 2), (5, 4)])
def test_chain_slicing(stand_in, thin_by, discard, thin):
    K, N, D, n = 3, 8, 2, 12
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1)
    last = s.run_mcmc(_p0(K, N, D), n, thin_by=thin_by)
    assert s.iteration == n and last.coords.shape == (K, N, D) and last.log_prob.shape == (K, N)
    steps = thin_by * np.arange(1, n + 1)[discard + thin - 1 :: thin]  # the stored steps the slice keeps
    rows = np.arange(K * N).reshape(K, N)
    want = (steps[:, None, None] * 1000.0 + rows[None])[..., None] + 0.1 * np.arange(D)
    chain = s.get_chain(discard=discard, thin=thin)
    assert chain.shape == (len(steps), K, N, D)
    assert np.array_equal(chain, want)
    flat = s.get_chain(discard=discard, thin=thin, flat=True)
    assert flat.shape == (K, len(steps) * N, D)
    for k in range(K):  # what the twin's get_chain(flat=True) gives: (step, walker) order
        assert np.array_equal(flat[k], want[:, k].reshape(-1, D))
    lp = s.get_log_prob(discard=discard, thin=thin)
    assert np.array_equal(lp, -(steps[:, None, None] * 1000.0 + rows[None]))
    assert np.array_equal(s.get_log_prob(discard=discard, thin=thin, flat=True)[1], lp[:, 1].ravel())
    acc = s.acceptance_fraction
    assert acc.shape == (K, N)
    assert np.array_equal(acc, ((rows % 2 == 0) * (n * thin_by) / n).astype(float))
    ls = s.get_last_sample()
    assert np.array_equal(ls.coords, last.coords) and np.array_equal(ls.log_prob, last.log_prob)


def test_generator_and_resume(stand_in):
    K, N, D = 2, 8, 2
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1)
    states = list(s.sample(_p0(K, N, D), iterations=4, thin_by=2))
    assert len(states) == 4 and s.iteration == 4 and states[-1].random_state[2] == 8
    s.run_mcmc(states[-1], 3, store=False, skip_initial_state_check=True)  # the stand-in's rows are collinear
    assert s.iteration == 4 and s._engine.step_count == 11
    s.run_mcmc(None, 2, skip_initial_state_check=True)
    assert s.iteration == 6
    s.reset()
    assert s.iteration == 0


def test_compute_log_prob_shapes(stand_in):
    s = emcee_b200.BatchSampler(3, 8, 2, models.GaussianIso(), seeds=1)
    x = _p0(3, 5, 2)
    assert np.array_equal(s.compute_log_prob(x), -np.sum(x**2, axis=2))
    with pytest.raises(ValueError, match="incompatible"):
        s.compute_log_prob(x[:2])


# ---- autocorrelation --------------------------------------------------------------------------------------------
def _ar1_chain(n, K, N, D, rhos, seed=3):
    rng = np.random.default_rng(seed)
    x = np.zeros((n, K, N, D))
    for t in range(1, n):
        x[t] = rhos[:, None, None] * x[t - 1] + rng.normal(size=(K, N, D))
    return x


def test_autocorr_per_ensemble(stand_in, caplog):
    K, N, D, n = 3, 8, 2, 400
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1)
    s.backend.reset(K * N, D)
    s.backend.grow(n, None)
    x = _ar1_chain(n, K, N, D, np.array([0.1, 0.5, 0.2]))
    s.backend.chain[:] = x.reshape(n, K * N, D)
    s.backend.iteration = n
    for discard, thin in [(0, 1), (50, 2)]:
        tau = s.get_autocorr_time(discard=discard, thin=thin, tol=5)
        assert tau.shape == (K, D)
        for k in range(K):
            want = autocorr.integrated_time(x[discard + thin - 1 :: thin, k], tol=5) * thin
            assert np.array_equal(tau[k], want)
    # ensemble 1 (rho = 0.99) fails tol = 50 over 400 steps; the others pass at tol = 20
    x[:, 1] = _ar1_chain(n, 1, N, D, np.array([0.995]), seed=4)[:, 0]
    s.backend.chain[:] = x.reshape(n, K * N, D)
    with pytest.raises(autocorr.AutocorrError, match=r"ensemble\(s\) \[1\]") as e:
        s.get_autocorr_time(tol=20)
    for k in range(K):
        assert np.array_equal(e.value.tau[k], autocorr.integrated_time(x[:, k], tol=20, quiet=True))
    with caplog.at_level(logging.WARNING):
        tau = s.get_autocorr_time(tol=20, quiet=True)
    assert "ensemble(s) [1]" in caplog.text
    assert np.array_equal(tau, e.value.tau)


# ---- the initial-state check ------------------------------------------------------------------------------------
def test_walkers_independent_batched(stand_in):
    K, N, D = 5, 10, 3
    x = _p0(K, N, D, seed=7)
    x[2, :, 1] = 4.0  # a constant parameter
    x[3, :, 2] = 2.0 * x[3, :, 0]  # dependent walkers
    x[4, 3, 0] = np.inf
    got = _walkers_independent(x)
    assert got.tolist() == [emcee_b200.walkers_independent(x[k]) for k in range(K)] == [True, True, False, False, False]
    s = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1)
    with pytest.raises(ValueError, match=r"linearly independent.*\(ensemble 2\)"):
        s.run_mcmc(x, 3)
    assert ("state",) not in s._engine.calls
    s.run_mcmc(x, 1, skip_initial_state_check=True)
    assert ("state",) in s._engine.calls


# ---- the batched callback ---------------------------------------------------------------------------------------
class _Lib(object):
    """``eb_callback_result`` of the library: copies the flattened result the trampoline hands over."""

    def __init__(self):
        self.got = None

    def eb_callback_result(self, h, lp, src, stride, m, stream):
        a = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_double)), shape=(m * stride // 8,))
        self.got = a[:: stride // 8][:m].copy()
        return _lib.EB_OK

    def eb_last_error(self, h):
        return b""


def test_batch_trampoline_host():
    K, m, D = 3, 4, 2
    seen, failure = [], [None]

    def fn(x):
        seen.append(x.shape)
        return np.sum(x, axis=2) * np.arange(1, K + 1)[:, None]

    cb = _lib.make_batch_trampoline(None, fn, _lib.EB_CALLBACK_HOST, failure, K)
    rows = np.arange(K * m * D, dtype=np.float64)
    lp = np.zeros(K * m)
    assert cb(None, rows.ctypes.data_as(_lib._dp), K * m, D, lp.ctypes.data_as(_lib._dp), None) == 0
    assert seen == [(K, m, D)] and failure[0] is None
    x = rows.reshape(K, m, D)
    assert np.array_equal(lp, (np.sum(x, axis=2) * np.arange(1, K + 1)[:, None]).ravel())


@pytest.mark.parametrize("out,err", [(np.zeros(12), NotImplementedError), (np.zeros((4, 3)), NotImplementedError),
                                     (np.zeros((3, 4, 1)), NotImplementedError),
                                     (np.zeros((3, 4), dtype=np.float32), TypeError)])
def test_batch_trampoline_shape_errors(out, err):
    failure = [None]
    cb = _lib.make_batch_trampoline(None, lambda x: out, _lib.EB_CALLBACK_HOST, failure, 3)
    rows = np.zeros(12 * 2)
    lp = np.zeros(12)
    assert cb(None, rows.ctypes.data_as(_lib._dp), 12, 2, lp.ctypes.data_as(_lib._dp), None) == 1
    assert isinstance(failure[0], err) and not lp.any()
    if err is NotImplementedError:
        assert "lp[nbatch, m] = (3, 4)" in str(failure[0])


class _Cai(object):
    def __init__(self, a, strides=None, shape=None):
        self.a = a
        self.__cuda_array_interface__ = {"shape": a.shape if shape is None else shape, "typestr": "<f8", "data": (a.ctypes.data, False),
                                         "strides": strides, "version": 3, "stream": None}


def test_batch_result_device_strides(monkeypatch):
    fake = _Lib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    base = np.arange(24, dtype=np.float64)
    _lib._batch_result(None, None, _Cai(base[:12].reshape(3, 4)), 3, 4, 2)
    assert np.array_equal(fake.got, base[:12])
    _lib._batch_result(None, None, _Cai(base, strides=(64, 16), shape=(3, 4)), 3, 4, 2)  # every other value
    assert np.array_equal(fake.got, base[::2])
    with pytest.raises(ValueError, match="one strided run"):
        _lib._batch_result(None, None, _Cai(base, strides=(8, 32), shape=(3, 4)), 3, 4, 2)
    with pytest.raises(NotImplementedError, match="returned shape"):
        _lib._batch_result(None, None, _Cai(base[:12]), 3, 4, 2)
