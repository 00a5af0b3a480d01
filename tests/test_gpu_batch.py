"""``BatchSampler`` on the GPU: every ensemble of a batch against its twin, an ``EnsembleSampler`` of the same seed
run from the same state.

Against twins that run the generic kernel (options ``tma_rows`` and ``dense_dmma`` off) the chains, log-probabilities,
acceptance fractions and final states are byte-equal: the batch kernel runs the generic kernel's per-walker code.
Against twins with the default kernel choice, accept masks and counts are equal and the coordinates and
log-probabilities meet DESIGN §3's tolerances."""

import numpy as np
import pytest

from util import load_golden

import emcee_b200
from emcee_b200 import models, moves
from gpu_util import device_model, device_moves
from test_gpu_parity import LP_ATOL, LP_RTOL, _tols

pytestmark = pytest.mark.gpu

STEPS = 50


def _icov(D, seed=5):
    a = np.random.default_rng(seed).normal(size=(D, D))
    return a @ a.T / D + np.eye(D)


MODELS = {
    "gauss_iso": lambda D: models.GaussianIso(),
    "gauss_dense": lambda D: models.GaussianDense(_icov(D), np.linspace(-0.5, 0.5, D)),
    "rosenbrock": lambda D: models.Rosenbrock(),
    "ring": lambda D: models.Ring(2.0, 0.5),
    "bounded": lambda D: models.Bounded(models.GaussianIso(), -1.5, 1.5),
}
MOVES = {
    "stretch": lambda P, r: moves.StretchMove(nsplits=P, randomize_split=r),
    "stretch_a3": lambda P, r: moves.StretchMove(a=3.0, nsplits=P, randomize_split=r),
    "de": lambda P, r: moves.DEMove(nsplits=P, randomize_split=r),
    "de_gamma0": lambda P, r: moves.DEMove(gamma0=0.7, nsplits=P, randomize_split=r),
    "snooker": lambda P, r: moves.DESnookerMove(randomize_split=r),
}
SHAPES = [(32, 5), (37, 3), (64, 8)]
KS = [1, 3, 64]
NSPLITS = [2, 3, 7, 32]


def _cases():
    out = []
    for i, (mv, model) in enumerate((a, b) for a in MOVES for b in MODELS):
        N, D = SHAPES[i % 3]
        out.append((mv, model, KS[(i // 3) % 3], N, D, NSPLITS[i % 4], i % 2 == 0, [1, 3][(i // 2) % 2]))
    return out


# Large ensembles, each reaching a branch of batch.cu the rows of _cases() do not:
#   N = 1 025, 2 048     batch_split_table_kernel runs a second chunk of TABLE_THREADS = 1 024 walkers
#   D = 20, 60, 130      lanes_per_walker = 8, 16, 32
#   D = 300, snooker x dense: 8 groups x 5 rows x 300 doubles = 96 000 bytes of shared memory, above the 48 KB default
#   D = 700, snooker x dense: 224 000 bytes at 256 threads, so the launch halves to 128 threads (112 000 bytes)
#   32 splits of 100 walkers, K = 3
# (a red-blue move needs at least twice as many walkers as dimensions)
LARGE_CASES = [("stretch", "gauss_iso", 2, 1025, 3, 2, True, 1), ("de", "ring", 2, 2048, 4, 3, True, 1),
               ("stretch", "rosenbrock", 3, 48, 20, 2, True, 1), ("de_gamma0", "gauss_dense", 2, 128, 60, 2, False, 1),
               ("stretch_a3", "ring", 2, 260, 130, 3, True, 2), ("snooker", "gauss_dense", 2, 600, 300, 4, True, 1),
               ("snooker", "gauss_dense", 2, 1400, 700, 4, False, 1), ("de", "gauss_iso", 3, 100, 4, 32, True, 1)]


def _p0(K, N, D, seed=11):
    return 0.7 * np.random.default_rng(seed).normal(size=(K, N, D))


def _seeds(K, base=1234):
    return [base + 7919 * k for k in range(K)]


def _twin(N, D, model, move, seed, generic=True):
    s = emcee_b200.EnsembleSampler(N, D, model, moves=move, seed=seed)
    if generic:
        s._engine.set_option("tma_rows", 0)
        s._engine.set_option("dense_dmma", 0)
    return s


def _assert_twin(b, k, t, last_b, last_t):
    assert np.array_equal(b.get_chain()[:, k], t.get_chain())
    assert np.array_equal(b.get_log_prob()[:, k], t.get_log_prob())
    assert np.array_equal(b.acceptance_fraction[k], t.acceptance_fraction)
    assert np.array_equal(last_b.coords[k], last_t.coords)
    assert np.array_equal(last_b.log_prob[k], last_t.log_prob)


@pytest.mark.parametrize("mv,model,K,N,D,P,rand,thin_by", _cases() + LARGE_CASES)
def test_twins_exact(mv, model, K, N, D, P, rand, thin_by):
    seeds = _seeds(K)
    p0 = _p0(K, N, D)
    b = emcee_b200.BatchSampler(K, N, D, MODELS[model](D), moves=MOVES[mv](P, rand), seeds=seeds)
    last = b.run_mcmc(p0, STEPS, thin_by=thin_by, skip_initial_state_check=True)
    assert b.get_chain().shape == (STEPS, K, N, D)
    assert last.random_state[2] == STEPS * thin_by
    for k in range(K):
        t = _twin(N, D, MODELS[model](D), MOVES[mv](P, rand), seeds[k])
        lt = t.run_mcmc(p0[k], STEPS, thin_by=thin_by, skip_initial_state_check=True)
        _assert_twin(b, k, t, last, lt)


@pytest.mark.parametrize("model,mv,N,D", [("gauss_dense", "stretch", 64, 8), ("gauss_iso", "stretch", 64, 8),
                                          ("ring", "de", 32, 5), ("rosenbrock", "stretch_a3", 37, 3)])
def test_twins_default_kernels(model, mv, N, D):
    K = 5
    seeds = _seeds(K, 99)
    p0 = _p0(K, N, D, 3)
    b = emcee_b200.BatchSampler(K, N, D, MODELS[model](D), moves=MOVES[mv](2, True), seeds=seeds)
    b.run_mcmc(p0, STEPS, skip_initial_state_check=True)
    for k in range(K):
        t = _twin(N, D, MODELS[model](D), MOVES[mv](2, True), seeds[k], generic=False)
        t.run_mcmc(p0[k], STEPS, skip_initial_state_check=True)
        assert np.array_equal(b.backend.accepted.reshape(K, N)[k], t.backend.accepted)
        np.testing.assert_allclose(b.get_chain()[:, k], t.get_chain(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(b.get_log_prob()[:, k], t.get_log_prob(), rtol=LP_RTOL, atol=LP_ATOL)


@pytest.mark.parametrize("name", ["stretch_iso_32x5", "de_rosen_40x4", "snooker_iso_40x4", "stretch_iso_nsplits7_61x5",
                                  "stretch_iso_nsplits32_32x3", "stretch_iso_odd_37x3"])
def test_golden_at_nonzero_index(name):
    g = load_golden(name)
    N, D, seed = int(g["nwalkers"]), int(g["ndim"]), int(g["seed"])
    K, j = 4, 2
    seeds = [seed + 1 + k for k in range(K)]
    seeds[j] = seed
    p0 = _p0(K, N, D)
    p0[j] = g["p0"]
    (mv, _), = device_moves(g["moves"], g)
    b = emcee_b200.BatchSampler(K, N, D, device_model(str(g["model_kind"]), g=g), moves=mv, seeds=seeds)
    n = g["chain"].shape[0]
    b.run_mcmc(p0, n, skip_initial_state_check=True)
    exact, rtol, atol = _tols(g)
    if exact:
        assert np.array_equal(b.get_chain()[:, j], g["chain"])
    else:
        np.testing.assert_allclose(b.get_chain()[:, j], g["chain"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(b.get_log_prob()[:, j], g["log_prob"], rtol=max(rtol, LP_RTOL), atol=max(10 * atol, LP_ATOL))
    assert np.array_equal(b.backend.accepted.reshape(K, N)[j], g["accepted"].sum(axis=0))


# ---- user functions ---------------------------------------------------------------------------------------------
# Each row's value is computed with the same operations in both arrangements -- elementwise, with the sum over the
# small parameter axis taken term by term in a fixed order -- so the batch and its twins get the same bytes.
def _lp(x, mu):  # numpy or torch arrays
    d = x - mu[..., None, :]
    lp = -0.5 * (d[..., 0] * d[..., 0])
    for e in range(1, x.shape[-1]):
        lp = lp - 0.5 * (d[..., e] * d[..., e])
    return lp


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("mv", ["stretch", "de", "snooker"])
def test_callbacks(where, mv):
    K, N, D = 3, 32, 4
    seeds = _seeds(K, 5)
    data = np.random.default_rng(2).normal(size=(K, D))  # per-ensemble data: the mean of each ensemble's target
    p0 = _p0(K, N, D, 4)
    calls = []
    if where == "device":
        torch = pytest.importorskip("torch")
        mu_t = torch.as_tensor(data, device="cuda")

        def fn(x):
            calls.append(tuple(x.shape))
            return _lp(torch.as_tensor(x, device="cuda"), mu_t)

        def twin_fn(k):
            return models.CudaArrayFunction(lambda x: _lp(torch.as_tensor(x, device="cuda"), mu_t[k]))

        wrap = models.CudaArrayFunction
    else:
        def fn(x):
            calls.append(x.shape)
            return _lp(x, data)

        def twin_fn(k):
            return models.HostFunction(lambda x: _lp(x, data[k]), vectorize=True)

        def wrap(f):
            return models.HostFunction(f, vectorize=True)

    b = emcee_b200.BatchSampler(K, N, D, wrap(fn), moves=MOVES[mv](2, True), seeds=seeds)
    last = b.run_mcmc(p0, 20, skip_initial_state_check=True)
    P = 4 if mv == "snooker" else 2
    assert calls == [(K, N, D)] + [(K, N // P, D)] * (20 * P)  # the initial state, then once per half-step
    for k in range(K):
        t = emcee_b200.EnsembleSampler(N, D, twin_fn(k), moves=MOVES[mv](2, True), seed=seeds[k])
        lt = t.run_mcmc(p0[k], 20, skip_initial_state_check=True)
        _assert_twin(b, k, t, last, lt)
    x = _p0(K, 6, D, 9)
    calls.clear()
    assert np.array_equal(b.compute_log_prob(x), _lp(x, data))
    assert calls == [(K, 6, D)]


def test_callback_bad_shape():
    b = emcee_b200.BatchSampler(2, 16, 2, models.HostFunction(lambda x: np.zeros(x.shape[0] * x.shape[1]),
                                                              vectorize=True), seeds=1)
    with pytest.raises(NotImplementedError, match=r"lp\[nbatch, m\]"):
        b.run_mcmc(_p0(2, 16, 2), 2, skip_initial_state_check=True)


# ---- errors and resume ------------------------------------------------------------------------------------------
def test_nan_in_one_ensemble():
    """Ensemble j's rows turn NaN at the 31st call of the function, and so do its twin's: the initial state, then two
    calls a step, so the 31st is the second half-step of the step after the 14th."""
    K, N, D, j = 3, 32, 3, 1
    seeds = _seeds(K, 77)
    p0 = _p0(K, N, D, 8)

    def counted(nan_rows):
        calls = [0]

        def fn(x):
            calls[0] += 1
            lp = _lp(x, np.zeros(D))
            return np.where(nan_rows & (calls[0] == 31), np.nan, lp)

        return models.HostFunction(fn, vectorize=True)

    b = emcee_b200.BatchSampler(K, N, D, counted((np.arange(K) == j)[:, None]), seeds=seeds)
    t = emcee_b200.EnsembleSampler(N, D, counted(True), seed=seeds[j])
    errs = []
    for s, x in ((b, p0), (t, p0[j])):
        with pytest.raises(ValueError) as e:
            s.run_mcmc(x, STEPS, skip_initial_state_check=True)
        errs.append(str(e.value))
    assert errs[0] == errs[1] == "Probability function returned NaN"
    assert b.iteration == t.iteration == 14
    assert b.random_state[2] == t.random_state[2] == 14
    assert b.backend.random_state[2] == t.backend.random_state[2] == 14
    assert np.array_equal(b.get_chain()[:, j], t.get_chain())
    assert np.array_equal(b.get_log_prob()[:, j], t.get_log_prob())


def test_dependent_walkers_named():
    K, N, D = 4, 16, 3
    p0 = _p0(K, N, D)
    p0[2, :, 1] = 3.0 * p0[2, :, 0]
    b = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1)
    with pytest.raises(ValueError, match=r"\(ensemble 2\)"):
        b.run_mcmc(p0, 5)
    assert b.iteration == 0


def test_split_calls_and_resume():
    K, N, D = 6, 32, 5
    p0 = _p0(K, N, D)
    one = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40)
    one.run_mcmc(p0, 50, skip_initial_state_check=True)
    two = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40)
    two.run_mcmc(p0, 25, skip_initial_state_check=True)
    mid = two.get_last_sample()
    two.run_mcmc(None, 25)
    assert np.array_equal(one.get_chain(), two.get_chain())
    assert np.array_equal(one.acceptance_fraction, two.acceptance_fraction)
    # a random_state round trip on a fresh sampler resumes exactly
    three = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=1)
    three.random_state = mid.random_state
    three.run_mcmc(emcee_b200.State(mid.coords, log_prob=mid.log_prob), 25, skip_initial_state_check=True)
    assert np.array_equal(three.get_chain(), one.get_chain()[25:])
    # the generator gives the same steps
    four = emcee_b200.BatchSampler(K, N, D, models.Ring(2.0, 0.5), moves=moves.DEMove(), seeds=40)
    for _ in four.sample(p0, iterations=50, skip_initial_state_check=True):
        pass
    assert np.array_equal(four.get_chain(), one.get_chain())


def test_impossible_batch():
    with pytest.raises(MemoryError):
        emcee_b200.BatchSampler(2**20, 32, 1000, models.GaussianIso(), seeds=1)
    b = emcee_b200.BatchSampler(2, 16, 2, models.GaussianIso(), seeds=1)
    b.run_mcmc(_p0(2, 16, 2), 3, skip_initial_state_check=True)
    assert b.iteration == 3


def test_unsupported_engine_calls():
    b = emcee_b200.BatchSampler(2, 16, 2, models.GaussianIso(), seeds=1)
    for call in (lambda e: e.set_option("tma_rows", 1), lambda e: e.trace_config(1),
                 lambda e: e.window_config(4, 1), lambda e: e.reservoir_config(4, 1)):
        with pytest.raises(NotImplementedError, match="batch context"):
            call(b._engine)


# ---- scale ------------------------------------------------------------------------------------------------------
def test_scale_8192():
    K, N, D = 8192, 32, 5
    seeds = _seeds(K, 3)
    p0 = _p0(K, N, D, 21)
    b = emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=seeds)
    last = b.run_mcmc(p0, 20, skip_initial_state_check=True)
    for k in np.random.default_rng(0).choice(K, 12, replace=False).tolist() + [0, K - 1]:
        t = _twin(N, D, models.GaussianIso(), moves.StretchMove(), seeds[k])
        lt = t.run_mcmc(p0[k], 20, skip_initial_state_check=True)
        _assert_twin(b, k, t, last, lt)
