"""The running reservoir (``EnsembleSampler.enable_reservoir`` / ``reservoir`` / ``reservoir_count``;
``eb_reservoir_config``, ``eb_reservoir_read``, ``eb_reservoir_read_to``) against the rows the same run stores.

* Exact oracle: a run stores every ``every``-th step into a host ``Backend`` while the reservoir records the same
  steps; the tag-10 keys of every stored (step, walker) in numpy, ordered by ``np.lexsort``, give the first K rows,
  and the reservoir equals them with ``==``: K from 1 to more than all rows, odd and even N, every kernel path and
  move kind, a host function and a captured torch graph.
* Invariance: one call, many calls and ``sample()`` step by step give the same bytes, across table chunks and many
  compactions; ``size=K`` cut to k rows is ``size=k``.
* Nothing else moves: chain, trace and histograms are the same bytes with the reservoir on; ``cuda=True`` equals the
  host read.
* Edge cases: ``iterations=None``, re-enabling, ``every=0``, pickling, a graph model's NaN, an impossible size.
"""
import pickle

import numpy as np
import pytest

from reservoir_ref import reservoir_keys, reservoir_order

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, models, moves

pytestmark = pytest.mark.gpu

SEED = 0x5E5E


def _cb_iso(x):
    return -0.5 * np.sum(np.square(x), axis=1)


def _dense(D):
    rng = np.random.default_rng(D)
    a = rng.standard_normal((D, D))
    return models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)), np.linspace(-1, 1, D))


def _graph_iso(D):
    from test_gpu_graph_function import Capture, iso_columns

    return models.CudaGraphFunction(Capture(iso_columns, D))


CASES = {
    # name: (N, D, model, moves, expected kernel name)
    "dense_dmma": (96, 16, lambda: _dense(16), None, "dense_dmma"),
    "tma_rows": (64, 8, lambda: models.GaussianIso(), None, "tma_rows"),
    "generic_odd": (37, 3, lambda: models.GaussianIso(), None, "generic"),
    "de_snooker": (48, 6, lambda: models.Rosenbrock(),
                   lambda: [(moves.DEMove(), 0.7), (moves.DESnookerMove(), 0.3)], None),
    "walk_gaussian": (41, 4, lambda: models.GaussianIso(),
                      lambda: [(moves.WalkMove(s=5), 0.5), (moves.GaussianMove(0.3), 0.5)], None),
    "kde": (64, 4, lambda: models.GaussianIso(), lambda: moves.KDEMove(), None),
    "host_fn": (32, 5, lambda: models.HostFunction(_cb_iso, vectorize=True), None, "callback"),
    "graph_fn": (33, 5, lambda: _graph_iso(5), None, None),
}


def _make(case, backend=None, seed=SEED):
    N, D, model, mv, _ = CASES[case]
    return emcee_b200.EnsembleSampler(N, D, model(), moves=None if mv is None else mv(), seed=seed, backend=backend)


def _p0(case):
    N, D = CASES[case][:2]
    return np.random.default_rng(N * D).standard_normal((N, D)) * 0.5 + 0.1


def _expected(s, every, K):
    """the first K rows, in the reservoir's order, of the steps s stored (thin_by=every from step 0)"""
    chain, lp = s.get_chain(), s.get_log_prob()
    n, N = lp.shape
    steps = every * np.arange(1, n + 1, dtype=np.uint64)
    key = np.concatenate([reservoir_keys(SEED, int(t), np.arange(N)) for t in steps])
    step = np.repeat(steps, N)
    walker = np.tile(np.arange(N, dtype=np.int64), n)
    o = reservoir_order(key, step, walker)[:K]
    return chain.reshape(n * N, -1)[o], lp.reshape(-1)[o], step[o], walker[o]


def _same(r, want):
    coords, lp, step, walker = want
    assert r.step.dtype == np.uint64 and r.walker.dtype == np.int64
    assert r.coords.shape == coords.shape and r.log_prob.shape == lp.shape
    assert np.array_equal(r.step, step) and np.array_equal(r.walker, walker)
    assert r.coords.tobytes() == coords.tobytes() and r.log_prob.tobytes() == lp.tobytes()


def _bytes(r):
    return [np.asarray(f).tobytes() for f in r]


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("case", list(CASES))
def test_oracle(case, every):
    N = CASES[case][0]
    total = N * 12 // every
    for K in sorted({1, 7, N - 1, N, 3 * N + 5, total + 3}):
        s = _make(case)
        s.enable_reservoir(K, every)
        st = _p0(case)
        for _ in range(2):  # two calls of 6 steps (run_mcmc runs thin_by steps per stored one): stored == recorded
            st = s.run_mcmc(st, 6 // every, thin_by=every, skip_initial_state_check=True)
        want = CASES[case][4]
        if want is not None:
            assert s._engine.last_kernel_name() == want
        assert s.reservoir_count() == total
        _same(s.reservoir(), _expected(s, every, K))


@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma"])
@pytest.mark.parametrize("K", [50, 300])
def test_invariance(case, K):
    n = 130  # across two 64-step table chunks; K = 50 compacts before almost every record, K = 300 every few
    p0 = _p0(case)
    runs = []
    for split in ([n], [1, 63, 66], [5] * 26):
        s = _make(case)
        s.enable_reservoir(K)
        st = p0
        for m in split:
            st = s.run_mcmc(st, m, store=False, skip_initial_state_check=True)
        runs.append(s)
    s = _make(case)
    s.enable_reservoir(K)
    for _ in s.sample(p0, iterations=n, store=False, skip_initial_state_check=True):
        pass
    runs.append(s)
    N = CASES[case][0]
    assert all(r.reservoir_count() == n * N for r in runs)
    first = _bytes(runs[0].reservoir())
    for r in runs[1:]:
        assert _bytes(r.reservoir()) == first
    # reading again changes nothing
    assert _bytes(runs[0].reservoir()) == first
    # the prefix property: the first k rows are the reservoir of size k
    full = runs[0].reservoir()
    for k in (1, 7, 33):
        s = _make(case)
        s.enable_reservoir(k)
        s.run_mcmc(p0, n, store=False, skip_initial_state_check=True)
        assert _bytes(s.reservoir()) == [np.asarray(f)[:k].tobytes() for f in full]


@pytest.mark.parametrize("backend", [Backend, DeviceBackend])
@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma", "generic_odd"])
def test_nothing_else_moves(case, backend):
    D = CASES[case][1]
    out = []
    for on in (False, True):
        s = _make(case, backend())
        s.enable_trace(2)
        s.enable_histograms([(-4.0, 4.0)] * D, bins=16, every=2)
        if on:
            s.enable_reservoir(40, 2)
        s.run_mcmc(_p0(case), 20, skip_initial_state_check=True)
        out.append([s.get_chain().tobytes(), s.get_log_prob().tobytes(), s.backend.accepted.tobytes(),
                    _bytes(s.trace()), s.histogram()[0].tobytes(), s.random_state])
        if on:
            r, d = s.reservoir(), s.reservoir(cuda=True)
            assert isinstance(d.coords, emcee_b200.DeviceArray) and isinstance(d.log_prob, emcee_b200.DeviceArray)
            assert d.coords.get().tobytes() == r.coords.tobytes() and d.log_prob.get().tobytes() == r.log_prob.tobytes()
            assert np.array_equal(d.step, r.step) and np.array_equal(d.walker, r.walker)
    assert out[0] == out[1]


def test_iterations_none():
    case, N = "tma_rows", CASES["tma_rows"][0]
    s = _make(case)
    s.enable_reservoir(100)
    for i, _ in enumerate(s.sample(_p0(case), iterations=None, store=False, skip_initial_state_check=True)):
        if i + 1 == 20:
            break
    assert s.reservoir_count() == 20 * N
    t = _make(case)
    t.run_mcmc(_p0(case), 20, skip_initial_state_check=True)
    _same(s.reservoir(), _expected(t, 1, 100))


def test_lifecycle():
    case, N = "generic_odd", CASES["generic_odd"][0]
    s = _make(case)
    s.enable_reservoir(20, 2)
    st = s.run_mcmc(_p0(case), 10, store=False, skip_initial_state_check=True)
    kept = _bytes(s.reservoir())
    # every = 0 keeps the contents and records nothing more
    s.enable_reservoir(20, 0)
    st = s.run_mcmc(st, 6, store=False)
    assert s.reservoir_count() == 5 * N and _bytes(s.reservoir()) == kept
    # re-enabling clears
    s.enable_reservoir(20, 2)
    assert s.reservoir_count() == 0 and s.reservoir().coords.shape == (0, CASES[case][1])
    s.run_mcmc(st, 4, store=False)
    r = s.reservoir()
    assert s.reservoir_count() == 2 * N and set(r.step.tolist()) <= {18, 20}
    # an impossible size: MemoryError, and the reservoir and the sampler stay as they were
    kept = _bytes(s.reservoir())
    with pytest.raises(MemoryError):
        s.enable_reservoir(2**40)
    assert _bytes(s.reservoir()) == kept
    s.run_mcmc(None, 2, store=False)
    assert s.reservoir_count() == 3 * N
    # pickling drops the contents
    u = pickle.loads(pickle.dumps(s))
    with pytest.raises(RuntimeError, match="not enabled"):
        u.reservoir()
    u.enable_reservoir(5)
    u.run_mcmc(None, 1, store=False)
    assert u.reservoir_count() == N and u.reservoir().step.size == 5


def test_graph_nan_keeps_the_rows_before_it():
    from test_gpu_graph_function import Capture, NanAtCall

    N, D, e = 40, 4, 9  # the NaN falls in the first half-step of step e
    p0 = np.random.default_rng(1).standard_normal((N, D)) * 0.3

    def make(at):
        return emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(Capture(NanAtCall(at), D)),
                                          moves=moves.StretchMove(randomize_split=False), seed=SEED)

    s = make(1 + 2 * (e - 1) + 1)  # the initial state, two half-steps per step, then the first call of step e
    s.enable_reservoir(30)
    with pytest.raises(ValueError, match="NaN"):
        s.run_mcmc(p0, 20, store=False, skip_initial_state_check=True)
    t = make(0)
    t.enable_reservoir(30)
    t.run_mcmc(p0, e - 1, store=False, skip_initial_state_check=True)
    assert s.reservoir_count() == t.reservoir_count() == (e - 1) * N
    assert _bytes(s.reservoir()) == _bytes(t.reservoir())
