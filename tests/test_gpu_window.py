"""The running window (``EnsembleSampler.enable_window`` / ``window``; ``eb_window_config``, ``eb_window_chain``) against
the chain the same run stores.

* Twins: a ``store=False`` run with the window enabled and a run of the same seed that stores every step in a
  ``DeviceBackend``.  The window's reads equal ``get_chain(thin=every)[-size:]`` of the twin byte for byte, flat or
  not, over a grid of ``discard`` / ``thin`` and with ``cuda=True``; its ``steps`` are the twin's step counters.
  Every kernel path and move kind.
* Analyses: a reference ``DeviceBackend`` filled by ``save_step`` with exactly the window's steps gives the same
  percentiles, moments, histograms and autocorrelation time (``/ every``), slices across the wrap included.
* Accept counts, resume from ``get_last_sample()``, invariance across call splits, ``sample(thin_by=3)`` and
  ``iterations=None``, nothing else moving with the window on, a graph model's NaN, an impossible size, and the
  flagship ensemble.
"""
import numpy as np
import pytest

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, State, models, moves

pytestmark = pytest.mark.gpu

SEED = 0x3D1E


def _dense(D):
    rng = np.random.default_rng(D)
    a = rng.standard_normal((D, D))
    return models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)), np.linspace(-1, 1, D))


def _graph_iso(D):
    from test_gpu_graph_function import Capture, iso_columns

    return models.CudaGraphFunction(Capture(iso_columns, D))


def _gauss_mh(coords, random):
    return coords + 0.3 * random.standard_normal(coords.shape), np.zeros(coords.shape[0])


def _host_iso(x):
    return -0.5 * np.sum(np.square(x), axis=1)


CASES = {
    # name: (N, D, model, moves)
    "dense_dmma": (4096, 128, lambda: _dense(128), None),
    "tma_rows": (64, 8, lambda: models.GaussianIso(), None),
    "generic_odd": (37, 3, lambda: models.GaussianIso(), None),
    "bounded": (48, 4, lambda: models.Bounded(models.GaussianIso(), np.full(4, -2.5), np.full(4, 3.5)), None),
    "walk_gaussian": (41, 4, lambda: models.GaussianIso(),
                      lambda: [(moves.WalkMove(s=5), 0.5), (moves.GaussianMove(0.3), 0.5)]),
    "kde": (64, 4, lambda: models.GaussianIso(), lambda: moves.KDEMove()),
    "host_fn": (32, 3, lambda: models.HostFunction(_host_iso, vectorize=True), None),
    "graph_fn": (33, 5, lambda: _graph_iso(5), None),
    "user_move": (32, 4, lambda: models.GaussianIso(), lambda: moves.MHMove(moves.HostProposal(_gauss_mh))),
}


def _make(case, backend=None, seed=SEED):
    N, D, model, mv = CASES[case]
    return emcee_b200.EnsembleSampler(N, D, model(), moves=None if mv is None else mv(), seed=seed, backend=backend)


def _p0(case):
    N, D = CASES[case][:2]
    return np.random.default_rng(N * D).standard_normal((N, D)) * 0.5 + 1.0


def _twin(case, steps):
    t = _make(case, DeviceBackend())
    t.run_mcmc(_p0(case), steps)
    return t


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _expected(t, every, size):
    """(coords, log_prob, steps) the window must hold: the twin's every `every`-th step, the last `size` of them"""
    x, lp = t.get_chain(thin=every)[-size:], t.get_log_prob(thin=every)[-size:]
    steps = np.arange(1, t.iteration + 1, dtype=np.uint64)[every - 1 :: every][-size:]
    return x, lp, steps


SLICES = [(0, 1), (1, 1), (0, 2), (3, 2), (2, 5), (0, 50), (7, 3)]


def _check_reads(w, t, every, size):
    x, lp, steps = _expected(t, every, size)
    n = len(x)
    assert w.iteration == n and _same(w.steps, steps)
    assert w.random_state == ("philox4x32-10", SEED, int(steps[-1]))
    assert _same(w.get_chain(), x) and _same(w.get_log_prob(), lp)
    assert _same(w.get_chain(flat=True), x.reshape(-1, x.shape[2]))
    assert _same(w.get_value("log_prob", flat=True), lp.reshape(-1))
    assert w.get_blobs() is None
    for discard, thin in SLICES:
        sl = slice(discard + thin - 1, None, thin)
        assert _same(w.get_chain(discard=discard, thin=thin), x[sl]), (discard, thin)
        assert _same(w.get_log_prob(discard=discard, thin=thin), lp[sl]), (discard, thin)
        if len(x[sl]):
            assert _same(w.get_chain(discard=discard, thin=thin, cuda=True).get(), x[sl])
            assert _same(w.get_log_prob(discard=discard, thin=thin, flat=True, cuda=True).get(), lp[sl].reshape(-1))
    last = w.get_last_sample()
    assert _same(last.coords, x[-1]) and _same(last.log_prob, lp[-1]) and last.random_state == w.random_state
    last = w.get_last_sample(cuda=True)
    assert _same(last.coords.get(), x[-1]) and _same(last.log_prob.get(), lp[-1])


def _reference(w, t, every, size):
    """a DeviceBackend holding exactly the window's steps, saved one by one"""
    x, lp, _ = _expected(t, every, size)
    ref = DeviceBackend()
    ref.reset(*w.shape)
    ref.grow(len(x), None)
    for k in range(len(x)):
        ref.save_step(State(x[k], log_prob=lp[k]), np.zeros(w.nwalkers, dtype=bool))
    return ref


def _check_analyses(w, ref, every, slices=((0, 1), (2, 3), (1, 2))):
    for discard, thin in slices:
        kw = dict(discard=discard, thin=thin)
        if ref.get_chain(**kw).shape[0] == 0:
            continue
        q = [2.5, 50, 97.5]
        assert _same(w.get_percentile(q, **kw), ref.get_percentile(q, **kw))
        assert _same(w.get_percentile(q, name="log_prob", **kw), ref.get_percentile(q, name="log_prob", **kw))
        for a, b in zip(w.get_moments(**kw), ref.get_moments(**kw)):
            assert _same(a, b)
        for a, b in zip(w.get_histogram(bins=12, **kw), ref.get_histogram(bins=12, **kw)):
            assert _same(a, b)
        for a, b in zip(w.get_histogram2d(bins=6, **kw)[:2], ref.get_histogram2d(bins=6, **kw)[:2]):
            assert _same(a, b)
        if ref.get_chain(**kw).shape[0] >= 2:
            got = w.get_autocorr_time(quiet=True, **kw) / every
            assert _same(got, ref.get_autocorr_time(quiet=True, **kw))


TWINS = [
    # case, every, size, steps
    ("dense_dmma", 1, 5, 23),
    ("tma_rows", 3, 7, 60),
    ("generic_odd", 1, 16, 40),
    ("bounded", 1, 9, 50),
    ("walk_gaussian", 3, 6, 45),
    ("kde", 1, 8, 30),
    ("host_fn", 3, 5, 33),
    ("graph_fn", 1, 6, 25),
    ("user_move", 1, 11, 27),
]


@pytest.mark.parametrize("case,every,size,steps", TWINS)
def test_twins(case, every, size, steps):
    s = _make(case)
    s.enable_window(size, every)
    s.run_mcmc(_p0(case), steps, store=False)
    w = s.window()
    assert w.recorded == steps // every and w.every == every
    t = _twin(case, steps)
    _check_reads(w, t, every, size)
    _check_analyses(w, _reference(w, t, every, size), every)


@pytest.mark.parametrize("size", [1, 10, 19, 20, 21, 64])
def test_sizes_around_the_run(size):
    """size 1, below, equal to and above the 20 recorded steps, one call wrapping the ring several times"""
    s = _make("tma_rows")
    s.enable_window(size)
    s.run_mcmc(_p0("tma_rows"), 20, store=False)
    w = s.window()
    assert (w.recorded, w.iteration) == (20, min(size, 20))
    t = _twin("tma_rows", 20)
    _check_reads(w, t, 1, size)
    ref = _reference(w, t, 1, size)
    # slices that straddle the wrap (origin 20 % size), and every slot
    _check_analyses(w, ref, 1, slices=((0, 1), (1, 2), (0, 3), (size // 2, 1)))


def _window_after(case, cut, size=9, every=1, total=40):
    s = _make(case)
    s.enable_window(size, every)
    st = _p0(case)
    if cut == "one":
        s.run_mcmc(st, total, store=False)
    elif cut == "many":
        done = 0
        for k in [1, 4, 1, 9, 2, 13]:
            st = s.run_mcmc(st, k, store=False)
            done += k
        s.run_mcmc(st, total - done, store=False)
    elif cut == "sample":
        for _ in s.sample(st, iterations=total, store=False):
            pass
    elif cut == "sample_thin":
        assert total % 3 == 0
        for _ in s.sample(st, iterations=total // 3, thin_by=3, store=False):
            pass
    elif cut == "unbounded":
        for k, _ in enumerate(s.sample(st, iterations=None, store=False)):
            if k + 1 == total:
                break
    w = s.window()
    return w.recorded, w.steps, w.get_chain(), w.get_log_prob(), w.accepted


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma"])
def test_call_splits(case, every):
    want = _window_after(case, "one", every=every, total=42)
    for cut in ("many", "sample", "sample_thin", "unbounded"):
        got = _window_after(case, cut, every=every, total=42)
        assert got[0] == want[0], cut
        for a, b in zip(got[1:], want[1:]):
            assert _same(a, b), cut


@pytest.mark.parametrize("stop", [5, 17, 31])
def test_unbounded_stopped_anywhere(stop):
    s = _make("generic_odd")
    s.enable_window(8, 3)
    for k, _ in enumerate(s.sample(_p0("generic_odd"), iterations=None, store=False)):
        if k + 1 == stop:
            break
    _check_reads(s.window(), _twin("generic_odd", stop), 3, 8)


@pytest.mark.parametrize("every", [1, 3])
def test_accepted(every):
    """the accept counts of the window's steps: per-step masks from a host Backend twin's accepted, summed over the
    recorded steps the window holds"""
    case, size, steps = "generic_odd", 7, 36
    s = _make(case)
    s.enable_window(size, every)
    s.run_mcmc(_p0(case), steps, store=False)
    w = s.window()
    t = _make(case, Backend())
    before, masks = np.zeros(CASES[case][0]), []
    for _ in t.sample(_p0(case), iterations=steps):
        masks.append(t.backend.accepted - before)
        before = t.backend.accepted.copy()
    kept = np.array(masks)[every - 1 :: every][-size:]
    assert _same(w.accepted, kept.sum(axis=0))
    assert _same(w.acceptance_fraction, kept.sum(axis=0) / len(kept))


@pytest.mark.parametrize("every", [1, 3])
def test_resume_from_last_sample(every):
    case, steps, more = "tma_rows", 30, 12
    s = _make(case)
    s.enable_window(4, every)
    s.run_mcmc(_p0(case), steps, store=False)
    last = s.window().get_last_sample()
    fresh = _make(case, DeviceBackend(), seed=12345)
    fresh.run_mcmc(last, more)
    t = _twin(case, steps + more)
    assert _same(fresh.get_chain(), t.get_chain()[steps:]) and _same(fresh.get_log_prob(), t.get_log_prob()[steps:])


def test_nothing_else_moves():
    out = []
    for on in (False, True):
        s = _make("dense_dmma", DeviceBackend())
        s.enable_trace(1)
        s.enable_reservoir(100, 2)
        s.enable_autocorr(8, 1)
        s.enable_histograms([(-4, 4)] * 128, bins=16, params2d=[0, 1, 2])
        if on:
            s.enable_window(6, 2)
        s.run_mcmc(_p0("dense_dmma"), 30)
        out.append((s.get_chain(), s.get_log_prob(), s.backend.accepted, s.trace().mean, s.reservoir().coords,
                    s.autocorr_function(), s.histogram()[0], s.histogram2d()[0]))
    for a, b in zip(*out):
        assert _same(a, b)


def test_graph_nan_stops_before_the_window_records_past_it():
    from test_gpu_graph_function import Capture, NanAtCall

    N, D, e = 40, 4, 9  # the NaN falls in the first half-step of step e
    p0 = np.random.default_rng(1).standard_normal((N, D)) * 0.3

    def make(at):
        return emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(Capture(NanAtCall(at), D)),
                                          moves=moves.StretchMove(randomize_split=False), seed=SEED)

    s = make(1 + 2 * (e - 1) + 1)  # the initial state, two half-steps per step, then the first call of step e
    s.enable_window(5)
    with pytest.raises(ValueError, match="NaN"):
        s.run_mcmc(p0, 20, store=False, skip_initial_state_check=True)
    t = make(0)
    t.enable_window(5)
    t.run_mcmc(p0, e - 1, store=False, skip_initial_state_check=True)
    w, v = s.window(), t.window()
    assert w.recorded == v.recorded == e - 1
    assert _same(w.steps, v.steps) and _same(w.get_chain(), v.get_chain()) and _same(w.accepted, v.accepted)


def test_lifecycle_and_impossible_size():
    s = _make("tma_rows")
    with pytest.raises(RuntimeError, match="not enabled"):
        s.window()
    s.enable_window(6, 1)
    st = s.run_mcmc(_p0("tma_rows"), 15, store=False)
    w = s.window()
    first = (w.steps, w.get_chain(), w.accepted)
    s.enable_window(6, 0)  # freezes
    st = s.run_mcmc(st, 10, store=False)
    assert w.recorded == 15 and all(_same(a, b) for a, b in zip(first, (w.steps, w.get_chain(), w.accepted)))
    with pytest.raises(MemoryError):
        s.enable_window(2 ** 40, 1)
    assert s._window == (6, 1) and w.recorded == 15
    assert all(_same(a, b) for a, b in zip(first, (w.steps, w.get_chain(), w.accepted)))
    with pytest.raises(ValueError):  # the ring refuses writes in the library too
        w._ch.write(0, np.zeros((64, 8)), np.zeros(64))
    with pytest.raises(ValueError):
        w._ch.grow(100)
    s.enable_window(3, 2)  # re-enable: recorded from scratch
    s.run_mcmc(st, 10, store=False)
    assert (w.recorded, w.iteration) == (5, 3) and w.steps.tolist() == [30, 32, 34]


def test_flagship_ensemble():
    """65 536 x 128 on dense_dmma with a small window"""
    N, D, steps, size = 65536, 128, 12, 3
    p0 = np.random.default_rng(0).standard_normal((N, D)) * 0.5

    def make(backend=None):
        return emcee_b200.EnsembleSampler(N, D, _dense(D), seed=SEED, backend=backend)

    s = make()
    s.enable_window(size, 2)
    s.run_mcmc(p0, steps, store=False)
    assert s._engine.last_kernel_name() == "dense_dmma"
    w = s.window()
    t = make(DeviceBackend())
    t.run_mcmc(p0, steps)
    x, lp, st = _expected(t, 2, size)
    assert _same(w.steps, st) and _same(w.get_chain(), x) and _same(w.get_log_prob(), lp)
    assert _same(w.get_chain(thin=2, cuda=True).get(), x[1::2])
