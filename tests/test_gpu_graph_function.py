"""``models.CudaGraphFunction`` on the GPU: a torch log-probability captured as CUDA graphs, launched by the engine
between its propose and accept kernels.

* twins: the same torch function as a ``CudaArrayFunction`` and as captured graphs gives byte-equal chains,
  log-probabilities, accept counts, random states and final states, over every move kind, odd ensembles with three
  splits, every storage path, the running statistics and ``compute_log_prob``;
* golden cases of the unmodified reference with the oracle targets written in torch, at the tolerances of
  ``test_gpu_callback.py``;
* errors (NaN log-probability, non-finite proposals) leave what the ``CudaArrayFunction`` twin leaves, and the graph
  never sees a non-finite row;
* pickling re-captures, the kernel variant, ``eb_model_set`` clearing the graphs.

Only well-formed graphs reach the engine here; the refusals are tested on the host (test_graph_function_host.py).
"""
import pickle

import numpy as np
import pytest

from test_gpu_callback import CASES, LP_ATOL, LP_RTOL, _golden, _tols
from gpu_util import device_moves

import emcee_b200
from emcee_b200 import _lib, models, moves

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover
    pytest.skip("torch has no CUDA", allow_module_level=True)


def iso_columns(x):
    """-0.5 sum(x^2), column by column: elementwise kernels only, so every row's value is the same bits at any m."""
    lp = torch.zeros(x.shape[0], dtype=torch.float64, device=x.device)
    for j in range(x.shape[1]):
        lp = lp + (x[:, j] * x[:, j]) * -0.5
    return lp


class Capture(object):
    """capture(m) for a torch function f: warm-up on a side stream, then one capture on a static x.  Records the row
    counts it was asked for; `seen_nonfinite` is a static flag the graph raises if it ever reads a non-finite row."""

    def __init__(self, f, ndim, strided=False):
        self.f, self.ndim, self.strided = f, ndim, strided
        self.calls = []
        self.seen = torch.zeros((), dtype=torch.bool, device="cuda")

    def body(self, x):
        self.seen.logical_or_(~torch.isfinite(x).all())
        lp = self.f(x)
        x.zero_()  # the graph may overwrite its input
        return lp

    def __call__(self, m):
        self.calls.append(m)
        if self.strided:  # a strided first axis for x, a strided lp
            x = torch.zeros((m, 2 * self.ndim), dtype=torch.float64, device="cuda")[:, : self.ndim]
        else:
            x = torch.zeros((m, self.ndim), dtype=torch.float64, device="cuda")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self.body(x)
        torch.cuda.current_stream().wait_stream(side)
        self.seen.zero_()
        if hasattr(self.f, "reset"):
            self.f.reset()  # the warm-up calls do not count
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            lp = self.body(x)
            if self.strided:
                buf = torch.empty(2 * m, dtype=torch.float64, device="cuda")
                buf[::2] = lp
                lp = buf[::2]
        torch.cuda.synchronize()
        if hasattr(self.f, "reset"):
            self.f.reset()
        return models.CapturedGraph(g.raw_cuda_graph_exec(), x, lp, owner=g)

    @property
    def seen_nonfinite(self):
        return bool(self.seen.item())


def array_fn(f):
    return models.CudaArrayFunction(lambda rows: f(torch.as_tensor(rows, device="cuda")))


class TorchStretch(moves.CudaArrayRedBlueMove):
    """A user red-blue move in torch: the draws on the host, the rows on the device."""

    def __init__(self, **kw):
        self.a = 2.0
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        S = torch.as_tensor(s, device="cuda")
        Cc = torch.cat([torch.as_tensor(x, device="cuda") for x in c])
        ns, nc, ndim = S.shape[0], Cc.shape[0], S.shape[1]
        zz = ((self.a - 1.0) * random.rand(ns) + 1) ** 2.0 / self.a
        rint = random.randint(nc, size=(ns,))
        cr = Cc[torch.as_tensor(rint, device="cuda")]
        return cr - (cr - S) * torch.as_tensor(zz, device="cuda")[:, None], (ndim - 1.0) * np.log(zz)


def _p0(N, D, seed=3, scale=1.0):
    return scale * np.random.default_rng(seed).standard_normal((N, D))


def _pair(N, D, make_moves, f=iso_columns, seed=11, strided=False, **kw):
    cap = Capture(f, D, strided=strided)
    a = emcee_b200.EnsembleSampler(N, D, array_fn(f), moves=make_moves(), seed=seed, **kw)
    kw = {k: (type(v)() if isinstance(v, emcee_b200.DeviceBackend) else v) for k, v in kw.items()}
    g = emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(cap), moves=make_moves(), seed=seed, **kw)
    return a, g, cap


def _assert_same(a, g, stored=True):
    if stored:
        assert a.backend.iteration == g.backend.iteration
    if stored and g.backend.iteration:
        assert a.get_chain().tobytes() == g.get_chain().tobytes()
        assert a.get_log_prob().tobytes() == g.get_log_prob().tobytes()
        assert np.array_equal(a.backend.accepted, g.backend.accepted)
        assert a.backend.random_state == g.backend.random_state
    assert a.random_state == g.random_state
    ca, la = a._engine.get_state()
    cg, lg = g._engine.get_state()
    assert ca.tobytes() == cg.tobytes() and la.tobytes() == lg.tobytes()
    assert np.array_equal(a._engine.naccepted(), g._engine.naccepted())


MOVES = {
    "stretch": lambda: moves.StretchMove(),
    "de": lambda: moves.DEMove(),
    "snooker": lambda: moves.DESnookerMove(),
    "walk": lambda: moves.WalkMove(s=4),
    "walk_all": lambda: moves.WalkMove(),
    "gaussian": lambda: moves.GaussianMove(0.3),
    "gaussian_sequential": lambda: moves.GaussianMove(np.full(5, 0.2), mode="sequential"),
    "kde": lambda: moves.KDEMove(),
    "user": lambda: TorchStretch(),
    "mix": lambda: [(moves.StretchMove(nsplits=3), 0.4), (moves.DEMove(), 0.3), (moves.GaussianMove(0.2), 0.3)],
}


@pytest.mark.parametrize("name", sorted(MOVES))
def test_twins_every_move(name):
    N, D, n = 48, 5, 12
    a, g, cap = _pair(N, D, MOVES[name])
    for s in (a, g):
        s.run_mcmc(_p0(N, D), n, thin_by=2, skip_initial_state_check=True)
    _assert_same(a, g)
    if name == "gaussian_sequential":
        assert a._moves[0].index == g._moves[0].index
    if name != "user":  # a user move reports itself ("user_move where=device")
        assert g._engine.last_kernel_variant().endswith("where=graph")
    assert not cap.seen_nonfinite


@pytest.mark.parametrize("how", ["store_false", "backend", "device_backend", "sample", "sample_device_backend",
                                 "strided"])
def test_twins_odd_ensemble_three_splits(how):
    N, D, n = 37, 3, 10
    kw = {"backend": emcee_b200.DeviceBackend()} if "device_backend" in how else {}
    a, g, cap = _pair(N, D, lambda: moves.StretchMove(nsplits=3), strided=how == "strided", **kw)
    assert cap.calls == [12, 13, 37]
    for s in (a, g):
        if how.startswith("sample"):
            for _ in s.sample(_p0(N, D), iterations=n, thin_by=2, skip_initial_state_check=True):
                pass
        else:
            s.run_mcmc(_p0(N, D), n, thin_by=2, store=how != "store_false", skip_initial_state_check=True)
    _assert_same(a, g, stored=how != "store_false")


def test_twins_running_statistics():
    N, D, n = 40, 3, 30
    a, g, _ = _pair(N, D, lambda: moves.StretchMove())
    for s in (a, g):
        s.enable_moments(every=2)
        s.enable_histograms(range=[(-4.0, 4.0)] * D, bins=12, every=3)
        s.enable_trace(every=1)
        s.run_mcmc(_p0(N, D), n, store=False, skip_initial_state_check=True)
    ma, mg = a.moments(), g.moments()
    for x, y in zip(ma, mg):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    assert np.array_equal(a.histogram()[0], g.histogram()[0])
    assert np.array_equal(a.trace().step, g.trace().step)
    assert a.trace().mean.tobytes() == g.trace().mean.tobytes()
    assert a.trace().log_prob_max.tobytes() == g.trace().log_prob_max.tobytes()
    _assert_same(a, g, stored=False)


@pytest.mark.parametrize("m", [5, 32, 32 * 2 + 7])
def test_compute_log_prob_host_and_cuda(m):
    N, D = 32, 4
    a, g, cap = _pair(N, D, lambda: moves.StretchMove())
    x = _p0(m, D, seed=m)
    la, _ = a.compute_log_prob(x)
    lg, _ = g.compute_log_prob(x)
    assert la.tobytes() == lg.tobytes()
    xt = torch.as_tensor(x, device="cuda")
    da, _ = a.compute_log_prob(xt)
    dg, _ = g.compute_log_prob(xt)
    assert da.get().tobytes() == dg.get().tobytes() == la.tobytes()
    assert not cap.seen_nonfinite


def _torch_target(g):
    kind = str(g["model_kind"])
    if kind == "gauss_iso":
        return lambda x: -0.5 * (x * x).sum(-1)
    if kind == "gauss_dense":
        icov = torch.as_tensor(np.asarray(g["model_icov"], dtype=np.float64), device="cuda")
        mean = torch.as_tensor(np.asarray(g["model_mean"], dtype=np.float64), device="cuda")

        def dense(x):
            d = x - mean
            return -0.5 * ((d @ icov) * d).sum(-1)  # cuBLAS: the captured GEMM may differ in the last bits

        return dense
    a, b = (float(v) for v in g["model_params"])
    if kind == "rosenbrock":
        def rosen(x):
            x0, x1 = x[:, :-1], x[:, 1:]
            t = x1 - x0 * x0
            u = a - x0
            return -(b * (t * t) + u * u).sum(-1)

        return rosen

    def ring(x):
        d = torch.sqrt((x * x).sum(-1)) - a
        return -(d * d) / (2.0 * b * b)

    return ring


@pytest.mark.parametrize("case", [c for c in CASES if c.startswith("g:")])
def test_golden_run_mcmc(case):
    g, _ = _golden(case)
    N, D = int(g["nwalkers"]), int(g["ndim"])
    cap = Capture(_torch_target(g), D)
    s = emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(cap), moves=device_moves(g["moves"], g),
                                   seed=int(g["seed"]))
    nsteps = g["chain"].shape[0]
    exact, rtol, atol = _tols(g)
    s.run_mcmc(g["p0"], nsteps, skip_initial_state_check=True)
    chain, lps = s.get_chain(), s.get_log_prob()
    if exact:
        assert np.array_equal(chain, g["chain"])
    else:
        np.testing.assert_allclose(chain, g["chain"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(lps, g["log_prob"], rtol=max(rtol, LP_RTOL), atol=max(10 * atol, LP_ATOL))
    assert np.array_equal(s.backend.accepted, g["accepted"].sum(axis=0))
    assert not cap.seen_nonfinite


# ---- errors ------------------------------------------------------------------------------------------------------
def nan_beyond(limit):
    """iso_columns, except NaN for every row whose first coordinate exceeds `limit`."""

    def f(x):
        lp = iso_columns(x)
        return torch.where(x[:, 0] > limit, torch.full_like(lp, float("nan")), lp)

    return f


N_ERR, D_ERR, SEED_ERR = 40, 4, 0xE1


def _err_pair(f, backend=None, make_moves=lambda: moves.StretchMove(randomize_split=False)):
    return _pair(N_ERR, D_ERR, make_moves, f=f, seed=SEED_ERR,
                 **({} if backend is None else {"backend": backend}))


def _fail_both(a, g, exc, match, run):
    for s in (a, g):
        with pytest.raises(exc, match=match) as e:
            run(s)
        s._msg = str(e.value)
    assert a._msg == g._msg


@pytest.mark.parametrize("make_moves", [lambda: moves.StretchMove(randomize_split=False),
                                        lambda: [(moves.StretchMove(nsplits=3), 0.5), (moves.WalkMove(s=3), 0.3),
                                                 (moves.GaussianMove(np.full(D_ERR, 0.3), mode="sequential"), 0.2)]],
                         ids=["stretch", "mix"])
@pytest.mark.parametrize("stats", [False, True])
def test_nan_stops_at_its_half_step(make_moves, stats):
    a, g, cap = _err_pair(nan_beyond(1.2), make_moves=make_moves)
    if stats:
        for s in (a, g):
            s.enable_moments(every=1)
            s.enable_trace(every=2)
    _fail_both(a, g, ValueError, "Probability function returned NaN",
               lambda s: s.run_mcmc(_p0(N_ERR, D_ERR, scale=0.3), 60, skip_initial_state_check=True))
    assert 0 < g.backend.iteration < 60
    _assert_same(a, g)
    for s in (a, g):
        s._after = [m.index for m in s._moves if hasattr(m, "_advance")]
    assert a._after == g._after
    if stats:
        assert [np.asarray(v).tobytes() for v in a.moments()] == [np.asarray(v).tobytes() for v in g.moments()]
        assert np.array_equal(a.trace().step, g.trace().step)
        assert a.trace().mean.tobytes() == g.trace().mean.tobytes()
    assert not cap.seen_nonfinite


class NanAtCall(object):
    """iso_columns with a call counter in device memory: call number `at` (1 = the initial state; 0 = never) returns
    NaN in its middle row.  A captured graph increments the counter itself, so it fails at the same half-step as the
    CudaArrayFunction twin, wherever that falls, whatever the host does in between."""

    def __init__(self, at):
        self.at = at
        self.count = torch.zeros((), dtype=torch.int64, device="cuda")

    def reset(self):
        self.count.zero_()

    def __call__(self, x):
        self.count.add_(1)
        lp = iso_columns(x)
        m = x.shape[0]
        hit = (self.count == self.at) & (torch.arange(m, device=x.device) == m // 2)
        return torch.where(hit, torch.full_like(lp, float("nan")), lp)


def _mix_seq():
    return [(moves.StretchMove(nsplits=3), 0.5), (moves.WalkMove(s=3), 0.3),
            (moves.GaussianMove(np.full(D_ERR, 0.3), mode="sequential"), 0.2)]


def _mix_vec():
    """_mix_seq without state carried from step to step, so that a resumed run continues the chain exactly."""
    return [(moves.StretchMove(nsplits=3), 0.5), (moves.WalkMove(s=3), 0.3), (moves.GaussianMove(0.3), 0.2)]


def _calls_through(make_moves, nsteps):
    """How many calls the initial state and the first `nsteps` steps of the error schedule make."""
    f = NanAtCall(0)
    s = emcee_b200.EnsembleSampler(N_ERR, D_ERR, array_fn(f), moves=make_moves(), seed=SEED_ERR)
    s.run_mcmc(_p0(N_ERR, D_ERR), nsteps, store=False, skip_initial_state_check=True)
    return int(f.count.item())


# (run_mcmc arguments, backend, iterations, the step the NaN falls in).  In each the host reads the graph's error
# state only several steps after the failing one: at the end of the call (store=False), before the next stored step
# (thin_by=3: the NaN falls in an unstored step), or at the start of the next chunk of 512 steps.
LATE = {
    "store_false": (dict(store=False), None, 60, 23),
    "thin_by3": (dict(thin_by=3), None, 30, 21),
    "thin_by3_device_backend": (dict(thin_by=3), emcee_b200.DeviceBackend, 30, 21),
    "next_chunk": (dict(store=False), None, 1100, 515),
}


@pytest.mark.parametrize("case", sorted(LATE))
def test_nan_found_later_rolls_back_like_the_twin(case):
    kw, backend, n, e = LATE[case]
    at = _calls_through(_mix_seq, e) + 1  # the first call of step e
    fa, fg = NanAtCall(at), NanAtCall(at)
    cap = Capture(fg, D_ERR)
    bk = (lambda: {}) if backend is None else (lambda: {"backend": backend()})
    a = emcee_b200.EnsembleSampler(N_ERR, D_ERR, array_fn(fa), moves=_mix_seq(), seed=SEED_ERR, **bk())
    g = emcee_b200.EnsembleSampler(N_ERR, D_ERR, models.CudaGraphFunction(cap), moves=_mix_seq(), seed=SEED_ERR,
                                   **bk())
    _fail_both(a, g, ValueError, "Probability function returned NaN",
               lambda s: s.run_mcmc(_p0(N_ERR, D_ERR), n, skip_initial_state_check=True, **kw))
    assert a._engine.get_rng() == g._engine.get_rng() == (SEED_ERR, e)
    assert int(fg.count.item()) > at  # the graph ran on past the failing step before the host looked
    _assert_same(a, g, stored=kw.get("store", True))
    if kw.get("store", True):
        assert g.backend.iteration == e // kw["thin_by"]
    assert [m.index for m in a._moves if hasattr(m, "_advance")] == [m.index for m in g._moves
                                                                      if hasattr(m, "_advance")]
    assert not cap.seen_nonfinite


def test_nonfinite_proposal_raises_before_the_call():
    p0 = _p0(N_ERR, D_ERR)
    p0[0] = 1e308
    p0[1] = -1e308
    a, g, cap = _err_pair(iso_columns)
    _fail_both(a, g, ValueError, "At least one parameter value was",
               lambda s: s.run_mcmc(p0, 5, skip_initial_state_check=True))
    _assert_same(a, g)
    assert not cap.seen_nonfinite
    x = _p0(3, D_ERR)
    x[1, 2] = np.inf
    _fail_both(a, g, ValueError, "At least one parameter value was infinite", lambda s: s.compute_log_prob(x))
    assert not cap.seen_nonfinite


@pytest.mark.parametrize("thin_by", [1, 3])
@pytest.mark.parametrize("device_backend", [False, True])
@pytest.mark.parametrize("path", ["run_mcmc", "sample"])
def test_nan_error_and_resume_is_exact(path, device_backend, thin_by):
    n, e = 60 // thin_by, 31  # iterations; the step the NaN falls in (unstored with thin_by=3)
    at = _calls_through(_mix_vec, e) + 1
    bk = (lambda: {"backend": emcee_b200.DeviceBackend()}) if device_backend else (lambda: {})
    fa, fg = NanAtCall(at), NanAtCall(at)
    cap = Capture(fg, D_ERR)
    a = emcee_b200.EnsembleSampler(N_ERR, D_ERR, array_fn(fa), moves=_mix_vec(), seed=SEED_ERR, **bk())
    g = emcee_b200.EnsembleSampler(N_ERR, D_ERR, models.CudaGraphFunction(cap), moves=_mix_vec(), seed=SEED_ERR,
                                   **bk())

    def run(s):
        if path == "run_mcmc":
            s.run_mcmc(_p0(N_ERR, D_ERR), n, thin_by=thin_by, skip_initial_state_check=True)
        else:
            for _ in s.sample(_p0(N_ERR, D_ERR), iterations=n, thin_by=thin_by, skip_initial_state_check=True):
                pass

    _fail_both(a, g, ValueError, "Probability function returned NaN", run)
    k = g.backend.iteration
    assert k == e // thin_by
    _assert_same(a, g)
    assert a._engine.get_rng() == g._engine.get_rng() == (SEED_ERR, e)
    # resuming from the last stored sample continues the uninterrupted chain of the graph model bit for bit (the
    # counter is past the failing call, so the graph returns no more NaN)
    ref = emcee_b200.EnsembleSampler(N_ERR, D_ERR, models.CudaGraphFunction(Capture(NanAtCall(0), D_ERR)),
                                     moves=_mix_vec(), seed=SEED_ERR, **bk())
    ref.run_mcmc(_p0(N_ERR, D_ERR), k + 5, thin_by=thin_by, skip_initial_state_check=True)
    g.run_mcmc(g.get_last_sample(), 5, thin_by=thin_by)
    assert g.get_chain().tobytes() == ref.get_chain().tobytes()
    assert g.get_log_prob().tobytes() == ref.get_log_prob().tobytes()
    assert np.array_equal(g.backend.accepted, ref.backend.accepted)
    assert not cap.seen_nonfinite


# ---- pickling, re-capture, variant, model replacement -------------------------------------------------------------
CAPTURES = []


def module_capture(m):
    """A picklable capture function (module level)."""
    c = Capture(iso_columns, 3)
    CAPTURES.append(m)
    return c(m)


def test_pickle_recaptures_and_continues():
    N, D = 24, 3
    del CAPTURES[:]
    s = emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(module_capture),
                                   moves=[(moves.StretchMove(), 0.5), (moves.DEMove(nsplits=3), 0.5)], seed=5)
    assert CAPTURES == [8, 12, 24]
    s.run_mcmc(_p0(N, D), 6, skip_initial_state_check=True)
    t = pickle.loads(pickle.dumps(s))
    assert CAPTURES == [8, 12, 24, 8, 12, 24]
    s.run_mcmc(None, 6)
    t.run_mcmc(None, 6)
    assert s.get_chain().tobytes() == t.get_chain().tobytes()
    assert s.random_state == t.random_state


def test_kernel_variant_and_model_replacement():
    N, D = 16, 3
    cap = Capture(iso_columns, D)
    s = emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(cap), seed=2)
    s.run_mcmc(_p0(N, D), 2, skip_initial_state_check=True)
    assert s._engine.last_kernel_name() == "callback"
    assert s._engine.last_kernel_variant().endswith("where=graph")
    # eb_model_set clears the graphs: the device model runs, and the static buffers are no longer written
    before = cap.calls[:]
    bufs = [(g.x.clone(), g.lp.clone()) for g in s._engine._cb]
    s._engine.set_model("gauss_iso", [])
    s._engine.set_state(_p0(N, D), None)
    s._engine.step(s._schedule(), 2)
    torch.cuda.synchronize()
    assert s._engine.last_kernel_name() != "callback"
    assert cap.calls == before
    for g, (x, lp) in zip(s._engine._cb, bufs):
        assert torch.equal(g.x, x) and torch.equal(g.lp, lp)
    # and back: a new set of graphs
    s._load_model()
    s._engine.set_state(_p0(N, D), None)
    s._engine.step(s._schedule(), 1)
    assert s._engine.last_kernel_variant().endswith("where=graph")
    assert _lib.EB_CALLBACK_GRAPH == 2
