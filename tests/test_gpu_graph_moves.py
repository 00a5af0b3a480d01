"""Captured proposals on the GPU (``moves.CudaGraphRedBlueMove``, ``moves.CudaGraphProposal``): a torch proposal
captured as a CUDA graph and launched by the engine between its gather and its accept.

* draws: a graph that returns its draws as the proposal, from ``log_prob = -inf`` so that every proposal lands in the
  state, leaves the purpose-9 draws of ``graph_draws`` (uniform: bit for bit; normal: to a few ulps, since the device
  and numpy round log / sin / cos apart), and a graph that copies its ``s`` and ``c`` aside shows the boolean-mask
  gathers of the oracle's split;
* twins: the same torch proposal run eagerly as ``CudaArrayRedBlueMove`` / ``CudaArrayProposal``, fed
  ``graph_draws`` for its ``(step, split)``, and captured, gives byte-equal chains, log-probabilities, accept counts,
  random states and live states over models, dimensions, schedules, backends and calling patterns;
* errors: inf / NaN proposals at a chosen half-step leave what the twin leaves; NaN factors reject without an error;
  pickling re-captures and continues.

Only well-formed captures reach the engine here; the refusals are tested on the host (test_graph_moves_host.py)."""
import pickle

import numpy as np
import pytest

from graph_draws_ref import graph_draws
from oracle import philox as px

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover
    pytest.skip("torch has no CUDA", allow_module_level=True)


def _t(x):
    return torch.as_tensor(x, device="cuda")


# ---- torch proposals: f(s, c, draws) -> (q, factors), the same ops eagerly and inside a graph ------------------------
def stretch(s, c, d, a=2.0):
    ns, D = s.shape
    zz = ((a - 1.0) * d[:, 0] + 1.0) ** 2 / a
    idx = torch.clamp((d[:, 1] * c.shape[0]).long(), max=c.shape[0] - 1)
    cr = c[idx]
    return cr - (cr - s) * zz[:, None], (D - 1.0) * torch.log(zz)


def de(s, c, d):
    ns, D = s.shape
    nc = c.shape[0]
    g0 = 2.38 / np.sqrt(2.0 * D)
    gamma = g0 * (1.0 + 0.2 * (d[:, 0] - 0.5))
    i1 = torch.clamp((d[:, 1] * nc).long(), max=nc - 1)
    i2 = torch.clamp((d[:, 2] * (nc - 1)).long(), max=nc - 2)
    i2 = i2 + (i2 >= i1).long()
    return s + gamma[:, None] * (c[i1] - c[i2]), torch.zeros(ns, dtype=torch.float64, device=s.device)


def mh_walk(s, c, d):
    return s + 0.6 * (d - 0.5), torch.zeros(s.shape[0], dtype=torch.float64, device=s.device)


PROPS = {"stretch": (stretch, 2), "de": (de, 3)}


class Capture(object):
    """capture(ns, counts) / capture(ns) for a torch proposal f: static s, c, draws, warm-up on a side stream, one
    capture.  `strided` gives every buffer a strided first axis."""

    def __init__(self, f, N, D, ndraws, strided=False, record=False):
        self.f, self.N, self.D, self.ndraws, self.strided, self.record = f, N, D, ndraws, strided, record
        self.calls, self.recs = [], {}

    def _buf(self, m, n):
        if self.strided:
            return torch.zeros((m, n + 2), dtype=torch.float64, device="cuda")[:, :n]
        return torch.zeros((m, n), dtype=torch.float64, device="cuda")

    def body(self, s, c, d):
        if self.record:  # copy the inputs aside
            rec = self.recs[s.shape[0]]
            rec[0].copy_(s)
            if c is not None:
                rec[1].copy_(c)
            if d is not None:
                rec[2].copy_(d)
        return self.f(s, c, d)

    def __call__(self, ns, counts=None):
        self.calls.append((ns, counts))
        nc = self.N - ns if counts is not None else 0
        s = self._buf(ns, self.D)
        c = self._buf(nc, self.D) if nc else None
        d = self._buf(ns, self.ndraws) if self.ndraws else None
        if d is not None:
            d.fill_(0.5)
        if self.record:
            self.recs[ns] = (s.clone(), None if c is None else c.clone(), None if d is None else d.clone())
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self.body(s, c, d)
        torch.cuda.current_stream().wait_stream(side)
        if hasattr(self.f, "reset"):
            self.f.reset()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            q, f = self.body(s, c, d)
            if self.strided:
                qb = torch.empty((ns, self.D + 1), dtype=torch.float64, device="cuda")
                qb[:, : self.D] = q
                fb = torch.empty(2 * ns, dtype=torch.float64, device="cuda")
                fb[::2] = f
                q, f = qb[:, : self.D], fb[::2]
        torch.cuda.synchronize()
        if hasattr(self.f, "reset"):
            self.f.reset()
        return moves.CapturedProposal(g.raw_cuda_graph_exec(), s, c, d, q, f, owner=g)


def _call_id(random):
    """(seed, step, split) of a user proposal call, from the counter of its ``random`` (moves.user_random)."""
    st = random.get_state(legacy=False)["state"]
    return int(st["key"][0]), int(st["counter"][1]), int(st["counter"][2])


class EagerTwin(moves.CudaArrayRedBlueMove):
    """The same torch proposal, called by the engine once per half-step with ``graph_draws`` of that half-step."""

    def __init__(self, f, ndraws, draw="uniform", **kw):
        self.f, self.ndraws, self.draw = f, ndraws, draw
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        seed, step, split = _call_id(random)
        S = _t(s)
        Cc = torch.cat([_t(x) for x in c])
        d = _t(graph_draws(seed, step, split, S.shape[0], self.draw, self.ndraws)) if self.ndraws else None
        return self.f(S, Cc, d)


def eager_mh(f, ndraws, draw="uniform"):
    def prop(coords, random):
        seed, step, split = _call_id(random)
        S = _t(coords)
        d = _t(graph_draws(seed, step, split, S.shape[0], draw, ndraws)) if ndraws else None
        return f(S, None, d)

    return moves.MHMove(moves.CudaArrayProposal(prop))


def move_pair(kind, N, D, draw="uniform", strided=False, **kw):
    """(eager move, captured move) of proposal `kind` ("stretch", "de", "mh")."""
    if kind == "mh":
        return (eager_mh(mh_walk, D, draw),
                moves.MHMove(moves.CudaGraphProposal(Capture(mh_walk, N, D, D, strided), ndraws=D, draw=draw)))
    f, nd = PROPS[kind]
    return (EagerTwin(f, nd, draw, **kw),
            moves.CudaGraphRedBlueMove(Capture(f, N, D, nd, strided), ndraws=nd, draw=draw, **kw))


def _p0(N, D, seed=3, scale=1.0):
    return scale * np.random.default_rng(seed).standard_normal((N, D))


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


def _twins(N, D, model, schedule, seed=11, **kw):
    """Two samplers whose schedules differ only in eager / captured user moves; `schedule(pair)` builds one."""
    mk = lambda: model() if callable(model) else model  # noqa: E731
    a = emcee_b200.EnsembleSampler(N, D, mk(), moves=schedule(0), seed=seed, **kw)
    kw = {k: (type(v)() if isinstance(v, emcee_b200.DeviceBackend) else v) for k, v in kw.items()}
    g = emcee_b200.EnsembleSampler(N, D, mk(), moves=schedule(1), seed=seed, **kw)
    return a, g


# ---- the draws and the gathers --------------------------------------------------------------------------------------
def _run_from_minus_inf(s, x, step):
    """One step from x with log_prob = -inf everywhere: every proposal is accepted."""
    s._engine.set_rng(s._engine.get_rng()[0], step)
    st = emcee_b200.State(x, log_prob=np.full(len(x), -np.inf))
    s.run_mcmc(st, 1, store=False, skip_initial_state_check=True)
    return s._engine.get_state()[0]


@pytest.mark.parametrize("draw", ["uniform", "normal"])
@pytest.mark.parametrize("N,P", [(37, 2), (41, 3), (33, 5)])
def test_draws_and_gathers(draw, N, P):
    D = 4
    seed = 0xD4
    for ndraws in (1, 2, 3, D, 2 * D + 1):
        def f(s, c, d):
            q = s.clone()
            m = min(ndraws, D)
            q[:, :m] = d[:, :m]
            return q, torch.zeros(s.shape[0], dtype=torch.float64, device=s.device)

        cap = Capture(f, N, D, ndraws, record=True)
        s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(),
                                       moves=moves.CudaGraphRedBlueMove(cap, ndraws=ndraws, draw=draw, nsplits=P),
                                       seed=seed)
        sizes = [(N - j + P - 1) // P for j in range(P)]
        last = {ns: max(j for j in range(P) if sizes[j] == ns) for ns in set(sizes)}  # the split a capture ran last
        for step in (0, 5, 2 ** 33 + 1):
            x0 = _p0(N, D, seed=step % 97)
            x1 = _run_from_minus_inf(s, x0, step)
            inds = px.split_assignment(seed, step, N, P, True)
            m = min(ndraws, D)
            before = x0.copy()
            for j in range(P):
                ref = graph_draws(seed, step, j, sizes[j], draw, ndraws)
                got = x1[inds == j][:, :m]
                if draw == "uniform":
                    assert got.tobytes() == ref[:, :m].tobytes()
                else:
                    assert np.allclose(got, ref[:, :m], rtol=1e-14, atol=1e-300)
                if last[sizes[j]] == j:
                    rs, rc, rd = (t.cpu().numpy() for t in cap.recs[sizes[j]])
                    assert rs.tobytes() == before[inds == j].tobytes()
                    assert rc.tobytes() == np.concatenate([before[inds == k] for k in range(P) if k != j]).tobytes()
                    if draw == "uniform":
                        assert rd.tobytes() == ref.tobytes()
                    else:
                        assert np.allclose(rd, ref, rtol=1e-14, atol=1e-300)
                before[inds == j] = x1[inds == j]
            assert x1.tobytes() == before.tobytes()


def test_mh_draws_in_walker_order():
    N, D, seed = 37, 3, 0xAB
    for draw in ("uniform", "normal"):
        cap = Capture(lambda s, c, d: (d[:, :D].clone(), torch.zeros(s.shape[0], dtype=torch.float64,
                                                                      device=s.device)), N, D, 2 * D + 1)
        s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=seed,
                                       moves=moves.MHMove(moves.CudaGraphProposal(cap, ndraws=2 * D + 1, draw=draw)))
        for step in (0, 3):
            x1 = _run_from_minus_inf(s, _p0(N, D), step)
            ref = graph_draws(seed, step, 0, N, draw, 2 * D + 1)[:, :D]
            if draw == "uniform":
                assert x1.tobytes() == ref.tobytes()
            else:
                assert np.allclose(x1, ref, rtol=1e-14, atol=1e-300)


# ---- twins --------------------------------------------------------------------------------------------------------
def _torch_iso(x):
    return -0.5 * (x * x).sum(dim=1)


MODELS = {
    "iso": lambda D: models.GaussianIso(),
    "dense": lambda D: models.GaussianDense(np.eye(D) + 0.3),
    "rosen": lambda D: models.Rosenbrock(),
    "bounded": lambda D: models.Bounded(models.GaussianIso(), -np.full(D, 1.5), np.full(D, 1.5)),
    "host": lambda D: models.HostFunction(lambda x: -0.5 * np.sum(x * x, axis=1), vectorize=True),
    "cuda_blobs": lambda D: models.CudaArrayFunction(
        lambda x: (lambda t: (_torch_iso(t), t[:, 0] * 2.0))(_t(x)), blobs_dtype=np.float64),
}


def _graph_model(D):
    from test_gpu_graph_function import Capture as LpCapture, iso_columns

    return models.CudaGraphFunction(LpCapture(iso_columns, D))


@pytest.mark.parametrize("model", sorted(MODELS) + ["graph_fn"])
@pytest.mark.parametrize("kind", ["stretch", "de", "mh"])
def test_twins_models(model, kind):
    N, D = 41, 5
    mk = _graph_model if model == "graph_fn" else MODELS[model]
    pair = move_pair(kind, N, D, **({} if kind == "mh" else {"nsplits": 3}))
    a, g = _twins(N, D, lambda: mk(D), lambda k: pair[k])
    for s in (a, g):
        s.run_mcmc(_p0(N, D, scale=0.5), 12, skip_initial_state_check=True)
    _assert_same(a, g)
    if model == "cuda_blobs":
        assert a.get_blobs().tobytes() == g.get_blobs().tobytes()
    assert g._engine.last_kernel_variant() == "user_move where=graph"


@pytest.mark.parametrize("D", [1, 33, 257])
def test_twins_dimensions_and_strides(D):
    N = 2 * D + 7
    for strided in (False, True):
        pair = move_pair("stretch", N, D, strided=strided, live_dangerously=True)
        a, g = _twins(N, D, models.GaussianIso, lambda k: pair[k])
        for s in (a, g):
            s.run_mcmc(_p0(N, D, scale=0.3), 6, skip_initial_state_check=True)
        _assert_same(a, g)


def _mixed(N, D, pairs):
    return lambda k: [(moves.StretchMove(), 0.3), (pairs[0][k], 0.25), (moves.DEMove(), 0.15), (pairs[1][k], 0.2),
                      (moves.GaussianMove(np.full(D, 0.2), mode="sequential"), 0.1)]


@pytest.mark.parametrize("device_backend", [False, True])
@pytest.mark.parametrize("path", ["run_mcmc", "sample", "resume"])
def test_twins_mixed_schedule_backends_and_paths(device_backend, path):
    N, D = 40, 4
    pairs = [move_pair("stretch", N, D), move_pair("mh", N, D)]
    kw = {"backend": emcee_b200.DeviceBackend()} if device_backend else {}
    a, g = _twins(N, D, models.Rosenbrock, _mixed(N, D, pairs), **kw)
    for s in (a, g):
        if path == "run_mcmc":
            s.run_mcmc(_p0(N, D, scale=0.3), 30, thin_by=3, skip_initial_state_check=True)
        elif path == "sample":
            for _ in s.sample(_p0(N, D, scale=0.3), iterations=20, thin_by=2, skip_initial_state_check=True):
                pass
        else:
            s.run_mcmc(_p0(N, D, scale=0.3), 7, skip_initial_state_check=True)
            s.run_mcmc(None, 5)
            s.run_mcmc(None, 9)
    _assert_same(a, g)
    if path == "resume":  # several calls equal one call
        one = emcee_b200.EnsembleSampler(N, D, models.Rosenbrock(), moves=_mixed(N, D, [move_pair("stretch", N, D),
                                                                                      move_pair("mh", N, D)])(1),
                                         seed=11, **({"backend": emcee_b200.DeviceBackend()} if device_backend else {}))
        one.run_mcmc(_p0(N, D, scale=0.3), 21, skip_initial_state_check=True)
        assert one.get_chain().tobytes() == g.get_chain().tobytes()
        assert one.get_log_prob().tobytes() == g.get_log_prob().tobytes()
        assert one.random_state == g.random_state
        assert one._engine.get_state()[0].tobytes() == g._engine.get_state()[0].tobytes()


def test_twins_large_dense():
    N, D = 65536, 128
    rng = np.random.default_rng(1)
    A = rng.standard_normal((D, D)) / np.sqrt(D)
    model = lambda: models.GaussianDense(A @ A.T + np.eye(D))  # noqa: E731
    pair = move_pair("stretch", N, D)
    a, g = _twins(N, D, model, lambda k: pair[k])
    for s in (a, g):
        s.run_mcmc(_p0(N, D, scale=0.5), 3, store=False, skip_initial_state_check=True)
    _assert_same(a, g, stored=False)


# ---- errors -------------------------------------------------------------------------------------------------------
class BadAt(object):
    """The stretch proposal, except that call number `at` (one call per half-step, counted on the device) returns
    `value` in row 3 of q, or in every factor when `where == "f"`."""

    def __init__(self, at, value, where="q"):
        self.at, self.value, self.where = at, value, where
        self.n = torch.zeros((), dtype=torch.int64, device="cuda")

    def reset(self):
        self.n.zero_()

    def __call__(self, s, c, d):
        q, f = stretch(s, c, d)
        self.n.add_(1)
        hit = self.n == self.at
        if self.where == "f":
            return q, torch.where(hit, torch.full_like(f, self.value), f)
        r = torch.arange(q.shape[0], device=q.device)[:, None]
        e = torch.arange(q.shape[1], device=q.device)[None, :]
        return torch.where(hit & (r == 3) & (e == 1), torch.full_like(q, self.value), q), f


def _bad_pair(N, D, at, value, where="q"):
    fa, fg = BadAt(at, value, where), BadAt(at, value, where)
    eager = EagerTwin(fa, 2, randomize_split=False)
    fa.reset()
    cap = Capture(fg, N, D, 2)
    return eager, moves.CudaGraphRedBlueMove(cap, ndraws=2, randomize_split=False)


@pytest.mark.parametrize("value,match", [(np.inf, "infinite"), (np.nan, "NaN")])
@pytest.mark.parametrize("case", ["store", "thin3", "device_thin3", "nostore", "mixed"])
def test_nonfinite_proposal_leaves_what_the_twin_leaves(value, match, case):
    N, D, at = 40, 4, 23  # call 23: step 11, split 0 with a pure two-split schedule
    pair = _bad_pair(N, D, at, value)
    if case == "mixed":
        sched = lambda k: [(moves.StretchMove(), 0.4), (pair[k], 0.6)]  # noqa: E731
    else:
        sched = lambda k: pair[k]  # noqa: E731
    kw = {"backend": emcee_b200.DeviceBackend()} if case == "device_thin3" else {}
    a, g = _twins(N, D, models.GaussianIso, sched, seed=0xE1, **kw)
    msgs = []
    for s in (a, g):
        with pytest.raises(ValueError, match=match) as e:
            if case == "nostore":
                s.run_mcmc(_p0(N, D), 40, store=False, skip_initial_state_check=True)
            else:
                s.run_mcmc(_p0(N, D), 40, thin_by=1 if case in ("store", "mixed") else 3,
                           skip_initial_state_check=True)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]
    _assert_same(a, g, stored=case != "nostore")
    assert a._engine.get_rng() == g._engine.get_rng()


def _mixed_err(k, pair, D):
    return [(moves.StretchMove(), 0.3), (moves.DEMove(), 0.1), (moves.WalkMove(s=3), 0.05),
            (moves.GaussianMove(np.full(D, 0.2), mode="sequential"), 0.1), (pair[k], 0.45)]


@pytest.mark.parametrize("value,match", [(np.inf, "infinite"), (np.nan, "NaN")])
@pytest.mark.parametrize("model", ["iso", "dense", "host"])
@pytest.mark.parametrize("case", ["nostore", "thin3", "device_thin3", "sample_thin3"])
def test_error_in_a_mixed_schedule_freezes_the_state(value, match, model, case):
    """Built-in steps after a captured proposal's error must not move the state before the host sees the error:
    with store=False or thin_by=3 no stored step synchronises between the failing half-step and the built-in steps
    the schedule picks after it."""
    N, D, at = 40, 4, 7
    pair = _bad_pair(N, D, at, value)
    mk = {"iso": models.GaussianIso, "dense": lambda: models.GaussianDense(np.eye(D) + 0.3),
          "host": lambda: models.HostFunction(lambda x: -0.5 * np.sum(x * x, axis=1), vectorize=True)}[model]
    kw = {"backend": emcee_b200.DeviceBackend()} if case == "device_thin3" else {}
    a, g = _twins(N, D, mk, lambda k: _mixed_err(k, pair, D), seed=0xE2, **kw)
    msgs = []
    for s in (a, g):
        with pytest.raises(ValueError, match=match) as e:
            if case == "nostore":
                s.run_mcmc(_p0(N, D), 60, store=False, skip_initial_state_check=True)
            elif case == "sample_thin3":
                for _ in s.sample(_p0(N, D), iterations=20, thin_by=3, skip_initial_state_check=True):
                    pass
            else:
                s.run_mcmc(_p0(N, D), 20, thin_by=3, skip_initial_state_check=True)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]
    _assert_same(a, g, stored=case != "nostore")
    assert a._engine.get_rng() == g._engine.get_rng()
    assert a._moves[3].index == g._moves[3].index  # the sequential GaussianMove's dimension


def test_nan_factors_reject_without_error():
    N, D = 40, 4
    pair = _bad_pair(N, D, 5, np.nan, where="f")
    a, g = _twins(N, D, models.GaussianIso, lambda k: pair[k], seed=3)
    for s in (a, g):
        s.run_mcmc(_p0(N, D), 10, skip_initial_state_check=True)
    _assert_same(a, g)


CAPTURES = []


def module_capture(ns, counts):
    """A picklable capture function (module level)."""
    CAPTURES.append((ns, counts))
    return Capture(stretch, 24, 3, 2)(ns, counts)


def test_pickle_recaptures_and_continues():
    N, D = 24, 3
    del CAPTURES[:]
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=5,
                                   moves=moves.CudaGraphRedBlueMove(module_capture, ndraws=2, nsplits=3))
    assert CAPTURES == [(8, (8, 8))]
    s.run_mcmc(_p0(N, D), 6, skip_initial_state_check=True)
    t = pickle.loads(pickle.dumps(s))
    assert CAPTURES == [(8, (8, 8))] * 2
    s.run_mcmc(None, 6)
    t.run_mcmc(None, 6)
    assert s.get_chain().tobytes() == t.get_chain().tobytes()
    assert s.random_state == t.random_state
    assert s._engine.last_kernel_name() == "user_move"
    assert s._engine.last_kernel_variant() == "user_move where=graph"
