"""User log-probability functions on the GPU (``models.HostFunction`` / ``models.CudaArrayFunction``):
the engine calls the function once per half-step with one split's proposals, between the propose and
the accept launches of the generic kernel.

* golden vectors of the unmodified reference (and the bounded ones), with the numpy target as the
  function: accept masks bit-exact, coordinates at the parity tolerances, every stored log_prob the
  bits the function returned for the accepted proposal;
* the call sequence equals the oracle's ``compute_log_prob`` inputs;
* the proposals the function sees are the bits the fused device-model kernel proposes;
* accept edges (+-inf), the timing of NaN and non-finite-parameter errors, user exceptions and resuming;
* map / pool / args / kwargs, every storage path, pickling, re-entrancy, refusals, CUDA-array mode.
"""
import pickle

import numpy as np
import pytest

from gpu_util import device_moves, single_step_tol
from oracle import redblue as rb
from oracle import targets as T
from oracle.bounded import Bounded as OracleBounded
from test_bounds_host import bounded_names, load_bounded
from util import golden_names, load_golden, oracle_moves, oracle_target

import emcee_b200
from emcee_b200 import _lib, models, moves

pytestmark = pytest.mark.gpu

LP_RTOL, LP_ATOL = 1e-12, 1e-12


class Recorder(object):
    """The target as a vectorised function that keeps every input and output."""

    def __init__(self, target):
        self.target = target
        self.inputs, self.outputs = [], []

    def __call__(self, x):
        self.inputs.append(np.array(x, copy=True))
        out = np.asarray(self.target(x), dtype=np.float64)
        self.outputs.append(out.copy())
        return out


def _tols(g):
    kinds = set(g["moves"][:, 0].astype(int))
    if kinds == {0}:
        return True, 0.0, 0.0
    if 2 in kinds:
        return False, 1e-5, 1e-6
    if kinds & {3, 4}:
        return False, 1e-9, 1e-11
    return False, 1e-12, 1e-12


def _golden(case):
    kind, name = case.split(":")
    if kind == "g":
        g = load_golden(name)
        return g, oracle_target(g)
    g = load_bounded(name)
    return g, OracleBounded(oracle_target(g), g["model_lower"], g["model_upper"])


def _sampler(g, fn, **kw):
    return emcee_b200.EnsembleSampler(int(g["nwalkers"]), int(g["ndim"]), fn, moves=device_moves(g["moves"], g),
                                      seed=int(g["seed"]), **kw)


def _check_lp_is_returned(rec, first_call, coords, lp, acc, prev_lp):
    """Accepted walkers hold the bits the function returned for their proposal, the others their old lp."""
    returned = {}
    for x, out in zip(rec.inputs[first_call:], rec.outputs[first_call:]):
        for row, v in zip(x, out):
            returned[row.tobytes()] = v
    for w in range(len(lp)):
        if acc[w]:
            assert lp[w].tobytes() == returned[coords[w].tobytes()].tobytes(), w
        else:
            assert lp[w].tobytes() == prev_lp[w].tobytes(), w


CASES = ["g:" + n for n in golden_names()] + ["b:" + n for n in bounded_names()]


@pytest.mark.parametrize("case", CASES)
def test_golden_single_steps(case):
    g, target = _golden(case)
    rec = Recorder(target)
    s = _sampler(g, models.HostFunction(rec, vectorize=True))
    eng = s._engine
    exact = _tols(g)[0]
    step_tol = single_step_tol(g)
    lp_tol = step_tol if step_tol > 1e-11 else LP_RTOL  # a rank-deficient Walk: its log-probs follow its coordinates
    prev_c, prev_lp = g["p0"], g["lp0"]
    for k in range(g["chain"].shape[0]):
        for m in s._moves:
            if hasattr(m, "index"):
                m.index = k % int(g["ndim"])
        eng.set_state(prev_c, prev_lp)
        eng.set_rng(int(g["seed"]), k)
        first = len(rec.inputs)
        acc = eng.step(s._schedule(), 1)
        coords, lp = eng.get_state()
        assert eng.last_kernel_name() == "callback"
        assert np.array_equal(acc, g["accepted"][k]), (case, k)
        if exact:
            assert np.array_equal(coords, g["chain"][k]), (case, k)
        else:
            np.testing.assert_allclose(coords, g["chain"][k], rtol=step_tol, atol=step_tol)
        np.testing.assert_allclose(lp, g["log_prob"][k], rtol=lp_tol, atol=max(lp_tol, LP_ATOL))
        _check_lp_is_returned(rec, first, coords, lp, acc, np.asarray(prev_lp, dtype=np.float64))
        prev_c, prev_lp = g["chain"][k], g["log_prob"][k]


@pytest.mark.parametrize("case", CASES)
def test_golden_run_mcmc_bulk(case):
    g, target = _golden(case)
    rec = Recorder(target)
    s = _sampler(g, models.HostFunction(rec, vectorize=True))
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
    # every stored log_prob is a value the function returned for that walker's coordinates
    returned = {}
    for x, out in zip(rec.inputs, rec.outputs):
        for row, v in zip(x, out):
            returned[row.tobytes()] = v.tobytes()
    for k in range(nsteps):
        for w in range(chain.shape[1]):
            assert lps[k, w].tobytes() == returned[chain[k, w].tobytes()]


@pytest.mark.parametrize("name", golden_names())
def test_call_sequence_matches_the_oracle(name):
    g = load_golden(name)
    orec, drec = Recorder(oracle_target(g)), Recorder(oracle_target(g))
    o = rb.OracleSampler(int(g["nwalkers"]), int(g["ndim"]), orec, oracle_moves(g), seed=int(g["seed"]))
    o.set_state(g["p0"])
    nsteps = min(6, g["chain"].shape[0])
    o.run(nsteps)
    s = _sampler(g, models.HostFunction(drec, vectorize=True))
    s.run_mcmc(g["p0"], nsteps, store=False, skip_initial_state_check=True)
    exact = _tols(g)[0]
    assert len(drec.inputs) == len(orec.inputs)
    assert drec.inputs[0].shape[0] == int(g["nwalkers"])  # the initial state: every walker
    for k, (a, b) in enumerate(zip(drec.inputs, orec.inputs)):
        assert a.shape == b.shape, (name, k)
        if exact:
            assert np.array_equal(a, b), (name, k)
        else:
            np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-11)


# ---- the proposals are the fused kernel's ------------------------------------------------------------------------
def _identity_case(move, N, D, taps, seed=0x1D):
    p0 = np.random.default_rng(N + D).standard_normal((N, D))
    lp0 = np.full(N, -np.inf)  # every proposal is accepted, so the state holds them all
    ref = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=move, seed=seed)
    rec = Recorder(T.GaussIso(D))
    cb = emcee_b200.EnsembleSampler(N, D, models.HostFunction(rec, vectorize=True), moves=move, seed=seed)
    for s in (ref, cb):
        if taps:
            s._engine.set_option("debug_taps", 1)
    for k in (0, 5):
        got = []
        for s in (ref, cb):
            s._engine.set_state(p0, lp0)
            s._engine.set_rng(seed, k)
            acc = s._engine.step(s._schedule(), 1)
            assert acc.all()
            got.append((s._engine.get_state()[0], s._engine.debug_taps() if taps else None))
        (xa, ta), (xb, tb) = got
        assert np.array_equal(xa, xb), k
        if taps:
            for key in ("partners", "scalar", "u_accept", "active"):
                assert np.array_equal(ta[key], tb[key]), key
            # the last call holds the last split's proposals, in ascending walker order
            assert np.array_equal(rec.inputs[-1], xa[ta["active"]])
            assert np.all(np.diff(ta["active"]) > 0)
        # every row the function saw in this step is one walker's proposal
        d = move.descriptor()
        ncalls = 1 if d["kind"] == "gaussian" else int(d["nsplits"])
        assert sum(len(x) for x in rec.inputs[-ncalls:]) == N
        assert {r.tobytes() for x in rec.inputs[-ncalls:] for r in x} == {r.tobytes() for r in xa}

    # the accept phase: a function returning the device model's own bits (eb_compute_log_prob runs the same
    # model code) from a finite start must give the device-model step exactly -- the accept uniforms, the strict
    # `>` and the update, for Walk / Gaussian too, whose taps the engine does not record
    lpdev = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=seed)._engine
    cb2 = emcee_b200.EnsembleSampler(N, D, models.HostFunction(lpdev.compute_log_prob, vectorize=True), moves=move,
                                     seed=seed)
    if taps:
        cb2._engine.set_option("debug_taps", 1)
    lp_start = lpdev.compute_log_prob(p0)
    for k in (0, 5):
        got = []
        for s in (ref, cb2):
            s._engine.set_state(p0, lp_start)
            s._engine.set_rng(seed, k)
            acc = s._engine.step(s._schedule(), 1)
            got.append((acc,) + s._engine.get_state() + (s._engine.debug_taps() if taps else None,))
        (acc_a, xa, la, ta), (acc_b, xb, lb, tb) = got
        assert np.array_equal(acc_a, acc_b) and np.array_equal(xa, xb) and np.array_equal(la, lb), k
        if taps:
            for key in ("partners", "scalar", "u_accept", "active"):
                assert np.array_equal(ta[key], tb[key]), key


def _full_cov(D):
    a = np.random.default_rng(D).standard_normal((D, D))
    return 0.01 * (a @ a.T) + 0.1 * np.eye(D)


IDENTITY = [
    ("stretch", lambda P, D: moves.StretchMove(nsplits=P), True),
    ("de", lambda P, D: moves.DEMove(nsplits=P), True),
    ("snooker", lambda P, D: moves.DESnookerMove(), True),
    ("walk", lambda P, D: moves.WalkMove(nsplits=P), False),
    ("walk_subset", lambda P, D: moves.WalkMove(s=4, nsplits=P), False),
    ("gauss_scalar", lambda P, D: moves.GaussianMove(0.3), False),
    ("gauss_diag_random", lambda P, D: moves.GaussianMove(np.linspace(0.1, 0.4, D), mode="random", factor=1.5), False),
    ("gauss_sequential", lambda P, D: moves.GaussianMove(np.linspace(0.1, 0.4, D), mode="sequential"), False),
    ("gauss_full", lambda P, D: moves.GaussianMove(_full_cov(D)), False),
]


@pytest.mark.parametrize("D", [1, 33, 257])
@pytest.mark.parametrize("P", [2, 3, 5])
@pytest.mark.parametrize("kind,make,taps", IDENTITY, ids=[c[0] for c in IDENTITY])
def test_proposals_identical_to_the_device_model(kind, make, taps, P, D):
    if kind.startswith("gauss") and P != 2:
        pytest.skip("GaussianMove has no splits")
    if kind == "snooker" and P != 2:
        pytest.skip("DESnookerMove always uses 4 splits")
    if kind == "walk_subset" and D > 64:
        pytest.skip("WalkMove helper subsets are limited to ndim <= 64")
    N = max(2 * D + 1, 41) | 1  # odd
    _identity_case(make(P, D), N, D, taps)


# ---- accept edges (red_blue.py:96-101) -----------------------------------------------------------------------------
@pytest.mark.parametrize(
    "lp_old, lp_new, accepted",
    [(0.0, -np.inf, False), (-np.inf, -3.0, True), (0.0, np.inf, True), (np.inf, np.inf, False), (np.inf, 1.0, False)],
)
def test_accept_edges(lp_old, lp_new, accepted):
    N, D = 32, 3
    p0 = np.random.default_rng(1).standard_normal((N, D))
    s = emcee_b200.EnsembleSampler(N, D, models.HostFunction(lambda x: np.full(len(x), lp_new), vectorize=True),
                                   seed=3)
    s._engine.set_state(p0, np.full(N, lp_old))
    acc = s._engine.step(s._schedule(), 1)
    coords, lp = s._engine.get_state()
    assert np.all(acc == accepted)
    if accepted:
        assert np.all(lp == lp_new) and not np.array_equal(coords, p0)
    else:
        assert np.array_equal(coords, p0) and np.array_equal(lp, np.full(N, lp_old))


# ---- error timing ------------------------------------------------------------------------------------------------
class FailAt(object):
    """GaussIso, except that call number `call` (0 = the initial state) returns NaN or raises."""

    def __init__(self, D, call, what):
        self.t, self.call, self.what, self.n, self.armed = T.GaussIso(D), call, what, 0, True
        self.inputs = []

    def __call__(self, x):
        self.inputs.append(np.array(x, copy=True))
        n, self.n = self.n, self.n + 1
        out = self.t(x)
        if self.armed and n == self.call:
            self.armed = False
            if self.what == "nan":
                out = out.copy()
                out[len(out) // 2] = np.nan
            else:
                raise self.what("user failure at call %d" % n)
        return out


class UserError(Exception):
    pass


N_ERR, D_ERR, SEED_ERR = 40, 4, 0xE1


def _err_sampler(fn, backend=None):
    return emcee_b200.EnsembleSampler(N_ERR, D_ERR, models.HostFunction(fn, vectorize=True),
                                      moves=moves.StretchMove(randomize_split=False), seed=SEED_ERR, backend=backend)


def _p0():
    return np.random.default_rng(7).standard_normal((N_ERR, D_ERR))


def _twin(nsteps):
    s = _err_sampler(T.GaussIso(D_ERR))
    s.run_mcmc(_p0(), nsteps, skip_initial_state_check=True)
    return s


@pytest.mark.parametrize("k,j", [(3, 1), (2, 0)])
def test_nan_stops_at_its_half_step(k, j):
    s = _err_sampler(FailAt(D_ERR, 1 + 2 * k + j, "nan"))
    with pytest.raises(ValueError, match="Probability function returned NaN"):
        s.run_mcmc(_p0(), 6, skip_initial_state_check=True)
    tw = _twin(k + 1)
    assert s.backend.iteration == k
    assert np.array_equal(s.get_chain(), tw.get_chain()[:k]) and np.array_equal(s.get_log_prob(), tw.get_log_prob()[:k])
    assert s._engine.get_rng()[1] == k
    coords, _ = s._engine.get_state()
    before = tw.get_chain()[k - 1] if k else _p0()
    after = tw.get_chain()[k]
    even, odd = np.arange(0, N_ERR, 2), np.arange(1, N_ERR, 2)  # unshuffled splits: walker w is in split w % 2
    if j == 1:
        assert np.array_equal(coords[even], after[even]) and np.array_equal(coords[odd], before[odd])
    else:
        assert np.array_equal(coords, before)


def test_nonfinite_proposal_raises_before_the_call():
    p0 = _p0()
    p0[0] = 1e308
    p0[1] = -1e308
    rec = Recorder(T.GaussIso(D_ERR))
    s = _err_sampler(rec)
    with pytest.raises(ValueError, match="At least one parameter value was"):
        s.run_mcmc(p0, 5, skip_initial_state_check=True)
    assert all(np.isfinite(x).all() for x in rec.inputs)


@pytest.mark.parametrize("device_backend", [False, True])
@pytest.mark.parametrize("path", ["run_mcmc", "sample"])
def test_user_exception_propagates_and_resume_is_exact(path, device_backend):
    k, j, n = 3, 1, 7
    fn = FailAt(D_ERR, 1 + 2 * k + j, UserError)
    s = _err_sampler(fn, backend=emcee_b200.DeviceBackend() if device_backend else None)
    with pytest.raises(UserError, match="user failure"):
        if path == "run_mcmc":
            s.run_mcmc(_p0(), n, skip_initial_state_check=True)
        else:
            for _ in s.sample(_p0(), iterations=n, skip_initial_state_check=True):
                pass
    tw = _twin(n)
    assert s.backend.iteration == k
    assert np.array_equal(s.get_chain(), tw.get_chain()[:k])
    assert np.array_equal(s.get_log_prob(), tw.get_log_prob()[:k])
    tk = _twin(k)
    assert np.array_equal(s.backend.accepted, tk.backend.accepted)
    assert s.backend.random_state == ("philox4x32-10", SEED_ERR, k)
    s.run_mcmc(s.get_last_sample(), n - k)
    assert np.array_equal(s.get_chain(), tw.get_chain()) and np.array_equal(s.get_log_prob(), tw.get_log_prob())
    assert np.array_equal(s.backend.accepted, tw.backend.accepted)


# ---- map, pool, args, inputs -----------------------------------------------------------------------------------
class RecordingPool(object):
    def __init__(self):
        self.calls = 0

    def map(self, f, it):
        self.calls += 1
        return list(map(f, it))


def _shifted(x, c, scale=1.0):
    d = np.asarray(x) - c
    return -0.5 * scale * np.sum(d * d, axis=-1)


def _run(fn, n=6, **kw):
    s = emcee_b200.EnsembleSampler(32, 5, fn, seed=0x3A, **kw)
    s.run_mcmc(np.random.default_rng(2).standard_normal((32, 5)), n, skip_initial_state_check=True)
    return s


def test_map_and_pool_equal_vectorize():
    ref = _run(models.HostFunction(_shifted, vectorize=True, args=(0.25,), kwargs={"scale": 2.0}))
    pool = RecordingPool()
    for fn in (models.HostFunction(_shifted, args=(0.25,), kwargs={"scale": 2.0}),
               models.HostFunction(_shifted, pool=pool, args=(0.25,), kwargs={"scale": 2.0})):
        s = _run(fn)
        assert np.array_equal(s.get_chain(), ref.get_chain()) and np.array_equal(s.get_log_prob(), ref.get_log_prob())
    assert pool.calls == 1 + 6 * 2  # initial state + two splits per step


def test_input_is_fresh():
    kept = []

    def mutating(x):
        kept.append(x)
        out = T.GaussIso(5)(x)
        x[:] = 1e6  # the function owns x
        return out

    ref = _run(models.HostFunction(T.GaussIso(5), vectorize=True))
    s = _run(models.HostFunction(mutating, vectorize=True))
    assert np.array_equal(s.get_chain(), ref.get_chain())
    assert len({id(x) for x in kept}) == len(kept) and all(np.all(x == 1e6) for x in kept)


# ---- storage paths -----------------------------------------------------------------------------------------------
def _fn():
    return models.HostFunction(T.GaussIso(5), vectorize=True)


def _p0s():
    return np.random.default_rng(4).standard_normal((32, 5))


@pytest.mark.parametrize("how", ["thin_by", "thin", "store_false", "device_backend", "moments", "sample_thin_by"])
def test_storage_paths_match_backend(how):
    ref = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
    ref.run_mcmc(_p0s(), 12, skip_initial_state_check=True)
    chain, lps = ref.get_chain(), ref.get_log_prob()
    if how == "device_backend":
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B, backend=emcee_b200.DeviceBackend())
        s.run_mcmc(_p0s(), 12, skip_initial_state_check=True)
        assert np.array_equal(s.get_chain(), chain) and np.array_equal(s.get_log_prob(), lps)
        assert np.array_equal(s.backend.accepted, ref.backend.accepted)
    elif how == "thin_by":
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
        s.run_mcmc(_p0s(), 4, thin_by=3, skip_initial_state_check=True)
        assert np.array_equal(s.get_chain(), chain[2::3]) and np.array_equal(s.get_log_prob(), lps[2::3])
    elif how == "sample_thin_by":
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
        for _ in s.sample(_p0s(), iterations=4, thin_by=3, skip_initial_state_check=True):
            pass
        assert np.array_equal(s.get_chain(), chain[2::3])
    elif how == "thin":
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
        s.run_mcmc(_p0s(), 12, thin=3, skip_initial_state_check=True)
        assert np.array_equal(s.get_chain(), chain[2::3])
    elif how == "store_false":
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
        last = s.run_mcmc(_p0s(), 12, store=False, skip_initial_state_check=True)
        assert np.array_equal(last.coords, chain[-1]) and np.array_equal(last.log_prob, lps[-1])
    else:
        s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=0x5B)
        s.enable_moments(1)
        s.run_mcmc(_p0s(), 12, store=False, skip_initial_state_check=True)
        mean, cov, n = s.moments()
        flat = chain.reshape(-1, 5)
        assert n == flat.shape[0]
        np.testing.assert_allclose(mean, flat.mean(0), rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(cov, np.cov(flat, rowvar=False), rtol=1e-10, atol=1e-13)


# ---- pickling, re-entrancy, compute_log_prob, refusals -----------------------------------------------------------
def test_pickled_sampler_continues_identically():
    a = emcee_b200.EnsembleSampler(32, 5, models.HostFunction(_shifted, args=(0.5,), pool=RecordingPool()), seed=9)
    a.run_mcmc(_p0s(), 4, skip_initial_state_check=True)
    b = pickle.loads(pickle.dumps(a))
    assert b.log_prob_fn.pool is None
    a.run_mcmc(None, 5)
    b.run_mcmc(None, 5)
    assert np.array_equal(a.get_chain(), b.get_chain()) and np.array_equal(a.get_log_prob(), b.get_log_prob())


def test_reentrant_call_is_refused():
    holder = {}

    def fn(x):
        holder["s"].compute_log_prob(x)
        return T.GaussIso(5)(x)

    s = emcee_b200.EnsembleSampler(32, 5, models.HostFunction(fn, vectorize=True), seed=1)
    holder["s"] = s
    with pytest.raises(RuntimeError, match="inside a log-probability callback"):
        s.compute_log_prob(_p0s())


def test_compute_log_prob():
    rec = Recorder(T.GaussIso(5))
    s = emcee_b200.EnsembleSampler(32, 5, models.HostFunction(rec, vectorize=True), seed=1)
    x = np.random.default_rng(5).standard_normal((3, 4, 5))
    lp, blobs = s.compute_log_prob(x)
    assert blobs is None and lp.dtype == np.float64 and lp.shape == (3, 4)
    assert np.array_equal(lp, T.GaussIso(5)(x)) and rec.inputs[-1].shape == (12, 5)
    for bad, msg in ((np.inf, "infinite"), (np.nan, "NaN")):
        y = x.copy()
        y[1, 2, 3] = bad
        n = len(rec.inputs)
        with pytest.raises(ValueError, match=msg):
            s.compute_log_prob(y)
        assert len(rec.inputs) == n  # the function never saw the row
    nan_fn = models.HostFunction(lambda x: np.full(len(x), np.nan), vectorize=True)
    with pytest.raises(ValueError, match="Probability function returned NaN"):
        emcee_b200.EnsembleSampler(32, 5, nan_fn, seed=1).compute_log_prob(x)


def test_refusals():
    s = emcee_b200.EnsembleSampler(32, 5, _fn(), seed=1)
    with pytest.raises(NotImplementedError):
        s.attach(None)
    with pytest.raises(TypeError):
        models.Bounded(_fn(), -1.0, 1.0)
    with pytest.raises(NotImplementedError):
        s._engine.set_bounds(-np.ones(5), np.ones(5))
    blobs = emcee_b200.EnsembleSampler(32, 5, models.HostFunction(lambda x: (-0.5 * np.sum(x * x), 1.0)), seed=1)
    with pytest.raises(NotImplementedError, match="blobs"):
        blobs.run_mcmc(_p0s(), 2, skip_initial_state_check=True)
    wrong = emcee_b200.EnsembleSampler(32, 5, models.HostFunction(lambda x: np.zeros(len(x) + 1), vectorize=True),
                                       seed=1)
    with pytest.raises(ValueError, match="shape"):
        wrong.run_mcmc(_p0s(), 2, skip_initial_state_check=True)


def test_kernel_name_and_variant():
    s = _run(_fn(), n=2)
    assert s._engine.last_kernel_name() == "callback"
    assert s._engine.last_kernel_variant() == "callback G=4 where=host"


# ---- CUDA-array mode ---------------------------------------------------------------------------------------------
def _torch():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("torch has no CUDA")
    return torch


def _iso_columns_np(x):
    lp = np.zeros(x.shape[0])
    for j in range(x.shape[1]):
        lp = lp + (x[:, j] * x[:, j]) * -0.5
    return lp


class V3Result(object):
    """A torch result re-exported with interface version 3 and the stream its last write was enqueued on."""

    def __init__(self, t, stream):
        self.t = t
        cai = dict(t.__cuda_array_interface__)
        cai.update(version=3, stream=stream.cuda_stream or 1)
        self.__cuda_array_interface__ = cai


SLEEP_CYCLES = 20_000_000  # ~10 ms: the final write of the result lands long after the function returns


def _torch_iso(torch, mode, sleep):
    """The column loop of _iso_columns_np in torch.  mode: "current" (torch's current stream, an interface v2
    result that names no stream), "side" (a side stream, a strided v2 view, no hand-back to the current stream),
    "v3" (a side stream, named in a v3 interface).  With `sleep`, the stream sleeps before the result's final
    write, so an engine that does not wait for it reads stale memory."""
    stream = torch.cuda.Stream() if mode != "current" else None

    def body(rows):
        x = torch.as_tensor(rows, device="cuda")
        lp = torch.zeros(x.shape[0], dtype=torch.float64, device="cuda")
        for j in range(x.shape[1]):
            lp = lp + (x[:, j] * x[:, j]) * -0.5
        x.zero_()  # the rows are the function's scratch copy: overwriting them changes nothing
        if sleep:
            torch.cuda._sleep(SLEEP_CYCLES)
        if mode == "current":
            return lp * 1.0
        buf = torch.full((2 * x.shape[0],), float("nan"), dtype=torch.float64, device="cuda")
        buf[::2] = lp
        return buf[::2] if mode == "side" else V3Result(buf[::2], stream)

    def f(rows):
        if stream is None:
            return body(rows)
        with torch.cuda.stream(stream):
            return body(rows)

    return f


@pytest.mark.parametrize("mode", ["current", "side", "v3"])
def test_cuda_array_function_waits_for_its_result(mode):
    torch = _torch()
    N, D = 64, 7
    p0 = np.random.default_rng(8).standard_normal((N, D))
    mv = [(moves.StretchMove(), 0.5), (moves.DEMove(), 0.3), (moves.WalkMove(), 0.2)]
    host = emcee_b200.EnsembleSampler(N, D, models.HostFunction(_iso_columns_np, vectorize=True), moves=mv, seed=11)
    dev = emcee_b200.EnsembleSampler(N, D, models.CudaArrayFunction(_torch_iso(torch, mode, True)), moves=mv, seed=11)
    host.run_mcmc(p0, 10, skip_initial_state_check=True)
    dev.run_mcmc(p0, 10, skip_initial_state_check=True)
    assert dev._engine.last_kernel_variant().endswith("where=device")
    assert np.array_equal(dev.get_chain(), host.get_chain())
    assert np.array_equal(dev.get_log_prob(), host.get_log_prob())
    assert np.array_equal(dev.backend.accepted, host.backend.accepted)


def test_cuda_array_function_large_rows():
    """32 MiB of rows per split: torch reads them on its own stream as soon as the function starts."""
    torch = _torch()
    N, D = 16384, 128
    p0 = np.random.default_rng(9).standard_normal((N, D))
    host = emcee_b200.EnsembleSampler(N, D, models.HostFunction(_iso_columns_np, vectorize=True), seed=12)
    dev = emcee_b200.EnsembleSampler(N, D, models.CudaArrayFunction(_torch_iso(torch, "current", False)), seed=12)
    a = host.run_mcmc(p0, 3, store=False, skip_initial_state_check=True)
    b = dev.run_mcmc(p0, 3, store=False, skip_initial_state_check=True)
    assert np.array_equal(a.coords, b.coords) and np.array_equal(a.log_prob, b.log_prob)


def test_cuda_array_function_numpy_result_and_errors():
    _torch()
    dev = emcee_b200.EnsembleSampler(32, 5, models.CudaArrayFunction(lambda rows: np.zeros(rows.shape[0])), seed=2)
    lp, _ = dev.compute_log_prob(_p0s())
    assert np.array_equal(lp, np.zeros(32))
    bad = emcee_b200.EnsembleSampler(32, 5, models.CudaArrayFunction(lambda rows: np.zeros(3)), seed=2)
    with pytest.raises(ValueError, match="shape"):
        bad.compute_log_prob(_p0s())
