"""User-written proposals on the GPU: ``RedBlueMove`` subclasses overriding ``get_proposal`` (numpy and torch),
``MHMove(HostProposal / CudaArrayProposal)``, against the unmodified reference's golden runs of the same functions
(``tests/golden/user_moves``) and against ``UserOracle`` (the reference's step loop in numpy with the same move
objects and the draw specification, pinned to those golden runs on the CPU):

* accept counts and coordinates bit-exact, device-model log-probabilities to 1e-12, callback ones bit-exact;
* the rows ``get_proposal`` sees equal the reference's boolean-mask gathers;
* torch moves give the numpy move's chain bit for bit, on a side stream and as v3 stream-named results too;
* errors stop at their half-step and ``run_mcmc`` resumes the uninterrupted chain; storage paths agree;
* the statistical gate of the reference for a user stretch and a user MH move.
"""
import pickle

import numpy as np
import pytest
import torch

from oracle import gen_golden_user_moves as gen
from oracle import targets as T
from oracle.bounded import Bounded as OracleBounded
from user_moves_ref import (NumpyDE, NumpyStretch, Recording, UserOracle, WithSetup, gauss_mh, gauss_mh_symmetric,
                            golden_cases, golden_moves, load_case, oracle_moves)

import emcee_b200
from emcee_b200 import DeviceBackend, models, moves

pytestmark = pytest.mark.gpu

SEED = 0x5EED


def device_model(kind, target):
    if kind == "gauss_iso":
        return models.GaussianIso()
    if kind == "gauss_dense":
        return models.GaussianDense(target.icov, target.mean)
    if kind == "rosenbrock":
        return models.Rosenbrock(target.a, target.b)
    if kind == "ring":
        return models.Ring(target.radius, target.sigma)
    raise ValueError(kind)


def make_moves(name, **kw):
    if name == "stretch":
        return [(NumpyStretch(**kw), 1.0)]
    if name == "de":
        return [(NumpyDE(**kw), 1.0)]
    if name == "mh":
        return [(moves.MHMove(moves.HostProposal(gauss_mh)), 1.0)]
    if name == "mix":  # user moves between the built-in ones
        return [(NumpyStretch(**kw), 0.3), (moves.StretchMove(), 0.3), (moves.DEMove(), 0.2),
                (moves.MHMove(moves.HostProposal(gauss_mh)), 0.2)]
    raise ValueError(name)


def run_both(model, target, p0, mv, nsteps, **kw):
    N, D = p0.shape
    s = emcee_b200.EnsembleSampler(N, D, model, moves=mv, seed=SEED)
    s.run_mcmc(p0, nsteps, skip_initial_state_check=True, **kw)
    o = UserOracle(N, D, target, oracle_moves(mv), seed=SEED)
    o.set_state(p0)
    chain = []
    for _ in range(nsteps):
        o.run(1)
        chain.append(o.coords.copy())
    return s, o, np.array(chain)


def check(s, o, chain, exact_lp):
    np.testing.assert_array_equal(s.get_chain(), chain)
    np.testing.assert_array_equal(s.backend.accepted, o.naccepted.astype(np.float64))
    lp = s.get_log_prob()[-1]
    if exact_lp:
        np.testing.assert_array_equal(lp, o.log_prob)
    else:
        np.testing.assert_allclose(lp, o.log_prob, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("how", ["device_model", "host_function"])
@pytest.mark.parametrize("name", golden_cases())
def test_golden(name, how):
    # the unmodified reference's runs of the same user functions (oracle/gen_golden_user_moves.py)
    (name, N, D, kind, spec, nsteps), g = load_case(name)
    target = gen.case_target(kind, D)
    model = device_model(kind, target) if how == "device_model" else models.HostFunction(target, vectorize=True)
    s = emcee_b200.EnsembleSampler(N, D, model, moves=golden_moves(spec), seed=int(g["seed"]))
    prev, k = np.zeros(N), 0
    for _ in s.sample(g["p0"], iterations=nsteps, skip_initial_state_check=True):
        now = s.backend.accepted.copy()
        np.testing.assert_array_equal((now - prev) > 0.5, g["accepted"][k])
        prev, k = now, k + 1
    np.testing.assert_array_equal(s.get_chain(), g["chain"])
    if how == "host_function":
        np.testing.assert_array_equal(s.get_log_prob(), g["log_prob"])
    else:
        np.testing.assert_allclose(s.get_log_prob(), g["log_prob"], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("kind", ["gauss_iso", "gauss_dense", "rosenbrock", "ring"])
@pytest.mark.parametrize("mname", ["stretch", "de", "mh", "mix"])
def test_device_models(kind, mname):
    target, p0 = T.make_config(kind, 48, 6)
    s, o, chain = run_both(device_model(kind, target), target, p0, make_moves(mname), 25)
    check(s, o, chain, False)
    if mname == "mix":  # the last step may have drawn a built-in move
        assert s._engine.last_kernel_name() in ("user_move", "generic", "tma_rows")
    else:
        assert s._engine.last_kernel_name() == "user_move"


@pytest.mark.parametrize("N,D,nsplits,rand", [(37, 3, 2, True), (37, 3, 3, False), (41, 5, 5, True),
                                              (64, 8, 3, True), (33, 4, 2, False)])
def test_splits_and_odd_sizes(N, D, nsplits, rand):
    target, p0 = T.make_config("gauss_iso", N, D)
    mv = make_moves("stretch", nsplits=nsplits, randomize_split=rand)
    s, o, chain = run_both(models.GaussianIso(), target, p0, mv, 20)
    check(s, o, chain, False)
    assert s._engine.last_kernel_variant() == "user_move where=host"


def test_bounded_model():
    target, p0 = T.make_config("gauss_iso", 40, 4)
    lo, hi = -1.5 * np.ones(4), 1.5 * np.ones(4)
    p0 = np.clip(p0, -1.4, 1.4)
    mv = make_moves("mix")
    s, o, chain = run_both(models.Bounded(models.GaussianIso(), lo, hi), OracleBounded(target, lo, hi), p0, mv, 30)
    check(s, o, chain, False)


@pytest.mark.parametrize("blobs", [False, True])
@pytest.mark.parametrize("mname", ["stretch", "mh", "mix"])
def test_host_function(blobs, mname):
    target, p0 = T.make_config("rosenbrock", 40, 4)

    def f(x):
        lp = target(x)
        # with blobs: one (lp, blob) pair per row (ensemble.py:498-547), the blob being the row's lp
        return [(float(v), float(v)) for v in lp] if blobs else lp

    model = models.HostFunction(f, vectorize=True, blobs_dtype=np.float64 if blobs else None)
    s, o, chain = run_both(model, target, p0, make_moves(mname), 20)
    check(s, o, chain, True)
    if blobs:  # every walker's blob is the record of the proposal it holds
        np.testing.assert_array_equal(s.get_blobs(), s.get_log_prob())


def test_rows_seen_equal_boolean_mask_gathers():
    target, p0 = T.make_config("ring", 45, 4)
    rec_e, rec_o = Recording(nsplits=3), Recording(nsplits=3)
    s = emcee_b200.EnsembleSampler(45, 4, models.Ring(target.radius, target.sigma), moves=rec_e, seed=SEED)
    s.run_mcmc(p0, 6, skip_initial_state_check=True, store=False)
    o = UserOracle(45, 4, target, [(rec_o, 1.0)], seed=SEED)
    o.set_state(p0)
    o.run(6)
    assert len(rec_e.calls) == len(rec_o.calls) == 18
    for (s1, c1), (s2, c2) in zip(rec_e.calls, rec_o.calls):
        np.testing.assert_array_equal(s1, s2)
        assert len(c1) == len(c2) == 2
        for a, b in zip(c1, c2):
            np.testing.assert_array_equal(a, b)


def test_setup_sees_each_steps_ensemble():
    target, p0 = T.make_config("gauss_iso", 32, 5)
    m = WithSetup()
    s = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=m, seed=SEED)
    states = [p0]
    for st in s.sample(p0, iterations=5, skip_initial_state_check=True, store=False):
        states.append(st.coords.copy())
    assert len(m.setups) == 5
    for seen, want in zip(m.setups, states[:-1]):
        np.testing.assert_array_equal(seen, want)


# ---- torch moves ---------------------------------------------------------------------------------------------

class V3(object):
    """A CUDA-array result that names its producer's stream (interface v3)."""

    def __init__(self, t, stream):
        self.t = t
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, version=3, stream=stream.cuda_stream)


class TorchStretch(moves.CudaArrayRedBlueMove):
    """NumpyStretch op by op: the draws and zz on the host, the row arithmetic in torch."""

    def __init__(self, how="current", **kw):
        self.a, self.how = 2.0, how
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        S = torch.as_tensor(s, device="cuda")
        Cc = torch.cat([torch.as_tensor(x, device="cuda") for x in c])
        ns, nc, ndim = S.shape[0], Cc.shape[0], S.shape[1]
        zz = ((self.a - 1.0) * random.rand(ns) + 1) ** 2.0 / self.a
        factors = (ndim - 1.0) * np.log(zz)
        rint = random.randint(nc, size=(ns,))
        side = torch.cuda.Stream() if self.how != "current" else torch.cuda.current_stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            torch.cuda._sleep(2_000_000)  # the result is late: the engine must wait for it
            cr = Cc[torch.as_tensor(rint, device="cuda")]
            q = cr - (cr - S) * torch.as_tensor(zz, device="cuda")[:, None]
            f = torch.as_tensor(factors, device="cuda")
        if self.how == "v3":
            return V3(q, side), V3(f, side)
        return q, (f if self.how != "numpy_f" else factors)


def torch_mh(coords, random):
    x = torch.as_tensor(coords, device="cuda")
    noise = torch.as_tensor(0.3 * random.randn(*x.shape), device="cuda")
    return x + noise, torch.as_tensor(0.25 * random.randn(x.shape[0]), device="cuda")


@pytest.mark.parametrize("how", ["current", "side", "v3", "numpy_f"])
def test_torch_move_equals_numpy_move(how):
    target, p0 = T.make_config("gauss_dense", 64, 8)
    model = device_model("gauss_dense", target)
    a = emcee_b200.EnsembleSampler(64, 8, model, moves=[(TorchStretch(how), 1.0)], seed=SEED)
    b = emcee_b200.EnsembleSampler(64, 8, model, moves=[(NumpyStretch(), 1.0)], seed=SEED)
    a.run_mcmc(p0, 12, skip_initial_state_check=True)
    b.run_mcmc(p0, 12, skip_initial_state_check=True)
    np.testing.assert_array_equal(a.get_chain(), b.get_chain())
    np.testing.assert_array_equal(a.get_log_prob(), b.get_log_prob())
    assert a._engine.last_kernel_variant() == "user_move where=device"


def test_torch_mh_equals_numpy_mh_with_callback_model():
    target, p0 = T.make_config("ring", 48, 4)
    f = models.HostFunction(target, vectorize=True)
    a = emcee_b200.EnsembleSampler(48, 4, f, moves=moves.MHMove(moves.CudaArrayProposal(torch_mh)), seed=SEED)
    b = emcee_b200.EnsembleSampler(48, 4, f, moves=moves.MHMove(moves.HostProposal(gauss_mh)), seed=SEED)
    a.run_mcmc(p0, 15, skip_initial_state_check=True)
    b.run_mcmc(p0, 15, skip_initial_state_check=True)
    np.testing.assert_array_equal(a.get_chain(), b.get_chain())
    np.testing.assert_array_equal(a.get_log_prob(), b.get_log_prob())


def test_large_dense_torch_move():
    # the torch move on the GPU against the numpy move it restates in the numpy driver
    N, D, steps = 65536, 128, 3
    target, p0 = T.make_config("gauss_dense", N, D)
    s = emcee_b200.EnsembleSampler(N, D, device_model("gauss_dense", target), moves=TorchStretch("side"), seed=SEED)
    s.run_mcmc(p0, steps, skip_initial_state_check=True)
    o = UserOracle(N, D, target, [(NumpyStretch(), 1.0)], seed=SEED)
    o.set_state(p0)
    o.run(steps)
    np.testing.assert_array_equal(s.get_chain()[-1], o.coords)
    np.testing.assert_array_equal(s.backend.accepted, o.naccepted.astype(np.float64))
    np.testing.assert_allclose(s.get_log_prob()[-1], o.log_prob, rtol=1e-11, atol=1e-9)


# ---- errors, resume, storage --------------------------------------------------------------------------------
class Boom(Exception):
    pass


class FailAt(NumpyStretch):
    def __init__(self, at, **kw):
        super().__init__(**kw)
        self.at, self.n = at, 0

    def get_proposal(self, s, c, random):
        self.n += 1
        if self.n == self.at:
            raise Boom("half-step %d" % self.n)
        return super().get_proposal(s, c, random)


@pytest.mark.parametrize("bulk", [True, False])
def test_exception_stops_at_its_half_step_and_resume_is_exact(bulk):
    target, p0 = T.make_config("gauss_iso", 32, 5)
    n, k = 12, 7
    ref = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=NumpyStretch(), seed=SEED)
    ref.run_mcmc(p0, n, skip_initial_state_check=True)
    m = FailAt(2 * k + 2)  # the second split of step k + 1 (1-based) fails
    s = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=m, seed=SEED)
    with pytest.raises(Boom, match="half-step %d" % (2 * k + 2)):
        if bulk:
            s.run_mcmc(p0, n, skip_initial_state_check=True)
        else:
            for _ in s.sample(p0, iterations=n, skip_initial_state_check=True):
                pass
    assert s.iteration == k
    assert s._engine.get_rng()[1] == k
    np.testing.assert_array_equal(s.get_chain(), ref.get_chain()[:k])
    s.run_mcmc(s.get_last_sample(), n - k, skip_initial_state_check=True)
    np.testing.assert_array_equal(s.get_chain(), ref.get_chain())
    np.testing.assert_array_equal(s.get_log_prob(), ref.get_log_prob())


def test_nonfinite_proposal_raises_before_any_log_prob():
    calls = []

    def f(x):
        calls.append(len(x))
        return -0.5 * np.sum(x * x, axis=1)

    def bad(coords, random):
        q = coords + random.randn(*coords.shape)
        q[3, 1] = np.inf
        return q, np.zeros(len(q))

    target, p0 = T.make_config("gauss_iso", 32, 5)
    for model in (models.GaussianIso(), models.HostFunction(f, vectorize=True)):
        s = emcee_b200.EnsembleSampler(32, 5, model, moves=moves.MHMove(moves.HostProposal(bad)), seed=SEED)
        n0 = len(calls)
        with pytest.raises(ValueError, match="At least one parameter value was infinite"):
            s.run_mcmc(p0, 3, skip_initial_state_check=True)
        assert len(calls) == n0 + (1 if model.__class__ is models.HostFunction else 0)  # only the initial state


def test_nan_factors_are_rejected_not_errors():
    def nanf(coords, random):
        return coords + random.randn(*coords.shape), np.full(len(coords), np.nan)

    target, p0 = T.make_config("gauss_iso", 32, 5)
    s = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=moves.MHMove(moves.HostProposal(nanf)), seed=1)
    s.run_mcmc(p0, 5, skip_initial_state_check=True)
    assert s.backend.accepted.sum() == 0
    np.testing.assert_array_equal(s.get_last_sample().coords, p0)


@pytest.mark.parametrize("backend", ["host", "device"])
def test_store_thin_by_matches_store_false(backend):
    target, p0 = T.make_config("gauss_dense", 64, 6)
    model = device_model("gauss_dense", target)
    mv = make_moves("mix")
    b = DeviceBackend() if backend == "device" else None
    a = emcee_b200.EnsembleSampler(64, 6, model, moves=mv, seed=SEED, backend=b)
    last = a.run_mcmc(p0, 3, thin_by=10, skip_initial_state_check=True)
    c = emcee_b200.EnsembleSampler(64, 6, model, moves=make_moves("mix"), seed=SEED)
    st = p0
    for _ in range(3):
        st = c.run_mcmc(st, 10, store=False, skip_initial_state_check=True)
        np.testing.assert_array_equal(a.get_chain()[_], st.coords)
    np.testing.assert_array_equal(last.coords, st.coords)
    np.testing.assert_array_equal(last.log_prob, st.log_prob)
    # sample() agrees with run_mcmc
    d = emcee_b200.EnsembleSampler(64, 6, model, moves=make_moves("mix"), seed=SEED)
    for st2 in d.sample(p0, iterations=30, skip_initial_state_check=True):
        pass
    np.testing.assert_array_equal(st2.coords, st.coords)


def test_pickled_sampler_continues_the_chain():
    target, p0 = T.make_config("gauss_iso", 32, 5)
    mv = [(NumpyStretch(), 0.5), (moves.MHMove(moves.HostProposal(gauss_mh)), 0.5)]
    a = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=mv, seed=SEED)
    a.run_mcmc(p0, 5, skip_initial_state_check=True)
    b = pickle.loads(pickle.dumps(a))
    a.run_mcmc(None, 5)
    b.run_mcmc(None, 5)
    np.testing.assert_array_equal(a.get_chain(), b.get_chain())


def test_calls_into_the_engine_from_a_proposal_are_refused():
    holder = {}

    def reenter(coords, random):
        holder["s"].compute_log_prob(coords)
        return coords, np.zeros(len(coords))

    target, p0 = T.make_config("gauss_iso", 32, 5)
    s = emcee_b200.EnsembleSampler(32, 5, models.GaussianIso(), moves=moves.MHMove(moves.HostProposal(reenter)))
    holder["s"] = s
    with pytest.raises(RuntimeError, match="inside a user proposal"):
        s.run_mcmc(p0, 1, skip_initial_state_check=True)


# ---- statistics (tests/integration/test_proposal.py:31-102 of the reference) ---------------------------------
def _test_normal(mv, ndim=1, nwalkers=32, nsteps=2000, seed=1234):
    from scipy import stats

    p0 = np.random.RandomState(seed).randn(nwalkers, ndim)
    s = emcee_b200.EnsembleSampler(nwalkers, ndim, models.GaussianIso(), moves=mv, seed=seed)
    s.run_mcmc(p0, nsteps, skip_initial_state_check=True)
    acc = s.acceptance_fraction
    assert np.all((acc < 0.9) * (acc > 0.1)), acc
    samps = s.get_chain(flat=True)
    assert np.all(np.abs(np.mean(samps, axis=0)) < 0.08), "Incorrect mean"
    assert np.all(np.abs(np.std(samps, axis=0) - 1) < 0.05), "Incorrect standard deviation"
    if ndim == 1:
        ks, _ = stats.kstest(samps[:, 0], "norm")
        assert ks < 0.05, "The K-S test failed"


def _test_uniform(mv, nwalkers=32, nsteps=2000, seed=1234):
    # a uniform start on the normal target: the chain must leave [0, 1], i.e. "fail" the uniform K-S test
    from scipy import stats

    rs = np.random.RandomState(seed)
    p0 = rs.rand(nwalkers, 1)
    s = emcee_b200.EnsembleSampler(nwalkers, 1, models.GaussianIso(), moves=mv, seed=seed)
    s.run_mcmc(p0, nsteps, skip_initial_state_check=True)
    acc = s.acceptance_fraction
    assert np.all((acc < 0.9) * (acc > 0.1)), acc
    samps = s.get_chain(flat=True)
    rs.shuffle(samps)
    ks, _ = stats.kstest(samps[::100, 0], "uniform")
    assert ks > 0.1, "The K-S test failed"


def _stat_moves():
    return [NumpyStretch(), moves.MHMove(moves.HostProposal(gauss_mh_symmetric))]


@pytest.mark.parametrize("k", [0, 1], ids=["stretch", "mh"])
@pytest.mark.parametrize("ndim", [1, 3])
def test_normal_target_statistics(k, ndim):
    _test_normal(_stat_moves()[k], ndim=ndim)


@pytest.mark.parametrize("k", [0, 1], ids=["stretch", "mh"])
def test_uniform_start_statistics(k):
    _test_uniform(_stat_moves()[k])
