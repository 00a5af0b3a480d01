"""Launch counts and kernel names of every path the step driver dispatches, other than the dense Gaussian stretch
run test_gpu_variants models step by step.

Each case runs one stepping call on a fresh engine (fewer than 64 steps, so exactly one split-table build) and
checks ``last_step_timing()[1]``, ``last_kernel_name()`` and ``last_kernel_variant()`` against counts written out
per path:

* a device-model half-step: one generic or tma_rows launch per split;
* WalkMove: per split the shift, the moment sums (two), the factorisation and the shared proposal (five) when every
  walker draws from the whole complement, one subset proposal with a helper subset; then the accept;
* GaussianMove: the proposal and the accept, plus the shared shift of a full covariance;
* a user RedBlueMove: per split the gather and the accept; a user MHMove: one accept;
* a log-probability function: per split the propose and the accept launches, the blob select behind every accept
  when the state has blobs;
* moments: two launches per accumulation and the shift once; histograms: one per recorded step, plus one for the
  log-probabilities and one for the parameter pairs; the trace: two per recorded step.
"""
import re

import numpy as np
import pytest
import torch

from oracle import redblue as rb
from test_gpu_variants import LaunchModel
from user_moves_ref import NumpyStretch, WithSetup, gauss_mh

import emcee_b200
from emcee_b200 import DeviceBackend, models, moves

pytestmark = pytest.mark.gpu

N, D, SEED = 48, 5, 0xD41E
TABLE = 1  # the split-table build of the first chunk


def lanes(D):
    g = 4
    while g < 32 and g * 4 < D:
        g <<= 1
    return g


def p0(n=N, d=D):
    return 0.5 * np.random.default_rng(7).standard_normal((n, d))


def lp_rows(x):
    x = np.asarray(x)
    return -0.5 * np.sum(x * x, axis=-1)


def host_fn(blobs=False):
    if blobs:
        return models.HostFunction(lambda x: (float(lp_rows(x)), float(x[0])), blobs_dtype=float)
    return models.HostFunction(lp_rows, vectorize=True)


def device_fn(blobs=False):
    def f(rows):
        x = torch.as_tensor(rows, device="cuda")
        lp = -0.5 * (x * x).sum(1)
        return (lp, torch.stack([x[:, 0], x[:, -1]], dim=1)) if blobs else lp

    return models.CudaArrayFunction(f, blobs_dtype="f8" if blobs else None)


def model(kind, blobs=False):
    if kind == "iso":
        return models.GaussianIso()
    if kind == "host":
        return host_fn(blobs)
    if kind == "device":
        return device_fn(blobs)
    raise ValueError(kind)


def callback_variant(kind):
    return "callback G=%d where=%s" % (lanes(D), kind)


def run(mdl, mv, nsteps, options=(), n=N, d=D, setup=None, **kw):
    s = emcee_b200.EnsembleSampler(n, d, mdl, moves=mv, seed=SEED, **kw.pop("sampler", {}))
    for k, v in options:
        s._engine.set_option(k, v)
    if setup is not None:
        setup(s)
    s.run_mcmc(p0(n, d), nsteps, skip_initial_state_check=True, **kw)
    eng = s._engine
    return s, eng.last_step_timing()[1], eng.last_kernel_name(), eng.last_kernel_variant()


# ---- device models ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mv,P", [(moves.StretchMove(), 2), (moves.StretchMove(nsplits=3), 3), (moves.DEMove(), 2),
                                  (moves.DESnookerMove(), 4)], ids=["stretch", "stretch3", "de", "snooker"])
@pytest.mark.parametrize("store", [False, True])
def test_generic(mv, P, store):
    nsteps, thin_by = 7, 2
    kw = {"thin_by": thin_by} if store else {}
    _, launches, name, variant = run(model("iso"), mv, nsteps, options=[("tma_rows", 0)], store=store, **kw)
    assert launches == TABLE + nsteps * (thin_by if store else 1) * P
    assert name == "generic"
    assert variant == "generic G=%d" % lanes(D)


def test_tma_rows():
    nsteps = 5
    _, launches, name, variant = run(model("iso"), moves.StretchMove(), nsteps, n=256, d=16)
    assert launches == TABLE + nsteps * 2
    assert name == "tma_rows"
    assert re.fullmatch(r"tma_rows R=\d+ epl=\d+ own_reg=[01] warps=\d+", variant), variant


@pytest.mark.parametrize("s_arg", [None, 3], ids=["complement", "subset"])
@pytest.mark.parametrize("P", [2, 3])
def test_walk(s_arg, P):
    nsteps = 6
    _, launches, name, variant = run(model("iso"), moves.WalkMove(s=s_arg, nsplits=P), nsteps)
    propose = 5 if s_arg is None else 1
    assert launches == TABLE + nsteps * P * (propose + 1)
    assert (name, variant) == ("walk", "walk")


@pytest.mark.parametrize("cov,extra", [(0.1, 0), (np.full(D, 0.1), 0), (0.1 * np.eye(D) + 0.01, 1)],
                         ids=["scalar", "diagonal", "full"])
def test_gaussian(cov, extra):
    nsteps = 9
    _, launches, name, variant = run(model("iso"), moves.GaussianMove(cov), nsteps)
    assert launches == TABLE + nsteps * (2 + extra)
    assert (name, variant) == ("gaussian", "gaussian")


# ---- user proposals ---------------------------------------------------------------------------------------------


class DeviceStretch(moves.CudaArrayRedBlueMove):
    """NumpyStretch on rows read through their CUDA-array interface."""

    def __init__(self, **kw):
        self.a, self.setups = 2.0, 0
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        s = torch.as_tensor(s, device="cuda").cpu().numpy()
        c = [torch.as_tensor(x, device="cuda").cpu().numpy() for x in c]
        return NumpyStretch(a=self.a).get_proposal(s, c, random)


class DeviceStretchSetup(DeviceStretch):
    def setup(self, coords):
        torch.as_tensor(coords, device="cuda")
        self.setups += 1


def device_mh(coords, random):
    return gauss_mh(torch.as_tensor(coords, device="cuda").cpu().numpy(), random)


def user_move(where, setup, P):
    if where == "host":
        return (WithSetup if setup else NumpyStretch)(nsplits=P)
    return (DeviceStretchSetup if setup else DeviceStretch)(nsplits=P)


@pytest.mark.parametrize("mdl", ["iso", "host", "device"])
@pytest.mark.parametrize("setup", [False, True], ids=["plain", "setup"])
@pytest.mark.parametrize("where", ["host", "device"])
def test_user_red_blue(where, setup, mdl):
    nsteps, P = 4, 3
    mv = user_move(where, setup, P)
    _, launches, name, variant = run(model(mdl), mv, nsteps)
    assert launches == TABLE + nsteps * P * 2
    assert (name, variant) == ("user_move", "user_move where=%s" % where)
    if setup:
        assert len(mv.setups) == nsteps if where == "host" else mv.setups == nsteps


@pytest.mark.parametrize("mdl", ["iso", "host", "device"])
@pytest.mark.parametrize("where", ["host", "device"])
def test_user_mh(where, mdl):
    nsteps = 5
    prop = moves.HostProposal(gauss_mh) if where == "host" else moves.CudaArrayProposal(device_mh)
    _, launches, name, variant = run(model(mdl), moves.MHMove(prop), nsteps)
    assert launches == TABLE + nsteps
    assert (name, variant) == ("user_move", "user_move where=%s" % where)


@pytest.mark.parametrize("where", ["host", "device"])
def test_user_blobs(where):
    nsteps, P = 3, 2
    _, launches, _, _ = run(model(where, blobs=True), user_move("host", False, P), nsteps)
    assert launches == TABLE + nsteps * P * 3
    _, launches, _, _ = run(model(where, blobs=True), moves.MHMove(moves.HostProposal(gauss_mh)), nsteps)
    assert launches == TABLE + nsteps * 2


# ---- log-probability functions ------------------------------------------------------------------------------------


@pytest.mark.parametrize("blobs", [False, True], ids=["plain", "blobs"])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("mv,P", [(moves.StretchMove(), 2), (moves.DEMove(nsplits=3), 3), (moves.DESnookerMove(), 4)],
                         ids=["stretch", "de", "snooker"])
def test_callback_red_blue(mv, P, where, blobs):
    nsteps = 5
    _, launches, name, variant = run(model(where, blobs), mv, nsteps)
    assert launches == TABLE + nsteps * P * (2 + blobs)
    assert (name, variant) == ("callback", callback_variant(where))


@pytest.mark.parametrize("blobs", [False, True], ids=["plain", "blobs"])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("s_arg", [None, 3], ids=["complement", "subset"])
def test_callback_walk(s_arg, where, blobs):
    nsteps, P = 4, 2
    _, launches, name, variant = run(model(where, blobs), moves.WalkMove(s=s_arg), nsteps)
    propose = 5 if s_arg is None else 1
    assert launches == TABLE + nsteps * P * (propose + 1 + blobs)
    assert (name, variant) == ("callback", callback_variant(where))


@pytest.mark.parametrize("blobs", [False, True], ids=["plain", "blobs"])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("cov,extra", [(0.1, 0), (0.1 * np.eye(D) + 0.01, 1)], ids=["scalar", "full"])
def test_callback_gaussian(cov, extra, where, blobs):
    nsteps = 6
    _, launches, name, variant = run(model(where, blobs), moves.GaussianMove(cov), nsteps)
    assert launches == TABLE + nsteps * (2 + extra + blobs)
    assert (name, variant) == ("callback", callback_variant(where))


# ---- running statistics -------------------------------------------------------------------------------------------


def stat_launches(what, every, nsteps):
    recorded = nsteps // every
    if what == "moments":
        return 2 * recorded + (recorded > 0)
    if what == "hist":
        return recorded
    if what == "hist_lp_pairs":
        return 3 * recorded
    if what == "trace":
        return 2 * recorded
    raise ValueError(what)


def enable(what, every):
    def f(s):
        d = s.ndim
        if what == "moments":
            s.enable_moments(every)
        elif what == "hist":
            s.enable_histograms([(-3.0, 3.0)] * d, bins=8, every=every)
        elif what == "hist_lp_pairs":
            s.enable_histograms([(-3.0, 3.0)] * d, bins=8, every=every, log_prob_range=(-20.0, 0.0),
                                params2d=[0, 2, 4])
        else:
            s.enable_trace(every)

    return f


STATS = ["moments", "hist", "hist_lp_pairs", "trace"]


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("what", STATS)
def test_statistics_generic(what, every):
    nsteps, P = 10, 2
    _, launches, name, _ = run(model("iso"), moves.StretchMove(), nsteps, options=[("tma_rows", 0)],
                               setup=enable(what, every), store=False)
    assert launches == TABLE + nsteps * P + stat_launches(what, every, nsteps)
    assert name == "generic"


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("what", STATS)
def test_statistics_callback_walk(what, every):
    nsteps, P = 7, 2
    _, launches, name, _ = run(model("host", blobs=True), moves.WalkMove(s=3), nsteps, setup=enable(what, every),
                               store=False)
    assert launches == TABLE + nsteps * P * 3 + stat_launches(what, every, nsteps)
    assert name == "callback"


def dense_model(n, d):
    a = np.random.default_rng(3).standard_normal((d, d))
    icov = np.linalg.inv(a @ a.T / d + np.eye(d))
    return models.GaussianDense(icov)


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("what", STATS)
@pytest.mark.parametrize("group", [1, 4])
def test_statistics_dense_dmma(what, every, group):
    # a dense_dmma group ends at every step whose statistics are due, as at a stored step
    n, d, nsteps = 256, 16, 11
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    expect, variant = LaunchModel(n, SEED, sm).call([rb.Stretch()], [1.0], 0, nsteps, group, moments_every=every)
    if what != "moments":
        expect += stat_launches(what, every, nsteps) - stat_launches("moments", every, nsteps)
    _, launches, name, got = run(dense_model(n, d), moves.StretchMove(), nsteps, n=n, d=d,
                                 options=[("dmma_group", group)], setup=enable(what, every), store=False)
    assert launches == expect
    assert (name, got) == ("dense_dmma", variant)


@pytest.mark.parametrize("thin_by", [1, 3])
@pytest.mark.parametrize("group", [1, 4])
@pytest.mark.parametrize("backend", ["host", "device"])
def test_store_dense_dmma(backend, group, thin_by):
    # a stored step ends a dense_dmma group; the store itself is no counted launch
    n, d, nsteps = 256, 16, 4
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    expect, variant = LaunchModel(n, SEED, sm).call([rb.Stretch()], [1.0], 0, nsteps * thin_by, group,
                                                    sync_every=thin_by)
    kw = {"sampler": {"backend": DeviceBackend()}} if backend == "device" else {}
    _, launches, name, got = run(dense_model(n, d), moves.StretchMove(), nsteps, n=n, d=d,
                                 options=[("dmma_group", group)], thin_by=thin_by, **kw)
    assert launches == expect
    assert (name, got) == ("dense_dmma", variant)
