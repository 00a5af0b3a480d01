"""Box priors (``models.Bounded`` -> ``eb_model_set_bounds``) on every log-probability path.

A bounded model's log-probability is the model's value inside the closed box ``lower <= x <= upper`` and exactly
``-inf`` outside.  Every kernel that evaluates a model applies the box where it holds the proposal:

* golden vectors of the unmodified reference on bounded targets (``tests/golden/bounded/``), stepwise and bulk;
* every row of the ``test_gpu_variants`` cell table under a binding box with some walkers starting outside, against
  the oracle (``oracle.bounded.Bounded``), with the cell asserted; a box that never binds (+-1e300) must give the
  bits of the unbounded run;
* dense Gaussian: dense_dmma at several D with and without a mean, grouped launches, the CUDA-core kernel;
  WalkMove and GaussianMove (the generic kernel's precomputed proposals);
* ``compute_log_prob`` on the generic and the dense_dmma log-prob kernels: rows on a bound, one ulp outside, +-0.0
  bounds, one-sided bounds, row counts 8k +- 1;
* the reference's errors for non-finite coordinates, none for rows outside the box;
* statistics: a diagonal Gaussian in a box on dense_dmma has truncated-normal marginals, a half-normal on a
  tma_rows register cell has half-normal ones (error bars from independent replica ensembles).
"""
import os

import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T
from oracle.bounded import Bounded as OracleBounded

from gpu_util import device_model, device_moves, move_rows_from_oracle
from test_bounds_host import bounded_names, load_bounded
from test_gpu_variants import CELLS
from util import oracle_target

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu


def _sampler(g_or_model, N, D, dmoves, seed, lower=None, upper=None):
    m = g_or_model if lower is None else models.Bounded(g_or_model, lower, upper)
    return emcee_b200.EnsembleSampler(N, D, m, moves=dmoves, seed=seed)


# ---- 1. golden vectors of the reference ------------------------------------------------------------------------
def _golden_tols(g):
    # as test_gpu_parity._tols
    kinds = set(g["moves"][:, 0].astype(int))
    if kinds == {0}:
        return True, 0.0, 0.0
    if 2 in kinds:
        return False, 1e-5, 1e-6
    if kinds & {3, 4}:
        return False, 1e-9, 1e-11
    return False, 1e-12, 1e-12


def _golden_sampler(g):
    inner = device_model(str(g["model_kind"]), g=g)
    return _sampler(inner, int(g["nwalkers"]), int(g["ndim"]), device_moves(g["moves"], g), int(g["seed"]),
                    g["model_lower"], g["model_upper"])


@pytest.mark.parametrize("name", bounded_names())
def test_bounded_golden_stepwise(name):
    g = load_bounded(name)
    s = _golden_sampler(g)
    exact, rtol, atol = _golden_tols(g)
    lp0, _ = s.compute_log_prob(g["p0"])
    assert np.array_equal(np.isneginf(lp0), np.isneginf(g["lp0"]))
    np.testing.assert_allclose(lp0, g["lp0"], rtol=1e-12, atol=1e-12)
    prev = np.zeros(int(g["nwalkers"]))
    for k, state in enumerate(s.sample(g["p0"], iterations=g["chain"].shape[0], skip_initial_state_check=True)):
        now = s.backend.accepted.copy()
        assert np.array_equal((now - prev) > 0.5, g["accepted"][k]), (name, k)
        prev = now
        if exact:
            assert np.array_equal(state.coords, g["chain"][k]), (name, k)
        else:
            np.testing.assert_allclose(state.coords, g["chain"][k], rtol=rtol, atol=atol, err_msg="%s %d" % (name, k))
        assert np.array_equal(np.isneginf(state.log_prob), np.isneginf(g["log_prob"][k])), (name, k)
        np.testing.assert_allclose(state.log_prob, g["log_prob"][k], rtol=max(rtol, 1e-12), atol=max(10 * atol, 1e-12))


@pytest.mark.parametrize("name", bounded_names())
def test_bounded_golden_run_mcmc_bulk(name):
    g = load_bounded(name)
    s = _golden_sampler(g)
    exact, rtol, atol = _golden_tols(g)
    s.run_mcmc(g["p0"], g["chain"].shape[0], skip_initial_state_check=True)
    if exact:
        assert np.array_equal(s.get_chain(), g["chain"])
    else:
        np.testing.assert_allclose(s.get_chain(), g["chain"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(s.get_log_prob(), g["log_prob"], rtol=max(rtol, 1e-12), atol=max(10 * atol, 1e-12))
    assert np.array_equal(s.backend.accepted, g["accepted"].sum(axis=0))


def test_bounded_sampler_pickles_with_its_box():
    import pickle

    g = load_bounded("bounded_halfnormal_iso_32x5")
    s = _golden_sampler(g)
    s2 = pickle.loads(pickle.dumps(s))
    lp, _ = s2.compute_log_prob(g["p0"])
    assert np.array_equal(np.isneginf(lp), np.isneginf(g["lp0"]))


# ---- 2. every kernel cell under a box ----------------------------------------------------------------------------
def _box_and_p0(target, p0, seed):
    """A box that binds in every parameter (about 1 sd below and 1.3 sd above the centre of p0), p0 clipped into
    it, and three walkers moved outside."""
    c, sd = float(np.mean(p0)), float(np.std(p0))
    lo = np.full(p0.shape[1], c - sd)
    hi = np.full(p0.shape[1], c + 1.3 * sd)
    p = np.clip(p0, lo + 1e-3 * sd, hi - 1e-3 * sd)
    N, D = p.shape
    for k, r in enumerate((0, N // 3, N - 1)):
        p[r, (r + k) % D] = hi[0] + 0.5 * sd if k % 2 else lo[0] - 0.5 * sd
    return lo, hi, p


def _check(s, o, last, stretch_only, snooker, target):
    if stretch_only:
        assert np.array_equal(last.coords, o.coords)
    else:
        tol = 1e-6 if snooker else 1e-11
        np.testing.assert_allclose(last.coords, o.coords, rtol=tol, atol=tol)
    assert np.array_equal(np.isneginf(last.log_prob), np.isneginf(o.log_prob))
    np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-6 if snooker else 1e-11, atol=1e-9 if snooker else 1e-11)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    np.testing.assert_allclose(last.log_prob, target(last.coords), rtol=1e-11, atol=1e-11)


def _bounded_row(kind, N, D, omoves, nsteps, seed, dmodel=None, target=None, p0=None, options=(), dmoves=None,
                 stretch_only=None):
    """Run (model, box) on the device and on the oracle; then the never-binding box against the unbounded model."""
    if target is None:
        target, p0 = T.make_config(kind, N, D)
    if dmodel is None:
        dmodel = device_model(kind, target=target)
    if dmoves is None:
        dmoves = device_moves(move_rows_from_oracle(omoves))
    if stretch_only is None:
        stretch_only = all(m.kind == "stretch" for m, _ in omoves)
    snooker = any(m.kind == "snooker" for m, _ in omoves)
    lo, hi, pb = _box_and_p0(target, p0, seed)
    bt = OracleBounded(target, lo, hi)
    o = rb.OracleSampler(N, D, bt, omoves, seed=seed)
    o.set_state(pb)
    assert np.isneginf(o.log_prob).sum() == 3
    o.run(nsteps)
    s = _sampler(dmodel, N, D, dmoves, seed, lo, hi)
    for k, v in options:
        s._engine.set_option(k, v)
    last = s.run_mcmc(pb, nsteps, store=False, skip_initial_state_check=True)
    _check(s, o, last, stretch_only, snooker, bt)
    variant = s._engine.last_kernel_variant()

    # a box that never binds: the bits of the unbounded model, on the same cell
    runs = []
    for box in ((None, None), (-1e300, 1e300)):
        r = _sampler(dmodel, N, D, dmoves, seed, *box)
        for k, v in options:
            r._engine.set_option(k, v)
        lr = r.run_mcmc(p0, nsteps, store=False, skip_initial_state_check=True)
        runs.append((lr.coords.copy(), lr.log_prob.copy(), r._engine.naccepted(), r._engine.last_kernel_variant()))
    for a, b in zip(runs[0], runs[1]):
        assert np.array_equal(a, b)
    assert runs[0][3] == variant
    return s, variant


@pytest.mark.parametrize("model,N,D,omoves,variant", [c[1:] for c in CELLS], ids=[c[0] for c in CELLS])
def test_bounded_tma_cell(model, N, D, omoves, variant):
    _, got = _bounded_row(model, N, D, omoves, 4, seed=0xB0 + N + D)
    assert got == variant


@pytest.mark.parametrize("own", [1, 0])
def test_bounded_own_reg_options(own):
    _, got = _bounded_row("rosenbrock", 334, 32, [(rb.Stretch(), 1.0)], 4, seed=0xB1, options=(("tma_own_reg", own),))
    assert got == "tma_rows R=8 epl=8 own_reg=%d warps=16" % own


def _dense(D, mean, N, seed=0):
    base, p0 = T.make_config("gauss_dense", N, D)
    mu = np.linspace(-0.7, 1.3, D) if mean else None
    t = T.GaussDense(base.icov, mu)
    return t, (p0 if mu is None else p0 + mu)


DMMA_CASES = [(8, False), (24, True), (64, False), (64, True), (120, True), (128, False), (128, True)]


@pytest.mark.parametrize("D,mean", DMMA_CASES, ids=["D%d%s" % (d, "-mean" if m else "") for d, m in DMMA_CASES])
def test_bounded_dense_dmma(D, mean):
    N = 8 * 37 * 2 + 2  # partial tiles
    t, p0 = _dense(D, mean, N)
    s, variant = _bounded_row("gauss_dense", N, D, [(rb.Stretch(), 1.0)], 5, seed=0xD0 + D, target=t, p0=p0)
    assert variant.startswith("dense_dmma nhalf_max=1 ")
    # stored log-probabilities are those of compute_log_prob at the same coordinates
    c, lp = s._engine.get_state()
    assert np.array_equal(s.compute_log_prob(c)[0], lp)


@pytest.mark.parametrize("group", [2, 3])
def test_bounded_dense_dmma_grouped(group):
    D, N = 64, 1026
    t, p0 = _dense(D, True, N)
    _, variant = _bounded_row("gauss_dense", N, D, [(rb.Stretch(), 1.0)], 6, seed=0xD7, target=t, p0=p0,
                              options=(("dmma_group", group),))
    assert variant.startswith("dense_dmma nhalf_max=%d " % group)


@pytest.mark.parametrize("D,options", [(20, ()), (136, ()), (64, (("dense_dmma", 0),))], ids=["D20", "D136", "D64-dmma-off"])
def test_bounded_dense_cuda_core(D, options):
    N = 301
    t, p0 = _dense(D, True, N)
    G = 4
    while G < 32 and G * 4 < D:
        G *= 2
    _, variant = _bounded_row("gauss_dense", N, D, [(rb.Stretch(), 1.0)], 5, seed=0xDC + D, target=t, p0=p0,
                              options=options)
    assert variant == "generic G=%d" % G


def test_bounded_debug_taps_generic():
    _, variant = _bounded_row("ring", 301, 32, [(rb.Stretch(), 1.0)], 4, seed=0xDB, options=(("debug_taps", 1),))
    assert variant == "generic G=8"


@pytest.mark.parametrize(
    "kind,D,omove,dmove,variant",
    [
        ("rosenbrock", 4, rb.Walk(s=None), moves.WalkMove(), "walk"),
        ("ring", 8, rb.Walk(s=6), moves.WalkMove(s=6), "walk"),
        ("gauss_iso", 5, rb.Gaussian(0.3, "vector", None), moves.GaussianMove(0.3), "gaussian"),
        ("rosenbrock", 6, rb.Gaussian(0.05, "random", 2.0), moves.GaussianMove(0.05, mode="random", factor=2.0),
         "gaussian"),
    ],
    ids=["walk-all-rosen", "walk-s6-ring", "gauss-vector-iso", "gauss-random-rosen"],
)
def test_bounded_walk_gaussian(kind, D, omove, dmove, variant):
    N = 64
    # the WalkMove / GaussianMove tolerances of test_gpu_parity (normals through device log / sincos)
    target, p0 = T.make_config(kind, N, D)
    lo, hi, pb = _box_and_p0(target, p0, 0)
    bt = OracleBounded(target, lo, hi)
    o = rb.OracleSampler(N, D, bt, [(omove, 1.0)], seed=0xAA + D)
    o.set_state(pb)
    o.run(20)
    s = _sampler(device_model(kind, target=target), N, D, [(dmove, 1.0)], 0xAA + D, lo, hi)
    last = s.run_mcmc(pb, 20, store=False, skip_initial_state_check=True)
    assert s._engine.last_kernel_variant() == variant
    np.testing.assert_allclose(last.coords, o.coords, rtol=1e-9, atol=1e-11)
    assert np.array_equal(np.isneginf(last.log_prob), np.isneginf(o.log_prob))
    np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-9, atol=1e-11)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))


# ---- 3. compute_log_prob on each path ----------------------------------------------------------------------------
LP_PATHS = [
    ("iso-D5", "gauss_iso", 5, ()),
    ("ring-D32", "ring", 32, ()),
    ("rosen-D64", "rosenbrock", 64, ()),
    ("dense-D37-generic", "gauss_dense", 37, ()),
    ("dense-D64-dmma", "gauss_dense", 64, ()),
    ("dense-D128-dmma", "gauss_dense", 128, ()),
    ("dense-D64-dmma-off", "gauss_dense", 64, (("dense_dmma", 0),)),
]


def _edge_rows(lo, hi, M, rng):
    """M rows inside [lo, hi] (finite parts), with single coordinates set exactly on a bound, one ulp outside,
    or to -0.0 / +0.0."""
    D = lo.size
    flo = np.where(np.isfinite(lo), lo, -2.0)
    fhi = np.where(np.isfinite(hi), hi, 2.0)
    x = flo + (fhi - flo) * rng.uniform(0.05, 0.95, (M, D))
    for r in range(M):
        k = rng.integers(D)
        pick = r % 7
        if pick == 0 and np.isfinite(lo[k]):
            x[r, k] = lo[k]
        elif pick == 1 and np.isfinite(hi[k]):
            x[r, k] = hi[k]
        elif pick == 2 and np.isfinite(lo[k]):
            x[r, k] = np.nextafter(lo[k], -np.inf)
        elif pick == 3 and np.isfinite(hi[k]):
            x[r, k] = np.nextafter(hi[k], np.inf)
        elif pick == 4:
            x[r, k] = -0.0
        elif pick == 5:
            x[r, k] = 0.0
    return x


@pytest.mark.parametrize("kind,D,options", [c[1:] for c in LP_PATHS], ids=[c[0] for c in LP_PATHS])
def test_bounded_compute_log_prob(kind, D, options):
    rng = np.random.default_rng(D)
    target, _ = T.make_config(kind, 64, D)
    dmodel = device_model(kind, target=target)
    # finite two-sided, one-sided both ways, +-0.0 bounds, and infinite parameters
    lo = rng.uniform(-1.5, -0.2, D)
    hi = rng.uniform(0.2, 1.5, D)
    lo[::5] = 0.0
    hi[1::5] = -0.0
    lo[1::5] = -1.0
    lo[2::5] = -np.inf
    hi[3::5] = np.inf
    lo[4::7], hi[4::7] = -np.inf, np.inf
    bt = OracleBounded(target, lo, hi)
    plain = _sampler(dmodel, 64, D, None, 1)
    boxed = _sampler(dmodel, 64, D, None, 1, lo, hi)
    for s in (plain, boxed):
        for k, v in options:
            s._engine.set_option(k, v)
    for M in (1, 7, 8, 9, 63, 64, 65, 1023):
        x = _edge_rows(lo, hi, M, rng)
        ref_in = bt.inbox(x)
        lp_plain, _ = plain.compute_log_prob(x)
        lp_box, _ = boxed.compute_log_prob(x)
        assert np.array_equal(np.isneginf(lp_box), ~ref_in), M
        assert np.array_equal(lp_box[ref_in], lp_plain[ref_in]), M  # bit-identical inside
        if M >= 63:
            assert 0 < ref_in.sum() < M


def test_bounded_compute_log_prob_kernels_agree():
    """dense_dmma's log-prob kernel (the path that stores log-probs) and its CUDA-core fallback mark the same rows."""
    D = 64
    t, _ = _dense(D, True, 64)
    lo, hi = np.full(D, -0.5), np.full(D, 2.0)
    rng = np.random.default_rng(5)
    x = _edge_rows(lo, hi, 257, rng)
    a = _sampler(device_model("gauss_dense", target=t), 64, D, None, 1, lo, hi)
    b = _sampler(device_model("gauss_dense", target=t), 64, D, None, 1, lo, hi)
    b._engine.set_option("dense_dmma", 0)
    la, lb = a.compute_log_prob(x)[0], b.compute_log_prob(x)[0]
    assert np.array_equal(np.isneginf(la), np.isneginf(lb))
    np.testing.assert_allclose(la, lb, rtol=1e-11, atol=1e-11)


def test_set_bounds_clears_and_model_set_resets():
    D = 8
    e = _sampler(models.GaussianIso(), 32, D, None, 1)._engine
    x = np.full((4, D), 2.0)
    assert np.isfinite(e.compute_log_prob(x)).all()
    e.set_bounds(np.full(D, -1.0), np.full(D, 1.0))
    assert np.isneginf(e.compute_log_prob(x)).all()
    e.set_bounds(None, None)
    assert np.isfinite(e.compute_log_prob(x)).all()
    e.set_bounds(np.full(D, -1.0), np.full(D, 1.0))
    e.set_model("gauss_iso", np.zeros(0))
    assert np.isfinite(e.compute_log_prob(x)).all()
    for lo, hi in ((np.full(D, np.nan), np.ones(D)), (np.ones(D), np.ones(D)), (np.ones(D), np.zeros(D))):
        with pytest.raises(ValueError):
            e.set_bounds(lo, hi)


# ---- 4. errors ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,D", [("gauss_iso", 5), ("gauss_dense", 64), ("ring", 32)])
def test_bounded_nonfinite_coordinates_still_raise(kind, D):
    target, _ = T.make_config(kind, 64, D)
    s = _sampler(device_model(kind, target=target), 64, D, None, 1, np.full(D, -1.0), np.full(D, 1.0))
    x = np.zeros((9, D))
    x[3, 1] = 5.0  # outside: no error
    assert np.isneginf(s.compute_log_prob(x)[0][3])
    for bad, msg in ((np.inf, "infinite"), (-np.inf, "infinite"), (np.nan, "NaN")):
        y = x.copy()
        y[4, 0] = bad
        with pytest.raises(ValueError, match=msg):
            s.compute_log_prob(y)
    y = x.copy()
    y[4, 0], y[6, 2] = np.inf, np.nan  # both: the infinite one first (ensemble.py:476-479)
    with pytest.raises(ValueError, match="infinite"):
        s.compute_log_prob(y)


def test_out_of_box_row_never_raises_nan():
    """An indefinite precision matrix gives inf - inf = NaN at huge coordinates; outside the box the value is -inf
    and nothing is raised, while the unbounded model raises the reference's NaN error."""
    icov = np.diag([1.0, -1.0])
    x = np.array([[1e200, 1e200], [0.5, 0.5]])
    plain = _sampler(models.GaussianDense(icov), 8, 2, None, 1)
    with pytest.raises(ValueError, match="NaN"):
        plain.compute_log_prob(x)
    boxed = _sampler(models.GaussianDense(icov), 8, 2, None, 1, -1.0, 1.0)
    lp = boxed.compute_log_prob(x)[0]
    assert np.isneginf(lp[0]) and lp[1] == 0.0


# ---- 5. statistics -----------------------------------------------------------------------------------------------
def _replica_moments(make_sampler, draw_p0, mean, var, R=16, nstore=200, thin=10, nsig=6.0):
    """Per-parameter chain mean and second moment about the exact mean, against the exact mean and variance.

    Ensemble moves couple the walkers and these targets mix slowly near the walls, so an error bar from the
    per-walker autocorrelation time is too small: the numpy oracle, which steps exactly as the reference does,
    lands 8 such sigmas from the exact half-normal moments.  The error bar here is the spread of R independent
    ensembles (different seeds and initial draws)."""
    est = []
    for r in range(R):
        s = make_sampler(r)
        s.run_mcmc(draw_p0(r), nstore, thin_by=thin, skip_initial_state_check=True)
        chain = s.get_chain()
        assert np.isfinite(s.get_log_prob()).all()
        est.append((chain.mean(axis=(0, 1)), ((chain - mean) ** 2).mean(axis=(0, 1))))
        variant = s._engine.last_kernel_variant()
        s._engine.close()
    est = np.array(est)  # [R, 2, D]
    m, sd = est.mean(axis=0), est.std(axis=0, ddof=1) / np.sqrt(R)
    dev = np.abs(m - np.stack([mean, var])) / sd
    assert np.all(dev < nsig), "max dev/sigma: mean %.2f, variance %.2f" % (dev[0].max(), dev[1].max())
    return variant


def test_truncated_gaussian_on_dense_dmma():
    from scipy import stats

    D, N = 64, 512
    sig = np.linspace(0.5, 2.0, D)
    lo, hi = -np.full(D, 1.0), np.linspace(0.3, 3.0, D)
    dist = stats.truncnorm(lo / sig, hi / sig, scale=sig)
    icov = np.diag(1.0 / sig**2)
    variant = _replica_moments(
        lambda r: _sampler(models.GaussianDense(icov), N, D, None, 0x7C00 + r, lo, hi),
        lambda r: dist.rvs(size=(N, D), random_state=np.random.default_rng(1100 + r)),  # stationary from the start
        dist.mean(), dist.var())
    assert variant.startswith("dense_dmma")


def test_half_normal_on_tma_register_cell():
    D, N = 32, 512
    variant = _replica_moments(
        lambda r: _sampler(models.GaussianIso(), N, D, None, 0x7D00 + r, 0.0, np.inf),
        lambda r: np.abs(np.random.default_rng(1200 + r).standard_normal((N, D))),
        np.full(D, np.sqrt(2.0 / np.pi)), np.full(D, 1.0 - 2.0 / np.pi))
    assert variant == "tma_rows R=8 epl=8 own_reg=1 warps=16"
