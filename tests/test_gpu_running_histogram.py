"""Running histograms (``EnsembleSampler.enable_histograms`` / ``histogram`` / ``histogram2d``;
``eb_histograms_config``, ``eb_histograms``) against numpy and against stored twins, compared with
``np.array_equal`` and equal dtypes.

* Golden chains of the reference (stretch, exact on this engine): ``run_mcmc(store=False)`` with ``every`` 1 and 3
  equals ``np.histogram`` / ``np.histogram2d`` of ``g["chain"][every - 1::every]`` and its log-probabilities.
* Twins, one per kernel path: the counting run equals ``get_histogram(thin=every)`` / ``get_histogram2d`` of a
  same-seed run stored into ``Backend()`` and ``DeviceBackend()``; split runs, ``sample(thin_by=3)``, a run that
  stores while it counts, ``iterations=0``.
* Edges: data outside the range and on its last edge, ``bins`` 1 / 4096 and 128 (2-D), float32 range scalars, a
  range narrower than the data.
* Lifecycle and refusals, and 65 536 x 128 on ``dense_dmma``.
"""
import pickle

import numpy as np
import pytest

from gpu_util import golden_sampler
from test_bounds_host import load_bounded
from test_gpu_bounds import _golden_sampler as bounded_golden_sampler
from user_moves_ref import NumpyStretch, gauss_mh
from util import load_golden

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, models, moves
from emcee_b200.dist import Rendezvous

pytestmark = pytest.mark.gpu


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, list):
            assert g == w
            continue
        assert g.dtype == w.dtype and g.shape == w.shape
        assert np.array_equal(g, w)


def _cut(x, lo=10, hi=80, dtype=float):
    """ranges that cut the data (some values outside): percentiles of each column"""
    a, b = np.percentile(x.reshape(-1, x.shape[-1]), [lo, hi], axis=0)
    return [(dtype(u), dtype(v)) for u, v in zip(a, b)]


def _lp_cut(lp, dtype=float):
    """a range of the log-probabilities whose ends lie halfway between two values: the golden log-probabilities
    equal this engine's to about 1e-11 (not bit for bit), so a value on an edge could fall either side"""
    f = np.unique(lp[np.isfinite(lp)])
    k1, k2 = len(f) // 20, len(f) - 2 - len(f) // 20
    return dtype((f[k1] + f[k1 + 1]) / 2), dtype((f[k2] + f[k2 + 1]) / 2)


# ---- golden chains of the reference -----------------------------------------------------------------------------
GOLDEN = ["stretch_iso_32x5", "stretch_dense_mean_96x16", "stretch_ring_80x6", "stretch_iso_odd_37x3",
          "bounded/bounded_stretch_dense_mean_96x16"]


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("name", GOLDEN)
def test_golden(name, every):
    if name.startswith("bounded/"):
        g = load_bounded(name.split("/")[1])
        s = bounded_golden_sampler(g)
    else:
        g = load_golden(name)
        s = golden_sampler(g)
    chain, lp = g["chain"], g["log_prob"]
    D = chain.shape[2]
    rng, lprng = _cut(chain), _lp_cut(lp)
    params = list(range(D))[::-1][: min(D, 6)]
    s.enable_histograms(rng, 20, every, lprng, params, 16)
    s.run_mcmc(g["p0"], chain.shape[0], store=False, skip_initial_state_check=True)
    if "dense" in name:
        assert s._engine.last_kernel_name() == "dense_dmma"
    flat = chain[every - 1 :: every].reshape(-1, D)
    flp = lp[every - 1 :: every].ravel()
    assert s.histogram_count == flat.shape[0]
    want = [np.histogram(flat[:, d], 20, rng[d]) for d in range(D)]
    _same(s.histogram(), (np.array([h for h, _ in want]), np.array([e for _, e in want])))
    _same(s.histogram(name="log_prob"), np.histogram(flp, 20, lprng))
    h2, e2, pairs = s.histogram2d()
    assert pairs == [(params[i], params[j]) for i in range(len(params)) for j in range(i + 1, len(params))]
    for k, (i, j) in enumerate(pairs):
        h, ei, ej = np.histogram2d(flat[:, i], flat[:, j], 16, [rng[i], rng[j]])
        assert h.dtype == h2.dtype and np.array_equal(h2[k], h)
        assert np.array_equal(e2[params.index(i)], ei) and np.array_equal(e2[params.index(j)], ej)


# ---- twins against stored runs ----------------------------------------------------------------------------------
def _cb_iso(x):
    return -0.5 * np.sum(np.square(x), axis=1)


def _torch_iso(rows):
    import torch

    x = torch.as_tensor(rows, device="cuda")
    return (x * x).sum(dim=1) * -0.5


CASES = {
    # name: (N, D, model, moves, expected kernel name)
    "tma_rows": (64, 8, lambda: models.GaussianIso(), None, "tma_rows"),
    "generic": (37, 3, lambda: models.GaussianIso(), None, "generic"),
    "dense_dmma": (96, 16, "dense", None, "dense_dmma"),
    "walk": (48, 4, lambda: models.GaussianIso(), lambda: moves.WalkMove(s=5), "walk"),
    "gaussian": (40, 4, lambda: models.GaussianIso(), lambda: moves.GaussianMove(0.3), "gaussian"),
    "de_snooker": (48, 6, lambda: models.Rosenbrock(),
                   lambda: [(moves.DEMove(), 0.7), (moves.DESnookerMove(), 0.3)], "tma_rows"),
    "host_fn": (32, 5, lambda: models.HostFunction(_cb_iso, vectorize=True), None, "callback"),
    "cuda_array_fn": (32, 5, lambda: models.CudaArrayFunction(_torch_iso), None, "callback"),
    "user_move": (32, 5, lambda: models.GaussianIso(),
                  lambda: [(NumpyStretch(), 0.5), (moves.MHMove(moves.HostProposal(gauss_mh)), 0.5)], None),
}


def _make(case, backend=None, seed=0x4157):
    N, D, model, mv, _ = CASES[case]
    if model == "dense":
        rng = np.random.default_rng(D)
        a = rng.standard_normal((D, D))
        cov = a @ a.T / D + np.eye(D)
        model = lambda: models.GaussianDense(np.linalg.inv(cov), np.linspace(-1, 1, D))  # noqa: E731
    return emcee_b200.EnsembleSampler(N, D, model(), moves=None if mv is None else mv(), seed=seed, backend=backend)


def _p0(case):
    N, D = CASES[case][:2]
    return np.random.default_rng(N * D).standard_normal((N, D)) * 0.5 + 0.1


def _enable(s, case, every, bins=20, bins2=12, f32=False, lp=True, params=True):
    """enable_histograms with ranges that cut the data of a short run of the same case; returns its arguments"""
    D = CASES[case][1]
    ref = _make(case)
    ref.run_mcmc(_p0(case), 12, store=True, skip_initial_state_check=True)
    dt = np.float32 if f32 else float
    cfg = dict(range=_cut(ref.get_chain(), dtype=dt), bins=bins, every=every,
               log_prob_range=_lp_cut(ref.get_log_prob(), dtype=dt) if lp else None,
               params2d=([D - 1, 0, D // 2] if D > 2 else [1, 0]) if params else None, bins2d=bins2)
    s.enable_histograms(**cfg)
    return cfg


def _check_twins(s, case, cfg, total):
    """s counted the first `total` steps from the start; its twins store every step and read thin=every"""
    every = cfg["every"]
    twins = []
    for backend in (Backend(), DeviceBackend()):
        t = _make(case, backend)
        t.run_mcmc(_p0(case), total, skip_initial_state_check=True)
        twins.append(t)
    assert np.array_equal(twins[0].get_chain(), twins[1].get_chain())
    for t in twins:
        _same(s.histogram(), t.get_histogram(cfg["bins"], cfg["range"], thin=every))
        if cfg["log_prob_range"] is not None:
            _same(s.histogram(name="log_prob"),
                  t.get_histogram(cfg["bins"], cfg["log_prob_range"], thin=every, name="log_prob"))
        if cfg["params2d"] is not None:
            _same(s.histogram2d(), t.get_histogram2d(cfg["params2d"], cfg["bins2d"], cfg["range"], thin=every))
    assert s.histogram_count == (total // every) * CASES[case][0]


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("case", list(CASES))
def test_twin_run_mcmc(case, every):
    s = _make(case)
    cfg = _enable(s, case, every)
    calls = (7, 5)  # two calls; the second starts off the cadence when every = 3
    st = _p0(case)
    for n in calls:
        st = s.run_mcmc(st, n, store=False, skip_initial_state_check=True)
    want = CASES[case][4]
    if want is not None:
        assert s._engine.last_kernel_name() == want
    _check_twins(s, case, cfg, sum(calls))


@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma", "host_fn"])
def test_twin_sample_thin_by_and_storing(case):
    """sample(thin_by=3) as a generator, storing into a Backend while counting every step, then iterations=0"""
    s = _make(case)
    cfg = _enable(s, case, 1)
    n = 0
    for _ in s.sample(_p0(case), iterations=4, thin_by=3, skip_initial_state_check=True):
        n += 1
    assert n == 4 and s.iteration == 4
    assert list(s.sample(s.get_last_sample(), iterations=0, skip_initial_state_check=True)) == []
    _check_twins(s, case, cfg, 12)
    # a run that stores while it counts, every 3rd step of 9 into a DeviceBackend: its own chain is what it counted
    s2 = _make(case, DeviceBackend())
    c2 = _enable(s2, case, 3)
    s2.run_mcmc(_p0(case), 3, skip_initial_state_check=True, thin_by=3)
    _same(s2.histogram(), s2.get_histogram(c2["bins"], c2["range"]))
    _same(s2.histogram(name="log_prob"), s2.get_histogram(c2["bins"], c2["log_prob_range"], name="log_prob"))
    _same(s2.histogram2d(), s2.get_histogram2d(c2["params2d"], c2["bins2d"], c2["range"]))


# ---- edge values --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bins,bins2,f32", [(1, 1, False), (4096, 128, False), (20, 128, True), (7, 3, True)])
def test_edges(bins, bins2, f32):
    case = "tma_rows"
    s = _make(case)
    cfg = _enable(s, case, 2, bins=bins, bins2=bins2, f32=f32)
    s.run_mcmc(_p0(case), 8, store=False, skip_initial_state_check=True)
    _check_twins(s, case, cfg, 8)


def test_last_edge_and_narrow_range():
    """a range whose top is the largest value counted (the last edge: counted in the last bin), and one whose
    bottom is the smallest value, against numpy on the twin's stored steps"""
    case = "generic"
    D = CASES[case][1]
    t = _make(case, Backend())
    t.run_mcmc(_p0(case), 6, skip_initial_state_check=True)
    flat = t.get_chain(flat=True)
    rng = [(float(np.percentile(flat[:, d], 40)), float(flat[:, d].max())) for d in range(D)]
    rng[1] = (float(flat[:, 1].min()), float(np.percentile(flat[:, 1], 45)))
    s = _make(case)
    s.enable_histograms(rng, 9, 1, None, [0, 1, 2], 5)
    s.run_mcmc(_p0(case), 6, store=False, skip_initial_state_check=True)
    _same(s.histogram(), t.get_histogram(9, rng))
    _same(s.histogram2d(), t.get_histogram2d([0, 1, 2], 5, rng))
    assert s.histogram()[0][0, -1] >= 1  # the maximum sits on the last edge


def test_float32_top_edge_truncation():
    """float32 range scalars: numpy's norm_denom is the float32 difference, and a value at the top edge gives
    f > bins, truncated into the last bin -- as get_histogram counts it"""
    case = "generic"
    D = CASES[case][1]
    t = _make(case, Backend())
    t.run_mcmc(_p0(case), 5, skip_initial_state_check=True)
    flat = t.get_chain(flat=True)
    rng = [(np.float32(-0.3), np.float32(flat[:, d].max())) for d in range(D)]
    s = _make(case)
    s.enable_histograms(rng, 20)
    s.run_mcmc(_p0(case), 5, store=False, skip_initial_state_check=True)
    try:
        want = t.get_histogram(20, rng)
    except Exception as e:  # noqa: B902 -- numpy's IndexError: the running count raises ValueError on read
        assert isinstance(e, IndexError)
        with pytest.raises(ValueError, match="truncated bin index is above bins"):
            s.histogram()
        return
    _same(s.histogram(), want)


# ---- lifecycle and refusals ------------------------------------------------------------------------------------
def test_lifecycle():
    case = "tma_rows"
    s = _make(case)
    with pytest.raises(RuntimeError, match="not enabled"):
        s.histogram()
    with pytest.raises(RuntimeError, match="not enabled"):
        s.histogram_count
    _enable(s, case, 1, lp=False, params=False)
    with pytest.raises(RuntimeError, match="log_prob_range"):
        s.histogram(name="log_prob")
    with pytest.raises(RuntimeError, match="params2d"):
        s.histogram2d()
    st = s.run_mcmc(_p0(case), 4, store=False, skip_initial_state_check=True)
    assert s.histogram_count == 4 * 64
    # re-enabling zeroes the counts
    _enable(s, case, 2)
    assert s.histogram_count == 0 and not s.histogram()[0].any() and not s.histogram2d()[0].any()
    st = s.run_mcmc(st, 4, store=False)
    assert s.histogram_count == 2 * 64
    # every=0: counts nothing, readable
    _enable(s, case, 0)
    st = s.run_mcmc(st, 3, store=False)
    assert s.histogram_count == 0 and not s.histogram()[0].any()
    # pickling drops the counts
    s2 = pickle.loads(pickle.dumps(s))
    with pytest.raises(RuntimeError, match="not enabled"):
        s2.histogram()
    s2.run_mcmc(st, 2, store=False)
    with pytest.raises(RuntimeError, match="not enabled"):
        s2.histogram2d()
    # a bad range keeps the previous configuration
    with pytest.raises(ValueError, match="need a \\(lo, hi\\) range"):
        s.enable_histograms(None)
    assert s.histogram_count == 0


def test_counting_leaves_the_chain_alone():
    """the same seed with and without counting: the same chain and the same kernel"""
    out = []
    for on in (False, True):
        s = _make("dense_dmma", Backend())
        if on:
            _enable(s, "dense_dmma", 2)
        s.run_mcmc(_p0("dense_dmma"), 10, skip_initial_state_check=True)
        out.append(s)
    assert np.array_equal(out[0].get_chain(), out[1].get_chain())
    assert np.array_equal(out[0].get_log_prob(), out[1].get_log_prob())


def test_sharded_refused_both_ways():
    s = _make("tma_rows")
    _enable(s, "tma_rows", 1)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(Rendezvous())
    s = _make("tma_rows")
    s.attach(Rendezvous())
    with pytest.raises(NotImplementedError, match="sharded"):
        _enable(s, "tma_rows", 1)


def test_oversized_pairs_memory_error():
    """2 048 parameters, all pairs at 128 bins: 2 096 128 * 128^2 * 8 bytes = 275 GB of counts"""
    D = 2048
    s = emcee_b200.EnsembleSampler(2 * D + 2, D, models.GaussianIso(), seed=3)
    with pytest.raises(MemoryError, match="bytes free"):
        s.enable_histograms([(-1, 1)] * D, 10, params2d=list(range(D)), bins2d=128)
    with pytest.raises(RuntimeError, match="not enabled"):
        s.histogram()


# ---- at scale ------------------------------------------------------------------------------------------------------
def test_scale_dense_dmma_65536x128():
    N, D, steps = 65536, 128, 20
    rng = np.random.default_rng(5)
    a = rng.standard_normal((D, D))
    cov = a @ a.T / D + np.eye(D)
    icov = np.linalg.inv(cov)
    p0 = rng.standard_normal((N, D))
    r = [(-4.0, 4.0)] * D
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(icov), seed=9)
    s.enable_histograms(r, 20, 1, (-400.0, -20.0), list(range(16)), 20)
    s.run_mcmc(p0, steps, store=False, skip_initial_state_check=True)
    assert s._engine.last_kernel_name() == "dense_dmma"
    t = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(icov), seed=9, backend=DeviceBackend())
    t.run_mcmc(p0, steps, skip_initial_state_check=True)
    _same(s.histogram(), t.get_histogram(20, r))
    _same(s.histogram(name="log_prob"), t.get_histogram(20, (-400.0, -20.0), name="log_prob"))
    _same(s.histogram2d(), t.get_histogram2d(list(range(16)), 20, r))
    assert s.histogram_count == steps * N
