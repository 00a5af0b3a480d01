"""``DeviceBackend``: the stored chain kept in GPU memory (``eb_chain``), against the host ``Backend``.

* Twin runs: the same seed, model and moves once into ``Backend()`` and once into ``DeviceBackend()`` must give
  equal bits for every read (``get_chain`` / ``get_log_prob`` over a grid of ``discard`` / ``thin`` / ``flat``,
  the last sample, ``accepted``, ``acceptance_fraction``, ``iteration``), driven through ``run_mcmc``, resumes that
  make several segments, ``iterations = 0``, a ``store=False`` run, ``sample(thin_by=3)`` and the deprecated
  ``thin=``; one case per kernel path.
* The reference's golden chains stored into a ``DeviceBackend``, under the comparisons of ``test_gpu_parity`` and
  ``test_gpu_bounds``.
* Autocorrelation read in place (``eb_chain_autocorr``) against the host route, exactly, including a chain wider
  than one FFT slab and longer than one segment.
* Restart through an initialised backend, pickling, and the error contracts.
"""
import pickle

import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T

from gpu_util import device_model, device_moves, move_rows_from_oracle
from test_bounds_host import bounded_names, load_bounded
from test_gpu_bounds import _box_and_p0, _golden_tols
from test_gpu_parity import _tols
from util import golden_names, load_golden

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, autocorr, models, moves

pytestmark = pytest.mark.gpu


# ---- twin runs -------------------------------------------------------------------------------------------------
def _reads_equal(h, d):
    assert d.iteration == h.iteration
    if h.iteration == 0:
        for s in (h, d):
            with pytest.raises(AttributeError, match="store == True"):
                s.get_chain()
        return
    it = h.iteration
    for discard in sorted({0, 1, 3, it // 2, it - 1, it, it + 4}):
        for thin in (1, 2, 3, 7):
            for flat in (False, True):
                kw = dict(discard=discard, thin=thin, flat=flat)
                a, b = h.get_chain(**kw), d.get_chain(**kw)
                assert a.shape == b.shape and np.array_equal(a, b), kw
                a, b = h.get_log_prob(**kw), d.get_log_prob(**kw)
                assert a.shape == b.shape and np.array_equal(a, b), kw
    lh, ld = h.get_last_sample(), d.get_last_sample()
    assert np.array_equal(lh.coords, ld.coords) and np.array_equal(lh.log_prob, ld.log_prob)
    assert lh.random_state == ld.random_state
    assert np.array_equal(h.backend.accepted, d.backend.accepted)
    assert np.array_equal(h.acceptance_fraction, d.acceptance_fraction)
    assert d.get_blobs() is None


def _drive(s, p0):
    """run_mcmc, iterations = 0, store=False, three resumes (three more segments), sample() with thin_by = 3
    and the deprecated thin= on the per-yield path."""
    it0 = s.iteration
    last = s.run_mcmc(p0, 5, skip_initial_state_check=True)
    before = s.get_chain()
    assert s.run_mcmc(last, 0, skip_initial_state_check=True) is None  # nothing yielded, nothing stored
    s.run_mcmc(last, 4, store=False, skip_initial_state_check=True)
    assert np.array_equal(s.get_chain(), before) and s.iteration == it0 + 5
    s.run_mcmc(None, 3)
    s.run_mcmc(None, 2, thin_by=3)
    last = s.run_mcmc(None, 4)
    for last in s.sample(last, iterations=3, thin_by=3):
        pass
    for last in s.sample(last, iterations=6, thin=2):
        pass
    assert s.iteration == it0 + 5 + 3 + 2 + 4 + 3 + 3


def _twin(make, p0, drive=_drive):
    h, d = make(Backend()), make(DeviceBackend())
    drive(h, p0)
    drive(d, p0)
    _reads_equal(h, d)
    assert d.backend.nbytes > 0
    return h, d


def _sampler_factory(N, D, model, dmoves, seed, options=()):
    def make(backend):
        s = emcee_b200.EnsembleSampler(N, D, model, moves=dmoves, seed=seed, backend=backend)
        for k, v in options:
            s._engine.set_option(k, v)
        return s

    return make


def test_twin_dense_dmma_128():
    N, D = 512, 128
    target, p0 = T.make_config("gauss_dense", N, D)
    h, d = _twin(_sampler_factory(N, D, models.GaussianDense(target.icov), None, 0x51), p0)
    assert d._engine.last_kernel_name() == "dense_dmma"


def test_twin_grouped_dense_dmma_launch_count():
    N, D = 1026, 64
    target, p0 = T.make_config("gauss_dense", N, D)
    make = _sampler_factory(N, D, models.GaussianDense(target.icov), None, 0x52, options=(("dmma_group", 4),))

    def drive(s, p0):
        s.run_mcmc(p0, 4, thin_by=3, skip_initial_state_check=True)
        s.launches = s._engine.last_step_timing()[1]
        assert s._engine.last_kernel_variant().startswith("dense_dmma nhalf_max=4 ")
        _drive(s, s.get_last_sample())

    h, d = _twin(make, p0, drive)
    assert d.launches == h.launches


def test_twin_tma_rows_register_ring_32():
    N, D = 2 * (8 * 20 + 1), 32
    target, p0 = T.make_config("ring", N, D)
    h, d = _twin(_sampler_factory(N, D, device_model("ring", target=target), None, 0x53), p0)
    assert d._engine.last_kernel_variant().startswith("tma_rows R=8 epl=8 own_reg=1")


def test_twin_generic_odd_ndim():
    N, D = 301, 37
    target, p0 = T.make_config("gauss_iso", N, D)
    h, d = _twin(_sampler_factory(N, D, models.GaussianIso(), None, 0x54), p0)
    assert d._engine.last_kernel_name() == "generic"


def test_twin_rosenbrock_de_snooker():
    N, D = 512, 16
    target, p0 = T.make_config("rosenbrock", N, D)
    dm = device_moves(move_rows_from_oracle([(rb.DE(), 0.8), (rb.Snooker(), 0.2)]))
    _twin(_sampler_factory(N, D, models.Rosenbrock(), dm, 0x55), p0)


def test_twin_walk_gaussian_mix():
    N, D = 64, 4
    target, p0 = T.make_config("ring", N, D)
    dm = [(moves.WalkMove(s=6), 0.4), (moves.GaussianMove(0.05, mode="sequential"), 0.3), (moves.StretchMove(), 0.3)]
    h, d = _twin(_sampler_factory(N, D, device_model("ring", target=target), dm, 0x56), p0)


def test_twin_bounded_stores_minus_inf():
    N, D = 2 * (8 * 20 + 1), 32
    target, p0 = T.make_config("ring", N, D)
    lo, hi, pb = _box_and_p0(target, p0, 0)
    model = models.Bounded(device_model("ring", target=target), lo, hi)
    h, d = _twin(_sampler_factory(N, D, model, None, 0x57), pb)
    assert np.isneginf(d.get_log_prob()[0]).any()


# ---- golden chains ---------------------------------------------------------------------------------------------
def _golden_device(g, model):
    s = emcee_b200.EnsembleSampler(int(g["nwalkers"]), int(g["ndim"]), model, moves=device_moves(g["moves"], g),
                                   seed=int(g["seed"]), backend=DeviceBackend())
    s.run_mcmc(g["p0"], g["chain"].shape[0], skip_initial_state_check=True)
    return s


def _golden_compare(s, g, exact, rtol, atol):
    if exact:
        assert np.array_equal(s.get_chain(), g["chain"])
    else:
        np.testing.assert_allclose(s.get_chain(), g["chain"], rtol=rtol, atol=atol)
    assert np.array_equal(np.isneginf(s.get_log_prob()), np.isneginf(g["log_prob"]))
    np.testing.assert_allclose(s.get_log_prob(), g["log_prob"], rtol=max(rtol, 1e-12), atol=max(10 * atol, 1e-12))
    assert np.array_equal(s.backend.accepted, g["accepted"].sum(axis=0))


@pytest.mark.parametrize("name", golden_names())
def test_golden_into_device_backend(name):
    g = load_golden(name)
    s = _golden_device(g, device_model(str(g["model_kind"]), g=g))
    _golden_compare(s, g, *_tols(g))


@pytest.mark.parametrize("name", bounded_names())
def test_bounded_golden_into_device_backend(name):
    g = load_bounded(name)
    model = models.Bounded(device_model(str(g["model_kind"]), g=g), g["model_lower"], g["model_upper"])
    s = _golden_device(g, model)
    _golden_compare(s, g, *_golden_tols(g))


# ---- autocorrelation -------------------------------------------------------------------------------------------
def _tau_or_error(f):
    try:
        return "ok", f()
    except autocorr.AutocorrError as e:
        return "short", e.tau


def _same_tau(h, d, grid):
    for discard, thin in grid:
        for quiet in (False, True):
            kh = _tau_or_error(lambda: h.get_autocorr_time(discard=discard, thin=thin, quiet=quiet))
            kd = _tau_or_error(lambda: d.get_autocorr_time(discard=discard, thin=thin, quiet=quiet))
            kb = _tau_or_error(lambda: d.backend.get_autocorr_time(discard=discard, thin=thin, quiet=quiet))
            assert kh[0] == kd[0] == kb[0], (discard, thin, quiet)
            assert np.array_equal(kh[1], kd[1]) and np.array_equal(kh[1], kb[1]), (discard, thin, quiet)


def test_autocorr_matches_host_route():
    N, D = 64, 3
    target, p0 = T.make_config("gauss_iso", N, D)
    make = _sampler_factory(N, D, models.GaussianIso(), None, 0x61)
    h, d = make(Backend()), make(DeviceBackend())
    for s in (h, d):
        s.run_mcmc(p0, 150, skip_initial_state_check=True)
        s.run_mcmc(None, 90)
        s.run_mcmc(None, 60, thin_by=2)
    grid = [(0, 1), (140, 1), (50, 3), (10, 7), (0, 40)]
    _same_tau(h, d, grid)
    # a short window raises on both routes with the same estimate
    with pytest.raises(autocorr.AutocorrError):
        d.get_autocorr_time(discard=280)
    for s in (h, d):
        with pytest.raises(ValueError):
            s.get_autocorr_time(discard=400)  # no stored step left


def test_autocorr_wider_than_one_slab_two_segments():
    # 8192 walkers x 8 parameters x 640 steps: ~300 KB of FFT scratch per walker, so a ~1 GiB slab holds
    # 3573 walkers and the ensemble takes three slabs; two run_mcmc calls make two segments.  (Slabs of more
    # than 65 535 series are covered by test_gpu_autocorr_exact.py.)
    N, D = 8192, 8
    target, p0 = T.make_config("gauss_iso", N, D)
    make = _sampler_factory(N, D, models.GaussianIso(), None, 0x62)
    h, d = make(Backend()), make(DeviceBackend())
    for s in (h, d):
        s.run_mcmc(p0, 400, skip_initial_state_check=True)
        s.run_mcmc(None, 240)
    wb = (1 << 30) // ((2048 * 16 + 640 * 8) * D)
    assert wb < N and wb * D < 65536
    _same_tau(h, d, [(0, 1), (40, 2)])  # 640 and 300 steps: three and two slabs


# ---- restart and pickling --------------------------------------------------------------------------------------
def test_restart_through_initialised_backend():
    N, D = 64, 5
    target, p0 = T.make_config("gauss_iso", N, D)
    make = _sampler_factory(N, D, models.GaussianIso(), None, 0x71)
    out = []
    for b in (Backend(), DeviceBackend()):
        s1 = make(b)
        s1.run_mcmc(p0, 7, skip_initial_state_check=True)
        s2 = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), backend=b, seed=12345)
        assert s2.iteration == 7
        s2.run_mcmc(None, 6)
        out.append(s2)
    _reads_equal(*out)
    assert out[1].iteration == 13


def test_pickled_sampler_keeps_the_chain_and_continues():
    N, D = 96, 6
    target, p0 = T.make_config("ring", N, D)
    make = _sampler_factory(N, D, device_model("ring", target=target), None, 0x72)
    loaded = []
    for b in (Backend(), DeviceBackend()):
        s = make(b)
        s.run_mcmc(p0, 9, skip_initial_state_check=True)
        s2 = pickle.loads(pickle.dumps(s))
        assert np.array_equal(s2.get_chain(), s.get_chain()) and np.array_equal(s2.backend.accepted, s.backend.accepted)
        s2.run_mcmc(None, 5)
        loaded.append(s2)
    _reads_equal(*loaded)
    assert isinstance(loaded[1].backend, DeviceBackend)


# ---- contracts -------------------------------------------------------------------------------------------------
def _small(backend, seed=0x81, N=32, D=5):
    return emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=seed, backend=backend)


def test_read_before_store_raises_like_host():
    s = _small(DeviceBackend())
    for f in (s.get_chain, s.get_log_prob, s.get_last_sample):
        with pytest.raises(AttributeError, match="store == True"):
            f()
    s.run_mcmc(np.random.default_rng(0).normal(size=(32, 5)), 3, store=False)
    with pytest.raises(AttributeError, match="store == True"):
        s.get_chain()


def test_shape_mismatch_and_device_mismatch():
    b = DeviceBackend()
    s = _small(b)
    s.run_mcmc(np.random.default_rng(0).normal(size=(32, 5)), 2)
    with pytest.raises(ValueError, match="incompatible with the shape"):
        emcee_b200.EnsembleSampler(34, 5, models.GaussianIso(), backend=b)
    with pytest.raises(ValueError, match="device"):
        _small(DeviceBackend(device=1))


def test_blobs_refused():
    b = DeviceBackend()
    b.reset(32, 5)
    with pytest.raises(NotImplementedError):
        b.grow(3, np.zeros(3))
    b.grow(1, None)
    st = emcee_b200.State(np.zeros((32, 5)), log_prob=np.zeros(32), blobs=np.zeros(32))
    with pytest.raises(NotImplementedError):
        b.save_step(st, np.zeros(32, dtype=bool))


def test_save_step_matches_host_backend():
    rng = np.random.default_rng(3)
    h, d = Backend(), DeviceBackend()
    for b in (h, d):
        b.reset(33, 7)  # odd N * D: unaligned tails of the slot copies
        b.grow(2, None)
    for k in range(5):
        if k == 2:
            for b in (h, d):
                b.grow(3, None)
        st = emcee_b200.State(rng.normal(size=(33, 7)), log_prob=rng.normal(size=33), random_state=("r", k))
        acc = rng.random(33) < 0.4
        for b in (h, d):
            b.save_step(st, acc)
    for kw in (dict(), dict(discard=1, thin=2), dict(flat=True, thin=3)):
        assert np.array_equal(h.get_chain(**kw), d.get_chain(**kw))
        assert np.array_equal(h.get_log_prob(**kw), d.get_log_prob(**kw))
    assert np.array_equal(h.accepted, d.accepted) and d.iteration == 5
    assert np.array_equal(h.get_last_sample().coords, d.get_last_sample().coords)
    assert d.get_last_sample().random_state == ("r", 4)
    with pytest.raises(ValueError, match="invalid coordinate dimensions"):
        d.save_step(emcee_b200.State(np.zeros((33, 6)), log_prob=np.zeros(33)), np.zeros(33, dtype=bool))


def test_grow_beyond_device_memory_then_run():
    b = DeviceBackend()
    s = _small(b)
    p0 = np.random.default_rng(1).normal(size=(32, 5))
    s.run_mcmc(p0, 3)
    held = b.nbytes
    # 10^12 slots of 32 x 5 doubles: more than the device holds in total, refused before any allocation
    with pytest.raises(MemoryError, match="bytes"):
        b.grow(10**12, None)
    assert b.nbytes == held
    s.run_mcmc(None, 4)
    assert s.iteration == 7 and s.get_chain().shape == (7, 32, 5)


def test_close_frees_and_refuses():
    b = DeviceBackend()
    s = _small(b)
    s.run_mcmc(np.random.default_rng(2).normal(size=(32, 5)), 3)
    assert b.nbytes > 0
    b.close()
    assert b.nbytes == 0
    for f in (b.get_chain, lambda: b.accepted, lambda: b.grow(1, None), lambda: b.reset(32, 5), s.get_chain):
        with pytest.raises(ValueError, match="closed"):
            f()
    with pytest.raises(ValueError, match="closed"):
        s.run_mcmc(None, 2)


def test_attach_refused():
    s = _small(DeviceBackend())
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(None)


def test_abi_refusals():
    from emcee_b200 import _lib

    s = _small(DeviceBackend())
    s._engine.set_state(np.random.default_rng(4).normal(size=(32, 5)))
    sched = s._schedule()
    other = _lib.Chain(34, 5)
    other.grow(4)
    with pytest.raises(ValueError, match="the chain is"):
        s._engine.step_store_chain(sched, 2, 1, other, 0)
    ch = s.backend._ch
    ch.grow(4)
    with pytest.raises(ValueError, match="out of range"):
        s._engine.step_store_chain(sched, 5, 1, ch, 0)
    with pytest.raises(ValueError, match="Invalid thinning argument"):
        s._engine.step_store_chain(sched, 2, 0, ch, 0)
    with pytest.raises(ValueError, match="out of range"):
        ch.read(3, 1, 2)
    with pytest.raises(ValueError, match="out of range"):
        ch.read(0, 0, 2)
