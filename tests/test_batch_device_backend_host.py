"""Host side of a ``BatchSampler`` storing into a ``DeviceBackend``, and of its per-ensemble summaries: the
``backend=`` checks, the routing of stored steps to ``step_store_chain`` (bulk and generator paths), the accounting of
``iteration`` when a run stops early and result shapes, over a stand-in engine and chain; the host ``Backend``'s
``get_percentile`` / ``get_moments`` against per-ensemble numpy; and g++ builds of the segmented slab planning
(``acf_grid.h``) and of the segmented selection plan (``select_keys.h``)."""

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import DeviceBackend, _lib, models

from test_batch_host import _Engine, _p0

HERE = os.path.dirname(os.path.abspath(__file__))


class _Chain(object):
    """The calls ``DeviceBackend`` and ``BatchSampler`` make on ``_lib.Chain``, in host memory."""

    def __init__(self, nwalkers, ndim, device=0):
        self.nwalkers, self.ndim, self.device = nwalkers, ndim, device
        self.x = np.empty((0, nwalkers, ndim))
        self.lp = np.empty((0, nwalkers))
        self.acc = np.zeros(nwalkers)

    def close(self):
        pass

    def grow(self, nslots):
        if nslots > 10**6:
            raise MemoryError("stand-in: %d slots do not fit" % nslots)
        add = max(nslots - len(self.x), 0)
        self.x = np.concatenate([self.x, np.full((add, self.nwalkers, self.ndim), np.nan)])
        self.lp = np.concatenate([self.lp, np.full((add, self.nwalkers), np.nan)])

    def write(self, slot, coords, log_prob, accepted=None):
        self.x[slot], self.lp[slot] = coords, log_prob
        if accepted is not None:
            self.acc += accepted

    def read(self, first, stride, count, coords=True, log_prob=True):
        sl = slice(first, first + stride * count, stride) if count else slice(0, 0)
        return (self.x[sl].copy() if coords else None), (self.lp[sl].copy() if log_prob else None)

    def accepted(self):
        return self.acc.copy()


class _StoreEngine(_Engine):
    """``_Engine`` with ``step_store_chain``; ``fail_at`` (a step count) raises there, as a user function's error
    stops a run inside a step."""

    fail_at = None

    def _advance(self):
        if self.fail_at is not None and self.step_count + 1 == self.fail_at:
            raise ValueError("Probability function returned NaN")
        super()._advance()

    def step_store_chain(self, sched, nsteps, thin_by, chain, slot0):
        self.calls.append(("store_chain", nsteps, thin_by, slot0))
        k = slot0
        for j in range(nsteps):
            self._advance()
            if (j + 1) % thin_by == 0:
                chain.write(k, self.x, self.lp, np.arange(self.nwalkers) % 2 == 0)
                k += 1

    def step_store(self, sched, nsteps, thin_by, chain, log_prob, accepted):
        self.calls.append(("store_host", nsteps, thin_by))
        super().step_store(sched, nsteps, thin_by, chain, log_prob, accepted)


@pytest.fixture
def stand_in(monkeypatch):
    _StoreEngine.created, _StoreEngine.fail_at = [], None
    monkeypatch.setattr(_lib, "BatchEngine", _StoreEngine)
    monkeypatch.setattr(_lib, "Chain", _Chain)
    return _StoreEngine


def _batch(K=3, N=8, D=2, **kw):
    return emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, **kw)


# ---- backend= ---------------------------------------------------------------------------------------------------
def test_backend_checks(stand_in):
    with pytest.raises(ValueError, match="device 1"):
        _batch(backend=DeviceBackend(device=1))
    b = DeviceBackend()
    b.reset(7, 2)
    with pytest.raises(ValueError, match="incompatible"):
        _batch(backend=b)
    s = _batch(backend=DeviceBackend())
    assert s.backend.shape == (24, 2) and s.iteration == 0


def test_resume_from_initialised_backend(stand_in):
    one = _batch(backend=DeviceBackend())
    one.run_mcmc(_p0(3, 8, 2), 4, thin_by=2, skip_initial_state_check=True)
    two = emcee_b200.BatchSampler(3, 8, 2, models.GaussianIso(), seeds=[9, 9, 9], backend=one.backend)
    assert two.iteration == 4
    assert two.random_state[2] == 8 and np.array_equal(two.random_state[1], one.random_state[1])
    last = two.run_mcmc(None, 2, thin_by=2, skip_initial_state_check=True)  # the stand-in's walkers are dependent
    assert two.iteration == 6 and last.coords.shape == (3, 8, 2)
    assert np.array_equal(two.get_chain()[:4], one.get_chain()[:4])


# ---- routing and failure accounting --------------------------------------------------------------------------------
def test_routing(stand_in):
    s = _batch(backend=DeviceBackend())
    s.run_mcmc(_p0(3, 8, 2), 5, thin_by=3, skip_initial_state_check=True)
    assert s._engine.calls[-1] == ("store_chain", 15, 3, 0)
    for _ in s.sample(s.get_last_sample(), iterations=2, thin_by=2, skip_initial_state_check=True):
        pass
    assert s._engine.calls[-2:] == [("store_chain", 2, 2, 5), ("store_chain", 2, 2, 6)]
    assert s.iteration == 7
    h = _batch()
    h.run_mcmc(_p0(3, 8, 2), 5, skip_initial_state_check=True)
    assert h._engine.calls[-1] == ("store_host", 5, 1)
    # the stand-in writes step s of row r as s * 1000 + r: the stored steps are the thinned ones
    assert np.array_equal(s.get_log_prob()[:, 0, 0], -1000.0 * np.array([3, 6, 9, 12, 15, 17, 19]))


@pytest.mark.parametrize("bulk", [True, False])
def test_failure_keeps_stored_steps(stand_in, bulk):
    stand_in.fail_at = 8
    s = _batch(backend=DeviceBackend())
    with pytest.raises(ValueError, match="NaN"):
        if bulk:
            s.run_mcmc(_p0(3, 8, 2), 5, thin_by=2, skip_initial_state_check=True)
        else:
            for _ in s.sample(_p0(3, 8, 2), iterations=5, thin_by=2, skip_initial_state_check=True):
                pass
    assert s.iteration == 3  # steps 2, 4 and 6 were stored before step 8 failed
    assert s.get_chain().shape == (3, 3, 8, 2)
    if bulk:
        assert s.backend.random_state[2] == 6


def test_result_shapes(stand_in):
    K, N, D = 3, 8, 2
    s = _batch(K, N, D, backend=DeviceBackend())
    s.run_mcmc(_p0(K, N, D), 6, skip_initial_state_check=True)
    assert s.get_chain().shape == (6, K, N, D) and s.get_log_prob().shape == (6, K, N)
    assert s.get_chain(flat=True, discard=2, thin=2).shape == (K, 2 * N, D)
    assert s.get_log_prob(flat=True).shape == (K, 6 * N)
    assert s.acceptance_fraction.shape == (K, N)
    assert s.get_last_sample().coords.shape == (K, N, D)
    h = _batch(K, N, D)
    h.run_mcmc(_p0(K, N, D), 6, skip_initial_state_check=True)
    with pytest.raises(TypeError, match="DeviceBackend"):
        h.get_chain(cuda=True)
    assert h.get_percentile([16, 50, 84]).shape == (K, 3, D)
    assert h.get_percentile(50, name="log_prob").shape == (K,)
    mean, cov, n = h.get_moments()
    assert mean.shape == (K, D) and cov.shape == (K, D, D) and n == 6 * N


# ---- host Backend summaries -----------------------------------------------------------------------------------------
class _Random(_Engine):
    """Stored steps of random numbers, so that the summaries see distinct values."""

    def _advance(self):
        self.step_count += 1
        rng = np.random.default_rng(self.step_count)
        self.x = rng.normal(size=(self.nwalkers, self.ndim))
        self.lp = rng.normal(size=self.nwalkers)


@pytest.mark.parametrize("discard,thin", [(0, 1), (3, 2)])
def test_host_percentile_and_moments(monkeypatch, discard, thin):
    monkeypatch.setattr(_lib, "BatchEngine", _Random)
    K, N, D = 4, 6, 3
    s = _batch(K, N, D)
    s.run_mcmc(_p0(K, N, D), 12, skip_initial_state_check=True)
    flat = s.get_chain(flat=True, discard=discard, thin=thin)
    flat_lp = s.get_log_prob(flat=True, discard=discard, thin=thin)
    for q in ([16, 50, 84], 0, 100, [[5, 50], [95, 99]]):
        got = s.get_percentile(q, discard=discard, thin=thin)
        for k in range(K):
            assert np.array_equal(got[k], np.percentile(flat[k], q, axis=0))
            assert np.array_equal(s.get_percentile(q, discard=discard, thin=thin, name="log_prob")[k],
                                  np.percentile(flat_lp[k], q, axis=0))
    mean, cov, n = s.get_moments(discard=discard, thin=thin)
    assert n == flat.shape[1]
    for k in range(K):
        assert np.array_equal(mean[k], np.mean(flat[k], axis=0))
        assert np.array_equal(cov[k], np.cov(flat[k], rowvar=False))


def test_bad_q_and_empty_slices(monkeypatch):
    monkeypatch.setattr(_lib, "BatchEngine", _Random)
    K, N, D = 2, 6, 3
    s = _batch(K, N, D)
    s.run_mcmc(_p0(K, N, D), 4, skip_initial_state_check=True)
    with pytest.raises(ValueError, match="Percentiles must be in the range"):
        s.get_percentile([50, 101])
    with pytest.raises(ValueError, match="percentiles are taken of"):
        s.get_percentile(50, name="blobs")
    with pytest.raises(IndexError):
        s.get_percentile(50, discard=4)
    mean, cov, n = s.get_moments(discard=4)
    assert n == 0 and np.isnan(mean).all() and np.isnan(cov).all() and cov.shape == (K, D, D)


# ---- g++: segmented slab planning -----------------------------------------------------------------------------------
def _build(tmp_path_factory, name, src):
    out = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", src)],
                   check=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def acf_probe(tmp_path_factory):
    lib = _build(tmp_path_factory, "acfseg", "acf_segments_host.cpp")
    u64 = C.POINTER(C.c_uint64)
    lib.probe_acf_segment_slabs.restype = C.c_uint64
    lib.probe_acf_segment_slabs.argtypes = [C.c_uint64] * 4 + [u64, u64, u64, C.c_uint64]

    def slabs(n_t, nw, nd, nseg):
        cap = nw + 1
        w0, wn, blocks = (np.zeros(cap, dtype=np.uint64) for _ in range(3))
        n = lib.probe_acf_segment_slabs(n_t, nw, nd, nseg, *(a.ctypes.data_as(u64) for a in (w0, wn, blocks)), cap)
        return w0[:n].astype(int), wn[:n].astype(int), blocks[:n].astype(int)

    return slabs


@pytest.mark.parametrize("n_t,N,nd,K", [(100, 32, 5, 64), (2000, 32, 5, 4096), (1 << 20, 32, 5, 3),
                                        (1 << 22, 37, 2, 2), (300, 7, 1, 1), (1 << 21, 64, 1, 1), (50, 2, 1000, 500)])
def test_segment_slabs(acf_probe, n_t, N, nd, K):
    """Slabs cover the walkers in order; each holds whole segments or lies inside one segment; a segment's walkers
    are split exactly as the chain of that ensemble alone (nseg = 1, nw = N) is; the accumulate grid has one CTA
    row per (segment, parameter) the slab holds."""
    w0, wn, blocks = acf_probe(n_t, K * N, nd, K)
    assert w0[0] == 0 and np.array_equal(w0[1:], (w0 + wn)[:-1]) and w0[-1] + wn[-1] == K * N
    alone_w0, alone_wn, _ = acf_probe(n_t, N, nd, 1)
    whole = (w0 % N == 0) & (wn % N == 0)
    inside = w0 // N == (w0 + wn - 1) // N
    assert np.all(whole | inside)
    lag_tiles = (n_t + 255) // 256
    nks = (w0 + wn - 1) // N - w0 // N + 1
    assert np.array_equal(blocks, lag_tiles * nd * nks)
    for k in sorted({0, K // 2, K - 1}):
        part = [(a - k * N, b) for a, b in zip(w0, wn) if k * N <= a < (k + 1) * N and not whole[list(w0).index(a)]]
        if len(alone_w0) == 1:  # the segment fits in one slab alone: it is never split
            assert part == [] and any(a <= k * N < a + b for a, b in zip(w0, wn))
        else:
            assert part == list(zip(alone_w0, alone_wn))
    one_w0, one_wn, _ = acf_probe(n_t, K * N, nd, 1)  # nseg = 1: the slabs of the plain call
    if K == 1:
        assert np.array_equal(one_w0, w0) and np.array_equal(one_wn, wn)


# ---- g++: segmented selection plan ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sel_probe(tmp_path_factory):
    lib = _build(tmp_path_factory, "selseg", "select_segments_host.cpp")
    u64, dp = C.POINTER(C.c_uint64), C.POINTER(C.c_double)
    lib.probe_select_segments.restype = C.c_int
    lib.probe_select_segments.argtypes = [dp, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, u64, C.c_size_t,
                                          C.c_uint64, dp, C.POINTER(C.c_uint8)]
    return lib


@pytest.mark.parametrize("count,K,N,D,budget", [(5, 7, 8, 3, 1 << 20), (40, 3, 32, 2, 64), (3, 50, 4, 1, 1 << 20),
                                                (9, 2, 16, 40, 1000)])
def test_segmented_selection(sel_probe, count, K, N, D, budget):
    rng = np.random.default_rng(count * K + D)
    x = np.round(rng.normal(size=(count, K, N, D)), 2)  # ties
    x[1, K - 1, 2, D - 1] = np.nan
    n = count * N
    ranks = np.unique(np.r_[0, n - 1, rng.integers(0, n, 5)]).astype(np.uint64)
    out = np.empty((K, ranks.size, D))
    has_nan = np.zeros((K, D), dtype=np.uint8)
    passes = sel_probe.probe_select_segments(
        np.ascontiguousarray(x).ctypes.data_as(C.POINTER(C.c_double)), count, K, N, D,
        ranks.ctypes.data_as(C.POINTER(C.c_uint64)), ranks.size, budget, out.ctypes.data_as(C.POINTER(C.c_double)),
        has_nan.ctypes.data_as(C.POINTER(C.c_uint8)))
    assert passes > 0
    flat = np.swapaxes(x, 0, 1).reshape(K, n, D)
    want_nan = np.isnan(flat).any(axis=1)
    assert np.array_equal(has_nan.astype(bool), want_nan)
    for k in range(K):
        srt = np.sort(flat[k], axis=0)
        want = np.where(want_nan[k][None, :], np.nan, srt[ranks.astype(np.intp)] + 0.0)
        assert np.array_equal(out[k], want, equal_nan=True)
