"""Host side of the running reservoir (``EnsembleSampler.enable_reservoir`` / ``reservoir`` / ``reservoir_count``),
no GPU needed: argument checks and the lifecycle of the Python methods over a stand-in engine."""
import pickle

import numpy as np
import pytest

import emcee_b200
from emcee_b200.ensemble import Reservoir


class _Engine(object):
    """records what EnsembleSampler asks of the engine's reservoir functions"""

    def __init__(self, ndim):
        self.ndim, self.calls, self.offered, self.size = ndim, [], 0, 0

    def reservoir_config(self, size, every):
        self.calls.append((size, every))
        if every > 0 or not self.size:
            self.offered, self.size = 0, size

    def reservoir_count(self):
        return self.offered, min(self.offered, self.size)

    def reservoir_read(self, cuda=False):
        k = min(self.offered, self.size)
        coords = np.arange(k * self.ndim, dtype=np.float64).reshape(k, self.ndim)
        return coords, -np.arange(k, dtype=np.float64), np.arange(1, k + 1, dtype=np.uint64), np.arange(k)

    def get_rng(self):
        return 1, 0


def _sampler(ndim=3):
    s = object.__new__(emcee_b200.EnsembleSampler)
    s.ndim, s.nwalkers, s._rdv, s._hist, s._trace_every, s._reservoir_every = ndim, 8, None, None, None, None
    s._engine, s._pinned = _Engine(ndim), None
    return s


def test_reading_before_enabling():
    s = _sampler()
    for read in (s.reservoir, s.reservoir_count):
        with pytest.raises(RuntimeError, match="not enabled"):
            read()


@pytest.mark.parametrize("size", [0, -1])
def test_size_at_least_one(size):
    s = _sampler()
    with pytest.raises(ValueError, match="size must be >= 1"):
        s.enable_reservoir(size)
    assert s._engine.calls == [] and s._reservoir_every is None


@pytest.mark.parametrize("size", [1.0, "2", None, 2.5])
def test_size_must_be_an_index(size):
    s = _sampler()
    with pytest.raises(TypeError):
        s.enable_reservoir(size)
    assert s._engine.calls == [] and s._reservoir_every is None


@pytest.mark.parametrize("every", [1.0, "2", None, 2.5])
def test_every_must_be_an_index(every):
    s = _sampler()
    with pytest.raises(TypeError):
        s.enable_reservoir(4, every)
    assert s._engine.calls == [] and s._reservoir_every is None


def test_every_negative():
    s = _sampler()
    with pytest.raises(ValueError, match="every must be >= 0"):
        s.enable_reservoir(4, -1)
    assert s._engine.calls == []
    s.enable_reservoir(np.int64(5), np.int64(4))  # anything with __index__
    assert s._engine.calls == [(5, 4)] and s._reservoir_every == 4


def test_every_zero_keeps_the_contents():
    s = _sampler()
    s.enable_reservoir(10, 3)
    s._engine.offered = 16
    s.enable_reservoir(10, 0)
    assert s._engine.calls == [(10, 3), (10, 0)] and s._reservoir_every == 3
    assert s.reservoir_count() == 16 and s.reservoir().step.size == 10
    s.enable_reservoir(10, 2)  # every > 0 drops what was kept
    assert s._reservoir_every == 2 and s.reservoir_count() == 0 and s.reservoir().step.size == 0


def test_reservoir_fields():
    s = _sampler(ndim=3)
    s.enable_reservoir(5)
    s._engine.offered = 4
    r = s.reservoir()
    assert isinstance(r, Reservoir) and r._fields == ("coords", "log_prob", "step", "walker")
    assert r.coords.shape == (4, 3) and r.log_prob.shape == (4,) and r.step.dtype == np.uint64
    s._engine.offered = 40
    assert s.reservoir().coords.shape == (5, 3) and s.reservoir_count() == 40


def test_sharded_refused():
    s = _sampler()
    s._rdv = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.enable_reservoir(4)
    s = _sampler()
    s.backend = emcee_b200.Backend()
    s.enable_reservoir(4)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(object())


def test_contents_are_not_pickled():
    s = _sampler()
    s.enable_reservoir(4, 2)
    state = s.__getstate__()
    assert state["_reservoir_every"] is None and "_engine" not in state
    pickle.dumps(state)
