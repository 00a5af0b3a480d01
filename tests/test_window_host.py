"""Host side of the running window (``EnsembleSampler.enable_window`` / ``window``): the ring origin of the slot map
``csrc/chain_map.h`` built with g++ and driven against numpy indexing, and the Python lifecycle over a stand-in
engine."""

import ctypes as C
import os
import pickle
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200.backend import ChainWindow, slice_plan

HERE = os.path.dirname(os.path.abspath(__file__))
_P = C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("chainring") / "libchain_ring_probe.so")
    subprocess.run(
        ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", "chain_ring_host.cpp")],
        check=True,
    )
    lib = C.CDLL(out)
    lib.probe_ring_runs.restype = C.c_longlong
    lib.probe_ring_runs.argtypes = [_P, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _P, C.c_size_t]
    lib.probe_plain_runs.restype = C.c_longlong
    lib.probe_plain_runs.argtypes = [_P, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, _P, C.c_size_t]
    return lib


def _start(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)


def _runs(probe, sizes, first, stride, count, origin=None):
    start = _start(sizes)
    out = np.zeros((max(count, 1) + 2, 4), dtype=np.uint64)
    if origin is None:
        n = probe.probe_plain_runs(start.ctypes.data_as(_P), len(sizes), first, stride, count, out.ctypes.data_as(_P),
                                   out.shape[0])
    else:
        n = probe.probe_ring_runs(start.ctypes.data_as(_P), len(sizes), origin, first, stride, count,
                                  out.ctypes.data_as(_P), out.shape[0])
    return None if n < 0 else out[:n].astype(np.int64)


def _visited(runs, sizes, stride):
    """The physical slots the runs visit, in order; each run must stay inside its segment."""
    start = _start(sizes).astype(np.int64)
    slots, k = [], 0
    for seg, off, k0, n in runs:
        assert k0 == k and n >= 1
        s = start[seg] + off + stride * np.arange(n)
        assert off >= 0 and s[-1] < start[seg + 1]
        slots.extend(s.tolist())
        k += n
    return slots


def _window_case(probe, size, recorded, discard, thin):
    """The window of `recorded` steps in a ring of `size` slots, sliced like emcee: the physical slots visited must be
    np.arange(recorded)[-size:] sliced with discard + thin - 1 :: thin, mapped through (origin + i) % size."""
    filled = min(recorded, size)
    origin = recorded % size if recorded >= size else 0
    first, stride, count = slice_plan(filled, discard, thin)
    runs = _runs(probe, [size], first, stride, count, origin)
    assert runs is not None
    kept = np.arange(recorded)[-size:] if recorded else np.arange(0)
    logical = np.arange(filled)[discard + thin - 1 :: thin]
    want_steps = kept[discard + thin - 1 :: thin]
    got = _visited(runs, [size], stride)
    assert got == ((origin + logical) % size).tolist(), (size, recorded, discard, thin)
    # the physical slot of step t is t % size: the slots visited hold exactly the steps the slice names
    assert got == (want_steps % size).tolist()
    # a run never crosses the wrap, so a slice crossing it splits into at least two
    if count and any(s < g for s, g in zip(got[1:], got[:-1])):
        assert len(runs) >= 2


def test_ring_map_grid(probe):
    for size in (1, 2, 3, 5, 8):
        for recorded in range(0, 3 * size + 3):
            for discard in range(0, size + 2):
                for thin in (1, 2, 3, size + 1, size + 4):
                    _window_case(probe, size, recorded, discard, thin)


def test_ring_map_random(probe):
    rng = np.random.default_rng(7)
    for _ in range(3000):
        size = int(rng.integers(1, 64))
        recorded = int(rng.integers(0, 5 * size))
        discard = int(rng.integers(0, size + 3))
        thin = int(rng.integers(1, 2 * size + 3))
        _window_case(probe, size, recorded, discard, thin)


def test_ring_map_refusals(probe):
    assert _runs(probe, [5], 0, 0, 3, origin=2) is None  # stride 0
    assert _runs(probe, [5], 0, 1, 6, origin=2) is None  # beyond the capacity
    assert _runs(probe, [5], 4, 2, 2, origin=0) is None
    assert _runs(probe, [5], 0, 1, 1, origin=5) is None  # origin outside the ring
    assert _runs(probe, [5], 2**64 - 1, 2**63, 2, origin=1) is None  # the last slot overflows
    assert _runs(probe, [5], 0, 1, 0, origin=3).shape == (0, 4)  # an empty slice is always fine
    assert _runs(probe, [1], 0, 1, 1, origin=0).tolist() == [[0, 0, 0, 1]]


def test_origin_zero_is_the_plain_map(probe):
    """Origin 0 on a multi-segment chain gives exactly the runs of the map without an origin."""
    for sizes in ([20], [1] * 20, [7, 13], [3, 5, 4, 8], [1, 19], [19, 1], [2, 2, 2, 2, 2, 10]):
        for it in range(21):
            for discard in range(23):
                for thin in range(1, 8):
                    first, stride, count = slice_plan(it, discard, thin)
                    plain = _runs(probe, sizes, first, stride, count)
                    ring = _runs(probe, sizes, first, stride, count, origin=0)
                    assert plain is not None and np.array_equal(plain, ring), (sizes, it, discard, thin)


def test_origin_on_segments(probe):
    """A nonzero origin on a multi-segment chain visits (origin + i) mod capacity, each run inside a segment."""
    rng = np.random.default_rng(3)
    for sizes in ([7, 13], [3, 5, 4, 8], [1] * 6):
        cap = sum(sizes)
        for _ in range(300):
            origin = int(rng.integers(0, cap))
            it = int(rng.integers(0, cap + 1))
            first, stride, count = slice_plan(it, int(rng.integers(0, 5)), int(rng.integers(1, 6)))
            runs = _runs(probe, sizes, first, stride, count, origin)
            assert _visited(runs, sizes, stride) == ((origin + first + stride * np.arange(count)) % cap).tolist()


# ---- the Python methods over a stand-in engine -------------------------------------------------------------------
class _Engine(object):
    """The window calls of ``_lib.Engine``, keeping a host ring of step numbers."""

    def __init__(self, nwalkers=4, ndim=2):
        self.nwalkers, self.ndim, self.device = nwalkers, ndim, 0
        self.calls, self.size, self.every, self.n = [], None, 0, 0
        self.fail = False

    def window_config(self, size, every):
        if self.fail:
            raise MemoryError("no room")
        self.calls.append((size, every))
        if every > 0 or self.size is None:
            self.size, self.n = size, 0
        self.every = every

    def record(self, k):
        self.n += k

    def window_count(self):
        return self.n, min(self.n, self.size)

    def window_steps(self):
        filled = min(self.n, self.size)
        steps = np.arange(self.n - filled + 1, self.n + 1, dtype=np.uint64) * max(self.every, 1)
        return steps, np.full(filled, 9, dtype=np.uint64)

    def window_chain(self):
        return object()  # the ring's readers are the GPU tests' business

    def get_rng(self):
        return 9, 0


def _sampler(nwalkers=4, ndim=2):
    s = object.__new__(emcee_b200.EnsembleSampler)
    s.ndim, s.nwalkers, s._device, s._rdv = ndim, nwalkers, 0, None
    s._hist = s._trace_every = s._reservoir_every = s._autocorr = s._window = None
    s._engine, s._pinned = _Engine(nwalkers, ndim), None
    return s


def test_reading_before_enabling():
    s = _sampler()
    with pytest.raises(RuntimeError, match="not enabled"):
        s.window()


@pytest.mark.parametrize("size,every,err", [(0, 1, ValueError), (-2, 1, ValueError), (4, -1, ValueError),
                                            (4.0, 1, TypeError), ("4", 1, TypeError), (4, 1.5, TypeError),
                                            (None, 1, TypeError)])
def test_arguments(size, every, err):
    s = _sampler()
    with pytest.raises(err):
        s.enable_window(size, every)
    assert s._engine.calls == [] and s._window is None


def test_lifecycle():
    s = _sampler()
    s.enable_window(np.int64(5), np.int64(3))
    assert s._engine.calls == [(5, 3)] and s._window == (5, 3)
    w = s.window()
    assert isinstance(w, ChainWindow) and isinstance(w, emcee_b200.DeviceBackend)
    assert w.iteration == 0 and w.recorded == 0 and w.random_state is None and w.every == 3
    assert w.shape == (4, 2) and not w.has_blobs()
    with pytest.raises(AttributeError, match="store == True"):  # an empty window reads like an empty backend
        w.get_chain()
    s._engine.record(7)  # the view reads the live ring
    assert (w.iteration, w.recorded) == (5, 7) and w.get_blobs() is None
    assert w.steps.tolist() == [9, 12, 15, 18, 21] and w.steps.dtype == np.uint64
    assert w.random_state == ("philox4x32-10", 9, 21)
    s.enable_window(2, 0)  # every=0: keeps the size, the cadence and the contents
    assert s._window == (5, 3) and (w.iteration, w.recorded) == (5, 7) and w.every == 3
    s.enable_window(3, 2)  # every > 0: drops what was recorded
    assert s._window == (3, 2) and (w.iteration, w.recorded) == (0, 0) and w.every == 2


def test_impossible_size_changes_nothing():
    s = _sampler()
    s.enable_window(4, 2)
    s._engine.record(6)
    s._engine.fail = True
    with pytest.raises(MemoryError):
        s.enable_window(2**40, 1)
    assert s._window == (4, 2) and s.window().recorded == 6


def test_view_refuses_writes():
    s = _sampler()
    s.enable_window(4)
    w = s.window()
    for call in (lambda: w.reset(4, 2), lambda: w.grow(3, None), lambda: w.save_step(None, np.zeros(4)), w.close):
        with pytest.raises(TypeError, match="read-only"):
            call()
    with pytest.raises(TypeError, match="pickled"):
        pickle.dumps(w)


def test_sharded_refused():
    s = _sampler()
    s._rdv = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        s.enable_window(4)
    s = _sampler()
    s.backend = emcee_b200.Backend()
    s._cuda_results = False
    s.enable_window(4)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(object())


def test_window_is_not_pickled():
    s = _sampler()
    s.enable_window(4, 2)
    state = s.__getstate__()
    assert state["_window"] is None and "_engine" not in state
    pickle.dumps(state)
