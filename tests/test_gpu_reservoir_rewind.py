"""The running reservoir when the random state moves, at sizes past what it can address, and into caller memory.

* ``run_mcmc`` from an earlier state (its ``random_state`` moves the step counter back) empties the reservoir and
  keeps it enabled: what it keeps afterwards equals a twin that enabled the reservoir at that state.  Setting the
  same ``random_state`` again changes nothing; another seed empties it.
* ``size`` 2**32, 2**63 and 2**64 + 5 raise ``MemoryError`` and leave the reservoir and the sampler as they were.
* ``eb_reservoir_read_to`` into a destination that is 8 but not 16 bytes aligned equals the host read.
"""
import ctypes as C

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models

pytestmark = pytest.mark.gpu

SEED = 0x5E5F
N, D = 64, 8  # tma_rows, even ndim: the 16-byte row path


def _make():
    return emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED)


def _p0():
    return np.random.default_rng(5).standard_normal((N, D)) * 0.5


def _bytes(r):
    return [np.asarray(f).tobytes() for f in r]


@pytest.mark.parametrize("K", [1, 30, 200])
def test_rewound_step_counter_starts_again(K):
    s = _make()
    s.enable_reservoir(K)
    st5 = s.run_mcmc(_p0(), 5, store=False, skip_initial_state_check=True)
    s.run_mcmc(st5, 7, store=False)
    assert s.reservoir_count() == 12 * N
    s.run_mcmc(st5, 6, store=False)  # back to step 5: steps 6 .. 11 come again, with their old keys
    assert s.reservoir_count() == 6 * N and s.random_state[2] == 11
    t = _make()
    u5 = t.run_mcmc(_p0(), 5, store=False, skip_initial_state_check=True)
    assert u5.random_state == st5.random_state and u5.coords.tobytes() == st5.coords.tobytes()
    t.enable_reservoir(K)
    t.run_mcmc(u5, 6, store=False)
    assert t.reservoir_count() == 6 * N
    assert _bytes(s.reservoir()) == _bytes(t.reservoir())
    assert set(s.reservoir().step.tolist()) <= set(range(6, 12))


def test_same_state_keeps_another_seed_empties():
    s = _make()
    s.enable_reservoir(40)
    s.run_mcmc(_p0(), 4, store=False, skip_initial_state_check=True)
    kept = _bytes(s.reservoir())
    s.random_state = s.random_state  # the same (seed, step)
    tag, seed, step = s.random_state
    s.random_state = (tag, seed, step + 3)  # forward: no step comes twice
    assert s.reservoir_count() == 4 * N and _bytes(s.reservoir()) == kept
    s.random_state = (tag, seed ^ 1, step + 3)
    assert s.reservoir_count() == 0 and s.reservoir().step.size == 0
    s.run_mcmc(None, 2, store=False)
    assert s.reservoir_count() == 2 * N and s.reservoir().step.size == 40


@pytest.mark.parametrize("size", [2**32, 2**63, 2**63 + 7, 2**64 - 1, 2**64 + 5, 2**70])
def test_unaddressable_size(size):
    s = _make()
    s.enable_reservoir(20)
    st = s.run_mcmc(_p0(), 3, store=False, skip_initial_state_check=True)
    kept = _bytes(s.reservoir())
    with pytest.raises(MemoryError):
        s.enable_reservoir(size)
    assert _bytes(s.reservoir()) == kept and s.reservoir_count() == 3 * N
    s.run_mcmc(st, 2, store=False)
    assert s.reservoir_count() == 5 * N and s.reservoir().step.size == 20


def test_read_to_unaligned_destination():
    s = _make()
    s.enable_reservoir(50)
    s.run_mcmc(_p0(), 6, store=False, skip_initial_state_check=True)
    r = s.reservoir()
    k = r.step.size
    buf = _lib.DeviceArray((k * D + 1,), s._device)
    lp = _lib.DeviceArray((k + 1,), s._device)
    step = np.zeros(k, dtype=np.uint64)
    walker = np.zeros(k, dtype=np.int64)
    rc = _lib.lib().eb_reservoir_read_to(s._engine._h, C.c_void_p(buf._ptr + 8), C.c_void_p(lp._ptr + 8),
                                         step.ctypes.data_as(C.POINTER(C.c_uint64)),
                                         walker.ctypes.data_as(C.POINTER(C.c_int64)))
    assert rc == 0
    assert buf.get()[1:].tobytes() == r.coords.reshape(-1).tobytes()
    assert lp.get()[1:].tobytes() == r.log_prob.tobytes()
    assert np.array_equal(step, r.step) and np.array_equal(walker, r.walker)
