"""CUDA arrays in and out of the sampler on the GPU: initial states, ``compute_log_prob``, ``cuda_results=True``
states and ``DeviceBackend`` reads with ``cuda=True``, against the host forms of the same calls.

* Twin runs, bit-exact: host-in / host-out against CUDA-in / CUDA-out with the same seed give equal bytes for every
  state, the accept counts and the stored chain, on a registered model (``tma_rows`` and ``dense_dmma``), a
  ``models.Bounded`` box and a ``CudaArrayFunction``, through ``run_mcmc`` (``thin_by > 1``) and ``sample``.
* Device reads equal host reads for every ``discard`` / ``thin`` / ``flat`` of a chain grown in three segments,
  the empty slice and ``get_last_sample`` included.
* ``compute_log_prob`` of CUDA arrays equals the host result; ``m = 0``, a strided first axis, the reference's
  errors for non-finite coordinates and a NaN initial log_prob.
* Ordering and ownership: an initial state written late on a torch side stream (interface v2 and a v3 object naming
  the stream), ``torch.as_tensor`` sharing a ``DeviceArray``'s pointer and outliving it, memory returned.
* Refusals: sharded samplers, CUDA-array states with blobs, blob functions in ``compute_log_prob``, pointers the
  engine cannot take.
"""
import gc

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import DeviceArray, DeviceBackend, State, models
from emcee_b200.dist import Rendezvous

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

SEED = 0xCA1


def _torch_iso(rows):
    x = torch.as_tensor(rows, device="cuda")
    return (x * x).sum(dim=1) * -0.5


def _dense(D):
    rng = np.random.default_rng(D)
    a = rng.standard_normal((D, D))
    return models.GaussianDense(np.linalg.inv(a @ a.T / D + np.eye(D)), np.linspace(-1, 1, D))


CASES = {
    # name: (N, D, model, kernel the steps run)
    "tma_rows": (64, 8, lambda: models.GaussianIso(), "tma_rows"),
    "dense_dmma": (96, 16, lambda: _dense(16), "dense_dmma"),
    "bounded": (64, 6, lambda: models.Bounded(models.GaussianIso(), -np.ones(6), np.ones(6)), None),
    "cuda_function": (48, 5, lambda: models.CudaArrayFunction(_torch_iso), "callback"),
}


def _p0(N, D, seed=1):
    return np.random.default_rng(seed).uniform(-0.8, 0.8, (N, D))


def _host(a):
    return a.get() if isinstance(a, DeviceArray) else np.asarray(a)


def _same(a, b):
    a, b = _host(a), _host(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("case", sorted(CASES))
def test_twin_runs_bit_exact(case):
    N, D, make, kernel = CASES[case]
    p0 = _p0(N, D)
    h = emcee_b200.EnsembleSampler(N, D, make(), seed=SEED, backend=DeviceBackend())
    d = emcee_b200.EnsembleSampler(N, D, make(), seed=SEED, backend=DeviceBackend(), cuda_results=True)
    lh = h.run_mcmc(p0, 5, thin_by=2)
    ld = d.run_mcmc(torch.as_tensor(p0, device="cuda"), 5, thin_by=2)  # the initial-state check downloads once
    assert isinstance(ld.coords, DeviceArray) and isinstance(ld.log_prob, DeviceArray)
    _same(lh.coords, ld.coords)
    _same(lh.log_prob, ld.log_prob)
    assert lh.random_state == ld.random_state
    if kernel is not None:
        assert d._engine.last_kernel_name() == kernel
    # the sample generator from the returned states, and a resume from the stored DeviceArray state
    for a, b in zip(h.sample(lh, iterations=3, thin_by=2), d.sample(ld, iterations=3, thin_by=2,
                                                                     skip_initial_state_check=True)):
        assert isinstance(b.coords, DeviceArray)
        _same(a.coords, b.coords)
        _same(a.log_prob, b.log_prob)
    _same(h.run_mcmc(None, 2).coords, d.run_mcmc(None, 2).coords)
    assert np.array_equal(h._engine.naccepted(), d._engine.naccepted())
    assert h.backend.accepted.tobytes() == d.backend.accepted.tobytes()
    assert h.iteration == d.iteration == 5 + 3 + 2
    _same(h.get_chain(), d.get_chain())
    _same(h.get_chain(), d.get_chain(cuda=True))
    _same(h.get_log_prob(), d.get_log_prob(cuda=True))


def _grown_in_three_segments():
    N, D = 40, 6
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED, backend=DeviceBackend())
    s.run_mcmc(_p0(N, D), 4, skip_initial_state_check=True)
    s.run_mcmc(None, 3)
    s.run_mcmc(None, 5)
    return s


def test_device_reads_equal_host_reads():
    s = _grown_in_three_segments()
    b = s.backend
    it = b.iteration
    for discard in sorted({0, 1, 3, 4, it // 2, it - 1, it, it + 4}):
        for thin in (1, 2, 3, 7):
            for flat in (False, True):
                kw = dict(discard=discard, thin=thin, flat=flat)
                for name in ("chain", "log_prob"):
                    host = b.get_value(name, **kw)
                    dev = b.get_value(name, cuda=True, **kw)
                    assert isinstance(dev, DeviceArray) and dev.shape == host.shape, kw
                    _same(host, dev)
                _same(s.get_chain(**kw), s.get_chain(cuda=True, **kw))
                _same(s.get_log_prob(**kw), s.get_log_prob(cuda=True, **kw))
    empty = s.get_chain(discard=it, cuda=True)
    assert empty.shape == (0, 40, 6) and empty.__cuda_array_interface__["data"][0] == 0
    lh, ld = s.get_last_sample(), s.get_last_sample(cuda=True)
    assert isinstance(ld.coords, DeviceArray) and ld.random_state == lh.random_state
    _same(lh.coords, ld.coords)
    _same(lh.log_prob, ld.log_prob)
    assert s.get_blobs(cuda=True) is None


@pytest.mark.parametrize("case", ["tma_rows", "dense_dmma", "cuda_function"])
def test_compute_log_prob_on_cuda_arrays(case):
    N, D, make, _ = CASES[case]
    s = emcee_b200.EnsembleSampler(N, D, make(), seed=SEED)
    x = np.random.default_rng(2).standard_normal((33, D))
    host, _ = s.compute_log_prob(x)
    dev, blobs = s.compute_log_prob(torch.as_tensor(x, device="cuda"))
    assert blobs is None and isinstance(dev, DeviceArray)
    _same(host, dev)
    wide = torch.zeros((33, 2 * D), dtype=torch.float64, device="cuda")
    wide[:, :D] = torch.as_tensor(x, device="cuda")
    _same(host, s.compute_log_prob(wide[:, :D])[0])  # rows 2 D apart
    _same(s.compute_log_prob(x[::3])[0], s.compute_log_prob(torch.as_tensor(x, device="cuda")[::3])[0])
    none, _ = s.compute_log_prob(torch.zeros((0, D), dtype=torch.float64, device="cuda"))
    assert none.shape == (0,) and none.get().shape == (0,)
    bad = torch.as_tensor(x, device="cuda").clone()
    bad[4, 1] = float("inf")
    with pytest.raises(ValueError, match="infinite"):
        s.compute_log_prob(bad)
    bad[4, 1] = float("nan")
    with pytest.raises(ValueError, match="NaN"):
        s.compute_log_prob(bad)


def test_nan_initial_log_prob_from_a_cuda_array():
    N, D = 32, 4
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED)
    x = torch.as_tensor(_p0(N, D), device="cuda")
    lp = torch.zeros(N, dtype=torch.float64, device="cuda")
    lp[17] = float("nan")
    with pytest.raises(ValueError, match="The initial log_prob was NaN"):
        s.run_mcmc(State(x, log_prob=lp), 1)
    # a given log_prob is taken as it is, like the host form
    lp[17] = 0.0
    h = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED)
    _same(h.run_mcmc(State(x.cpu().numpy(), log_prob=lp.cpu().numpy()), 3).coords,
          s.run_mcmc(State(x, log_prob=lp), 3).coords)


class V3(object):
    """A v3 interface naming the stream the values are written on."""

    def __init__(self, t, stream):
        cai = dict(t.__cuda_array_interface__)
        cai.update(version=3, stream=stream.cuda_stream or 1)
        self.__cuda_array_interface__ = cai
        self.t = t


@pytest.mark.parametrize("mode", ["v2", "v3"])
@pytest.mark.parametrize("check", [False, True])
def test_initial_state_written_late_on_a_side_stream(mode, check):
    N, D = 64, 8
    p0 = _p0(N, D)
    want = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED).run_mcmc(p0, 3, store=False)
    src = torch.as_tensor(p0, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        t = torch.zeros((N, D), dtype=torch.float64, device="cuda")
        torch.cuda._sleep(20_000_000)  # ~10 ms before the final write
        t.copy_(src)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED, cuda_results=True)
    got = s.run_mcmc(t if mode == "v2" else V3(t, side), 3, store=False, skip_initial_state_check=not check)
    _same(want.coords, got.coords)
    _same(want.log_prob, got.log_prob)


def test_device_arrays_are_shared_and_outlive_their_reference():
    N, D = 64, 8
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED, backend=DeviceBackend(), cuda_results=True)
    last = s.run_mcmc(_p0(N, D), 4, skip_initial_state_check=True)
    a = s.get_chain(cuda=True)
    want = a.get()
    t = torch.as_tensor(a, device="cuda")
    assert t.data_ptr() == a.__cuda_array_interface__["data"][0] and t.shape == a.shape
    c = torch.as_tensor(last.coords, device="cuda")
    assert c.data_ptr() == last.coords.__cuda_array_interface__["data"][0]
    want_c = last.coords.get()
    del a, last
    s._previous_state = None
    gc.collect()
    junk = [s.get_chain(cuda=True) for _ in range(4)]  # fresh allocations that would reuse freed memory
    for j in junk:
        j.__cuda_array_interface__
    assert np.array_equal(t.cpu().numpy(), want) and np.array_equal(c.cpu().numpy(), want_c)
    # and a consumer's own work on the array is visible through the interface
    t.mul_(2.0)
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), 2.0 * want)


def test_repeated_reads_return_the_memory():
    N, D = 4096, 64
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED, backend=DeviceBackend())
    s.run_mcmc(np.random.default_rng(3).standard_normal((N, D)), 32, skip_initial_state_check=True)
    nbytes = 32 * N * D * 8  # 64 MiB a read
    a = s.get_chain(cuda=True)
    del a
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        a = s.get_chain(cuda=True)
        assert a.nbytes == nbytes
        del a
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < nbytes  # less than one read's worth: nothing accumulates


def test_refusals():
    N, D = 32, 4
    x = torch.as_tensor(_p0(N, D), device="cuda")
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED, cuda_results=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(Rendezvous())
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED)
    s.attach(Rendezvous())
    with pytest.raises(NotImplementedError, match="sharded"):
        s.run_mcmc(x, 1, skip_initial_state_check=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.compute_log_prob(x)
    blob_fn = models.CudaArrayFunction(lambda rows: (_torch_iso(rows), torch.as_tensor(rows, device="cuda")[:, 0]),
                                       blobs_dtype=np.float64)
    b = emcee_b200.EnsembleSampler(N, D, blob_fn, seed=SEED)
    with pytest.raises(NotImplementedError, match="blobs"):
        b.run_mcmc(State(x, log_prob=torch.zeros(N, dtype=torch.float64, device="cuda"), blobs=np.zeros(N)), 1,
                   skip_initial_state_check=True)
    with pytest.raises(NotImplementedError, match="blobs_dtype"):
        b.compute_log_prob(x)
    # without a given log_prob the function's blobs of the initial evaluation become the state's, on the host
    st = b.run_mcmc(x, 2, skip_initial_state_check=True)
    assert isinstance(st.blobs, np.ndarray) and st.blobs.shape == (N,)


class HostMemory(object):
    """Host memory posing as a CUDA array: the engine checks the pointer itself."""

    def __init__(self, a):
        self.a = a
        self.__cuda_array_interface__ = {"shape": a.shape, "typestr": "<f8", "data": (a.ctypes.data, False),
                                         "strides": None, "version": 3, "stream": None}


def test_engine_refuses_memory_it_cannot_take():
    N, D = 32, 4
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=SEED)
    with pytest.raises(ValueError, match="not device memory"):
        s.run_mcmc(HostMemory(_p0(N, D)), 1, skip_initial_state_check=True)
    with pytest.raises(ValueError, match="not device memory"):
        s.compute_log_prob(HostMemory(_p0(N, D)))
    # the sampler is still usable
    assert s.run_mcmc(torch.as_tensor(_p0(N, D), device="cuda"), 1, skip_initial_state_check=True) is not None
