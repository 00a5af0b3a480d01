"""CUDA arrays in and out of the sampler, the parts that need no GPU: ``State`` keeps CUDA-array-interface objects as
they are, ``DeviceArray`` exposes the interface (v3) it promises, and every argument the CUDA-array paths refuse is
refused before any call reaches the engine.  The engine is a recording stand-in (the pattern of
``test_blobs_host.py``), so the pointers below are never dereferenced."""
import ctypes as C
import copy

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import DeviceArray, State, _lib, models

N, D = 8, 3


class RecordingLib(object):
    """Every engine call is recorded with its arguments and succeeds; eb_device_alloc hands out fake pointers."""

    def __init__(self):
        self.calls = []
        self.next_ptr = 0x10000

    def eb_device_alloc(self, device, nbytes, out):
        self.calls.append(("eb_device_alloc", device, nbytes))
        if nbytes:
            out._obj.value = self.next_ptr
            self.next_ptr += 0x10000
        return 0

    def eb_last_error(self, h):
        return b""

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name,) + args)
            return 0

        return call

    def names(self):
        return [c[0] for c in self.calls]


@pytest.fixture
def fake(monkeypatch):
    lib = RecordingLib()
    monkeypatch.setattr(_lib, "lib", lambda: lib)
    return lib


class Producer(object):
    """A CUDA array as torch / CuPy present one: the interface dict and, optionally, a device."""

    def __init__(self, shape, typestr="<f8", strides=None, ptr=0xA000, stream="absent", mask=None, device=None,
                 version=3):
        cai = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "strides": strides,
               "version": version}
        if stream != "absent":
            cai["stream"] = stream
        if mask is not None:
            cai["mask"] = mask
        self.__cuda_array_interface__ = cai
        if device is not None:
            self.device = device


class TorchDevice(object):
    def __init__(self, index):
        self.type, self.index = "cuda", index


def _sampler(fake, **kw):
    s = emcee_b200.EnsembleSampler(N, D, kw.pop("model", models.GaussianIso()), seed=1, **kw)
    del fake.calls[:]
    return s


# ---- State ------------------------------------------------------------------------------------------------------
def test_state_keeps_cuda_arrays_unconverted():
    x, lp = Producer((N, D)), Producer((N,))
    s = State(x, log_prob=lp, random_state="r")
    assert s.coords is x and s.log_prob is lp
    again = State(s)
    assert again.coords is x and again.log_prob is lp
    one = Producer((D,))  # a single row is not made 2-D either: np.atleast_2d would download it
    assert State(one).coords is one
    assert State(np.zeros(D)).coords.shape == (1, D)  # host arrays keep the reference's atleast_2d


# ---- DeviceArray ------------------------------------------------------------------------------------------------
def test_device_array_interface(fake):
    a = DeviceArray((N, D), device=0)
    cai = a.__cuda_array_interface__
    assert cai == {"shape": (N, D), "typestr": "<f8", "data": (0x10000, False), "strides": None, "version": 3,
                   "stream": None}
    assert a.shape == (N, D) and a.dtype == np.float64 and a.device == 0 and a.nbytes == N * D * 8 and len(a) == N
    assert fake.calls == [("eb_device_alloc", 0, N * D * 8)]
    del a
    (name, device, ptr), = fake.calls[1:]
    assert name == "eb_device_free" and device == 0 and ptr.value == 0x10000
    e = DeviceArray((0, D), device=0)
    assert e.__cuda_array_interface__["data"] == (0, False) and e.__cuda_array_interface__["shape"] == (0, D)
    assert e.get().shape == (0, D)
    del e
    assert fake.names()[-1] == "eb_device_alloc"  # nothing to free


def test_empty_device_array_needs_no_device():
    e = DeviceArray((0,), device=0)  # the real library: zero bytes touch no device
    assert e.__cuda_array_interface__["data"][0] == 0 and e.get().shape == (0,)
    assert copy.deepcopy(e).shape == (0,)


def test_device_array_get_and_copy_are_one_copy_each(fake):
    a = DeviceArray((N,), device=0)
    a.get()
    name, device, dst, src, width, pitch, rows, stream = fake.calls[-1]
    assert name == "eb_device_copy" and src.value == 0x10000 and (width, pitch, rows, stream) == (N * 8, N * 8, 1, 0)
    b = copy.deepcopy(a)
    assert b.__cuda_array_interface__["data"][0] != a.__cuda_array_interface__["data"][0]
    name, device, dst, src = fake.calls[-1][:4]
    assert name == "eb_device_copy" and src.value == 0x10000 and dst.value == b.__cuda_array_interface__["data"][0]


# ---- argument validation: nothing reaches the engine --------------------------------------------------------------
@pytest.mark.parametrize(
    "coords, exc, match",
    [
        (Producer((N, D + 1)), ValueError, "incompatible input dimensions"),
        (Producer((N - 1, D)), ValueError, "incompatible input dimensions"),
        (Producer((N, D), typestr="<f4"), TypeError, "float64"),
        (Producer((N, D), mask=Producer((N, D), typestr="|b1")), ValueError, "masked"),
        (Producer((N, D), strides=(8 * D * 2, 16)), ValueError, "contiguous"),
        (Producer((N, D), strides=(8 * D - 8, 8)), ValueError, "stride"),
        (Producer((N, D), strides=(8 * D + 4, 8)), ValueError, "stride"),
        (Producer((N, D), device=1), ValueError, "device 1"),
        (Producer((N, D), device=TorchDevice(1)), ValueError, "device 1"),
    ],
)
def test_initial_state_validation_reaches_no_engine_call(fake, coords, exc, match):
    s = _sampler(fake)
    with pytest.raises(exc, match=match):
        s.run_mcmc(coords, 1, skip_initial_state_check=True)
    if coords.__cuda_array_interface__["shape"][0] == N:  # compute_log_prob takes any number of rows
        with pytest.raises(exc, match=match):
            s.compute_log_prob(coords)
    assert fake.calls == []


def test_log_prob_validation_and_mixed_states(fake):
    s = _sampler(fake)
    x = Producer((N, D))
    for lp, exc in ((Producer((N + 1,)), ValueError), (Producer((N,), typestr="<i8"), TypeError),
                    (Producer((N,), strides=(4,)), ValueError), (np.zeros(N), TypeError)):
        with pytest.raises(exc):
            s.run_mcmc(State(x, log_prob=lp), 1, skip_initial_state_check=True)
    with pytest.raises(TypeError, match="both"):
        s.run_mcmc(State(np.zeros((N, D)), log_prob=Producer((N,))), 1, skip_initial_state_check=True)
    assert fake.calls == []


def test_blobs_refused(fake):
    s = _sampler(fake, model=models.CudaArrayFunction(lambda x: x, blobs_dtype=float))
    with pytest.raises(NotImplementedError, match="blobs"):
        s.run_mcmc(State(Producer((N, D)), log_prob=Producer((N,)), blobs=np.zeros(N)), 1,
                   skip_initial_state_check=True)
    with pytest.raises(NotImplementedError, match="blobs_dtype"):
        s.compute_log_prob(Producer((N, D)))
    assert fake.calls == []


def test_cuda_results_with_pinned_results_refused(fake):
    with pytest.raises(ValueError, match="cuda_results"):
        emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), cuda_results=True, pinned_results=True)
    assert fake.calls == []


def test_sharded_refused(fake):
    s = _sampler(fake, cuda_results=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.attach(object())
    s = _sampler(fake)
    s._rdv = object()  # what attach leaves behind
    with pytest.raises(NotImplementedError, match="sharded"):
        s.run_mcmc(Producer((N, D)), 1, skip_initial_state_check=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        s.compute_log_prob(Producer((N, D)))
    assert fake.calls == []


def test_host_backend_takes_no_cuda_argument(fake):
    s = _sampler(fake)
    s.backend.iteration = 1
    s.backend.chain = np.zeros((1, N, D))
    s.backend.log_prob = np.zeros((1, N))
    for call in (lambda: s.get_chain(cuda=True), lambda: s.get_log_prob(cuda=True),
                 lambda: s.get_last_sample(cuda=True)):
        with pytest.raises(TypeError):
            call()


# ---- what reaches the engine ---------------------------------------------------------------------------------------
def test_upload_passes_strides_and_stream(fake):
    s = _sampler(fake, cuda_results=True)
    x = Producer((N, D), strides=(8 * D * 2, 8), ptr=0xB000, stream=77)
    lp = Producer((N,), strides=(16,), ptr=0xC000, stream=None)
    out = s.run_mcmc(State(x, log_prob=lp), 0, skip_initial_state_check=True)
    assert out is None
    (name, h, xp, xs, lpp, ls, stream), = [c for c in fake.calls if c[0] == "eb_set_state_from"]
    assert (xp.value, xs, lpp.value, ls, stream) == (0xB000, 16 * D, 0xC000, 16, 77)
    assert "eb_set_state" not in fake.names()
    del fake.calls[:]
    v2 = Producer((N, D), version=2)  # no stream entry (torch): the engine waits for the whole device
    s.run_mcmc(v2, 0, skip_initial_state_check=True)
    (name, h, xp, xs, lpp, ls, stream), = [c for c in fake.calls if c[0] == "eb_set_state_from"]
    assert lpp is None and xs == 8 * D and stream == _lib.EB_STREAM_UNKNOWN
    # the initial-state check downloads the rows once, in the producer's order, before the upload
    del fake.calls[:]
    with pytest.raises(ValueError, match="condition number"):
        s.run_mcmc(Producer((N, D), ptr=0xD000, stream=5), 1)  # the fake download leaves zeros: a zero span
    name, device, dst, src, width, pitch, rows, stream = fake.calls[0]
    assert name == "eb_device_copy" and (src.value, width, pitch, rows, stream) == (0xD000, 8 * D, 8 * D, N, 5)
    assert "eb_set_state_from" not in fake.names()


def test_cuda_results_and_compute_log_prob_return_device_arrays(fake):
    s = _sampler(fake, cuda_results=True)
    last = s.run_mcmc(Producer((N, D)), 2, store=False, skip_initial_state_check=True)
    assert isinstance(last.coords, DeviceArray) and isinstance(last.log_prob, DeviceArray)
    assert last.coords.shape == (N, D) and last.log_prob.shape == (N,)
    assert "eb_get_state_to" in fake.names() and "eb_get_state" not in fake.names()
    del fake.calls[:]
    lp, blobs = s.compute_log_prob(Producer((5, D), strides=(8 * D * 3, 8), ptr=0xE000, stream=9))
    assert blobs is None and isinstance(lp, DeviceArray) and lp.shape == (5,)
    (name, h, xp, xs, m, out, stream), = [c for c in fake.calls if c[0] == "eb_compute_log_prob_from"]
    assert (xp.value, xs, m, stream) == (0xE000, 24 * D, 5, 9)


def test_header_declares_the_cuda_array_abi():
    handle = C.CDLL(_lib.LIB_PATH)
    for name in ("eb_device_alloc", "eb_device_free", "eb_device_copy", "eb_set_state_from", "eb_get_state_to",
                 "eb_compute_log_prob_from", "eb_chain_read_to"):
        assert hasattr(handle, name), name
    assert _lib.lib().eb_abi_version() == 2
