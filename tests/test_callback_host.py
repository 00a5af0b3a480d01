"""User log-probability functions, the parts that need no GPU: the wrappers' validation and
semantics (the reference's ``_scalar`` and blob rules, ``ensemble.py:486-512,703-713``), the
sampler's refusals, the ctypes trampoline against host buffers, and pickling."""
import ctypes as C
import pickle

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models


def _iso(x):
    return -0.5 * np.sum(np.asarray(x) ** 2, axis=-1)


def _shift(x, c, scale=1.0):
    return -0.5 * scale * np.sum((np.asarray(x) - c) ** 2, axis=-1)


class RecordingPool(object):
    def __init__(self):
        self.calls = 0

    def map(self, f, it):
        self.calls += 1
        return list(map(f, it))


# ---- wrappers ---------------------------------------------------------------------------
def test_wrapper_validation():
    with pytest.raises(TypeError):
        models.HostFunction(3.0)
    with pytest.raises(TypeError):
        models.CudaArrayFunction("not callable")
    with pytest.raises(TypeError):
        models.HostFunction(_iso, pool=object())
    h = models.HostFunction(_iso, vectorize=True, args=(1,), kwargs={"k": 2})
    assert h.where == "host" and h.vectorize and h.args == [1] and h.kwargs == {"k": 2}
    assert models.CudaArrayFunction(_iso).where == "device"
    # neither is a registered device model, so Bounded refuses them as before
    for w in (models.HostFunction(_iso), models.CudaArrayFunction(_iso)):
        with pytest.raises(TypeError):
            models.Bounded(w, -1.0, 1.0)


def test_plain_callables_still_refused_before_any_gpu():
    with pytest.raises(TypeError, match="HostFunction"):
        emcee_b200.EnsembleSampler(32, 5, _iso)
    with pytest.raises(TypeError, match="CudaArrayFunction"):
        emcee_b200.EnsembleSampler(32, 5, lambda x: 0.0)
    # the sampler's own pool / args / kwargs stay refused: they belong to the wrapper
    h = models.HostFunction(_iso)
    with pytest.raises(NotImplementedError, match="HostFunction"):
        emcee_b200.EnsembleSampler(32, 5, h, pool=RecordingPool())
    with pytest.raises(NotImplementedError):
        emcee_b200.EnsembleSampler(32, 5, h, args=(1,))
    with pytest.raises(NotImplementedError):
        emcee_b200.EnsembleSampler(32, 5, h, kwargs={"a": 1})
    with pytest.raises(NotImplementedError):
        emcee_b200.EnsembleSampler(32, 5, h, parameter_names=["a"] * 5)
    with pytest.raises(NotImplementedError):
        emcee_b200.EnsembleSampler(32, 5, h, blobs_dtype=float)


def test_vectorized_map_and_pool_agree():
    x = np.random.default_rng(0).standard_normal((7, 3))
    ref = _shift(x, 0.5, scale=2.0)
    vec = models.HostFunction(_shift, vectorize=True, args=(0.5,), kwargs={"scale": 2.0})
    row = models.HostFunction(_shift, args=(0.5,), kwargs={"scale": 2.0})
    pool = RecordingPool()
    pooled = models.HostFunction(_shift, pool=pool, args=(0.5,), kwargs={"scale": 2.0})
    for w in (vec, row, pooled):
        out = w.evaluate(x.copy())
        assert out.dtype == np.float64 and out.shape == (7,)
        assert np.array_equal(out, ref)
    assert pool.calls == 1


@pytest.mark.parametrize(
    "value, expected",
    [(1.5, 1.5), (np.float64(2.5), 2.5), (np.array([3.5]), 3.5), (np.array(4.5), 4.5), (7, 7.0),
     (np.float32(0.25), 0.25), (-np.inf, -np.inf)],
)
def test_scalar_rule(value, expected):
    f = models.HostFunction(lambda x: value)
    out = f.evaluate(np.zeros((3, 2)))
    assert out.dtype == np.float64 and np.array_equal(out, [expected] * 3)


def test_non_scalar_results_are_refused():
    with pytest.raises(ValueError, match="should return scalar"):
        models.HostFunction(lambda x: np.array([[1.0, 2.0]])).evaluate(np.zeros((2, 2)))
    with pytest.raises(ValueError):  # a string sniffs as blobs, then its first character is no float
        models.HostFunction(lambda x: "abc").evaluate(np.zeros((2, 2)))


@pytest.mark.parametrize("result", [lambda x: (0.0, 1.0), lambda x: [0.0, "blob"], lambda x: np.array([0.0, 1.0])])
def test_blobs_are_detected_and_refused(result):
    with pytest.raises(NotImplementedError, match="blobs"):
        models.HostFunction(result).evaluate(np.zeros((2, 2)))
    with pytest.raises(NotImplementedError, match="blobs"):
        models.HostFunction(lambda x: [result(r) for r in x], vectorize=True).evaluate(np.zeros((2, 2)))


def test_vectorized_result_rules():
    # a [M, 1] result: every row is a length-1 sequence -> no blobs, _scalar of each
    f = models.HostFunction(lambda x: -np.sum(x, axis=1, keepdims=True), vectorize=True)
    assert np.array_equal(f.evaluate(np.ones((3, 2))), [-2.0, -2.0, -2.0])
    ints = models.HostFunction(lambda x: np.arange(len(x)), vectorize=True)
    out = ints.evaluate(np.ones((3, 2)))
    assert out.dtype == np.float64 and np.array_equal(out, [0.0, 1.0, 2.0])


# ---- the trampoline against host buffers ----------------------------------------------
def _call(cb, x, lp):
    m, d = x.shape
    return cb(None, x.ctypes.data_as(_lib._dp), m, d, lp.ctypes.data_as(_lib._dp), None)


def test_host_trampoline_copies_rows_and_results():
    seen = []

    def evaluate(rows):
        seen.append(rows)
        out = -rows.sum(axis=1)
        rows[:] = 99.0  # the function owns its array: the engine's buffer is unaffected
        return out

    failure = [None]
    cb = _lib.make_trampoline(None, evaluate, _lib.EB_CALLBACK_HOST, failure)
    x = np.arange(12.0).reshape(4, 3)
    lp = np.full(4, np.nan)
    assert _call(cb, x, lp) == 0 and failure[0] is None
    assert np.array_equal(lp, -np.arange(12.0).reshape(4, 3).sum(axis=1))
    assert np.array_equal(x, np.arange(12.0).reshape(4, 3))
    assert seen[0].flags.owndata and seen[0].shape == (4, 3) and seen[0].dtype == np.float64


def test_host_trampoline_captures_exceptions():
    class Boom(Exception):
        pass

    def evaluate(rows):
        raise Boom("user error")

    failure = [None]
    cb = _lib.make_trampoline(None, evaluate, _lib.EB_CALLBACK_HOST, failure)
    x, lp = np.zeros((2, 2)), np.zeros(2)
    assert _call(cb, x, lp) != 0
    assert isinstance(failure[0], Boom) and failure[0].__traceback__ is not None


@pytest.mark.parametrize(
    "out, exc",
    [(np.zeros(3), ValueError), (np.zeros((2, 1)), ValueError), (np.zeros(2, dtype=np.float32), TypeError),
     (np.zeros(2, dtype=np.complex128), TypeError)],
)
def test_trampoline_checks_shape_and_dtype(out, exc):
    for where in (_lib.EB_CALLBACK_HOST, _lib.EB_CALLBACK_DEVICE):
        failure = [None]
        cb = _lib.make_trampoline(None, lambda rows: out, where, failure)
        x, lp = np.zeros((2, 2)), np.full(2, 7.0)
        assert _call(cb, x, lp) != 0
        assert isinstance(failure[0], exc), failure[0]
        assert np.array_equal(lp, [7.0, 7.0])  # nothing was written


def test_device_rows_interface_is_valid_only_during_the_call():
    kept = []

    def evaluate(rows):
        cai = rows.__cuda_array_interface__
        assert cai["shape"] == (2, 3) and cai["typestr"] == "<f8" and cai["version"] == 3
        assert cai["data"][1] is False and cai["stream"] == 1234
        kept.append(rows)
        return np.zeros(5)  # wrong shape: refused before any copy is attempted

    failure = [None]
    cb = _lib.make_trampoline(None, evaluate, _lib.EB_CALLBACK_DEVICE, failure)
    x, lp = np.zeros((2, 3)), np.zeros(2)
    assert cb(None, x.ctypes.data_as(_lib._dp), 2, 3, lp.ctypes.data_as(_lib._dp), C.c_void_p(1234)) != 0
    assert isinstance(failure[0], ValueError)
    with pytest.raises(RuntimeError, match="only valid during the call"):
        kept[0].__cuda_array_interface__


def test_engine_reraises_the_stored_exception_unchanged():
    class Boom(Exception):
        pass

    eng = _lib.Engine.__new__(_lib.Engine)  # no device: only the error mapping is exercised
    eng._h = C.c_void_p()
    err = Boom("from the callback")
    eng._cb_failure = [err]
    with pytest.raises(Boom) as info:
        eng._check(_lib.EB_ERR_CALLBACK)
    assert info.value is err and eng._cb_failure[0] is None


# ---- pickling ----------------------------------------------------------------------------
def test_pickling_drops_the_pool():
    pool = RecordingPool()
    h = models.HostFunction(_shift, vectorize=False, pool=pool, args=(0.5,), kwargs={"scale": 3.0})
    h2 = pickle.loads(pickle.dumps(h))
    assert h2.pool is None and h.pool is pool
    assert h2.fn is _shift and h2.args == [0.5] and h2.kwargs == {"scale": 3.0} and not h2.vectorize
    x = np.ones((3, 2))
    assert np.array_equal(h2.evaluate(x), h.evaluate(x))
    c2 = pickle.loads(pickle.dumps(models.CudaArrayFunction(_iso, args=(1,))))
    assert c2.fn is _iso and c2.args == [1] and c2.where == "device"


def test_header_declares_the_callback_abi():
    import os
    import re

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "emcee_b200.h")).read()
    assert re.search(r"EB_ERR_CALLBACK\s*=\s*-7", text)
    assert "#define EB_CALLBACK_HOST 0" in text and "#define EB_CALLBACK_DEVICE 1" in text
    handle = C.CDLL(_lib.LIB_PATH)
    assert hasattr(handle, "eb_model_set_callback") and hasattr(handle, "eb_callback_result")
    assert _lib.lib().eb_abi_version() == 2


class _Producer(object):
    def __init__(self, cai):
        self.__cuda_array_interface__ = cai


@pytest.mark.parametrize(
    "extra, stream",
    [({}, _lib.EB_STREAM_UNKNOWN),  # interface v2 (torch): no word on ordering -> wait for the whole device
     ({"version": 3, "stream": None}, 0), ({"version": 3, "stream": 1}, 1), ({"version": 3, "stream": 2}, 2),
     ({"version": 3, "stream": 0x7F00}, 0x7F00)],
)
def test_device_result_stream_encoding(monkeypatch, extra, stream):
    calls = []

    class FakeLib(object):
        def eb_callback_result(self, h, lp, src, stride, m, src_stream):
            calls.append((src.value, stride, m, src_stream))
            return 0

    monkeypatch.setattr(_lib, "lib", lambda: FakeLib())
    cai = {"shape": (4,), "typestr": "<f8", "data": (0x1000, False), "strides": (16,), "version": 2}
    cai.update(extra)
    _lib._device_result(None, None, _Producer(cai), 4)
    assert calls == [(0x1000, 16, 4, stream)]
