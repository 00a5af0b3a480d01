"""Blobs of user log-probability functions, the parts that need no GPU: the wrappers' blob rules
(restated from the reference's ``ensemble.py:498-547``), the fixed-width refusals, ``Backend``'s blob
storage (``backends/backend.py:157-231``), the trampoline handing records to the engine, and the
sampler's refusals."""
import ctypes as C
import pickle

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models
from emcee_b200.backend import Backend
from emcee_b200.state import State


def _lp(x):
    return -0.5 * float(np.sum(np.asarray(x) ** 2))


class Pool(object):
    def map(self, f, it):
        return list(map(f, it))


X = np.random.default_rng(0).standard_normal((6, 3))


# ---- the wrappers' blob rules (ensemble.py:498-547) ---------------------------------------------------
# blob = [r[1:] for r in results if len(r) > 1] (:506); log_prob = _scalar(r[0]) (:509); np.array(blob, dtype)
# (:535); size-1 axes after the first squeezed (:538-545).
@pytest.mark.parametrize(
    "blob_fn, shape",
    [  # the numeric cases of the reference's tests/unit/test_blobs.py::test_blob_shape
        (lambda x: np.arange(5.0) + x[0], (5,)),
        (lambda x: np.ones((5, 3)) * x[1], (5, 3)),
        (lambda x: np.ones((1, 5, 1, 3, 1)) * x[2], (5, 3)),
        (lambda x: float(x[0]), ()),
    ],
)
@pytest.mark.parametrize("how", ["map", "pool", "vectorize"])
def test_blob_shapes(blob_fn, shape, how):
    fn = lambda x: (_lp(x), blob_fn(x))  # noqa: E731
    if how == "vectorize":
        w = models.HostFunction(lambda xs: [fn(r) for r in xs], vectorize=True, blobs_dtype=float)
    else:
        w = models.HostFunction(fn, pool=Pool() if how == "pool" else None, blobs_dtype=float)
    lp, blobs = w.evaluate(X.copy())
    assert lp.dtype == np.float64 and np.array_equal(lp, [_lp(r) for r in X])
    assert blobs.dtype == np.float64 and blobs.shape == (6,) + shape
    for r, b in zip(X, blobs):
        assert np.array_equal(b, np.reshape(blob_fn(r), shape))


def test_vectorized_array_and_pair_results():
    # a [M, 1 + k] array: column 0 is log_prob, the rest each row's blob
    arr = models.HostFunction(lambda x: np.column_stack([-x.sum(1), x, 2 * x]), vectorize=True, blobs_dtype="f8")
    lp, b = arr.evaluate(X.copy())
    assert np.array_equal(lp, -X.sum(1)) and np.array_equal(b, np.column_stack([X, 2 * X]))
    # per-row (lp, a, b) tuples into a structured dtype
    dt = np.dtype([("a", "f8"), ("n", "i1")])
    rec = models.HostFunction(lambda x: (_lp(x), x[0], int(x[1] > 0)), blobs_dtype=dt)
    lp, b = rec.evaluate(X.copy())
    assert b.dtype == dt and b.shape == (6,) and np.array_equal(b["a"], X[:, 0])
    assert np.array_equal(b["n"], (X[:, 1] > 0).astype(np.int8))
    # a function declared with blobs that returns none: the trampoline refuses it (below); evaluate says None
    assert models.HostFunction(_lp, blobs_dtype=float).evaluate(X.copy())[1] is None


@pytest.mark.parametrize("dtype", [object, str, "U4", "S3", [("a", "f8"), ("s", "S2")], [("o", "O")]])
def test_variable_width_dtypes_refused(dtype):
    for cls in (models.HostFunction, models.CudaArrayFunction):
        with pytest.raises(NotImplementedError, match="fixed-width"):
            cls(_lp, blobs_dtype=dtype)


@pytest.mark.parametrize(
    "blob_fn",
    [lambda x: "face", lambda x: object(), lambda x: ("face", "surface"), lambda x: (np.ones(5), "face"),
     lambda x: np.ones(3 + int(x[0] > 0))],  # the reference's string / object / ragged cases, and ragged rows
)
def test_string_object_ragged_blobs_refused(blob_fn):
    w = models.HostFunction(lambda x: (_lp(x), blob_fn(x)), blobs_dtype=float)
    with pytest.raises(NotImplementedError, match="fixed-width"):
        w.evaluate(X.copy())


def test_wrappers_keep_blobs_dtype_through_pickling():
    h = pickle.loads(pickle.dumps(models.HostFunction(_lp, pool=Pool(), blobs_dtype=[("a", "<f4"), ("b", "i1")])))
    assert h.pool is None and h.blobs_dtype == np.dtype([("a", "<f4"), ("b", "i1")]) and h.blobs_dtype.itemsize == 5
    assert models.HostFunction(_lp).blobs_dtype is None


# ---- sampler refusals -------------------------------------------------------------------------------------------
def test_sampler_refusals_point_to_the_wrappers():
    with pytest.raises(NotImplementedError, match="blobs_dtype=") as info:
        emcee_b200.EnsembleSampler(32, 5, models.HostFunction(_lp), blobs_dtype=float)
    assert "HostFunction" in str(info.value)
    for cls in (models.HostFunction, models.CudaArrayFunction):
        with pytest.raises(NotImplementedError, match=r"Backend\(\)"):
            emcee_b200.EnsembleSampler(32, 5, cls(_lp, blobs_dtype=float), backend=emcee_b200.DeviceBackend())


# ---- Backend blob storage (backends/backend.py:157-231) -------------------------------------------------------
def _state(k, blobs):
    return State(np.full((4, 2), float(k)), log_prob=np.full(4, -float(k)), blobs=blobs, random_state=("r", k))


def test_backend_grow_save_and_read():
    b = Backend()
    b.reset(4, 2)
    dt = np.dtype([("a", "f8"), ("n", "i1")])
    blobs = np.zeros((4, 3), dtype=dt)
    b.grow(2, blobs)  # dtype (blobs.dtype, blobs.shape[1:]) (backend.py:178)
    assert b.has_blobs() and b.blobs.shape == (2, 4, 3) and b.blobs.dtype == dt
    for k in range(2):
        v = np.zeros((4, 3), dtype=dt)
        v["a"] = k
        b.save_step(_state(k, v), np.ones(4, dtype=bool))
    b.grow(3, blobs)  # concatenated (backend.py:180-185): stored records stay
    assert b.blobs.shape == (5, 4, 3) and np.all(b.blobs["a"][1] == 1)
    for k in range(2, 5):
        v = np.zeros((4, 3), dtype=dt)
        v["a"] = k
        b.save_step(_state(k, v), np.zeros(4, dtype=bool))
    assert b.get_blobs().shape == (5, 4, 3)
    assert np.array_equal(b.get_blobs(discard=1, thin=2)["a"][:, 0, 0], [2.0, 4.0])
    assert b.get_blobs(flat=True).shape == (20, 3)
    last = b.get_last_sample()
    assert np.all(last.blobs["a"] == 4) and last.blobs.shape == (4, 3) and len(last) == 4
    b2 = pickle.loads(pickle.dumps(b))
    assert np.array_equal(b2.get_blobs(), b.get_blobs()) and b2.has_blobs()


def test_backend_inconsistent_blobs():
    b = Backend()
    b.reset(4, 2)
    b.grow(1, np.zeros(4))
    with pytest.raises(ValueError, match="inconsistent use of blobs"):  # backend.py:159-160
        b.grow(1, None)
    with pytest.raises(ValueError, match="inconsistent use of blobs"):
        b.save_step(_state(0, None), np.zeros(4, dtype=bool))
    with pytest.raises(ValueError, match="invalid blobs size"):
        b.save_step(_state(0, np.zeros(3)), np.zeros(4, dtype=bool))
    with pytest.raises(ValueError):  # another record shape (the reference's concatenate fails)
        b.grow(1, np.zeros((4, 2)))
    with pytest.raises(ValueError):  # another dtype of the same size
        b.grow(1, np.zeros(4, dtype=np.int64))
    c = Backend()
    c.reset(4, 2)
    c.grow(1, None)
    c.save_step(_state(0, None), np.zeros(4, dtype=bool))
    with pytest.raises(ValueError, match="inconsistent use of blobs"):  # backend.py:161-162
        c.grow(1, np.zeros(4))
    with pytest.raises(ValueError):
        c.save_step(_state(1, np.zeros(4)), np.zeros(4, dtype=bool))


# ---- the trampoline hands the records to the engine -----------------------------------------------------------
class FakeLib(object):
    def __init__(self):
        self.calls = []

    def eb_callback_blobs(self, h, src, rec, stride, m, stream):
        data = C.string_at(src.value, stride * (m - 1) + rec) if m else b""
        self.calls.append((rec, stride, m, stream, data))
        return 0

    def eb_callback_result(self, h, lp, src, stride, m, stream):
        return 0


def _tramp(monkeypatch, evaluate, where, expect=None, dtype="f8"):
    fake = FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    sink = _lib.BlobSink(dtype)
    sink.expect = expect
    failure = [None]
    cb = _lib.make_trampoline(None, evaluate, where, failure, sink)
    x, lp = np.arange(6.0).reshape(3, 2), np.zeros(3)
    rc = cb(None, x.ctypes.data_as(_lib._dp), 3, 2, lp.ctypes.data_as(_lib._dp), None)
    return rc, failure[0], fake, sink, lp


def test_host_trampoline_writes_blobs(monkeypatch):
    dt = np.dtype([("s", "f8"), ("f", "i1")])
    w = models.HostFunction(lambda x: (-x.sum(), x.sum(), int(x[0] > 1)), blobs_dtype=dt)
    rc, err, fake, sink, lp = _tramp(monkeypatch, w.evaluate, _lib.EB_CALLBACK_HOST, dtype=dt)
    assert rc == 0 and err is None
    assert np.array_equal(lp, [-1.0, -5.0, -9.0])
    (rec, stride, m, stream, data), = fake.calls
    assert (rec, stride, m, stream) == (9, 9, 3, 0) and sink.last == (dt, ())
    got = np.frombuffer(data, dtype=dt)
    assert np.array_equal(got["s"], [1.0, 5.0, 9.0]) and np.array_equal(got["f"], [0, 1, 1])


def test_trampoline_refuses_missing_or_changed_blobs(monkeypatch):
    none = models.HostFunction(lambda x: -x.sum(), blobs_dtype="f8")
    rc, err, fake, _, lp = _tramp(monkeypatch, none.evaluate, _lib.EB_CALLBACK_HOST)
    assert rc != 0 and isinstance(err, ValueError) and "no blobs" in str(err) and not fake.calls
    two = models.HostFunction(lambda x: (-x.sum(), x), blobs_dtype="f8")
    rc, err, fake, _, _ = _tramp(monkeypatch, two.evaluate, _lib.EB_CALLBACK_HOST, expect=(np.dtype("f8"), (3,)))
    assert rc != 0 and isinstance(err, ValueError) and "shape" in str(err) and not fake.calls


class _Producer(object):
    def __init__(self, cai):
        self.__cuda_array_interface__ = cai


def test_device_trampoline_strides_and_streams(monkeypatch):
    lp_cai = {"shape": (3,), "typestr": "<f8", "data": (0x1000, False), "strides": None, "version": 2}
    buf = np.arange(24.0)  # host memory posing as a device array: only the pointer arithmetic is checked
    cai = {"shape": (3, 2), "typestr": "<f8", "data": (buf.ctypes.data, False), "strides": (64, 8), "version": 3,
           "stream": 77}
    rc, err, fake, sink, _ = _tramp(monkeypatch, lambda rows: (_Producer(lp_cai), _Producer(cai)),
                                    _lib.EB_CALLBACK_DEVICE)
    assert rc == 0 and err is None
    rec, stride, m, stream, _ = fake.calls[0]
    assert (rec, stride, m, stream) == (16, 64, 3, 77) and sink.last == (np.dtype("f8"), (2,))
    v2 = dict(cai, version=2)
    del v2["stream"]
    rc, _, fake, _, _ = _tramp(monkeypatch, lambda rows: (_Producer(lp_cai), _Producer(v2)), _lib.EB_CALLBACK_DEVICE)
    assert rc == 0 and fake.calls[0][3] == _lib.EB_STREAM_UNKNOWN
    bad = dict(cai, strides=(64, 16))  # a record that is not contiguous
    rc, err, _, _, _ = _tramp(monkeypatch, lambda rows: (_Producer(lp_cai), _Producer(bad)), _lib.EB_CALLBACK_DEVICE)
    assert rc != 0 and isinstance(err, ValueError) and "contiguous" in str(err)
    f4 = dict(cai, typestr="<f4")
    rc, err, _, _, _ = _tramp(monkeypatch, lambda rows: (_Producer(lp_cai), _Producer(f4)), _lib.EB_CALLBACK_DEVICE)
    assert rc != 0 and isinstance(err, TypeError)


class RecordingLib(object):
    """Every engine call is recorded and succeeds."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append(name)
            return 0

        return call


def _engine_without_device(monkeypatch, blobs_dtype):
    fake = RecordingLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    eng = _lib.Engine.__new__(_lib.Engine)
    eng._h, eng._cb_failure, eng.nwalkers, eng.ndim = C.c_void_p(), [None], 4, 2
    eng._blob_sink = None if blobs_dtype is None else _lib.BlobSink(blobs_dtype)
    eng._blob_layout = None
    return eng, fake


@pytest.mark.parametrize(
    "blobs",
    [np.array([object()] * 4, dtype=object),  # the reference's default for mixed blobs
     np.zeros(4, dtype=[("a", "f8"), ("o", "O")]),  # an object field
     np.array(["ab"] * 4)],
)
def test_state_blobs_of_variable_width_refused_before_upload(monkeypatch, blobs):
    eng, fake = _engine_without_device(monkeypatch, "f8")
    with pytest.raises(NotImplementedError, match="fixed-width"):
        eng.set_state(np.zeros((4, 2)), np.zeros(4), blobs)
    assert fake.calls == []  # nothing reached the engine, so no object pointer was ever copied as bytes


def test_state_blobs_of_another_dtype_refused_before_upload(monkeypatch):
    eng, fake = _engine_without_device(monkeypatch, [("a", "f8"), ("n", "i1")])
    for other in (np.zeros(4, dtype=np.int64), np.zeros((4, 9), dtype=np.uint8), np.zeros(4, dtype=[("b", "f8"), ("n", "i1")])):
        with pytest.raises(ValueError, match="declares"):
            eng.set_state(np.zeros((4, 2)), np.zeros(4), other)
    assert fake.calls == []
    nob, fake = _engine_without_device(monkeypatch, None)
    with pytest.raises(NotImplementedError, match="declares none"):
        nob.set_state(np.zeros((4, 2)), np.zeros(4), np.zeros(4))
    assert fake.calls == []
    # the declared dtype is uploaded, and becomes the live layout
    eng, fake = _engine_without_device(monkeypatch, "f4")
    eng.set_state(np.zeros((4, 2)), np.zeros(4), np.zeros((4, 1, 3), dtype=np.float32))
    assert fake.calls == ["eb_set_state", "eb_set_state_blobs"] and eng._blob_layout == (np.dtype("f4"), (3,))


def test_header_declares_the_blob_abi():
    handle = C.CDLL(_lib.LIB_PATH)
    for name in ("eb_callback_blobs", "eb_set_state_blobs", "eb_get_blobs", "eb_compute_log_prob_blobs",
                 "eb_step_store_blobs"):
        assert hasattr(handle, name), name
    assert _lib.lib().eb_abi_version() == 2
