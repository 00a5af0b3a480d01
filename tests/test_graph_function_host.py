"""``models.CudaGraphFunction``, the parts that need no GPU: the row counts the sampler captures graphs for, when it
captures them, the checks of every ``CapturedGraph`` before anything reaches the engine, and the refusals.  The
engine is a recording stand-in (the pattern of ``test_cuda_arrays_host.py``), so no pointer below is dereferenced."""
import pickle

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models, moves


class RecordingLib(object):
    """Every engine call is recorded with its arguments and succeeds."""

    def __init__(self):
        self.calls = []

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


class Array(object):
    """A CUDA array as torch presents one: the interface dict only."""

    def __init__(self, shape, typestr="<f8", strides=None, ptr=0xA000):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False),
                                          "strides": strides, "version": 2}


CALLS = []  # the row counts every FakeCapture was asked for, pickled copies included


class FakeCapture(object):
    """capture(m) -> a well-formed CapturedGraph of fake pointers, or what `bad(m, ndim)` returns."""

    def __init__(self, ndim, bad=None):
        self.ndim, self.bad = ndim, bad

    def __call__(self, m):
        CALLS.append(m)
        if self.bad is not None:
            return self.bad(m, self.ndim)
        return models.CapturedGraph(0x5000 + m, Array((m, self.ndim), ptr=0x100000 + 0x1000 * m),
                                    Array((m,), ptr=0x900000 + 0x1000 * m), owner="g%d" % m)


def _graphs_call(fake):
    (call,) = [c for c in fake.calls if c[0] == "eb_model_set_graphs"]
    _, h, arr, n = call
    return [(g.m, g.exec, g.x, g.x_row_stride_bytes, g.lp, g.lp_stride_bytes) for g in arr[:n]]


def _sampler(N, D, mv, bad=None, **kw):
    return emcee_b200.EnsembleSampler(N, D, models.CudaGraphFunction(FakeCapture(D, bad)), moves=mv, seed=1, **kw)


def _split_sizes(N, P):
    return set(np.bincount(np.arange(N) % P).tolist())


@pytest.mark.parametrize("N", [8, 9, 37, 64])
@pytest.mark.parametrize("P", [2, 3, 4])
def test_row_counts_red_blue(fake, N, P):
    del CALLS[:]
    s = _sampler(N, 3, moves.StretchMove(nsplits=P))
    want = sorted(_split_sizes(N, P) | {N})
    assert CALLS == want
    assert [g[0] for g in _graphs_call(fake)] == want
    assert s.log_prob_fn.capture.ndim == 3


@pytest.mark.parametrize("N", [11, 40])
def test_row_counts_mixed_schedule(fake, N):
    del CALLS[:]
    mv = [(moves.DEMove(nsplits=3), 0.3), (moves.GaussianMove(0.5), 0.3), (moves.WalkMove(nsplits=4), 0.2),
          (moves.DESnookerMove(), 0.2)]
    _sampler(N, 3, mv)
    assert CALLS == sorted(_split_sizes(N, 3) | _split_sizes(N, 4) | {N})
    del CALLS[:]
    _sampler(N, 3, moves.GaussianMove(0.5))  # proposes every walker at once: nwalkers only
    assert CALLS == [N]


def test_graph_descriptions_reach_the_engine(fake):
    def strided(m, ndim):
        return models.CapturedGraph(77 + m, Array((m, ndim), strides=(8 * (ndim + 2), 8), ptr=0x2000),
                                    Array((m,), strides=(24,), ptr=0x3000))

    del CALLS[:]
    _sampler(6, 2, moves.StretchMove(), bad=strided)
    assert _graphs_call(fake) == [(3, 80, 0x2000, 32, 0x3000, 24), (6, 83, 0x2000, 32, 0x3000, 24)]


def test_capture_runs_once_per_size_and_again_after_unpickling(fake):
    del CALLS[:]
    s = _sampler(10, 3, [(moves.StretchMove(), 0.5), (moves.DEMove(nsplits=3), 0.5)])
    assert CALLS == [3, 4, 5, 10]
    assert [c[0] for c in fake.calls].count("eb_model_set_graphs") == 1
    t = pickle.loads(pickle.dumps(s))
    assert CALLS == [3, 4, 5, 10, 3, 4, 5, 10]
    assert [c[0] for c in fake.calls].count("eb_model_set_graphs") == 2
    assert isinstance(t.log_prob_fn, models.CudaGraphFunction)
    # the engine keeps every CapturedGraph (and so its owner) alive while the graphs are the model
    assert sorted(g.owner for g in t._engine._cb) == ["g10", "g3", "g4", "g5"]


def _wrong_shape_x(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim + 1)), Array((m,)))


def _wrong_shape_lp(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim)), Array((m, 1)))


def _wrong_dtype(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim), typestr="<f4"), Array((m,)))


def _wrong_dtype_lp(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim)), Array((m,), typestr="<i8"))


def _strided_columns(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim), strides=(8, 8 * m)), Array((m,)))


def _short_row_stride(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim), strides=(8 * ndim - 8, 8)), Array((m,)))


def _odd_lp_stride(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim)), Array((m,), strides=(12,)))


def _exec_zero(m, ndim):
    return models.CapturedGraph(0, Array((m, ndim)), Array((m,)))


def _exec_not_int(m, ndim):
    return models.CapturedGraph("0x1234", Array((m, ndim)), Array((m,)))


def _host_x(m, ndim):
    return models.CapturedGraph(1, np.zeros((m, ndim)), Array((m,)))


def _host_lp(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim)), np.zeros(m))


def _not_captured(m, ndim):
    return (1, Array((m, ndim)), Array((m,)))


def _null_x(m, ndim):
    return models.CapturedGraph(1, Array((m, ndim), ptr=0), Array((m,)))


def _read_only_x(m, ndim):
    x = Array((m, ndim))
    x.__cuda_array_interface__["data"] = (0xA000, True)
    return models.CapturedGraph(1, x, Array((m,)))


BAD = [
    (_wrong_shape_x, ValueError, "x has shape"),
    (_wrong_shape_lp, ValueError, "lp has shape"),
    (_wrong_dtype, TypeError, "float64"),
    (_wrong_dtype_lp, TypeError, "float64"),
    (_strided_columns, ValueError, "contiguous"),
    (_short_row_stride, ValueError, "stride"),
    (_odd_lp_stride, ValueError, "stride"),
    (_exec_zero, ValueError, "non-zero cudaGraphExec_t"),
    (_exec_not_int, ValueError, "non-zero cudaGraphExec_t"),
    (_host_x, TypeError, "not a CUDA array"),
    (_host_lp, TypeError, "not a CUDA array"),
    (_not_captured, TypeError, "CapturedGraph"),
    (_null_x, ValueError, "null data pointer"),
    (_read_only_x, ValueError, "read-only"),
]


@pytest.mark.parametrize("bad,exc,match", BAD, ids=[b[0].__name__.lstrip("_") for b in BAD])
def test_malformed_graphs_are_refused_before_any_abi_call(fake, bad, exc, match):
    with pytest.raises(exc, match=match):
        _sampler(8, 3, moves.StretchMove(), bad=bad)
    assert fake.names() == ["eb_create"]  # nothing about the model reached the engine


def test_one_bad_size_refuses_the_whole_set(fake):
    def bad_at_8(m, ndim):
        return _exec_zero(m, ndim) if m == 8 else FakeCapture(ndim)(m)

    with pytest.raises(ValueError, match=r"capture\(8\) returned"):
        _sampler(8, 3, moves.StretchMove(), bad=bad_at_8)
    assert "eb_model_set_graphs" not in fake.names()


def test_refusals(fake):
    with pytest.raises(NotImplementedError, match="blobs"):
        models.CudaGraphFunction(FakeCapture(3), blobs_dtype=float)
    with pytest.raises(TypeError, match="callable"):
        models.CudaGraphFunction(None)
    fn = models.CudaGraphFunction(FakeCapture(3))
    assert isinstance(fn, models.CallbackFunction) and fn.blobs_dtype is None
    with pytest.raises(TypeError, match="captured graphs"):
        fn.evaluate(np.zeros((2, 3)))
    s = _sampler(8, 3, moves.StretchMove())
    with pytest.raises(NotImplementedError, match="cannot be sharded"):
        s.attach(None)
    assert "CudaGraphFunction" in models.__all__ and "CapturedGraph" in models.__all__
