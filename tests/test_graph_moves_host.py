"""Captured proposals (``moves.CudaGraphRedBlueMove``, ``moves.CudaGraphProposal``), the parts that need no GPU: the
``(ns, counts)`` the sampler captures, when it captures them, the checks of every ``CapturedProposal`` before anything
reaches the engine, the refusals, and the purpose-9 draws of the C++ header against their numpy statement.  The
engine is a recording stand-in (the pattern of ``test_graph_function_host.py``), so no pointer is dereferenced."""
import ctypes as C
import os
import pickle
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models, moves
from graph_draws_ref import graph_draws

HERE = os.path.dirname(os.path.abspath(__file__))


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

    def __init__(self, shape, typestr="<f8", strides=None, ptr=0xA000, readonly=False, device=None):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, readonly),
                                          "strides": strides, "version": 2}
        if device is not None:
            self.device = device


CALLS = []  # the arguments every FakeCapture was called with, pickled copies included


class FakeCapture(object):
    """capture(*args) -> a well-formed CapturedProposal of fake pointers, or what `bad(args, good)` returns."""

    def __init__(self, N, ndim, ndraws=0, bad=None):
        self.N, self.ndim, self.ndraws, self.bad = N, ndim, ndraws, bad

    def good(self, args):
        ns, D = args[0], self.ndim
        base = 0x100000 * (1 + len(CALLS))
        c = Array((self.N - ns, D), ptr=base + 0x1000) if len(args) > 1 else None
        d = Array((ns, self.ndraws), ptr=base + 0x2000) if self.ndraws else None
        return moves.CapturedProposal(0x5000 + len(CALLS), Array((ns, D), ptr=base), c, d,
                                      Array((ns, D), ptr=base + 0x3000), Array((ns,), ptr=base + 0x4000), owner=args)

    def __call__(self, *args):
        CALLS.append(args)
        g = self.good(args)
        return g if self.bad is None else self.bad(args, g)


def _graph_calls(fake):
    out = []
    for c in fake.calls:
        if c[0] == "eb_move_set_proposal_graphs":
            _, h, slot, draw, ndraws, arr, n = c
            out.append((slot, draw, ndraws, [(g.split, g.ns, g.exec, g.s, g.c or 0, g.draws or 0) for g in arr[:n]]))
    return out


def _sampler(N, D, mv, **kw):
    return emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=mv, seed=1, **kw)


def _redblue(N, D, nsplits=2, ndraws=0, bad=None, **kw):
    return moves.CudaGraphRedBlueMove(FakeCapture(N, D, ndraws, bad), ndraws=ndraws, nsplits=nsplits, **kw)


# ---- what is captured -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [9, 37, 63])
@pytest.mark.parametrize("P", [2, 3, 5])
def test_one_capture_per_distinct_split_shape(fake, N, P):
    CALLS.clear()
    _sampler(N, 3, _redblue(N, 3, nsplits=P, ndraws=3))
    sizes = [(N - j + P - 1) // P for j in range(P)]
    want = {(sizes[j], tuple(sizes[:j] + sizes[j + 1:])) for j in range(P)}
    assert sorted(CALLS) == sorted(want)  # each distinct (ns, counts) once
    ((slot, draw, ndraws, graphs),) = _graph_calls(fake)
    assert (slot, draw, ndraws) == (0, 0, 3)
    assert [g[0] for g in graphs] == list(range(P)) and [g[1] for g in graphs] == sizes
    for j, g in enumerate(graphs):  # splits of the same shape share one capture
        k = [s for s in range(P) if (sizes[s], tuple(sizes[:s] + sizes[s + 1:]))
             == (sizes[j], tuple(sizes[:j] + sizes[j + 1:]))][0]
        assert g[2:] == graphs[k][2:]
        assert g[4] != 0 and g[5] != 0


def test_mh_captures_the_ensemble_once(fake):
    CALLS.clear()
    _sampler(37, 4, moves.MHMove(moves.CudaGraphProposal(FakeCapture(37, 4), draw="normal")))
    assert CALLS == [(37,)]
    ((slot, draw, ndraws, graphs),) = _graph_calls(fake)
    assert (slot, draw, ndraws) == (0, 1, 0)
    assert graphs[0][:2] == (0, 37) and graphs[0][4] == 0 and graphs[0][5] == 0


def test_slots_shared_with_other_user_moves(fake):
    class Host(moves.RedBlueMove):
        def get_proposal(self, s, c, random):
            return s, np.zeros(len(s))

    N, D = 32, 3
    mv = [(moves.StretchMove(), 1.0), (Host(), 1.0), (_redblue(N, D), 1.0),
          (moves.MHMove(moves.CudaGraphProposal(FakeCapture(N, D))), 1.0)]
    s = _sampler(N, D, mv)
    assert [c[2] for c in fake.calls if c[0] == "eb_move_set_proposal"] == [0]
    assert [c[0] for c in _graph_calls(fake)] == [1, 2]
    assert [d["p0"] for d, _ in s._schedule() if d["kind"] in ("user", "user_mh")] == [0.0, 1.0, 2.0]
    assert [d["mode"] for d, _ in s._schedule() if d["kind"] == "user"] == [0, 0]


def test_too_many_user_moves_counts_graph_moves(fake):
    N, D = 16, 2
    mv = [_redblue(N, D) for _ in range(_lib.EB_MAX_PROPOSAL_SLOTS + 1)]
    with pytest.raises(NotImplementedError, match="at most 64 user moves"):
        _sampler(N, D, mv)
    assert "eb_move_set_proposal_graphs" not in fake.names()


def test_pickle_recaptures(fake):
    CALLS.clear()
    s = _sampler(37, 3, _redblue(37, 3, nsplits=3))
    first = list(CALLS)
    assert first
    CALLS.clear()
    s2 = pickle.loads(pickle.dumps(s))
    assert sorted(CALLS) == sorted(first)
    assert len(_graph_calls(fake)) == 2
    assert isinstance(s2._moves[0], moves.CudaGraphRedBlueMove)


# ---- checks of the captured objects ------------------------------------------------------------------------------
def _swap(name, value):
    def bad(args, g):
        setattr(g, name, value(args, g) if callable(value) else value)
        return g

    return bad


BAD = {
    "type": (lambda args, g: "nope", TypeError, "must return a moves.CapturedProposal"),
    "exec0": (_swap("exec", 0), ValueError, "exec is 0"),
    "exec_bool": (_swap("exec", True), ValueError, "exec is True"),
    "s_not_cuda": (_swap("s", np.zeros((4, 3))), TypeError, "s is not a CUDA array"),
    "s_shape": (_swap("s", lambda a, g: Array((a[0] + 1, 3))), ValueError, "s has shape"),
    "c_shape": (_swap("c", lambda a, g: Array((5, 3))), ValueError, "c has shape"),
    "c_none": (_swap("c", None), TypeError, "c is not a CUDA array"),
    "q_dtype": (_swap("q", lambda a, g: Array((a[0], 3), typestr="<f4")), TypeError, "float64"),
    "f_shape": (_swap("factors", lambda a, g: Array((a[0], 1))), ValueError, "factors has shape"),
    "s_readonly": (_swap("s", lambda a, g: Array((a[0], 3), readonly=True)), ValueError, "s is exported read-only"),
    "c_readonly": (_swap("c", lambda a, g: Array((32 - a[0], 3), readonly=True)), ValueError,
                   "c is exported read-only"),
    "draws_readonly": (_swap("draws", lambda a, g: Array((a[0], 2), readonly=True)), ValueError,
                       "draws is exported read-only"),
    "draws_shape": (_swap("draws", lambda a, g: Array((a[0], 3))), ValueError, "draws has shape"),
    "q_row_strided": (_swap("q", lambda a, g: Array((a[0], 3), strides=(48, 16))), ValueError, "contiguous"),
    "q_stride_short": (_swap("q", lambda a, g: Array((a[0], 3), strides=(16, 8))), ValueError, "at least a row"),
    "null_q": (_swap("q", lambda a, g: Array((a[0], 3), ptr=0)), ValueError, "q has a null data pointer"),
    "device": (_swap("factors", lambda a, g: Array((a[0],), device=1)), ValueError, "on CUDA device 1"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_malformed_captures_are_refused_before_the_engine(fake, case):
    bad, exc, match = BAD[case]
    with pytest.raises(exc, match=match):
        _sampler(32, 3, [moves.StretchMove(), _redblue(32, 3, ndraws=2, bad=bad)])
    assert "eb_move_set_proposal_graphs" not in fake.names()


def test_mh_capture_must_not_pass_c_or_unused_draws(fake):
    bad_c = _swap("c", lambda a, g: Array((1, 3)))
    with pytest.raises(ValueError, match="c; it must be None for an MHMove"):
        _sampler(32, 3, moves.MHMove(moves.CudaGraphProposal(FakeCapture(32, 3, bad=bad_c))))
    bad_d = _swap("draws", lambda a, g: Array((32, 1)))
    with pytest.raises(ValueError, match="draws; it must be None when ndraws == 0"):
        _sampler(32, 3, moves.MHMove(moves.CudaGraphProposal(FakeCapture(32, 3, bad=bad_d))))
    assert "eb_move_set_proposal_graphs" not in fake.names()


def test_strided_buffers_pass_their_strides(fake):
    def strided(args, g):
        g.s = Array((args[0], 3), strides=(32, 8), ptr=0x7000)
        return g

    _sampler(32, 3, _redblue(32, 3, bad=strided))
    (call,) = [c for c in fake.calls if c[0] == "eb_move_set_proposal_graphs"]
    arr = call[5]
    assert arr[0].s == 0x7000 and arr[0].s_row_stride_bytes == 32 and arr[0].q_row_stride_bytes == 24
    assert arr[0].factors_stride_bytes == 8


# ---- refusals ----------------------------------------------------------------------------------------------------
def test_construction_refusals():
    cap = FakeCapture(8, 2)
    with pytest.raises(NotImplementedError, match="at most 524288 draws"):
        moves.CudaGraphRedBlueMove(cap, ndraws=2**19 + 1)
    moves.CudaGraphRedBlueMove(cap, ndraws=2**19)
    with pytest.raises(NotImplementedError, match="at most 524288 draws"):
        moves.CudaGraphProposal(cap, ndraws=2**19 + 1)
    with pytest.raises(ValueError, match="ndraws must be >= 0"):
        moves.CudaGraphRedBlueMove(cap, ndraws=-1)
    with pytest.raises(TypeError, match="ndraws must be an int"):
        moves.CudaGraphProposal(cap, ndraws=2.0)
    with pytest.raises(ValueError, match="'uniform' or 'normal'"):
        moves.CudaGraphRedBlueMove(cap, draw="gamma")
    with pytest.raises(TypeError, match="callable"):
        moves.CudaGraphRedBlueMove(3)

    class WithSetup(moves.CudaGraphRedBlueMove):
        def setup(self, coords):
            pass

    with pytest.raises(NotImplementedError, match="no setup hook"):
        WithSetup(cap)


def test_outside_the_sampler_and_attach_are_refused(fake):
    N, D = 16, 2
    mv = _redblue(N, D)
    s = _sampler(N, D, mv)
    with pytest.raises(NotImplementedError, match="runs on one GPU"):
        s.attach(object())
    with pytest.raises(NotImplementedError, match="inside EnsembleSampler.sample"):
        mv.propose(s.model, emcee_b200.State(np.zeros((N, D))))
    prop = moves.CudaGraphProposal(FakeCapture(N, D))
    with pytest.raises(NotImplementedError, match="captured proposal runs as a CUDA graph"):
        prop(np.zeros((N, D)), None)
    with pytest.raises(NotImplementedError, match="inside EnsembleSampler.sample"):
        moves.MHMove(prop).propose(s.model, emcee_b200.State(np.zeros((N, D))))


def test_descriptor_is_a_user_move_without_setup():
    d = moves.CudaGraphRedBlueMove(FakeCapture(8, 2), nsplits=3, randomize_split=False).descriptor()
    assert d["kind"] == "user" and d["nsplits"] == 3 and d["randomize_split"] is False and d["mode"] == 0


# ---- the purpose-9 draws: C++ header against numpy -----------------------------------------------------------------
@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("probe") / "libgraph_draws_probe.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", "graph_draws_host.cpp")],
                   check=True)
    return C.CDLL(out)


def _probe(probe, seed, step, split, rows, draw, ndraws):
    out = np.zeros((rows, ndraws))
    probe.probe_graph_draws(C.c_uint64(seed), C.c_uint64(step), C.c_uint32(split), C.c_int64(rows),
                            C.c_int(draw == "normal"), C.c_int64(ndraws), out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


@pytest.mark.parametrize("ndraws", [1, 2, 3, 7, 10])
@pytest.mark.parametrize("seed,step,split", [(0, 0, 0), (0x656D636565B200, 12345678901, 3), (2**64 - 1, 2**40 + 7, 31)])
def test_graph_draws_match_the_header(probe, seed, step, split, ndraws):
    u = graph_draws(seed, step, split, 65, "uniform", ndraws)
    assert np.array_equal(u, _probe(probe, seed, step, split, 65, "uniform", ndraws))
    assert np.all((u >= 0) & (u < 1))
    z = graph_draws(seed, step, split, 65, "normal", ndraws)
    h = _probe(probe, seed, step, split, 65, "normal", ndraws)
    # the same words and the same expression; libm and numpy may round log / sin / cos apart by an ulp or so
    assert np.all(np.abs(z - h) <= 8 * np.finfo(float).eps * np.maximum(np.abs(z), 1e-300) + 1e-300)


def test_graph_draws_layout():
    from oracle import philox as px

    seed, step, split = 9, 77, 2
    u = graph_draws(seed, step, split, 5, "uniform", 5)
    for k in range(3):  # call k holds draws 2k, 2k + 1; the last call of an odd count keeps its first half
        w0, w1, w2, w3 = px.draw_words(seed, step, px.sub_split(split, k), 9, np.arange(5))
        assert np.array_equal(u[:, 2 * k], px.u53(w0, w1))
        if 2 * k + 1 < 5:
            assert np.array_equal(u[:, 2 * k + 1], px.u53(w2, w3))
    assert np.array_equal(graph_draws(seed, step, split, [3, 1], "uniform", 5), u[[3, 1]])
    z = graph_draws(seed, step, split, 5, "normal", 2)
    w0, w1, w2, w3 = px.draw_words(seed, step, split, 9, np.arange(5))
    assert np.array_equal(z[:, 0], px.box_muller(px.u53(w0, w1), px.u53(w2, w3)))
    # distinct from purpose 6 on the same counter, and different splits / steps give different draws
    assert not np.array_equal(z, px.normals(seed, step, split, np.arange(5), 2))
    assert not np.array_equal(u, graph_draws(seed, step, split + 1, 5, "uniform", 5))
    assert not np.array_equal(u, graph_draws(seed, step + 1, split, 5, "uniform", 5))
