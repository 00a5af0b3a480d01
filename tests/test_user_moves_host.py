"""User-written proposals, the parts that need no GPU: which moves are user moves, the wrappers, the schedule
entries they pack to, the ``random`` stream, the trampoline's checks of ``(q, factors)`` (through a recording fake
library), the refusals, and the numpy driver the GPU tests compare against."""
import ctypes as C
import os
import pickle

import numpy as np
import pytest

from oracle import gen_golden_user_moves as gen
from user_moves_ref import (NumpyStretch, UserOracle, WithSetup, gauss_mh, golden_cases, golden_moves, load_case,
                            oracle_moves)

import emcee_b200
from emcee_b200 import _lib, models, moves
from emcee_b200.backend import Backend
from emcee_b200.moves.user import user_move_spec


def test_user_moves_are_recognised_and_builtins_are_not():
    for m in (moves.StretchMove(), moves.DEMove(), moves.DESnookerMove(), moves.WalkMove(), moves.GaussianMove(1.0)):
        assert user_move_spec(m) is None
        assert m.descriptor()["kind"] not in ("user", "user_mh")
    kind, where, _, setup = user_move_spec(NumpyStretch(nsplits=3, randomize_split=False))
    assert (kind, where, setup) == ("user", "host", None)
    d = NumpyStretch(nsplits=3, randomize_split=False, live_dangerously=True).descriptor()
    assert d["kind"] == "user" and d["nsplits"] == 3 and not d["randomize_split"] and d["live_dangerously"]
    assert d["mode"] == 0 and WithSetup().descriptor()["mode"] == 1
    assert user_move_spec(WithSetup())[3] is not None

    class OnDevice(moves.CudaArrayRedBlueMove):
        def get_proposal(self, s, c, random):
            return s, None

    assert user_move_spec(OnDevice())[:2] == ("user", "device")
    # a subclass that does not override get_proposal is no user move: the reference's error
    with pytest.raises(NotImplementedError, match="implemented by subclasses"):
        moves.CudaArrayRedBlueMove().descriptor()


def test_wrappers_and_the_bare_callable():
    with pytest.raises(NotImplementedError, match="HostProposal"):
        moves.MHMove(gauss_mh)
    with pytest.raises(TypeError):
        moves.HostProposal(3)
    h, d = moves.MHMove(moves.HostProposal(gauss_mh)), moves.MHMove(moves.CudaArrayProposal(gauss_mh), ndim=4)
    assert user_move_spec(h)[:2] == ("user_mh", "host") and user_move_spec(d)[:2] == ("user_mh", "device")
    assert h.descriptor()["kind"] == "user_mh" and d.ndim == 4
    h._advance(5, 3)  # the sampler's stateful-move hook leaves a user MHMove alone
    x = np.arange(6.0).reshape(3, 2)
    q, f = user_move_spec(h)[2](x, [], np.random.RandomState(0))
    q2, f2 = gauss_mh(x, np.random.RandomState(0))
    assert np.array_equal(q, q2) and np.array_equal(f, f2)


def test_schedule_packing():
    rows = [(dict(NumpyStretch(nsplits=3).descriptor(), p0=2.0), 0.5), (dict(WithSetup().descriptor(), p0=0.0), 1.0),
            (dict(moves.MHMove(moves.HostProposal(gauss_mh)).descriptor(), p0=1.0), 0.25)]
    arr = _lib.Engine.pack_moves(rows)
    assert [a.kind for a in arr] == [5, 5, 6]
    assert [a.p0 for a in arr] == [2.0, 0.0, 1.0]
    assert [a.mode for a in arr] == [0, 1, 0] and arr[0].nsplits == 3 and arr[2].weight == 0.25


def test_random_is_a_pure_function_of_seed_step_split():
    a, b = moves.user_random(7, 3, 1), moves.user_random(7, 3, 1)
    assert np.array_equal(a.rand(5), b.rand(5)) and np.array_equal(a.randn(4), b.randn(4))
    assert not np.array_equal(moves.user_random(7, 3, 0).rand(5), moves.user_random(7, 3, 1).rand(5))
    assert not np.array_equal(moves.user_random(7, 4, 1).rand(5), moves.user_random(7, 3, 1).rand(5))
    assert not np.array_equal(moves.user_random(8, 3, 1).rand(5), moves.user_random(7, 3, 1).rand(5))
    # numpy's own Philox4x64, keyed by the engine seed, counter (0, step, split, 8)
    ref = np.random.RandomState(np.random.Philox(key=2**64 - 5, counter=[0, 11, 2, 8]))
    r = moves.user_random(-5, 11, 2)
    assert np.array_equal(r.randint(1000, size=6), ref.randint(1000, size=6))
    for name in ("rand", "randn", "randint", "choice", "shuffle", "uniform", "multivariate_normal"):
        assert callable(getattr(r, name))


def _raw(seed, step, split, n):
    return moves.user_random(seed, step, split)._bit_generator.random_raw(n)


@pytest.mark.parametrize("seed,step,split", [(0x5EED, 10, 0), (1, 0, 0), (2**64 - 1, 2**40, 3)])
def test_streams_of_different_calls_are_disjoint(seed, step, split):
    # Philox4x64 advances counter word 0 per 4-draw block: with (step, split) in that word, the stream of step + 1
    # would be the stream of step shifted by one block, and a walker's proposal noise would repeat from step to step
    n = 100_000
    a = _raw(seed, step, split, n)
    for other in (_raw(seed, step + 1, split, n), _raw(seed, step, split + 1, n)):
        assert np.intersect1d(a, other).size == 0
    x, y = moves.user_random(seed, step, split).randn(4096), moves.user_random(seed, step + 1, split).randn(4096)
    assert np.intersect1d(x, y).size == 0


class FakeLib(object):
    def __init__(self):
        self.calls = []

    def eb_proposal_result(self, h, q, qs, f, fs, m, stream):
        self.calls.append((q.value, qs, f.value, fs, m, stream))
        return 0


def _host_call(monkeypatch, propose, ns=3, ndim=2, counts=(2, 1)):
    monkeypatch.setattr(_lib, "lib", lambda: FakeLib())
    failure = [None]
    seen = {}

    def wrapped(s, c, random):
        seen["s"], seen["c"], seen["u"] = s, c, random.rand()
        return propose(s, c, random)

    cb = _lib.make_proposal_trampoline(None, wrapped, None, _lib.EB_CALLBACK_HOST, failure, [99])
    rows = np.arange((ns + sum(counts)) * ndim, dtype=np.float64).reshape(-1, ndim)
    q, f = np.zeros((ns, ndim)), np.zeros(ns)
    cnt = np.array(counts, dtype=np.int64)
    rc = cb(None, 4, 1, rows.ctypes.data_as(_lib._dp), ns, rows[ns:].ctypes.data_as(_lib._dp),
            cnt.ctypes.data_as(C.POINTER(C.c_int64)), len(counts), ndim, q.ctypes.data_as(_lib._dp),
            f.ctypes.data_as(_lib._dp), None)
    return rc, failure[0], seen, rows, q, f


def test_host_trampoline_hands_over_the_sets_and_the_stream(monkeypatch):
    rc, err, seen, rows, q, f = _host_call(monkeypatch, lambda s, c, r: (s + 1.0, np.full(len(s), 0.5)))
    assert rc == 0 and err is None
    assert np.array_equal(seen["s"], rows[:3]) and [len(x) for x in seen["c"]] == [2, 1]
    assert np.array_equal(seen["c"][0], rows[3:5]) and np.array_equal(seen["c"][1], rows[5:6])
    assert seen["u"] == moves.user_random(99, 4, 1).rand()
    assert np.array_equal(q, rows[:3] + 1.0) and np.array_equal(f, [0.5] * 3)


@pytest.mark.parametrize("out,exc,msg", [
    (lambda s: (s[:-1], np.zeros(len(s))), ValueError, "shape"),
    (lambda s: (s.astype(np.float32), np.zeros(len(s))), TypeError, "float64"),
    (lambda s: (s, np.zeros(len(s) + 1)), ValueError, "factors of shape"),
    (lambda s: (s, np.zeros(len(s), dtype=np.int64)), TypeError, "float64 factors"),
    (lambda s: s, ValueError, r"\(q, factors\)"),
])
def test_host_trampoline_checks_the_result(monkeypatch, out, exc, msg):
    rc, err, _, _, q, f = _host_call(monkeypatch, lambda s, c, r: out(s))
    assert rc != 0 and isinstance(err, exc) and err.args and __import__("re").search(msg, str(err))
    assert not q.any() and not f.any()


def test_user_exception_is_kept_unchanged(monkeypatch):
    class Boom(Exception):
        pass

    def boom(s, c, r):
        raise Boom("x")

    rc, err, _, _, _, _ = _host_call(monkeypatch, boom)
    assert rc != 0 and isinstance(err, Boom)


class _Producer(object):
    def __init__(self, cai):
        self.__cuda_array_interface__ = cai


def test_device_trampoline_streams_and_strides(monkeypatch):
    fake = FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    failure = [None]

    def cai(shape, stream=None, strides=None, version=3):
        d = dict(shape=shape, typestr="<f8", data=(4096, False), strides=strides, version=version)
        if version == 3:
            d["stream"] = stream
        return d

    def run(q, f):
        fake.calls.clear()
        cb = _lib.make_proposal_trampoline(None, lambda s, c, r: (q, f), None, _lib.EB_CALLBACK_DEVICE, failure, [1])
        cnt = np.array([4], dtype=np.int64)
        rc = cb(None, 0, 0, C.cast(C.c_void_p(1 << 20), _lib._dp), 3, C.cast(C.c_void_p((1 << 20) + 48), _lib._dp),
                cnt.ctypes.data_as(C.POINTER(C.c_int64)), 1, 2, None, None, C.c_void_p(77))
        return rc

    assert run(_Producer(cai((3, 2), stream=5)), _Producer(cai((3,), stream=5))) == 0
    assert fake.calls[0][1:] == (16, 4096, 8, 3, 5)
    assert run(_Producer(cai((3, 2), strides=(32, 8), version=2)), np.zeros(3)) == 0
    assert fake.calls[0][1] == 32 and fake.calls[0][5] == _lib.EB_STREAM_UNKNOWN
    assert run(_Producer(cai((3, 2), stream=5)), _Producer(cai((3,), stream=6))) == 0
    assert fake.calls[0][5] == _lib.EB_STREAM_UNKNOWN  # two producers: wait for the whole device
    assert run(_Producer(cai((3, 2), strides=(32, 16))), np.zeros(3)) == 1
    assert isinstance(failure[0], ValueError) and "contiguous" in str(failure[0])
    assert run(np.zeros((3, 3)), np.zeros(3)) == 1 and isinstance(failure[0], ValueError)


def test_attach_refuses_user_moves():
    s = emcee_b200.EnsembleSampler.__new__(emcee_b200.EnsembleSampler)
    s.backend, s.log_prob_fn = Backend(), models.GaussianIso()
    s._moves = [moves.StretchMove(), NumpyStretch()]
    with pytest.raises(NotImplementedError, match="user proposal"):
        s.attach(object())


def test_moves_pickle():
    for m in (NumpyStretch(a=3.0, nsplits=5), moves.MHMove(moves.HostProposal(gauss_mh), ndim=3)):
        m2 = pickle.loads(pickle.dumps(m))
        a, b = m.descriptor(), m2.descriptor()
        for d in (a, b):  # p0 (the slot the sampler fills in) and p1 are NaN
            assert np.isnan(d.pop("p0")) and np.isnan(d.pop("p1"))
        assert a == b
        assert user_move_spec(m2)[:2] == user_move_spec(m)[:2]


def test_header_declares_the_user_move_abi():
    handle = C.CDLL(_lib.LIB_PATH)
    for name in ("eb_move_set_proposal", "eb_proposal_result"):
        assert hasattr(handle, name), name
    assert _lib.MOVE_KINDS["user"] == 5 and _lib.MOVE_KINDS["user_mh"] == 6
    assert _lib.lib().eb_abi_version() == 2


def _run_oracle(case, g):
    name, N, D, kind, spec, nsteps = case
    o = UserOracle(N, D, gen.case_target(kind, D), oracle_moves(golden_moves(spec)), seed=int(g["seed"]))
    o.set_state(g["p0"])
    chain, lps, acc = [], [], []
    for _ in range(nsteps):
        acc.append(o.run(1))
        chain.append(o.coords.copy())
        lps.append(o.log_prob.copy())
    return np.array(chain), np.array(lps), np.array(acc)


@pytest.mark.parametrize("name", golden_cases())
def test_numpy_driver_reproduces_the_reference(name):
    # the driver the GPU tests compare against, against the unmodified reference's golden runs: bit for bit
    case, g = load_case(name)
    assert np.array_equal(g["p0"], gen.case_p0(name, case[1], case[2], case[3]))
    chain, lps, acc = _run_oracle(case, g)
    np.testing.assert_array_equal(chain, g["chain"])
    np.testing.assert_array_equal(lps, g["log_prob"])
    np.testing.assert_array_equal(acc, g["accepted"])


def test_random_is_the_generators_stream():
    for seed, step, split in ((gen.SEED, 0, 0), (2**64 - 1, 7, 4), (3, 2**40, 1)):
        assert np.array_equal(moves.user_random(seed, step, split).randn(7), gen.user_random(seed, step, split).randn(7))


@pytest.mark.skipif(not os.path.exists(gen.REF_ZIP), reason="the reference is not packaged (oracle/make_ref.py)")
@pytest.mark.parametrize("name", golden_cases())
def test_generator_reproduces_the_golden_files(name):
    case, g = load_case(name)
    new = gen.run_case(gen.import_reference(), *case)
    assert sorted(new) == sorted(g)
    for k in g:
        assert new[k].dtype == g[k].dtype and np.array_equal(new[k], g[k]), k


def test_user_moves_get_dense_proposal_slots():
    # slots count the user moves only, so a user move late in a long schedule still gets a valid slot
    s = emcee_b200.EnsembleSampler.__new__(emcee_b200.EnsembleSampler)
    s._moves = [moves.StretchMove()] * 70 + [NumpyStretch(), moves.MHMove(moves.HostProposal(gauss_mh))]
    s._raw_weights = np.ones(len(s._moves))
    s.ndim = 5
    sched = s._schedule()
    assert [d["p0"] for d, _ in sched[70:]] == [0.0, 1.0] and sched[0][0]["kind"] == "stretch"
    s._moves = [NumpyStretch() for _ in range(_lib.EB_MAX_PROPOSAL_SLOTS + 1)]
    with pytest.raises(NotImplementedError, match="at most 64 user moves"):
        s._load_moves()
