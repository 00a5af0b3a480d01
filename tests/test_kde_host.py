"""KDEMove on the host side: the descriptor and its bandwidth encoding (``include/emcee_b200.h``), the argument
refusals, which reach no ABI call, and the KDE shim (``oracle.kde.KdePhilox``), which still regenerates the
reference's existing golden fixtures bit for bit."""
import math
import os

import numpy as np
import pytest

import emcee_b200
from emcee_b200 import _lib, models, moves
from emcee_b200.backend import Backend
from kde_util import kde_names, load_kde
from oracle import gen_golden as gg
from oracle import gen_golden_kde as gk
from oracle import gen_golden_user_moves as gu
from oracle import kde as ok
from oracle import philox as px
from util import load_golden

NEED_REF = pytest.mark.skipif(not os.path.exists(gu.REF_ZIP), reason="the reference is not packaged (make_ref.py)")


class RecordingLib(object):
    """Stands in for the engine library: records every entry point looked up."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        self.calls.append(name)
        raise AssertionError("ABI call %s" % name)


@pytest.fixture
def recording(monkeypatch):
    rec = RecordingLib()
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


def test_descriptor_encodes_the_bandwidth():
    d = moves.KDEMove().descriptor()
    assert d["kind"] == "kde" and _lib.MOVE_KINDS["kde"] == 7
    assert d["nsplits"] == 2 and d["randomize_split"] and not d["live_dangerously"]
    assert math.isnan(d["p0"]) and math.isnan(d["p1"])
    assert math.isnan(moves.KDEMove("scott").descriptor()["p0"])
    d = moves.KDEMove("silverman", nsplits=5, randomize_split=False, live_dangerously=True).descriptor()
    assert (d["p0"], d["nsplits"], d["randomize_split"], d["live_dangerously"]) == (1.0, 5, False, True)
    for bw in (0.05, 2, np.float32(0.25)):
        d = moves.KDEMove(bw).descriptor()
        assert d["p0"] == 2.0 and d["p1"] == float(bw)
    arr = _lib.Engine.pack_moves([(moves.KDEMove(0.3, nsplits=3).descriptor(), 2.0)])
    assert (arr[0].kind, arr[0].nsplits, arr[0].p0, arr[0].p1, arr[0].weight) == (7, 3, 2.0, 0.3, 2.0)


def test_bad_bandwidths_are_refused_without_an_abi_call(recording):
    with pytest.raises(ValueError, match="`bw_method` should be 'scott', 'silverman', a scalar or a callable."):
        moves.KDEMove("Scott")
    for bad in (0.0, -1.0, float("nan"), float("inf"), True, [0.1], "0.1"):
        with pytest.raises(ValueError):
            moves.KDEMove(bad)
    with pytest.raises(NotImplementedError, match="callable bw_method"):
        moves.KDEMove(lambda kde: 0.5)
    assert recording.calls == []


def test_attach_refuses_kde_without_an_abi_call(recording):
    s = emcee_b200.EnsembleSampler.__new__(emcee_b200.EnsembleSampler)
    s.backend, s.log_prob_fn = Backend(), models.GaussianIso()
    s._moves = [moves.StretchMove(), moves.KDEMove()]
    with pytest.raises(NotImplementedError, match="KDEMove runs on one GPU"):
        s.attach(object())
    assert recording.calls == []


def test_kde_is_a_device_move():
    m = moves.KDEMove()
    assert isinstance(m, moves.RedBlueMove) and "KDEMove" in moves.__all__
    with pytest.raises(NotImplementedError):
        m.get_proposal(None, None, None)  # no host get_proposal: the sampler never takes it for a user move


def test_shim_is_a_random_state():
    shim = ok.KdePhilox(7)
    assert isinstance(shim, np.random.RandomState)
    assert shim.get_state() == ("philox4x32-10", 7, 0)


@NEED_REF
def test_extended_shim_regenerates_an_existing_fixture(tmp_path, monkeypatch):
    # WalkMove's multivariate_normal and DEMove's choice go through the methods KdePhilox overrides
    emcee = gu.import_reference()
    monkeypatch.setattr(gg, "OUT", str(tmp_path))
    monkeypatch.setattr(px, "PhiloxRandom", ok.KdePhilox)  # gen_golden.run_case takes the shim from oracle.philox
    for idx, case in enumerate(gg.case_list(emcee)):
        if case[0] in ("walk_all_rosen_40x4", "mix_walk_stretch_gauss_ring_64x4", "de_rosen_40x4"):
            gg.run_case(emcee, *case, seed=0x656D636565B200 + idx)
            new, old = dict(np.load(os.path.join(str(tmp_path), case[0] + ".npz"))), load_golden(case[0])
            assert sorted(new) == sorted(old)
            for k in old:
                same = np.array_equal(new[k], old[k], equal_nan=new[k].dtype.kind == "f")
                assert new[k].dtype == old[k].dtype and same, (case[0], k)


@NEED_REF
def test_generator_reproduces_the_kde_fixtures():
    emcee = gu.import_reference()
    cases = {c[0]: c for c in gk.case_list(emcee)}
    assert sorted(cases) == kde_names()
    for idx, name in enumerate(c[0] for c in gk.case_list(emcee)):
        new, old = gk.run_case(emcee, *cases[name], seed=gk.SEED0 + idx), load_kde(name)
        assert sorted(new) == sorted(old)
        for k in old:
            assert np.array_equal(new[k], old[k], equal_nan=new[k].dtype.kind == "f"), (name, k)
