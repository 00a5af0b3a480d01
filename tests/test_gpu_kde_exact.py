"""KDEMove's proposals and Hastings factors (``kde.cu``) against the high-precision references of ``kde_exact.py``,
under the first-order bounds derived in that module's docstring, at every tile geometry of ``kde_lse_kernel``.

How a split is observed.  The state carries ``log_prob = +inf`` for every walker outside the last split and
``-inf`` inside it.  Every earlier split's proposals then have lnpdiff = -inf and are rejected, so the last
split's complement is still the integer-valued input rows (``ExactCov``'s int64 path, at any ndim); every
proposal of the last split has lnpdiff = +inf and is accepted, so its walkers hold q bit for bit afterwards (the
test asserts their log-probabilities are finite).  With ``debug_taps`` the taps return the split's walkers, the
centre walker of each proposal and its factor.  ``(seed, step)`` vary through ``set_rng``: two pairs per row, one
above ndim 128.

Rows (``kde_exact.ROWS``; geometries for 132 SMs, the last split is the one observed):

=========  ===============================================================================================
d1         nc = 65: the second centre tile holds one centre; P = 130: the last point tile holds two
d33        two dimension chunks, the last of one column; nchunks = 2
d64        two full dimension chunks; nchunks = 3, last tile one centre (Silverman)
d100       four dimension chunks (last of 4); bw = 0.05: large |t|, the online rescale
ragged     tpc = 5, nchunks = 7, a short last chunk (4 tiles), last centre tile one centre
bench4096  tpc = 4, nchunks = 8
n16384     tpc = 43, nchunks = 3 (42 tiles in the last); one full dimension chunk
n65536     nchunks = 1: 512 tiles in one online log-sum-exp
d257       nine dimension chunks, the last of one column; five chunks of one tile, last tile 44 centres
d1024      ndim limit: 1024-thread inverse, 128 KiB of prepare shared memory, 32 dimension chunks,
           tpc = 2, nchunks = 9
ns3        three splits, nchunks = 11, ragged point and centre tiles
ns32       ns = 65, nc = 2015: 32 chunks of one tile
far        ensemble at 1e4 with unit spread: the x - mean cancellation
cond       complement covariance of condition number about 1e8
=========  ===============================================================================================

Factors are checked for both ends of the split, the ranks whose s or q row falls in the last point tile, and a
spread of 64 ranks (24 above ndim 128); proposals for every rank below ndim 128, the same ranks above.  The largest
error / bound of each class is printed and must stay below 1, with the row's wall time (reference included).
"""
import time

import numpy as np
import pytest

import kde_exact as KX
import proposals_exact as PX
from oracle import philox as px

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

SEED_STEPS = [(0x5EED, 0), (0xB200, 17)]
_SM = []


def sm_count():
    if not _SM:
        import torch

        _SM.append(int(torch.cuda.get_device_properties(0).multi_processor_count))
    return _SM[0]


class Tracker(object):
    """Largest |device - reference| / bound of one class."""

    def __init__(self, name):
        self.name, self.worst, self.n = name, 0.0, 0

    def check(self, err, bound, what):
        err = np.asarray(err, dtype=np.float64)
        bound = np.asarray(bound, dtype=np.float64)
        self.n += err.size
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(bound > 0, err / bound, np.where(err == 0, 0.0, np.inf))
        worst = float(np.max(ratio)) if ratio.size else 0.0
        self.worst = max(self.worst, worst)
        assert worst < 1.0, (what, worst, np.unravel_index(int(np.argmax(ratio)), ratio.shape))

    def report(self):
        print("  %s: %d elements, largest error / bound = %.3g" % (self.name, self.n, self.worst))
        assert self.n > 0 and self.worst < 1.0


def test_rows_cover_every_regime():
    """At this device's SM count the rows still pin every regime of ``kde_lse_kernel``'s geometry."""
    seen = KX.coverage(sm_count())
    assert KX.REQUIRED_REGIMES <= seen, KX.REQUIRED_REGIMES - seen


def _engine(N, D, bw, nsplits):
    mv = moves.KDEMove(bw, nsplits=nsplits, live_dangerously=True)
    eng = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=mv, seed=1)._engine
    eng.set_option("debug_taps", 1)
    return eng, mv.descriptor()


def _observe(eng, desc, X0, sets, seed, step):
    """One step with only the last split accepting: (X1, taps)."""
    act = sets[-1]
    lp = np.full(X0.shape[0], np.inf)
    lp[act] = -np.inf
    eng.set_state(X0, lp)
    eng.set_rng(seed, step)
    eng.step([(desc, 1.0)], 1)
    X1, lp1 = eng.get_state()
    assert np.all(np.isfinite(lp1[act])), "a proposal was not accepted: the state no longer shows every proposal"
    rest = np.setdiff1d(np.arange(X0.shape[0]), act)
    assert np.array_equal(X1[rest].view(np.uint64), X0[rest].view(np.uint64)), "an earlier split moved"
    taps = eng.debug_taps()
    assert np.array_equal(taps["active"], act)
    return X1, taps


def check_split(trq, trf, eng, X0, X1, taps, sets, seed, step, bw, plan, case=None):
    act, comp = sets[-1], np.concatenate(sets[:-1])
    ns, nc = len(act), len(comp)
    D = X0.shape[1]
    j = KX.centre_ranks(seed, step, len(sets) - 1, ns, nc)
    assert np.array_equal(taps["partners"][0], comp[j]), "kernel centres differ from the draw specification"
    if case is None:
        case = KX.Case(X0[comp], X0, bw, sm_count())
        case.pivots_ok()
    ranks = KX.checked_ranks(ns, plan, 64 if D <= 128 else 24)
    prop = np.arange(ns) if D < 128 else ranks
    z = PX.normals_mp(seed, step, len(sets) - 1, prop, D)
    q_dev = X1[act[prop]]
    q_ref = KX.proposal_reference(case, j[prop], z)
    err = np.abs(q_dev.astype(np.longdouble) - q_ref).astype(np.float64)
    trq.check(err, KX.proposal_bound(case, np.abs(PX.mp_to_f64(z)), np.abs(q_dev)), ("proposals", seed, step))
    S, Q = X0[act[ranks]], X1[act[ranks]]
    ref = KX.factor_reference(case, S, Q)
    bound = KX.factor_bounds(case, ref, S, Q, plan)
    trf.check(KX.factor_error(taps["scalar"][ranks], ref["f"]), bound, ("factors", seed, step))


@pytest.mark.parametrize("name", [r[0] for r in KX.ROWS])
def test_kde_exact(name):
    _, N, D, nsplits, bw, kind = KX.ROW[name]
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here (eps %g >= 1e-18)" % np.finfo(np.longdouble).eps)
    t0 = time.time()
    eng, desc = _engine(N, D, bw, nsplits)
    plan, ns, nc = KX.last_split_plan(N, nsplits, sm_count())
    print("\n%s: N=%d D=%d nsplits=%d bw=%s ns=%d nc=%d %s" % (name, N, D, nsplits, bw, ns, nc, KX.variant(plan)))
    trq = Tracker("proposals")
    trf = Tracker("factors")
    for seed, step in (SEED_STEPS if D <= 128 else SEED_STEPS[:1]):
        rng = np.random.default_rng(seed ^ (N * 1315423911 + D))
        X0 = KX.state(kind, N, D, rng)
        inds = px.split_assignment(seed, step, N, nsplits, True)
        sets = [np.flatnonzero(inds == k) for k in range(nsplits)]
        X1, taps = _observe(eng, desc, X0, sets, seed, step)
        assert eng.last_kernel_variant() == KX.variant(plan)
        check_split(trq, trf, eng, X0, X1, taps, sets, seed, step, bw, plan)
    trq.report()
    trf.report()
    print("  %.1f s (reference included)" % (time.time() - t0))


# ---- singular-factor decisions, both ways ---------------------------------------------------------------------------
def _mp_pivots(C):
    A = PX.ExactCov(C)
    L, piv = PX.chol_psd_mp(A.mp())
    return piv


@pytest.mark.parametrize("D", [16, 64])
def test_rank_deficient_complement_is_refused(D):
    """nc = D rows of rank D - 1 (``rankcap_rows``), N = 2 D: the exact factor drops the last pivot; the device
    raises at split 0 and leaves the state and the iteration as they were."""
    N, seed = 2 * D, 0x51
    rng = np.random.default_rng(D)
    inds = px.split_assignment(seed, 0, N, 2, True)
    sets = [np.flatnonzero(inds == k) for k in range(2)]
    X0 = np.round(rng.standard_normal((N, D)) * 16.0)
    X0[sets[1]] = PX.rankcap_rows(D, rng)  # split 0's complement
    assert len(_mp_pivots(X0[sets[1]])) == D - 1
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.KDEMove(live_dangerously=True), seed=seed)
    with pytest.raises(np.linalg.LinAlgError):
        s.run_mcmc(X0, 1, skip_initial_state_check=True)
    assert s.iteration == 0
    X1, _ = s._engine.get_state()
    assert np.array_equal(X1.view(np.uint64), X0.view(np.uint64))


def test_duplicated_column_is_refused():
    N, D, seed = 64, 8, 0x52
    rng = np.random.default_rng(5)
    X0 = np.round(rng.standard_normal((N, D)) * 16.0)
    X0[:, 5] = X0[:, 2]
    inds = px.split_assignment(seed, 0, N, 2, True)
    assert len(_mp_pivots(X0[inds == 1])) == D - 1
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.KDEMove(), seed=seed)
    with pytest.raises(np.linalg.LinAlgError):
        s.run_mcmc(X0, 1, skip_initial_state_check=True)
    assert s.iteration == 0


def near_singular_rows(n, D, rng):
    """``n`` integer rows whose covariance is full rank with a smallest pivot^2 a few 1e-9 of the largest
    diagonal: the last column is the one before it plus unit noise, at a scale of 3e4."""
    X = np.round(rng.standard_normal((n, D)) * 3.0e4)
    X[:, D - 1] = X[:, D - 2] + np.round(rng.standard_normal(n) * 6.0)
    return X


def test_near_singular_complement_runs_within_bound():
    """nc = D + 1 full-rank rows with a smallest pivot^2 of a few 1e-9 x the largest diagonal: clearly kept
    (``check_pivot_prefix``), so the device runs, and its factors and proposals are within the bounds."""
    D, seed, step = 8, 0x53, 3
    N = 2 * (D + 1)
    rng = np.random.default_rng(11)
    inds = px.split_assignment(seed, step, N, 2, True)
    sets = [np.flatnonzero(inds == k) for k in range(2)]
    X0 = np.round(rng.standard_normal((N, D)) * 16.0)
    X0[sets[0]] = near_singular_rows(D + 1, D, rng)  # the last split's complement
    case = KX.Case(X0[sets[0]], X0, None, sm_count())
    case.pivots_ok()
    d2 = np.diag(case.L) ** 2
    ratio = float(d2.min() / np.max(np.diag(case.Af)))
    print("smallest pivot^2 / largest diagonal = %.3g" % ratio)
    assert 1e-9 <= ratio < 1e-7
    eng, desc = _engine(N, D, None, 2)
    X1, taps = _observe(eng, desc, X0, sets, seed, step)
    plan = KX.kde_plan(len(sets[1]), len(sets[0]), sm_count())
    trq, trf = Tracker("proposals"), Tracker("factors")
    check_split(trq, trf, eng, X0, X1, taps, sets, seed, step, None, plan, case)
    trq.report()
    trf.report()
