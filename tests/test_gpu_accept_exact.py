"""The Metropolis accept decision of every half-step kernel, and the DE and snooker proposals, against
high-precision references, under first-order rounding-error bounds.

The decision.  Every kernel computes ``lnpdiff = fl(fl(factor + lp_new) - lp_old)`` and accepts iff
``lnpdiff > log u`` (red_blue.py:96-101, mh.py:57-58).  With ``A = fl(factor + lp_new)`` fixed, ``fl(A - L)`` is
monotone in ``L``, so for each walker there is one threshold ``L*``: the device accepts iff ``lp_old < L*``.  The
test finds it from outside:

1. observation run: every walker starts at ``log_prob = -inf``, so one step accepts every finite proposal, and the
   state then holds each walker's proposal ``q_dev`` and its log-probability, bit for bit;
2. per split k: the walkers of splits below k start at ``-inf`` again (they accept, so split k sees the same
   complement and makes the same proposals), the sampled walkers of split k start at a chosen ``L``, and the step
   is repeated with the same ``(seed, step)``.  The mask ``eng.step`` returns is the decision.  Each walker's
   threshold is bracketed between ``T - 4B`` (must accept) and ``T + 4B`` (must reject), then bisected, one step per
   round, until the bracket is narrower than ``B / 64`` or than one ulp of ``L``.  Splits above k are ignored;
3. reference: ``T = F + lp(q_dev) - ln u`` at 45 digits, with ``u`` the exact accept uniform of the draw
   specification, ``lp`` exact at the device's own proposal (``logprob_exact``), and ``F`` the exact Hastings factor
   at the device's inputs: ``(D - 1) ln zz`` for stretch (``zz`` the bit-exact double of the draw spec),
   ``(D - 1)(ln |q_dev - z| - ln |s - z|)`` for snooker, 0 for DE, Walk and Gaussian.

Bounds (u = 2^-53, gamma_n = n u / (1 - n u), first order; ``accept_exact.py`` evaluates them):

* dF, stretch: the device log within 1 ulp (2u |ln zz|, times D - 1 exactly) and the product: 3u |F|.
* dF, snooker: norm and qn = sqrt(sum fl(a - b)^2) through fma chains and a group tree of depth <= D carry
  eps = (2u + gamma_D) / 2 + u relative each; two logs add 2u |ln norm| + 2u |ln qn|, the subtraction
  u |ln qn - ln norm|, all times D - 1, and the product u |F|.
* dlp: the per-model bounds of ``test_gpu_logprob_exact.py`` (iso, ring, Rosenbrock, generic dense); the
  dense_dmma bound on that kernel.
* B = dF + dlp + u |F + lp| (A's rounding) + u |ln u| (the subtraction; at the threshold A - L = log u)
  + 2u |ln u| (the device log).
* The check: the largest accepted ``L`` may not exceed T + B, the smallest rejected one may not fall below T - B.
  The ratio printed is max(lo - T, T - hi) / B: for a device threshold at T + delta, about |delta| / B.

Proposals (same observation run; bookkeeping from ``oracle/redblue.py``: DE pairs, snooker triples, row order):

* DE, q = s + gamma (c1 - c0), gamma = g0 (1 + sigma n): the normal from the device's angle fl(2 pi u2) at 45
  digits, its device value within 7u |n| (log 1 ulp halved by sqrt, sqrt u, cos 2 ulp = 4u, the product u);
  |dgamma| <= g0 sigma 8u |n| + 2u |gamma|; |dq| <= |dgamma| |c1 - c0| + 2u |gamma (c1 - c0)| + u |q|.
* snooker: u_e = fl(d_e / norm) within eps_u = 2u + eps; dd = fl(u.z1) - fl(u.z2) within
  (eps_u + gamma_D) sum |u| (|z1| + |z2|) + u |dd| (the cancellation of z1 ~ z2 lives in that sum);
  |dq_e| <= gs (|u_e| |ddd| + |dd| |u_e| (eps_u + 2u)) + u |q_e|.
* mpmath references up to ndim 32, np.longdouble above with the same bound at its unit roundoff added.
* taps (debug_taps = 1, generic kernel, the last split): stretch zz and the accept uniform bit-exact, DE gamma within
  |dgamma|, snooker norm within eps norm.

Rows (three (seed, step) pairs each, at most 64 sampled walkers per split with the first and last active ranks;
``eb_last_kernel_variant`` asserted on every row):

==========================  ==================================================================================
generic-st37-iso-taps       generic kernel, odd ndim, stretch; zz / u taps
generic-de37-ring-taps      generic DE; gamma taps
generic-sn37-rosen-taps     generic snooker; norm taps
generic-dense130            generic kernel, dense Gaussian above the DMMA envelope
s16-iso / s32-rosen         tma_rows OWN_REG, R = 16 / 8
s128-ring / s96-iso         register path without OWN_REG (R = 2); strided path
s256-ring / s400-iso        R = 1 EPL = 8 (16 warps); R = 1 strided, 14 warps
de24 / de64 / de128 / de256 tma_rows DE, R = 8 / 2 / 1 strided, and the R = 1 register path
sn16 / sn64 / sn96 / sn200  tma_rows snooker, strided paths
sn256                       the snooker register path (R = 1, EPL = 8, 10 warps)
cross-s128 / cross-de128    more than G tiles per warp: batch crossings of prep_batch (sized from the SM count)
dmma-D8/64/128 (-mean)      dense_dmma, one half-step per launch
dmma-D64-group2             dmma_group = 2: both half-steps in one launch
dmma-D64-pdl0               programmatic dependent launch off
dmma-D64-box / s32-box      a box that never binds: the BOUNDED instantiations
gauss-diag-D5               GaussianMove, MOVE_PRECOMPUTED: walker-indexed u, no split table (mh.py)
walk-D8                     WalkMove, whole complement, both splits
rosen-far-s32               |lp| ~ 1e6: u |lp| dominates B
s16-a1.0001                 zz ~ 1, F ~ 0
de24-sigma1-gamma1          sigma = 1, gamma0 = 1: the normal's error reaches q
sn16-cluster                all walkers within 1e-7 of one point: s close to z (small norm), z1 ~ z2 (cancellation)
==========================  ==================================================================================

``test_snooker_s_equals_z_raises_like_the_reference``: every snooker cell with ``s == z`` in coordinates raises
``ValueError("At least one parameter value was NaN")``, as the reference does (its 0/0, ensemble.py:477-478).
"""
import time

import numpy as np
import pytest

import accept_exact as AX
from oracle import philox as px
from oracle import redblue as rb
from oracle import targets as T

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

SEED_STEPS = [(0x5EED, 0), (0xB200, 17), (7, 123456789)]
MAX_SAMPLE = 64
WORST = {}


class Tracker(object):
    """Largest error / bound of one class."""

    def __init__(self, name):
        self.name, self.worst, self.n = name, 0.0, 0

    def check(self, ratio, what):
        ratio = np.atleast_1d(np.asarray(ratio, dtype=np.float64))
        self.n += ratio.size
        worst = float(np.max(ratio)) if ratio.size else 0.0
        self.worst = max(self.worst, worst)
        assert worst < 1.0, (self.name, what, worst, int(np.argmax(ratio)))

    def report(self, cls):
        print("%s: %d values, largest error / bound = %.3g" % (self.name, self.n, self.worst))
        assert self.n > 0 and self.worst < 1.0
        WORST[cls] = max(WORST.get(cls, 0.0), self.worst)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for cls in sorted(WORST):
        print("largest error / bound, %s: %.3g" % (cls, WORST[cls]))


def _sm():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


def _tma(R, epl, own_reg, warps=16):
    return "tma_rows R=%d epl=%d own_reg=%d warps=%d" % (R, epl, own_reg, warps)


# ---- rows ------------------------------------------------------------------------------------------------------
# id, model, N (int, or a callable of the SM count), D, move, options, expected variant (None: checked by kernel
# name), state kind
ST = ("stretch", 2.0)
DE = ("de", 1e-5, None)
SN = ("snooker", 1.7)


def _cross_n(R):
    G = 32 // R
    return lambda sm: 2 * (R * (G * 16 * sm + 2 * sm) + 1)


ROWS = [
    ("generic-st37-iso-taps", "iso", 301, 37, ST, (("debug_taps", 1),), "generic G=16", "normal"),
    ("generic-de37-ring-taps", "ring", 301, 37, DE, (("debug_taps", 1),), "generic G=16", "normal"),
    ("generic-sn37-rosen-taps", "rosenbrock", 301, 37, SN, (("debug_taps", 1),), "generic G=16", "normal"),
    ("generic-dense130", "dense", 301, 130, ST, (), "generic G=32", "normal"),
    ("s16-iso", "iso", 2 * (16 * 8 + 1), 16, ST, (), _tma(16, 8, 1), "normal"),
    ("s32-rosen", "rosenbrock", 2 * (8 * 20 + 7), 32, ST, (), _tma(8, 8, 1), "normal"),
    ("s128-ring", "ring", 2 * (2 * 150 + 1), 128, ST, (), _tma(2, 8, 0), "normal"),
    ("s96-iso", "iso", 403, 96, ST, (), _tma(2, 0, 0), "normal"),
    ("s256-ring", "ring", 1029, 256, ST, (), _tma(1, 8, 0), "normal"),
    ("s400-iso", "iso", 1203, 400, ST, (), _tma(1, 0, 0, 14), "normal"),
    ("de24-iso", "iso", 301, 24, DE, (), _tma(8, 0, 0), "normal"),
    ("de64-ring", "ring", 413, 64, DE, (), _tma(2, 0, 0), "normal"),
    ("de128-iso", "iso", 517, 128, DE, (), _tma(1, 0, 0), "normal"),
    ("de256-ring", "ring", 1031, 256, DE, (), _tma(1, 8, 0, 13), "normal"),
    ("sn16-iso", "iso", 301, 16, SN, (), _tma(8, 0, 0), "normal"),
    ("sn64-rosen", "rosenbrock", 413, 64, SN, (), _tma(2, 0, 0), "normal"),
    ("sn96-iso", "iso", 517, 96, SN, (), _tma(1, 0, 0), "normal"),
    ("sn200-ring", "ring", 806, 200, SN, (), _tma(1, 0, 0, 13), "normal"),
    ("sn256-iso", "iso", 1030, 256, SN, (), _tma(1, 8, 0, 10), "normal"),
    ("cross-s128-iso", "iso", _cross_n(2), 128, ST, (), _tma(2, 8, 0), "normal"),
    ("cross-de128-rosen", "rosenbrock", _cross_n(1), 128, DE, (), _tma(1, 0, 0), "normal"),
    ("dmma-D8", "dense", 301, 8, ST, (), "dmma", "normal"),
    ("dmma-D8-mean", "dense-mean", 301, 8, ST, (), "dmma", "normal"),
    ("dmma-D64", "dense", 517, 64, ST, (), "dmma", "normal"),
    ("dmma-D64-mean", "dense-mean", 517, 64, ST, (), "dmma", "normal"),
    ("dmma-D128", "dense", 1001, 128, ST, (), "dmma", "normal"),
    ("dmma-D128-mean", "dense-mean", 1001, 128, ST, (), "dmma", "normal"),
    ("dmma-D64-group2", "dense-mean", 517, 64, ST, (("dmma_group", 2),), "dmma", "normal"),
    ("dmma-D64-pdl0", "dense", 517, 64, ST, (("pdl", 0),), "dmma", "normal"),
    ("dmma-D64-box", "dense-box", 517, 64, ST, (), "dmma", "normal"),
    ("s32-box", "rosenbrock-box", 2 * (8 * 20 + 7), 32, ST, (), _tma(8, 8, 1), "normal"),
    ("gauss-diag-D5", "iso", 1003, 5, ("gauss",), (), "gaussian", "normal"),
    ("walk-D8", "iso", 64, 8, ("walk",), (), "walk", "normal"),
    ("rosen-far-s32", "rosenbrock", 2 * (8 * 20 + 7), 32, ST, (), _tma(8, 8, 1), "far"),
    ("s16-a1.0001", "iso", 2 * (16 * 8 + 1), 16, ("stretch", 1.0001), (), _tma(16, 8, 1), "normal"),
    ("de24-sigma1-gamma1", "iso", 301, 24, ("de", 1.0, 1.0), (), _tma(8, 0, 0), "normal"),
    ("sn16-cluster", "iso", 301, 16, SN, (), _tma(8, 0, 0), "cluster"),
]


def _model(kind, D):
    """(device model, accept_exact.Model, state scale for 'normal' rows)."""
    if kind == "iso":
        return models.GaussianIso(), AX.Model("iso"), 1.0
    if kind == "ring":
        return models.Ring(5.0, 0.5), AX.Model("ring", (5.0, 0.5)), 5.0 / np.sqrt(D)
    if kind.startswith("rosenbrock"):
        m = models.Rosenbrock(1.0, 100.0)
        if kind.endswith("-box"):
            m = models.Bounded(m, np.full(D, -1e300), np.full(D, 1e300))
        return m, AX.Model("rosenbrock", (1.0, 100.0)), 0.1
    A = T.make_config("gauss_dense", 8, D)[0].icov
    mu = np.linspace(-0.5, 0.75, D) if kind == "dense-mean" else None
    m = models.GaussianDense(A, mu)
    if kind == "dense-box":
        m = models.Bounded(m, np.full(D, -1e300), np.full(D, 1e300))
    dmma = D % 8 == 0 and D <= 128
    return m, AX.Model("dense", A=A, mu=mu, dmma=dmma), 1.0


def _move(spec, D, nsplits=2):
    if spec[0] == "stretch":
        return moves.StretchMove(a=spec[1], nsplits=nsplits), rb.Stretch(a=spec[1], nsplits=nsplits)
    if spec[0] == "de":
        return (moves.DEMove(sigma=spec[1], gamma0=spec[2], nsplits=nsplits),
                rb.DE(sigma=spec[1], gamma0=spec[2], nsplits=nsplits))
    if spec[0] == "snooker":
        return moves.DESnookerMove(gammas=spec[1]), rb.Snooker(gammas=spec[1])
    if spec[0] == "walk":
        return moves.WalkMove(), rb.Walk()
    mv = moves.GaussianMove(np.linspace(0.01, 0.09, D))
    return mv, None


def _state(kind, model_kind, N, D, scale, rng):
    if kind == "far":
        return 5.0 + 0.1 * rng.standard_normal((N, D))
    if kind == "cluster":
        return 3.0 + 1e-7 * rng.standard_normal((N, D))
    X = rng.standard_normal((N, D)) * scale
    return X + 1.0 if model_kind.startswith("rosenbrock") else X


def _ranks(n):
    if n <= MAX_SAMPLE:
        return np.arange(n)
    return np.unique(np.r_[0, n - 1, np.linspace(0, n - 1, MAX_SAMPLE - 2).astype(np.int64)])


def _step(eng, X0, lp, desc, seed, step):
    eng.set_state(X0, lp)
    eng.set_rng(seed, step)
    return eng.step([(desc, 1.0)], 1)


def _check_variant(eng, variant, N, sm):
    if variant in ("walk", "gaussian"):
        assert eng.last_kernel_name() == variant
    elif variant == "dmma":
        assert eng.last_kernel_variant().startswith("dense_dmma nhalf_max="), eng.last_kernel_variant()
        grid = min(((N + 1) // 2 + 7) // 8, sm)
        assert eng.last_kernel_variant().endswith(" grid=%d" % grid), eng.last_kernel_variant()
    else:
        assert eng.last_kernel_variant() == variant


def _complement_state(X0, X1, sets, k):
    state = X0.copy()
    for j in range(k):
        state[sets[j]] = X1[sets[j]]
    return state


@pytest.mark.parametrize("model_kind,N,D,mspec,options,variant,skind", [r[1:] for r in ROWS], ids=[r[0] for r in ROWS])
def test_accept_threshold_exact(model_kind, N, D, mspec, options, variant, skind, nsplits=2):
    """nsplits (stretch and DE rows only) is left at the default here; test_gpu_splits.py runs rows at 7 splits."""
    if D > AX.MP_MAX_D and mspec[0] in ("de", "snooker") and not AX.PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here (eps %g >= 1e-18)" % np.finfo(np.longdouble).eps)
    t0 = time.time()
    sm = _sm()
    if callable(N):
        N = N(sm)
    dmodel, xm, scale = _model(model_kind, D)
    dmove, omove = _move(mspec, D, nsplits)
    desc = dmove.descriptor()
    eng = emcee_b200.EnsembleSampler(N, D, dmodel, seed=1)._engine
    for k, v in options:
        eng.set_option(k, v)
    taps = dict(options).get("debug_taps", 0)
    cls = variant.split(" ")[0] if variant.startswith(("generic", "tma_rows")) else (
        "dense_dmma" if variant == "dmma" else "precomputed")
    ta = Tracker("accept %s N=%d D=%d %s" % (variant, N, D, mspec))
    tq = Tracker("proposal %s N=%d D=%d %s" % (variant, N, D, mspec))
    tt = Tracker("taps N=%d D=%d %s" % (N, D, mspec))
    pairs = SEED_STEPS if N * D <= 4_000_000 else SEED_STEPS[:2]
    for seed, step in pairs:
        rng = np.random.default_rng(seed ^ (N * 7919 + D))
        X0 = _state(skind, model_kind, N, D, scale, rng)
        minus_inf = np.full(N, -np.inf)
        acc = _step(eng, X0, minus_inf, desc, seed, step)
        _check_variant(eng, variant, N, sm)
        X1, lp1 = eng.get_state()
        assert np.all(np.isfinite(lp1)) and acc.all(), "a proposal was not accepted: the state does not show it"
        if omove is None:  # MHMove: every walker in one set, accept uniform indexed by walker
            sets = [np.arange(N)]
        else:
            inds = px.split_assignment(seed, step, N, omove.nsplits, True)
            sets = [np.flatnonzero(inds == j) for j in range(omove.nsplits)]
        if taps:
            tap = eng.debug_taps()
        for k in range(len(sets)):
            act = sets[k]
            ranks = _ranks(len(act))
            walkers = act[ranks]
            state = _complement_state(X0, X1, sets, k)
            u = AX.accept_u(seed, step, k, ranks)
            if mspec[0] == "stretch":
                zz = AX.stretch_zz(mspec[1], seed, step, k, ranks)
            if mspec[0] in ("de", "snooker"):
                o = rb.OracleSampler(N, D, None, [(omove, 1.0)], seed=seed)
                o.coords = state
                sets_c = sets[:k] + sets[k + 1:]
                getattr(o, "_" + omove.kind)(omove, state[act], sets_c, step, k)
                otaps = o.taps
            if mspec[0] == "de":
                g0 = mspec[2] if mspec[2] is not None else 2.38 / np.sqrt(2.0 * D)
                n_mp, n = AX.de_normal_mp(seed, step, k, ranks)
            Ts, Bs = [], []
            for j, (r, w) in enumerate(zip(ranks, walkers)):
                q = X1[w]
                lp = xm.exact(q)
                dlp = xm.bound(q, lp)
                if mspec[0] == "stretch":
                    F, dF = AX.stretch_factor(zz[j], D)
                elif mspec[0] == "snooker":
                    z, z1, z2 = (state[otaps[key][r]] for key in ("z", "z1", "z2"))
                    F, dF = AX.snooker_factor(state[w], z, q, D)
                    q_ref, uref = AX.snooker_q_ref(state[w], z, z1, z2, mspec[1])
                    b = AX.snooker_q_bound(state[w], z, z1, z2, mspec[1], q) + AX.snooker_q_bound(
                        state[w], z, z1, z2, mspec[1], q, uref)
                    tq.check(AX.q_error(q, q_ref) / b, ("snooker q", seed, step, k, int(w)))
                else:
                    F, dF = AX.mpf(0.0), 0.0
                    if mspec[0] == "de":
                        c0, c1 = state[otaps["p0"][r]], state[otaps["p1"][r]]
                        g, dg = AX.de_gamma(g0, mspec[1], n_mp[j], n[j])
                        q_ref, uref = AX.de_q_ref(state[w], c0, c1, g)
                        b = AX.de_q_bound(state[w], c0, c1, g, dg, q, uref)
                        tq.check(AX.q_error(q, q_ref) / b, ("de q", seed, step, k, int(w)))
                        if taps and k == len(sets) - 1:
                            tt.check(AX.abs_err(tap["scalar"][r], g) / dg, ("gamma tap", int(w)))
                T_, B_ = AX.threshold(F, dF, lp, dlp, u[j])
                Ts.append(T_)
                Bs.append(B_)
                if taps and k == len(sets) - 1 and mspec[0] == "snooker":
                    nrm = AX.norm_exact(state[w], state[otaps["z"][r]])
                    tt.check(AX.abs_err(tap["scalar"][r], nrm) / (AX.norm_rel_err(D) * float(nrm)),
                             ("norm tap", int(w)))
            Bs = np.array(Bs)
            lp_run = minus_inf.copy()

            def decide(L):
                lp_run[walkers] = L
                return _step(eng, X0, lp_run, desc, seed, step)[walkers]

            lo, hi, bad = AX.bisect_thresholds(decide, Ts, Bs)
            assert bad.size == 0, ("threshold outside [T - 4B, T + 4B]", seed, step, k, walkers[bad],
                                   [float(Ts[i]) for i in bad], Bs[bad])
            ta.check([AX.bracket_ratio(a, b_, t, bb) for a, b_, t, bb in zip(lo, hi, Ts, Bs)],
                     ("threshold", seed, step, k))
            if taps and k == len(sets) - 1:
                assert np.array_equal(tap["active"][ranks], walkers)
                assert np.array_equal(tap["u_accept"][ranks].view(np.uint64), u.view(np.uint64))
                if mspec[0] == "stretch":
                    assert np.array_equal(tap["scalar"][ranks].view(np.uint64), zz.view(np.uint64))
                    tt.n += len(ranks)
    ta.report("accept threshold, " + cls)
    if mspec[0] in ("de", "snooker"):
        tq.report("%s proposal" % mspec[0])
    if taps:
        tt.report("taps")
    print("  %.1f s" % (time.time() - t0))


SNOOKER_CELLS = [
    # id, model, N, D, variant
    ("generic-D37", "rosenbrock", 301, 37, "generic G=16"),
    ("sn16", "iso", 301, 16, _tma(8, 0, 0)),
    ("sn64", "rosenbrock", 413, 64, _tma(2, 0, 0)),
    ("sn96", "iso", 517, 96, _tma(1, 0, 0)),
    ("sn200", "ring", 806, 200, _tma(1, 0, 0, 13)),
    ("sn256", "iso", 1030, 256, _tma(1, 8, 0, 10)),
]


@pytest.mark.parametrize("model_kind,N,D,variant", [c[1:] for c in SNOOKER_CELLS], ids=[c[0] for c in SNOOKER_CELLS])
def test_snooker_s_equals_z_raises_like_the_reference(model_kind, N, D, variant):
    """Every walker at the same point: s - z = 0, |s - z| = 0 and u = 0 / 0 (de_snooker.py:41-43), so every proposal
    is NaN.  The reference raises ValueError("At least one parameter value was NaN") from compute_log_prob
    (ensemble.py:477-478); so must every snooker cell, and the sampler stays usable."""
    dmodel, _, scale = _model(model_kind, D)
    target = T.make_config(model_kind if model_kind != "iso" else "gauss_iso", N, D)[0]
    X0 = np.tile(np.linspace(0.5, 1.5, D), (N, 1))
    o = rb.OracleSampler(N, D, target, [(rb.Snooker(), 1.0)], seed=3)
    o.set_state(X0)
    with np.errstate(invalid="ignore", divide="ignore"):
        with pytest.raises(ValueError) as ref:
            o.run(1)
    s = emcee_b200.EnsembleSampler(N, D, dmodel, moves=moves.DESnookerMove(), seed=3)
    with pytest.raises(ValueError) as dev:
        s.run_mcmc(X0, 1, store=False, skip_initial_state_check=True)
    assert str(dev.value) == str(ref.value) == "At least one parameter value was NaN"
    assert s._engine.last_kernel_variant() == variant
    X = _state("normal", model_kind, N, D, scale, np.random.default_rng(D))
    last = s.run_mcmc(X, 2, store=False, skip_initial_state_check=True)
    assert np.all(np.isfinite(last.log_prob))
