"""WalkMove and GaussianMove proposals (``moves_extra.cu``) and the chain moment sums (``launch_moments``, read by
``eb_moments``) against high-precision references, under first-order rounding-error bounds.

How a proposal is observed.  Debug taps do not cover these moves, so the state is set with ``log_prob = -inf`` for
every walker: every finite proposal then has ``lnpdiff = +inf`` and is accepted (red_blue.py:96-101, mh.py:57-58),
and after one step each walker's coordinates are its proposal, bit for bit (the test asserts that every
log-probability is finite afterwards).  In a two-split Walk step split 1's complement is split 0's proposals; both
are in the final state.  Cases vary ``(seed, step)`` through ``set_rng`` instead of running more steps.

Reference.  The bookkeeping comes from the oracle (``oracle/philox.py``: split sets, complement order, helper
subsets, the Philox words of every normal and the GaussianMove ``dim`` draws); the arithmetic is redone in high
precision (``proposals_exact.py``): normals with mpmath at 45 digits from the device's own theta = fl(2 pi u2);
covariances exactly (integer coordinates; split 1's non-integer complement through Python integers); the Cholesky
factor by the ``chol_psd`` rule (threshold 1e-12 max diag, rank cap s - 1) with mpmath up to ndim 32 and
``np.longdouble`` above (u_ld = 2^-64, added to every bound below as its own term).

Bounds (u = 2^-53, gamma_n = n u / (1 - n u); every bound is per element of q and first order in u):

* normals: log within 1 ulp (CUDA math library: 2u relative) halves under the square root, the correctly rounded
  sqrt adds u, sincos is within 2 ulp (4u |component|) and r * cos one more rounding: |dz| <= 7u |z|.
* moment sums (whole complement, one pass about the shift = device column mean of the whole ensemble):
  y = fl(x - shift) is off by u|y|; each sum runs through at most ``depth`` additions (rows staged by one CTA,
  the CTA partials, the final +=), so dS2 <= (2u + gamma_depth) |Y|^T |Y| and dS1 <= (u + gamma_depth) sum|y|;
  cov = (S2 - S1 S1^T / n) / (n - 1) adds the cancellation term (dS1 |S1|^T + |S1| dS1^T + 2u |S1| |S1|^T) / n
  and 2u |cov|.  Because |S1| is about the shift, a shift far from the complement (e.g. zero for an ensemble at
  1e6) inflates the error by |S1|^2 / n while the bound, which uses the intended shift, does not follow.
* helper subsets (two pass): the mean is off by dm <= (gamma_s + u) mean|x|, y by u|y|, the fma chain gamma_s:
  ((2u + gamma_s) |Y|^T |Y| + s dm dm^T) / (s - 1) + u |cov|.
* Cholesky: the computed factor is the exact one of cov + dA + E with |E| <= gamma_{D+1} |L| |L^T| (Higham,
  Thm 10.3); carried to L by dL = L Phi(L^-1 (dA + E) L^-T) (Phi: lower triangle, halved diagonal) bounded
  componentwise with |L^-1|.  With r < D pivots (rank cap or PSD input) the leading r x r block is perturbed
  that way and dL21 = (dA21 + E21 - L21 dL11^T) L11^-T; the dropped columns are exactly zero on both sides.
* q = fl(s + fl(L z)): |dL| |z| + (7u + gamma_{D+1}) |L| |z| (normals, fma chain) + u |q| (the __dadd_rn).
* GaussianMove, scalar / diagonal: sqrt of the variance, f * scale, * n and the normal: (df + 10u) |f scale n|
  + u |q|, with df the relative error of the host's f = exp(-lf + (lf + lf) u) (log, exp 2u each; the product and
  the sum u each).  Full covariance: the host factors the matrix in double (backward error as above, no cov
  rounding), v = f (L z) adds df + u, q = x + v one more u.  Where the step is small against x the last term
  dominates and is attained (a ratio near 1 at ndim 1 is that rounding, not a loose bound elsewhere).

Rows (test id: what it runs):

=====================================  ==========================================================================
walk-D1-odd / walk-D7-odd              whole complement, nwalkers 1003, nsplits 3; splits 0 and 1
walk-D32                               whole complement
walk-rankcap-D16 / -D128               nwalkers = 2 ndim + 1: split 0's complement has ndim rows, rank cap
                                       binds; the active split sits far from it, so that the dropped pivot is
                                       noise above the threshold and only the cap removes it
walk-D129                              two moment passes (blockIdx.y > 0)
walk-D511 / walk-D512                  cov_chol at 256 -> 1024 threads
walk-D770 / walk-D1024                 walk_shared_propose above 48 KB of shared memory
walk-offset1e6                         ensemble at 1e6 with unit spread
walk-cond1e8                           complement covariance of condition number ~1e8
subset-s2-D1, subset-s5-D12            helper subsets; s = 5 < ndim is rank deficient
subset-s64-D63                         odd ndim, s - 1 = ndim
subset-s4096-D64                       nwalkers 8194: opt-in shared memory of the subset kernel
mixed-D16                              nwalkers 1003, s = smallest complement: split 0 shared, split 1 subset
gauss-*                                scalar / diagonal / full; vector / random / sequential; factor none / 1.7;
                                       ndim 1, 2, 5 (nwalkers 1003: a partial last block), 257 and 1024 full;
                                       a zero variance; a PSD full covariance of rank ndim - 2
=====================================  ==========================================================================

Split 1 is checked at ndim <= 16.  The largest error / bound of every class is printed and must stay below 1.
The chain moments (``test_moments_exact``) carry their own derivation in that test's docstring.
"""
import math
import time

import mpmath
import numpy as np
import pytest

import proposals_exact as PX
from oracle import philox as px

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

U = PX.U


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
        print("%s: %d elements, largest error / bound = %.3g" % (self.name, self.n, self.worst))
        assert self.n > 0 and self.worst < 1.0


_SM = []


def sm_count():
    if not _SM:
        import torch

        _SM.append(int(torch.cuda.get_device_properties(0).multi_processor_count))
    return _SM[0]


def _engine(N, D):
    return emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=1)._engine


def _one_step(eng, X0, desc, seed, step):
    eng.set_state(X0, np.full(X0.shape[0], -np.inf))
    eng.set_rng(seed, step)
    eng.step([(desc, 1.0)], 1)
    X1, lp = eng.get_state()
    assert np.all(np.isfinite(lp)), "a proposal was not accepted: the state no longer shows every proposal"
    return X1


def _err(q_dev, q_ref):
    """|q_dev - q_ref| for a reference in mpf (object array) or longdouble."""
    if q_ref.dtype == object:
        with mpmath.workdps(PX.MP_DPS):
            return np.array([[float(abs(mpmath.mpf(float(a)) - b)) for a, b in zip(ra, rb)]
                             for ra, rb in zip(q_dev, q_ref)])
    return np.abs(q_dev.astype(np.longdouble) - q_ref).astype(np.float64)


def _mvn_ref(S, Lref, z):
    """s + L z in the reference's arithmetic: S [rows, D] float64, z [rows, D] mpf, Lref mpf or longdouble."""
    D = S.shape[1]
    if Lref.dtype == object:
        with mpmath.workdps(PX.MP_DPS):
            out = np.empty(S.shape, dtype=object)
            for i in range(S.shape[0]):
                for e in range(D):
                    out[i, e] = mpmath.mpf(float(S[i, e])) + mpmath.fsum(Lref[e, k] * z[i, k] for k in range(e + 1))
            return out
    return S.astype(np.longdouble) + PX.mp_to_ld(z) @ Lref.T


# ---- WalkMove ---------------------------------------------------------------------------------------------------
def _ints(rng, shape, spread):
    return np.round(rng.standard_normal(shape) * spread)


def _walk_state(kind, N, D, rng):
    if kind == "offset":
        return 1.0e6 + _ints(rng, (N, D), 1.0)
    if kind == "cond":
        q, _ = np.linalg.qr(rng.standard_normal((D, D)))
        return np.round((rng.standard_normal((N, D)) * np.logspace(0, 4, D)) @ q.T)
    return _ints(rng, (N, D), 16.0)


WALK_ROWS = [
    # id, N, D, nsplits, s, state kind
    ("walk-D1-odd", 1003, 1, 3, None, "int"),
    ("walk-D7-odd", 1003, 7, 3, None, "int"),
    ("walk-D32", 200, 32, 2, None, "int"),
    ("walk-rankcap-D16", 33, 16, 2, None, "far"),
    ("walk-rankcap-D128", 257, 128, 2, None, "far"),
    ("walk-D129", 300, 129, 2, None, "int"),
    ("walk-D511", 1086, 511, 2, None, "int"),
    ("walk-D512", 1088, 512, 2, None, "int"),
    ("walk-D770", 1604, 770, 2, None, "int"),
    ("walk-D1024", 2112, 1024, 2, None, "int"),
    ("walk-offset1e6", 64, 8, 2, None, "offset"),
    ("walk-cond1e8", 200, 24, 2, None, "cond"),
    ("subset-s2-D1", 64, 1, 2, 2, "int"),
    ("subset-s5-D12", 256, 12, 2, 5, "int"),
    ("subset-s64-D63", 256, 63, 2, 64, "int"),
    ("subset-s4096-D64", 8194, 64, 2, 4096, "int"),
    ("mixed-D16", 1003, 16, 2, 501, "int"),
]
SEED_STEPS = [(0x5EED, 0), (0xB200, 17), (7, 123456789)]


def _ranks(Ns, D, s0, Nc):
    cap = 64 if D <= PX.MP_MAX_D else 12
    if s0 != Nc:
        cap = min(cap, 6)
    if Ns <= cap:
        return np.arange(Ns)
    return np.unique(np.r_[0, Ns - 1, np.linspace(0, Ns - 1, cap - 2).astype(np.int64)])


def _check_walk_split(tr, X0, X1, sets, split, s, seed, step):
    N, D = X0.shape
    nsplits = len(sets)
    act = sets[split]
    state = X0.copy()
    for j in range(split):
        state[sets[j]] = X1[sets[j]]
    C = np.concatenate([state[sets[j]] for j in range(nsplits) if j != split])
    Nc = C.shape[0]
    s0 = Nc if s is None else int(s)
    ranks = _ranks(len(act), D, s0, Nc)
    z = PX.normals_mp(seed, step, split, ranks, D)
    zabs = np.abs(PX.mp_to_f64(z))
    S = state[act[ranks]]
    q_dev = X1[act[ranks]]
    if s0 == Nc:
        A = PX.ExactCov(C)
        L, Lref, piv, uref = PX.chol_reference(A, s0 - 1)
        Af = A.f64()
        r = min(D, Nc - 1)
        PX.check_pivot_prefix(L, piv, r, float(np.max(np.diag(Af))))
        shift = PX.colmean_device_order(state)
        depth = PX.moments_depth(Nc, D, sm_count(), 1)[0]
        Mcov = PX.cov_error_one_pass(C - shift, Nc, depth, Af)
        q_ref = _mvn_ref(S, Lref, z)
        bound = PX.mvn_bound(L, Mcov, r, zabs, np.abs(q_dev), uref)
        tr.check(_err(q_dev, q_ref), bound, ("split", split, "shared", seed, step))
        return
    for k, i in enumerate(ranks):
        inds = px.subset_indices(seed, step, split, int(i), Nc, s0)
        Cs = C[inds]
        A = PX.ExactCov(Cs)
        L, Lref, piv, uref = PX.chol_reference(A, s0 - 1)
        Af = A.f64()
        r = min(D, s0 - 1)
        PX.check_pivot_prefix(L, piv, r, float(np.max(np.diag(Af))))
        Mcov = PX.cov_error_two_pass(Cs, Af)
        q_ref = _mvn_ref(S[k:k + 1], Lref, z[k:k + 1])
        bound = PX.mvn_bound(L, Mcov, r, zabs[k:k + 1], np.abs(q_dev[k:k + 1]), uref)
        tr.check(_err(q_dev[k:k + 1], q_ref), bound, ("split", split, "subset", int(i), seed, step))


@pytest.mark.parametrize("N,D,nsplits,s,kind", [r[1:] for r in WALK_ROWS], ids=[r[0] for r in WALK_ROWS])
def test_walk_proposals_exact(N, D, nsplits, s, kind):
    if D > PX.MP_MAX_D and not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here (eps %g >= 1e-18)" % np.finfo(np.longdouble).eps)
    t0 = time.time()
    tr = Tracker("walk N=%d D=%d nsplits=%d s=%s %s" % (N, D, nsplits, s, kind))
    eng = _engine(N, D)
    desc = moves.WalkMove(s=s, nsplits=nsplits, live_dangerously=N < 2 * D).descriptor()
    pairs = SEED_STEPS if D <= 128 else SEED_STEPS[:2]
    for seed, step in pairs:
        rng = np.random.default_rng(seed ^ (N * 1315423911 + D))
        inds = px.split_assignment(seed, step, N, nsplits, True)
        sets = [np.flatnonzero(inds == j) for j in range(nsplits)]
        if kind == "far":
            X0 = _ints(rng, (N, D), 4.0)
            X0[sets[1]] = PX.rankcap_rows(D, rng)  # split 0's complement: D rows of rank D - 1
            X0[sets[0]] += 4096.0  # the shift (mean of all walkers) sits far from that complement
        else:
            X0 = _walk_state(kind, N, D, rng)
        X1 = _one_step(eng, X0, desc, seed, step)
        assert eng.last_kernel_name() == "walk"
        for split in range(nsplits if D <= 16 else 1):
            _check_walk_split(tr, X0, X1, sets, split, s, seed, step)
    tr.report()
    print("  %.1f s (reference included)" % (time.time() - t0))


def test_walk_cov_chol_time_at_1024():
    """One WalkMove step at ndim 1024, whole complement (one CTA factors the 1024 x 1024 covariance): printed
    for the record, not asserted."""
    N, D = 2112, 1024
    eng = _engine(N, D)
    X0 = _ints(np.random.default_rng(3), (N, D), 16.0)
    desc = moves.WalkMove().descriptor()
    _one_step(eng, X0, desc, 1, 0)
    ms = []
    for k in range(3):
        _one_step(eng, X0, desc, 1, k + 1)
        ms.append(eng.last_step_timing()[0])
    print("WalkMove step at %d x %d: %.2f ms (median of 3)" % (N, D, sorted(ms)[1]))


def test_walk_subset_refused_when_a_larger_complement_needs_the_subset_kernel():
    """nwalkers 257 in two splits: complements of 128 and 129 rows.  s = 128 is the smaller complement, so split 0
    runs the whole-complement kernel, but split 1 would run the helper-subset kernel at ndim 128 (264 712 B of
    shared memory): the documented refusal, before any kernel runs."""
    N, D = 257, 128
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), moves=moves.WalkMove(s=128), seed=1)
    X0 = np.random.default_rng(0).standard_normal((N, D))
    with pytest.raises(NotImplementedError, match="limited to ndim <= 64 and s <= 4096"):
        s.run_mcmc(X0, 1, store=False, skip_initial_state_check=True)
    # s above the envelope at small ndim, also at s = the smallest complement
    s = emcee_b200.EnsembleSampler(8195, 2, models.GaussianIso(), moves=moves.WalkMove(s=4097), seed=1)
    with pytest.raises(NotImplementedError, match="limited to ndim <= 64 and s <= 4096"):
        s.run_mcmc(np.random.default_rng(1).standard_normal((8195, 2)), 1, store=False, skip_initial_state_check=True)
    # equal complements: s = nc is the whole-complement path at any ndim
    s = emcee_b200.EnsembleSampler(256, D, models.GaussianIso(), moves=moves.WalkMove(s=128), seed=1)
    s.run_mcmc(np.random.default_rng(2).standard_normal((256, D)), 1, store=False, skip_initial_state_check=True)


# ---- GaussianMove -----------------------------------------------------------------------------------------------
def _psd_rank(D, k, rng):
    B = rng.standard_normal((D, k)) * 0.2
    return B @ B.T


def _dense_cov(D, rng):
    q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    return (q * np.linspace(0.01, 0.2, D)) @ q.T


GAUSS_ROWS = []
for _D in (1, 2, 5):
    for _form in ("scalar", "diag", "full"):
        if _form == "full" and _D == 1:
            continue
        for _mode in (("vector",) if _form == "full" else ("vector", "random", "sequential")):
            for _fac in (None, 1.7):
                GAUSS_ROWS.append(("gauss-%s-%s-D%d-f%s" % (_form, _mode, _D, _fac), 1003 if _D == 5 else 256, _D,
                                   _form, _mode, _fac))
GAUSS_ROWS += [
    ("gauss-full-vector-D257-f1.7", 300, 257, "full", "vector", 1.7),
    ("gauss-full-vector-D1024", 520, 1024, "full", "vector", None),
    ("gauss-diag0-random-D5", 1003, 5, "diag0", "random", 1.7),
    ("gauss-diag0-vector-D5", 1003, 5, "diag0", "vector", None),
    ("gauss-psd-vector-D16", 100, 16, "psd", "vector", 1.7),
]
_COV_CACHE = {}


@pytest.mark.parametrize("N,D,form,mode,factor", [r[1:] for r in GAUSS_ROWS], ids=[r[0] for r in GAUSS_ROWS])
def test_gaussian_proposals_exact(N, D, form, mode, factor):
    if D > PX.MP_MAX_D and not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here (eps %g >= 1e-18)" % np.finfo(np.longdouble).eps)
    rng = np.random.default_rng(D * 131 + len(form))
    if form == "scalar":
        cov = 0.04
    elif form in ("diag", "diag0"):
        cov = np.linspace(0.01, 0.09, D)
        if form == "diag0":
            cov[[0, D // 2]] = 0.0
    elif form == "full":
        cov = _dense_cov(D, rng)
    else:
        cov = _psd_rank(D, D - 2, rng)
    tr = Tracker("gaussian N=%d D=%d %s %s factor=%s" % (N, D, form, mode, factor))
    eng = _engine(N, D)
    mv = moves.GaussianMove(cov, mode=mode, factor=factor)
    mv.index = 3
    desc = mv.descriptor()
    full = np.ndim(cov) == 2
    if full:
        key = (D, form)
        if key not in _COV_CACHE:
            _COV_CACHE[key] = PX.chol_reference(cov, None)
        L, Lref, piv, uref = _COV_CACHE[key]
        r = D - 2 if form == "psd" else D
        PX.check_pivot_prefix(L, piv, r, float(np.max(np.diag(cov))))
        aL = np.abs(L)
        dL = PX.chol_perturbation(L, PX.backward_error(L) + PX.backward_error(L, uref) + uref * (aL @ aL.T), r)
    for seed, step in SEED_STEPS[:2]:
        X0 = rng.standard_normal((N, D)) + 0.5
        X0[X0 == 0] = 0.25  # no signed zeros: x + 0 must give x back bit for bit
        if full:
            X0[[1, N // 2, N - 1]] = 0.0  # walkers at the origin: q is the shared shift v itself
        X1 = _one_step(eng, X0, desc, seed, step)
        assert eng.last_kernel_name() == "gaussian"
        f, df = PX.factor_f(factor, seed, step)
        if mode == "random":
            w0, w1, _, _ = px.draw_words(seed, step, 0, px.TAG_PROP_B, np.arange(N))
            dim = px.bounded64(w0, w1, D)
        elif mode == "sequential":
            dim = np.full(N, 3 % D)
        else:
            dim = None
        rows = np.arange(N) if N * D <= 2048 else np.unique(np.r_[0, 1, N // 2, N - 1, rng.integers(0, N, 40)])
        if full:
            z = PX.normals_mp(seed, step, 0, [0], D)
            zabs = np.abs(PX.mp_to_f64(z))
            if Lref.dtype == object:
                with mpmath.workdps(PX.MP_DPS):
                    v = np.array([[f * mpmath.fsum(Lref[e, k] * z[0, k] for k in range(e + 1)) for e in range(D)]],
                                 dtype=object)
            else:
                v = np.longdouble(f) * (PX.mp_to_ld(z) @ Lref.T)
            vabs = np.abs(PX.mp_to_f64(v) if v.dtype == object else v.astype(np.float64))
            fl = float(f)
            bv = fl * (zabs @ dL.T + (PX.NORMAL_ERR + PX.gamma(D + 1) + PX.gamma(D + 2, uref)) * (zabs @ aL.T)) + (
                df + U + uref) * vabs
            q_ref = np.empty((len(rows), D), dtype=v.dtype)
            for k, w in enumerate(rows):
                q_ref[k] = (np.array([mpmath.mpf(float(a)) for a in X0[w]], dtype=object) + v[0]
                            if v.dtype == object else X0[w].astype(np.longdouble) + v[0])
            bound = bv + (U + uref) * np.abs(X1[rows])
            tr.check(_err(X1[rows], q_ref), bound, ("full", seed, step))
            origin = X1[[1, N // 2, N - 1]]
            assert np.array_equal(origin.view(np.uint64), np.broadcast_to(origin[0], origin.shape).view(np.uint64))
            continue
        z = PX.normals_mp(seed, step, 0, rows, D)
        zabs = np.abs(PX.mp_to_f64(z))
        var = np.broadcast_to(np.asarray(cov, dtype=np.float64), (D,))
        with mpmath.workdps(PX.MP_DPS):
            sig = [mpmath.sqrt(mpmath.mpf(float(c))) for c in var]
            q_ref = np.empty((len(rows), D), dtype=object)
            for k, w in enumerate(rows):
                for d in range(D):
                    q_ref[k, d] = mpmath.mpf(float(X0[w, d])) + f * sig[d] * z[k, d]
        step_abs = float(f) * np.sqrt(var)[None, :] * zabs
        bound = (df + 10 * U) * step_abs + U * np.abs(X1[rows])
        moved = np.ones((len(rows), D), dtype=bool) if dim is None else (np.arange(D)[None, :] == dim[rows][:, None])
        err = _err(X1[rows], q_ref)
        # every coordinate but the drawn one, and every zero-variance coordinate, is the input bit for bit
        still = ~moved | (var[None, :] == 0.0)
        assert np.array_equal(X1[rows][still].view(np.uint64), X0[rows][still].view(np.uint64))
        tr.check(np.where(moved, err, 0.0), np.where(moved, bound, 1.0), (form, mode, seed, step))
    tr.report()


# ---- chain moments ----------------------------------------------------------------------------------------------
MOMENT_ROWS = [
    # id, N, D, moments_every, steps per run_mcmc call, start
    ("mom-D129-partial-chunk-clipped-grid", 300, 129, 1, (10,), "near"),
    ("mom-D255-two-calls-every3", 520, 255, 3, (7, 8), "near"),
    ("mom-D520", 1050, 520, 1, (4,), "near"),
    ("mom-D1024", 2048, 1024, 1, (2,), "near"),
    ("mom-D129-drift-1e4-sigma", 300, 129, 1, (40,), "far"),
    ("mom-D129-outlier-first-row", 4096, 129, 1, (2,), "outlier"),
]


def _pair_sample(D, rng):
    """(i, j) pairs of the covariance that are compared: the diagonal, rows 0 and D - 1, and 2048 more."""
    i = np.r_[np.arange(D), np.zeros(D, np.int64), np.full(D, D - 1), rng.integers(0, D, 2048)]
    j = np.r_[np.arange(D), np.arange(D), np.arange(D), rng.integers(0, D, 2048)]
    return i, j


@pytest.mark.parametrize("N,D,every,calls,start", [r[1:] for r in MOMENT_ROWS], ids=[r[0] for r in MOMENT_ROWS])
def test_moments_exact(N, D, every, calls, start):
    """``eb_moments`` against a two-pass reference of the stored chain.

    The device folds the rows of every ``every``-th state into S1 = sum(y), S2 = sum(y y^T), y = fl(x - shift),
    with the shift fixed at the column mean of the first accumulated state (colmean_kernel's order, reproduced
    exactly here); then mean = shift + S1 / m and cov = (S2 - S1 S1^T / m) / (m - 1) on the host.  Bounds:
    mean: (u + gamma_depth) sum|y| / m + 2u |S1| / m + u |mean|; cov: the one-pass bound of the module docstring
    with depth = rows one CTA stages per accumulation + CTA partials + number of accumulations.  Reference:
    means as the exact column sums (``math.fsum`` of the values and of their residual) over m in longdouble;
    covariance two-pass in longdouble (pairwise sums) for the diagonal, two full rows and 2048 sampled entries,
    with gamma_m(u_ld) of the reference added to the bound.

    Drift: when the chain moves a distance delta from the shift, |S1| / m ~ delta and the cancellation term
    grows like gamma_depth delta^2 against a covariance of sigma^2: the bound alone reaches 1e-6 relative
    (north_star's bar for the chain moments) at delta ~ sqrt(1e-6 / gamma_depth) sigma, about 8e3 sigma at
    depth ~ 130; rounding that actually accumulates as a random walk loses the bar near 1e5 sigma.  The
    ``drift`` row starts 1e4 sigma from the mode and prints its worst relative error.  The ``outlier`` row
    puts walker 0 1e3 sigma from the rest, so that a shift taken from one row instead of the column mean
    would add u |x_0 - mean|^2 per entry, far above the bound."""
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here (eps %g >= 1e-18)" % np.finfo(np.longdouble).eps)
    rng = np.random.default_rng(N + D)
    X0 = rng.standard_normal((N, D))
    if start == "far":
        X0 += 1.0e4
    elif start == "outlier":
        X0[0] += 1.0e3
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=0x30 + D)
    s.enable_moments(every)
    st = X0
    for n in calls:
        st = s.run_mcmc(st, n, store=True, skip_initial_state_check=True)
    chain = s.get_chain()
    mean_d, cov_d, m, _ = s._engine.moments()
    rows = chain[every - 1::every]
    assert m == rows.shape[0] * N
    ncalls = rows.shape[0]
    X = rows.reshape(-1, D)
    shift = PX.colmean_device_order(rows[0])
    Y = X - shift
    depth, grid, CH = PX.moments_depth(N, D, sm_count(), ncalls)
    print("N=%d D=%d: %d accumulations, grid %d, CH %d, depth %d" % (N, D, ncalls, grid, CH, depth))
    # exact column sums: the rounded fsum plus the rounded residual
    hi = np.array([math.fsum(X[:, d]) for d in range(D)])
    lo = np.array([math.fsum(np.r_[X[:, d], -hi[d]]) for d in range(D)])
    mean_ref = (hi.astype(np.longdouble) + lo.astype(np.longdouble)) / np.longdouble(m)
    aY = np.abs(Y)
    S1 = Y.sum(axis=0)
    b_mean = (U + PX.gamma(depth)) * aY.sum(axis=0) / m + 2 * U * np.abs(S1) / m + (U + PX.ULD) * np.abs(mean_d)
    tm = Tracker("moments mean N=%d D=%d %s" % (N, D, start))
    tm.check(np.abs(mean_d.astype(np.longdouble) - mean_ref).astype(np.float64), b_mean, "mean")
    i, j = _pair_sample(D, rng)
    Xc = X.astype(np.longdouble) - mean_ref
    ref = np.empty(len(i), dtype=np.longdouble)
    P = np.empty(len(i))
    for a in range(0, len(i), 256):
        sl = slice(a, a + 256)
        ref[sl] = np.sum(Xc[:, i[sl]] * Xc[:, j[sl]], axis=0) / np.longdouble(m - 1)
        P[sl] = np.sum(aY[:, i[sl]] * aY[:, j[sl]], axis=0)
    aS1 = np.abs(S1)
    dS1 = (U + PX.gamma(depth)) * aY.sum(axis=0)
    cov_ref = ref.astype(np.float64)
    b_cov = ((2 * U + PX.gamma(depth)) * P + (dS1[i] * aS1[j] + aS1[i] * dS1[j]) / m
             + 2 * U * aS1[i] * aS1[j] / m) / (m - 1) + 2 * U * np.abs(cov_ref)
    b_cov += PX.gamma(m + 2, PX.ULD) * P / (m - 1)
    tc = Tracker("moments cov N=%d D=%d %s" % (N, D, start))
    err = np.abs(cov_d[i, j].astype(np.longdouble) - ref).astype(np.float64)
    tc.check(err, b_cov, "cov")
    scale = np.sqrt(np.abs(cov_ref[:D]))  # the diagonal comes first in the sample
    rel = float(np.max(err / (scale[i] * scale[j])))
    print("  largest |cov error| / sqrt(cov_ii cov_jj) = %.3g; drift of the final mean from the shift = %.3g"
          % (rel, float(np.max(np.abs(np.asarray(mean_ref, dtype=np.float64) - shift)))))
    tm.report()
    tc.report()
