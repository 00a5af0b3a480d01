"""The reference machinery of ``test_gpu_accept_exact.py`` checked on the CPU: the references against the numpy
oracle's proposals and Hastings factors; each bound against a planted error in a numpy emulation of the device
arithmetic (log u in single precision, a snooker factor with D for D - 1, emcee's historical u = d / sqrt(norm), a
single-precision cosine in the DE normal, zz one ulp off); and the bisection against an emulated decision."""
import numpy as np
import pytest

import accept_exact as AX
from oracle import philox as px
from oracle import redblue as rb

U = AX.U
needs_ld = pytest.mark.skipif(not AX.PX.longdouble_ok(), reason="np.longdouble is not wider than double here")


def _oracle_split(mv, N, D, seed, step, rng, shift=0.0, spread=1.0):
    X = shift + rng.standard_normal((N, D)) * spread
    o = rb.OracleSampler(N, D, None, [(mv, 1.0)], seed=seed)
    o.coords = X
    inds = px.split_assignment(seed, step, N, mv.nsplits, True)
    sets = [np.flatnonzero(inds == j) for j in range(mv.nsplits)]
    act = sets[0]
    with np.errstate(all="ignore"):
        q, fac = getattr(o, "_" + mv.kind)(mv, X[act], sets[1:], step, 0)
    return X, act, q, fac, o.taps


def _de_emulated(X, act, taps, mv, D, seed, step, cos=np.cos):
    """q of the generic DE kernel in numpy, with a replaceable cosine."""
    ranks = np.arange(len(act))
    b0, b1, b2, b3 = px.draw_words(seed, step, 0, px.TAG_PROP_B, ranks)
    u1, u2 = px.u53(b0, b1), px.u53(b2, b3)
    n = np.sqrt(-2.0 * np.log(1.0 - u1)) * cos(AX.TWO_PI * u2)
    g0 = mv.gamma0 if mv.gamma0 is not None else 2.38 / np.sqrt(2.0 * D)
    g = g0 * (1.0 + mv.sigma * n)
    return X[act] + g[:, None] * (X[taps["p1"]] - X[taps["p0"]])


@pytest.mark.parametrize("D", [5, pytest.param(48, marks=needs_ld)])
@pytest.mark.parametrize("sigma,gamma0", [(1e-5, None), (1.0, 1.0)])
def test_de_reference_agrees_with_the_oracle(D, sigma, gamma0):
    mv = rb.DE(sigma=sigma, gamma0=gamma0)
    seed, step = 11, 3
    X, act, q, _, taps = _oracle_split(mv, 64, D, seed, step, np.random.default_rng(D))
    ranks = np.arange(len(act))
    n_mp, n = AX.de_normal_mp(seed, step, 0, ranks)
    g0 = gamma0 if gamma0 is not None else 2.38 / np.sqrt(2.0 * D)
    worst_good, worst_bad = 0.0, 0.0
    bad = _de_emulated(X, act, taps, mv, D, seed, step,
                       cos=lambda t: np.cos(t.astype(np.float32)).astype(np.float64))
    for r in ranks:
        c0, c1 = X[taps["p0"][r]], X[taps["p1"][r]]
        g, dg = AX.de_gamma(g0, sigma, n_mp[r], n[r])
        q_ref, uref = AX.de_q_ref(X[act[r]], c0, c1, g)
        b = AX.de_q_bound(X[act[r]], c0, c1, g, dg, q[r], uref)
        worst_good = max(worst_good, float(np.max(AX.q_error(q[r], q_ref) / b)))
        worst_bad = max(worst_bad, float(np.max(AX.q_error(bad[r], q_ref) / b)))
    assert worst_good < 1.0, worst_good
    if sigma == 1.0:  # a single-precision cosine in the normal: caught only where the normal reaches q
        assert worst_bad > 1.0, worst_bad


@pytest.mark.parametrize("D", [6, pytest.param(40, marks=needs_ld)])
@pytest.mark.parametrize("kind", ["spread", "cluster"])
def test_snooker_reference_agrees_with_the_oracle(D, kind):
    mv = rb.Snooker()
    seed, step = 5, 8
    rng = np.random.default_rng(D + len(kind))
    if kind == "cluster":  # small norms and z1 ~ z2
        X, act, q, fac, taps = _oracle_split(mv, 96, D, seed, step, rng, 3.0, 1e-7)
    else:
        X, act, q, fac, taps = _oracle_split(mv, 96, D, seed, step, rng)
    gs = mv.gammas
    for r in range(len(act)):
        s, z, z1, z2 = X[act[r]], X[taps["z"][r]], X[taps["z1"][r]], X[taps["z2"][r]]
        q_ref, uref = AX.snooker_q_ref(s, z, z1, z2, gs)
        b = AX.snooker_q_bound(s, z, z1, z2, gs, q[r]) + AX.snooker_q_bound(s, z, z1, z2, gs, q[r], uref)
        assert np.all(AX.q_error(q[r], q_ref) < b), (r, np.max(AX.q_error(q[r], q_ref) / b))
        F, dF = AX.snooker_factor(s, z, q[r], D)
        assert AX.abs_err(fac[r], F) < dF, (r, AX.abs_err(fac[r], F), dF)
        # emcee's historical u = d / sqrt(norm): far outside the bound
        d = s - z
        nrm = np.sqrt(np.dot(d, d))
        u_bad = d / np.sqrt(nrm)
        q_bad = s + u_bad * gs * (np.dot(u_bad, z1) - np.dot(u_bad, z2))
        assert np.any(AX.q_error(q_bad, q_ref) > b)


def _emulated_threshold_case(D, a, seed, step, rng, xscale=1.0):
    """Stretch half-step quantities of split 0 at iso log-probabilities: (u, zz, lp_dev, lp exact, bound)."""
    ranks = np.arange(48)
    u = AX.accept_u(seed, step, 0, ranks)
    zz = AX.stretch_zz(a, seed, step, 0, ranks)
    X = rng.standard_normal((len(ranks), D)) * xscale
    m = AX.Model("iso")
    lp_dev = -0.5 * np.sum(X * X, axis=1)
    lp = [m.exact(x) for x in X]
    dlp = [m.bound(x, l) for x, l in zip(X, lp)]
    return u, zz, lp_dev, lp, dlp


def _emulated_ratios(D, u, zz, lp_dev, lp, dlp, log_u=np.log, zz_dev=None):
    """Bisected threshold of the emulated device decision fl(fl(F~ + lp~) - L) > log~(u), as ratios to B."""
    zz_dev = zz if zz_dev is None else zz_dev
    F_dev = (D - 1.0) * np.log(zz_dev)
    A = F_dev + lp_dev
    lu = log_u(u)
    TB = [AX.threshold(*AX.stretch_factor(zz[i], D), lp[i], dlp[i], u[i]) for i in range(len(u))]
    T, B = [t for t, _ in TB], np.array([b for _, b in TB])
    lo, hi, bad = AX.bisect_thresholds(lambda L: (A - L) > lu, T, B)
    if bad.size:
        return np.array([np.inf])
    return np.array([AX.bracket_ratio(lo[i], hi[i], T[i], B[i]) for i in range(len(u))])


def test_threshold_bound_holds_for_the_device_arithmetic_and_rejects_planted_errors():
    D, seed, step = 37, 0xB200, 5
    u, zz, lp_dev, lp, dlp = _emulated_threshold_case(D, 2.0, seed, step, np.random.default_rng(1))
    assert np.max(_emulated_ratios(D, u, zz, lp_dev, lp, dlp)) < 1.0
    # log u through float32
    f32 = lambda v: np.log(v.astype(np.float32)).astype(np.float64)
    assert np.max(_emulated_ratios(D, u, zz, lp_dev, lp, dlp, log_u=f32)) > 1.0
    # a = 1.0001 (zz ~ 1, F ~ 0) at small log-probabilities: zz one ulp off is caught
    u, zz, lp_dev, lp, dlp = _emulated_threshold_case(D, 1.0001, seed, step, np.random.default_rng(2), 1e-3)
    assert np.max(_emulated_ratios(D, u, zz, lp_dev, lp, dlp)) < 1.0
    off = np.nextafter(zz, np.inf)
    assert np.max(_emulated_ratios(D, u, zz, lp_dev, lp, dlp, zz_dev=off)) > 1.0


def test_snooker_factor_bound_rejects_d_for_d_minus_1():
    mv = rb.Snooker()
    D = 12
    X, act, q, fac, taps = _oracle_split(mv, 96, D, 9, 1, np.random.default_rng(4))
    caught = 0
    for r in range(len(act)):
        s, z = X[act[r]], X[taps["z"][r]]
        F, dF = AX.snooker_factor(s, z, q[r], D)
        assert AX.abs_err(fac[r], F) < dF
        wrong = fac[r] * D / (D - 1.0)
        caught += AX.abs_err(wrong, F) > dF
    assert caught >= len(act) - 2, caught


def test_bisection_finds_the_emulated_threshold_exactly():
    """The decision fl(A - L) > lu flips between two adjacent doubles, and the bisection returns them."""
    rng = np.random.default_rng(7)
    A = rng.standard_normal(40) * 100.0
    lu = np.log(rng.random(40))
    decide = lambda L: (A - L) > lu
    T = [AX.mpf(a) - AX.mpf(b) for a, b in zip(A, lu)]
    lo, hi, bad = AX.bisect_thresholds(decide, T, np.abs(A) * U + 4 * U)  # B / 64 is below one ulp of L
    assert bad.size == 0
    assert np.all(decide(lo)) and not np.any(decide(hi))
    assert np.all(np.nextafter(lo, np.inf) == hi)
