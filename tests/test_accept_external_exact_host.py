"""``accept_external_exact.py`` checked on the CPU: every rung of random ladders gives the lnpdiff it claims in both
orders, order-splitting triples really split, and the rung rule never contradicts ``accept_exact.threshold`` on
device-model inputs (nor an emulated device decision with its log(u) one ulp off either way)."""
import mpmath
import numpy as np
import pytest

import accept_exact as AX
import accept_external_exact as EX

U = AX.U
SEED_STEPS = [(0x5EED, 0), (0xB200, 17), (7, 123456789)]


def _u(seed, step, n):
    return AX.accept_u(seed, step, 0, np.arange(n))


def _inputs(kind, n, rng):
    """(F, lp_new) of one regime of magnitudes."""
    if kind == "small":
        return rng.normal(0.0, 1.0, n), -0.5 * rng.chisquare(5, n)
    if kind == "large":  # |lp| ~ 2^40: a coarse ladder
        return rng.normal(0.0, 3.0, n), -(2.0**40) * (1.0 + rng.uniform(0.01, 0.99, n))
    if kind == "zero":
        return np.zeros(n), -rng.uniform(0.0, 50.0, n)
    return rng.normal(0.0, 1e-3, n), -rng.uniform(1e-8, 1e-3, n)  # "tiny"


@pytest.mark.parametrize("order", EX.ORDERS)
@pytest.mark.parametrize("kind", ["small", "large", "zero", "tiny"])
@pytest.mark.parametrize("seed,step", SEED_STEPS)
def test_every_rung_gives_the_lnpdiff_claimed(order, kind, seed, step):
    n = 96
    rng = np.random.default_rng([seed, step, len(kind)])
    F, lp = _inputs(kind, n, rng)
    lnu = EX.ln_u(_u(seed, step, n))
    L, d = EX.ladder_all(F, lp, lnu, order)
    assert L.shape == d.shape == (9, n) and np.all(np.isfinite(L))
    for k in range(9):
        got = EX.lnpdiff(F, lp, L[k], order)
        assert np.array_equal(got.view(np.uint64), d[k].view(np.uint64)), (k, np.flatnonzero(got != d[k]))
    assert np.all(np.diff(d, axis=0) > 0), "rungs are not strictly increasing"
    assert np.all(np.diff(L, axis=0) < 0), "lp_old does not fall as the rungs rise"
    # rung 0 is the reachable value nearest ln u: the rungs on either side are no nearer
    with mpmath.workdps(AX.MP_DPS):
        for j, x in enumerate(lnu):
            r0 = abs(mpmath.mpf(float(d[4, j])) - x)
            assert r0 <= abs(mpmath.mpf(float(d[3, j])) - x) and r0 <= abs(mpmath.mpf(float(d[5, j])) - x)
    # no reachable value is skipped: nothing strictly between neighbouring rungs is reached by any lp_old between
    # theirs (checked on the doubles next to each rung's lp_old)
    for k in range(8):
        up = EX.lnpdiff(F, lp, EX._step(L[k + 1], 1), order)  # lp_old one double above rung k + 1's
        assert np.all((up <= d[k]) | (up == d[k + 1])), k


@pytest.mark.parametrize("order", EX.ORDERS)
def test_fine_factors_reach_every_ulp(order):
    n = 200
    rng = np.random.default_rng(5)
    lnu = EX.ln_u(_u(3, 11, n))
    if order == "red_blue":
        lp = -np.round(rng.chisquare(5, n) * 8) / 2  # integer rows: -0.5 sum q^2
    else:
        lp = -rng.uniform(0.0, 1e-3, n) * np.abs(EX.nearest(lnu))
    F = EX.fine_factors(lnu, lp, order, rng)
    L, d = EX.ladder_all(F, lp, lnu, order)
    dist = EX.distance_ulps(d, lnu)
    assert np.all(np.abs(dist[4]) <= 0.5 + 1e-9)
    assert np.all(np.abs(dist - EX.RUNGS[:, None] - dist[4]) <= 1 + 1e-9), "rungs further apart than one ulp"
    r = EX.rule(d, lnu)
    # the band is 2u |ln u| wide on each side, up to 2 ulps: rungs 3 and 4 ulps away are always decided
    assert np.all(r[:2] == -1) and np.all(r[7:] == 1), "rungs 3 ulps from ln u must be decided"
    assert np.mean(r[2:7] != 0) > 0.3


@pytest.mark.parametrize("integer_rows", [False, True])
@pytest.mark.parametrize("seed,step", SEED_STEPS)
def test_order_splitting_triples_split(seed, step, integer_rows):
    n = 256
    rng = np.random.default_rng([seed, step])
    lnu = EX.ln_u(_u(seed, step, n))
    if integer_rows:  # lp_new = -q^2 / 2 of an integer row, as a device GaussianIso computes it exactly
        q0 = np.floor(np.sqrt(2.0**41 * rng.uniform(1.05, 1.9, n)))
        lp_new = -0.5 * q0 * q0
    else:
        lp_new = -(2.0 ** rng.integers(40, 46, n)) * rng.uniform(1.01, 1.99, n)
    F, lp, L = EX.order_splitting_triples(lnu, lp_new)
    assert np.all(F != 0)
    d_rb = EX.lnpdiff(F, lp, L, "red_blue")
    d_mh = EX.lnpdiff(F, lp, L, "mh")
    # numpy's own evaluation, written out
    assert np.array_equal(d_rb, np.float64(F + lp) - L) and np.array_equal(d_mh, np.float64(lp - L) + F)
    r_rb, r_mh = EX.rule(d_rb[None], lnu)[0], EX.rule(d_mh[None], lnu)[0]
    assert np.all(r_rb != 0) and np.all(r_mh != 0), "a triple lands inside the band"
    assert np.all(r_rb == -r_mh), "the two orders agree"
    assert 0.2 < np.mean(r_rb == 1) < 0.8, "both directions of disagreement occur"


def _emulated(F_dev, lp, L, u, order, ulps):
    """The device's decision with its log(u) moved ``ulps`` doubles from the nearest double of ln u."""
    lnu_dev = EX._step(EX.nearest(EX.ln_u(u)), ulps)
    return EX.lnpdiff(F_dev, lp, L, order) > lnu_dev


@pytest.mark.parametrize("seed,step", SEED_STEPS)
@pytest.mark.parametrize("D", [5, 37])
def test_rule_agrees_with_the_threshold(seed, step, D):
    """Stretch factors and iso log-probabilities at device inputs: no rung the rule decides lies on the other side of
    accept_exact's threshold band, and an emulated device -- factor off by up to its bound, log(u) off by one ulp
    either way -- obeys the rule."""
    n = 64
    rng = np.random.default_rng([seed, step, D])
    u = AX.accept_u(seed, step, 0, np.arange(n))
    zz = AX.stretch_zz(2.0, seed, step, 0, np.arange(n))
    xm = AX.Model("iso")
    q = rng.standard_normal((n, D))
    lnu = EX.ln_u(u)
    Fs, dFs, lps, Ts, Bs = [], [], [], [], []
    for j in range(n):
        F, dF = AX.stretch_factor(zz[j], D)
        lp = xm.exact(q[j])
        dlp = xm.bound(q[j], lp)
        T, B = AX.threshold(F, dF, lp, dlp, u[j])
        Fs.append(float(F))
        dFs.append(dF)
        lps.append(float(lp))  # the device's lp, taken as exact here: the threshold carries its bound dlp
        Ts.append(T)
        Bs.append(B)
    Fs, dFs, lps = np.array(Fs), np.array(dFs), np.array(lps)
    for order in EX.ORDERS:
        L, d = EX.ladder_all(Fs, lps, lnu, order, EX.band_spacing(Fs, dFs, lps, lnu))
        r = EX.rule(d, lnu, EX.slack(Fs, dFs, lps, L, d))
        assert np.all(r[0] == -1) and np.all(r[8] == 1), "the outer rungs are not decided"
        with mpmath.workdps(AX.MP_DPS):
            for k in range(9):
                for j in range(n):
                    x = mpmath.mpf(float(L[k, j]))
                    if r[k, j] == 1:  # must accept: not above the threshold's must-reject line
                        assert x <= Ts[j] + Bs[j], (order, k, j)
                    if r[k, j] == -1:
                        assert x >= Ts[j] - Bs[j], (order, k, j)
        for sgn in (-1.0, 1.0):
            F_dev = Fs + sgn * dFs  # the factor at its bound
            for ulps in (-1, 0, 1):
                acc = np.stack([_emulated(F_dev, lps, L[k], u, order, ulps) for k in range(9)])
                assert np.all(acc[r == 1]) and not np.any(acc[r == -1]), (order, sgn, ulps)


def test_rule_catches_the_other_order():
    """A device that used the red-blue order where the mh order is due (or the reverse) fails on every triple."""
    n = 128
    lnu = EX.ln_u(_u(1, 2, n))
    rng = np.random.default_rng(9)
    F, lp, L = EX.order_splitting_triples(lnu, -(2.0**41) * rng.uniform(1.01, 1.99, n))
    for order, other in (("mh", "red_blue"), ("red_blue", "mh")):
        r = EX.rule(EX.lnpdiff(F, lp, L, order)[None], lnu)[0]
        wrong = EX.lnpdiff(F, lp, L, other) > EX.nearest(lnu)
        assert np.all(wrong[r == 1] == False) and np.all(wrong[r == -1] == True)  # noqa: E712
