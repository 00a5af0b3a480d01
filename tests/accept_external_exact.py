"""Exact ladders and rules for the Metropolis accept decision of the half-steps whose inputs come from outside the
kernel: a user log-probability function (``lp_new``), a user proposal's Hastings factor, the KDE factors
(``test_gpu_accept_external_exact.py`` holds the protocol and the table of rows; ``test_accept_external_exact_host.py``
checks this module on the CPU).

The device forms ``lnpdiff`` from three doubles in one of two orders and accepts iff ``lnpdiff > log~(u)``:

* ``red_blue``: ``fl(fl(F + lp_new) - lp_old)`` (red_blue.py:99; every red-blue and precomputed accept);
* ``mh``: ``fl(fl(lp_new - lp_old) + F)`` (mh.py:57; a user ``MHMove``).

With ``F`` and ``lp_new`` fixed, ``lnpdiff`` is a non-increasing function of ``lp_old``, so the doubles it can take
near ``ln u`` form a ladder: rung 0 is the one nearest ``ln u`` (45 digits), rung ``k`` the ``k``-th one above it
(``k < 0``: below).  Where every double near ``ln u`` can be reached (``|F + lp_new|`` or ``|lp_new - lp_old|`` no
larger than about ``|ln u|``), rung ``k`` is exactly ``k`` ulps from the double nearest ``ln u``; elsewhere the
rungs are as far apart as the rounding of the larger operands lets them be.

The only rounding the test cannot reproduce is the device's ``log(u)``, within 1 ulp (2u |ln u|): a rung at or above
``ln u + 2u |ln u|`` must accept, one at or below ``ln u - 2u |ln u|`` must reject, and the band between may go
either way.  A factor the device computed itself (stretch, snooker) widens the band by its own bound and by the
roundings its error moves through (``slack``)."""
import mpmath
import numpy as np

import accept_exact as AX

U = AX.U
MP_DPS = AX.MP_DPS
RUNGS = np.arange(-4, 5)
ORDERS = ("red_blue", "mh")
_MAG = np.int64(0x7FFFFFFFFFFFFFFF)


def lnpdiff(F, lp_new, lp_old, order):
    """The device's lnpdiff in float64 (numpy rounds each operation once, to nearest)."""
    F, lp_new, lp_old = (np.asarray(v, dtype=np.float64) for v in (F, lp_new, lp_old))
    with np.errstate(invalid="ignore", over="ignore"):
        if order == "red_blue":
            return (F + lp_new) - lp_old
        if order == "mh":
            return (lp_new - lp_old) + F
    raise ValueError(order)


def ln_u(u):
    """ln u at 45 digits, one mpf per accept uniform."""
    with mpmath.workdps(MP_DPS):
        return [mpmath.log(mpmath.mpf(float(v))) for v in np.atleast_1d(u)]


def nearest(x):
    """The doubles nearest a list of mpf."""
    return np.array([float(v) for v in x], dtype=np.float64)


def _key(x):
    """Doubles to int64 keys in the same order (-0.0 just below +0.0)."""
    b = np.asarray(x, dtype=np.float64).view(np.int64)
    return b ^ ((b >> 63) & _MAG)


def _unkey(k):
    k = np.asarray(k, dtype=np.int64)
    return (k ^ ((k >> 63) & _MAG)).view(np.float64)


def _step(x, n):
    """x moved n doubles up (n > 0) or down."""
    return _unkey(_key(x) + np.int64(n))


def _bracket(g, t, centre):
    """Keys (lo, hi) around ``centre`` with g(lo) > t >= g(hi), widened until they hold."""
    c = _key(centre)
    w = np.full(c.shape, 1 << 12, dtype=np.int64)
    for _ in range(24):  # up to 2^58 doubles either side: the keys stay inside int64
        lo, hi = c - w, c + w
        ok = (g(_unkey(lo)) > t) & (g(_unkey(hi)) <= t)
        if ok.all():
            return lo, hi
        w = np.where(ok, w, w * 4)
    raise AssertionError("no lp_old brackets the target lnpdiff")


def _first_at_most(g, t, centre):
    """The smallest lp_old (as a key) with g(lp_old) <= t: g there is the largest value g takes that is <= t."""
    lo, hi = _bracket(g, t, centre)
    while True:
        live = hi - lo > 1
        if not live.any():
            return hi
        mid = lo + (hi - lo) // 2
        at_most = g(_unkey(mid)) <= t
        hi = np.where(live & at_most, mid, hi)
        lo = np.where(live & ~at_most, mid, lo)


def _last_at_least(g, t, centre):
    """The largest lp_old (as a key) with g(lp_old) >= t: g there is the smallest value g takes that is >= t."""
    lo, hi = _bracket(g, _step(t, -1), centre)  # g(lo) >= t > g(hi)
    while True:
        live = hi - lo > 1
        if not live.any():
            return lo
        mid = lo + (hi - lo) // 2
        at_least = g(_unkey(mid)) >= t
        lo = np.where(live & at_least, mid, lo)
        hi = np.where(live & ~at_least, mid, hi)


def ladder_all(F, lp_new, lnu, order, spacing=0.0):
    """(lp_old[9, n], lnpdiff[9, n]) of rungs -4..4 for each walker: ``lnpdiff(F, lp_new, lp_old[k], order)`` is
    exactly ``lnpdiff[k]``, rung 0 is the value lnpdiff can take nearest ``ln u`` and rung k the k-th one above
    (below for k < 0).  ``lnu``: list of mpf (``ln_u``).  ``spacing`` (per walker, default 0) keeps rung k at least
    |k| spacing from the double nearest ln u, for a band wider than the ladder's steps."""
    F = np.atleast_1d(np.asarray(F, dtype=np.float64))
    lp_new = np.atleast_1d(np.asarray(lp_new, dtype=np.float64))
    t0 = nearest(lnu)
    g = lambda L: lnpdiff(F, lp_new, L, order)  # noqa: E731
    with np.errstate(over="ignore", invalid="ignore"):
        centre = lp_new + F - t0
    lo_k = _first_at_most(g, t0, centre)  # largest reachable value <= t0
    hi_k = _last_at_least(g, t0, centre)  # smallest reachable value >= t0
    d_lo, d_hi = g(_unkey(lo_k)), g(_unkey(hi_k))
    with mpmath.workdps(MP_DPS):
        take_hi = np.array([abs(mpmath.mpf(float(b)) - x) < abs(mpmath.mpf(float(a)) - x)
                            for a, b, x in zip(d_lo, d_hi, lnu)], dtype=bool)
    keys = np.empty((RUNGS.size,) + F.shape, dtype=np.int64)
    vals = np.empty((RUNGS.size,) + F.shape, dtype=np.float64)
    z = int(np.flatnonzero(RUNGS == 0)[0])
    keys[z] = np.where(take_hi, hi_k, lo_k)
    vals[z] = g(_unkey(keys[z]))
    spacing = np.broadcast_to(np.asarray(spacing, dtype=np.float64), F.shape)
    for j in range(z + 1, RUNGS.size):  # up: the smallest reachable value above the last rung
        t = np.maximum(_step(vals[j - 1], 1), t0 + RUNGS[j] * spacing)
        keys[j] = _last_at_least(g, t, _unkey(keys[j - 1]))
        vals[j] = g(_unkey(keys[j]))
    for j in range(z - 1, -1, -1):  # down: the largest reachable value below the last rung
        t = np.minimum(_step(vals[j + 1], -1), t0 + RUNGS[j] * spacing)
        keys[j] = _first_at_most(g, t, _unkey(keys[j + 1]))
        vals[j] = g(_unkey(keys[j]))
    return _unkey(keys), vals


def ladder(F, lp_new, lnu, order, k, spacing=0.0):
    """The lp_old doubles of rung ``k`` (-4..4) of ``ladder_all``."""
    return ladder_all(F, lp_new, lnu, order, spacing)[0][int(k) + 4]


def slack(F, dF, lp_new, lp_old, d):
    """How far the device's lnpdiff may lie from the test's when the device computed F itself, within dF of the exact
    factor whose nearest double the test used: dF + u |F| moves the first operation's result, which rounds once more
    (u |result| on each side), and the second operation rounds once more too.  0 where dF is 0 (F exact)."""
    F, lp_new, lp_old, d = (np.asarray(v, dtype=np.float64) for v in (F, lp_new, lp_old, d))
    dF = np.asarray(dF, dtype=np.float64)
    first = np.maximum(np.abs(F + lp_new), np.abs(lp_new - lp_old))
    return np.where(dF > 0, dF + U * np.abs(F) + 3 * U * first + 3 * U * np.abs(d), 0.0)


def band_spacing(F, dF, lp_new, lnu):
    """A rung spacing for ``ladder_all`` under a factor the device computed: half the band at rung 0, so that rungs
    +-3 and +-4 lie outside it."""
    t0 = nearest(lnu)
    F, lp_new = np.asarray(F, dtype=np.float64), np.asarray(lp_new, dtype=np.float64)
    return 0.5 * (AX.LOG_ERR * np.abs(t0) + slack(F, dF, lp_new, F + lp_new - t0, t0))


def rule(d, lnu, extra=0.0):
    """+1: the device must accept a rung whose lnpdiff is ``d``; -1: must reject; 0: either (the band
    ``ln u +- (2u |ln u| + extra)``).  ``d``: array [..., n] of doubles, ``lnu``: n mpf, ``extra``: broadcast to ``d``."""
    d = np.asarray(d, dtype=np.float64)
    extra = np.broadcast_to(np.asarray(extra, dtype=np.float64), d.shape)
    out = np.zeros(d.shape, dtype=np.int8)
    with mpmath.workdps(MP_DPS):
        for j, x in enumerate(lnu):
            for idx in np.ndindex(d.shape[:-1]):
                band = AX.LOG_ERR * abs(float(x)) + float(extra[idx + (j,)])
                delta = mpmath.mpf(float(d[idx + (j,)])) - x
                out[idx + (j,)] = 1 if delta >= band else (-1 if delta <= -band else 0)
    return out


def distance_ulps(d, lnu):
    """(d - ln u) in ulps of the double nearest ln u."""
    d = np.asarray(d, dtype=np.float64)
    t0 = nearest(lnu)
    with mpmath.workdps(MP_DPS):
        dist = np.array([[float(mpmath.mpf(float(a)) - x) for a, x in zip(row, lnu)]
                         for row in np.atleast_2d(d)])
    return (dist / np.spacing(np.abs(t0))).reshape(d.shape)


def order_splitting_triples(lnu, lp_new):
    """(F, lp_new, lp_old) per walker on which the two orders land on opposite sides of the band around ``ln u``.

    ``lp_new`` (doubles with 2^40 <= |lp_new| < 2^52, not a power of two) fixes the grid g = ulp(lp_new).  With c the
    multiple of g nearest ln u, r = ln u - c and F = r + sign(r) delta (|F| < g/2), lp_old = lp_new - c:

    * red_blue: F + lp_new rounds to lp_new, so lnpdiff = c exactly, on the side of ln u opposite to sign(r);
    * mh: lp_new - lp_old = c exactly, then c + F = ln u + sign(r) delta, on the side of sign(r).

    delta = min(g / 64, (g/2 - |r|) / 2) keeps |F| below g/2; both results then lie at least min(|r|, delta) from
    ln u, far outside the band (the construction refuses r within 2^-40 of 0 or of g/2)."""
    lp_new = np.asarray(lp_new, dtype=np.float64)
    g = np.spacing(np.abs(lp_new))
    assert np.all(np.abs(lp_new) >= 2.0**40) and np.all(np.abs(lp_new) < 2.0**52)
    assert np.all(np.spacing(np.abs(lp_new) - g) == g), "lp_new at the bottom of its binade"
    t0 = nearest(lnu)
    c = np.round(t0 / g) * g
    F = np.empty_like(lp_new)
    with mpmath.workdps(MP_DPS):
        for j, x in enumerate(lnu):
            r = x - mpmath.mpf(float(c[j]))
            margin = min(abs(float(r)), g[j] / 2 - abs(float(r)))
            if margin < 2.0**-40:
                raise ValueError("ln u sits on the grid of lp_new: choose another lp_new")
            delta = min(g[j] / 64, (g[j] / 2 - abs(float(r))) / 2)
            F[j] = float(r + mpmath.sign(r) * delta)
    return F, lp_new.copy(), lp_new - c


def fine_factors(lnu, lp_new, order, rng):
    """Factors under which every double near ln u is a rung: F + lp_new within 1 % of ln u (red_blue, so that
    lp_old is small), F itself within 1 % of ln u (mh, so that lp_new - lp_old is; this needs |lp_new| no larger than
    about 1 % of |ln u| too, or lp_new - lp_old moves in steps of ulp(lp_new))."""
    t0 = nearest(lnu)
    target = t0 * (1.0 + 0.01 * rng.uniform(-1.0, 1.0, t0.size))
    return target - np.asarray(lp_new, dtype=np.float64) if order == "red_blue" else target
