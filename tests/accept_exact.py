"""High-precision references and first-order rounding bounds for the Metropolis accept test of the red-blue and MH
moves and for the DE and snooker proposals (``test_gpu_accept_exact.py`` holds the derivation of the bounds and the
table of cases; ``test_accept_exact_host.py`` checks this module against the numpy oracle on the CPU).

Arithmetic of the references: the log-probability exactly (``logprob_exact``), logarithms, square roots and the
DE normal with ``mpmath`` at 45 digits; the proposals with ``mpmath`` up to ``MP_MAX_D`` columns and in
``np.longdouble`` above, whose own roundings (unit ``ULD``) are added to the bounds."""
import decimal
from fractions import Fraction

import mpmath
import numpy as np

import logprob_exact as LX
import proposals_exact as PX
from oracle import philox as px

U = PX.U
ULD = PX.ULD
UMP = PX.UMP
MP_DPS = PX.MP_DPS
MP_MAX_D = PX.MP_MAX_D
TWO_PI = PX.TWO_PI
LOG_ERR = 2 * U  # CUDA's log: 1 ulp, i.e. 2u relative to the result


def gamma(n, u=U):
    return n * u / (1.0 - n * u)


def mpf(v):
    """mpf of a double, Fraction or Decimal (at MP_DPS digits)."""
    with mpmath.workdps(MP_DPS):
        if isinstance(v, Fraction):
            return mpmath.mpf(v.numerator) / v.denominator
        if isinstance(v, decimal.Decimal):
            return mpmath.mpf(str(v))
        return mpmath.mpf(float(v))


# ---- draws -----------------------------------------------------------------------------------------------------
def accept_u(seed, step, split, index):
    """The accept uniform u53 of active rank (or, for MH moves, walker) ``index`` (red_blue.py:100, mh.py:58)."""
    w0, w1, _, _ = px.draw_words(seed, step, split, px.TAG_ACCEPT, np.asarray(index, dtype=np.uint64))
    return px.u53(w0, w1)


def stretch_zz(a, seed, step, split, index):
    """zz of stretch.py:30 as the draw specification defines it: every operation rounded once (bit-exact on the
    device, pinned by the oracle tests)."""
    w0, w1, _, _ = px.draw_words(seed, step, split, px.TAG_PROP_A, np.asarray(index, dtype=np.uint64))
    t = (a - 1.0) * px.u53(w0, w1) + 1.0
    return (t * t) / a


def de_normal_mp(seed, step, split, index):
    """The DE normal of active rank ``index`` (de.py:56): sqrt(-2 ln(1 - u1)) cos(fl(2 pi u2)) at 45 digits, from
    the device's own rounded angle.  Returns (list of mpf, float64 array)."""
    b0, b1, b2, b3 = px.draw_words(seed, step, split, px.TAG_PROP_B, np.asarray(index, dtype=np.uint64))
    u1 = px.u53(b0, b1)
    th = TWO_PI * px.u53(b2, b3)  # rounded once, as on the device
    out = []
    with mpmath.workdps(MP_DPS):
        for a, t in zip(u1.tolist(), th.tolist()):
            out.append(mpmath.sqrt(-2 * mpmath.log(1 - mpmath.mpf(a))) * mpmath.cos(mpmath.mpf(t)))
    return out, np.array([float(v) for v in out])


# ---- exact log-probabilities -----------------------------------------------------------------------------------
class Model(object):
    """One device model: ``exact(x)`` (mpf) and the kernel's bound ``bound(x)`` on |lp_dev - lp|."""

    def __init__(self, kind, params=(), A=None, mu=None, dmma=False):
        self.kind, self.params, self.dmma = kind, tuple(params), dmma
        if kind == "dense":
            self.A = np.asarray(A, dtype=np.float64)
            self.mu = np.zeros(self.A.shape[0]) if mu is None else np.asarray(mu, dtype=np.float64)
            self.Aint = LX._ints(self.A)
            self.L = np.linalg.cholesky(0.5 * (self.A + self.A.T))

    def exact(self, x):
        if self.kind == "iso":
            return mpf(LX.exact_iso(x))
        if self.kind == "ring":
            return mpf(LX.exact_ring(x, *self.params)[0])
        if self.kind == "rosenbrock":
            return mpf(LX.exact_rosen(x, *self.params))
        return mpf(LX.exact_dense(x, self.mu, self.Aint))

    def bound(self, x, lp):
        if self.kind == "iso":
            return LX.bound_iso(x)
        if self.kind == "ring":
            d = float(LX.exact_ring(x, *self.params)[1])
            return LX.bound_ring(x, self.params[0], self.params[1], d, abs(float(lp)))
        if self.kind == "rosenbrock":
            return LX.bound_rosen(x, *self.params)
        if self.dmma:
            return LX.bound_dense_dmma(x, self.mu, self.L)
        return LX.bound_dense_generic(x, self.mu, self.A)


# ---- Hastings factors --------------------------------------------------------------------------------------------
def stretch_factor(zz, D):
    """(F, |dF|): F = (D - 1) ln zz exactly for the double zz; the device's log is within 1 ulp (2u |ln zz|, times
    D - 1 exact) and the product rounds once."""
    with mpmath.workdps(MP_DPS):
        F = (D - 1) * mpmath.log(mpmath.mpf(float(zz)))
    f = abs(float(F))
    return F, LOG_ERR * f + U * f


def _sumsq_exact(a, b):
    """sum (a - b)^2 exactly, as an mpf (a, b: float64 rows)."""
    (na, nb), e = LX._ints(a, b)
    s = sum((int(x) - int(y)) ** 2 for x, y in zip(na.tolist(), nb.tolist()))
    with mpmath.workdps(MP_DPS):
        return mpmath.mpf(s) * mpmath.mpf(2) ** (2 * e)


def norm_rel_err(D, u=U):
    """Relative error of fl(sqrt(sum fl(a - b)^2)) with fma chains and a group tree of depth <= D: each square
    2u (the difference's rounding), the sum gamma_D, the square root halves that and adds u."""
    return (2 * u + gamma(D, u)) / 2 + u


def snooker_factor(s, z, q, D):
    """(F, |dF|): F = (D - 1)(ln |q - z| - ln |s - z|) at 45 digits with the device's q; |dF| carries the
    relative errors of norm and qn (``norm_rel_err``), two logs (2u |ln| each), the subtraction and the product."""
    with mpmath.workdps(MP_DPS):
        n2 = _sumsq_exact(s, z)
        m2 = _sumsq_exact(q, z)
        ln_n, ln_q = mpmath.log(n2) / 2, mpmath.log(m2) / 2
        F = (D - 1) * (ln_q - ln_n)
    a_n, a_q = abs(float(ln_n)), abs(float(ln_q))
    eps = norm_rel_err(D)
    dF = (D - 1) * (2 * eps + LOG_ERR * (a_n + a_q) + U * abs(float(ln_q - ln_n))) + U * abs(float(F))
    return F, dF


# ---- the accept threshold ----------------------------------------------------------------------------------------
def threshold(F, dF, lp, dlp, u):
    """(T, B): the device accepts iff fl(fl(F~ + lp~) - L) > log~(u), so for L below T - B it accepts and above
    T + B it rejects, with T = F + lp - ln u exactly and B = dF + dlp + u |F + lp| (the first addition)
    + u |ln u| (the subtraction: at the threshold A - L = log u) + 2u |ln u| (the device log)."""
    with mpmath.workdps(MP_DPS):
        lnu = mpmath.log(mpmath.mpf(float(u)))
        T = F + lp - lnu
    B = dF + dlp + U * abs(float(F + lp)) + 3 * U * abs(float(lnu))
    return T, B


def bracket_ratio(lo, hi, T, B):
    """How far the device's decision strays, in units of B: ``lo`` (accepted) may not lie above T + B, ``hi``
    (rejected) not below T - B.  A device threshold at T + delta gives about |delta| / B."""
    with mpmath.workdps(MP_DPS):
        return max(float(mpmath.mpf(float(lo)) - T), float(T - mpmath.mpf(float(hi))), 0.0) / B


def bisect_thresholds(decide, T, B):
    """Bracket and bisect the thresholds of a decision ``decide(L) -> bool array`` (accept iff L < threshold), all
    walkers at once: the bracket [T - 4B, T + 4B] must accept at its lower and reject at its upper end, then it is
    halved until narrower than B / 64 or one ulp.  Returns (lo, hi): lo accepted, hi rejected, and the indices of
    walkers whose bracket failed."""
    Tf = np.array([float(t) for t in T])
    lo, hi = Tf - 4 * B, Tf + 4 * B
    bad = np.flatnonzero(~decide(lo) | decide(hi))
    if bad.size:
        return lo, hi, bad
    for _ in range(200):
        live = (hi - lo > B / 64) & (np.nextafter(lo, hi) < hi)
        if not live.any():
            return lo, hi, bad
        mid = np.where(live, lo + (hi - lo) / 2, lo)
        acc = decide(mid)
        lo = np.where(live & acc, mid, lo)
        hi = np.where(live & ~acc, mid, hi)
    raise AssertionError("bisection did not converge")


# ---- DE ----------------------------------------------------------------------------------------------------------
def de_gamma(g0, sigma, n_mp, n):
    """(gamma exact, |dgamma|) of de.py:56, gamma = g0 (1 + sigma n): the normal within 7u |n| (log 2u halved by the
    square root, sqrt u, cos 4u, the product u), sigma n, 1 + and g0 * one rounding each."""
    with mpmath.workdps(MP_DPS):
        g = mpmath.mpf(g0) * (1 + mpmath.mpf(sigma) * n_mp)
    return g, g0 * sigma * (PX.NORMAL_ERR + U) * abs(n) + 2 * U * abs(float(g))


def de_q_ref(s, c0, c1, g):
    """q = s + gamma (c1 - c0) in mpmath (D <= MP_MAX_D) or longdouble; returns (q_ref, unit of the reference)."""
    D = s.size
    if D <= MP_MAX_D:
        with mpmath.workdps(MP_DPS):
            return np.array([mpmath.mpf(float(a)) + g * (mpmath.mpf(float(y)) - mpmath.mpf(float(x)))
                             for a, x, y in zip(s, c0, c1)], dtype=object), UMP
    gl = PX.mp_to_ld(np.array([g], dtype=object))[0]
    ld = np.longdouble
    return s.astype(ld) + gl * (c1.astype(ld) - c0.astype(ld)), ULD


def de_q_bound(s, c0, c1, g, dg, q, uref):
    """|dq| <= |dgamma| |c1 - c0| + 2u |gamma (c1 - c0)| + u |q|, plus the reference's own roundings."""
    diff = np.abs(c1 - c0)
    ag = abs(float(g))
    return dg * diff + (2 * U + 4 * uref) * ag * diff + (U + 2 * uref) * np.abs(q)


# ---- snooker -----------------------------------------------------------------------------------------------------
def snooker_q_ref(s, z, z1, z2, gs):
    """q = s + u gs (u.z1 - u.z2), u = (s - z) / |s - z| (de_snooker.py:41-44); returns (q_ref, unit)."""
    D = s.size
    if D <= MP_MAX_D:
        with mpmath.workdps(MP_DPS):
            m = [mpmath.mpf(float(v)) for v in s]
            d = [a - mpmath.mpf(float(b)) for a, b in zip(m, z)]
            nrm = mpmath.sqrt(mpmath.fsum(v * v for v in d))
            u = [v / nrm for v in d]
            dd = mpmath.fsum(a * mpmath.mpf(float(b)) for a, b in zip(u, z1)) - mpmath.fsum(
                a * mpmath.mpf(float(b)) for a, b in zip(u, z2))
            g = mpmath.mpf(float(gs))
            return np.array([a + v * g * dd for a, v in zip(m, u)], dtype=object), UMP
    ld = np.longdouble
    d = s.astype(ld) - z.astype(ld)
    u = d / np.sqrt(np.sum(d * d))
    dd = np.sum(u * z1.astype(ld)) - np.sum(u * z2.astype(ld))
    return s.astype(ld) + u * ld(gs) * dd, ULD


def snooker_q_bound(s, z, z1, z2, gs, q, unit=U):
    """Per-element bound on |fl(q) - q| for arithmetic of unit ``unit`` with sums of depth <= D + 2:
    u_e = fl(fl(s - z) / norm) within eps_u = 2 unit + norm_rel_err; dd = fl(u.z1) - fl(u.z2) within
    (eps_u + gamma_n) sum |u| (|z1| + |z2|) + unit |dd| (the cancellation of u.z1 - u.z2 is in the sum of
    magnitudes); q_e = s_e + fl(u_e gs) dd adds gs (|u_e| |ddd| + |dd| |u_e| (eps_u + 2 unit)) + unit |q_e|."""
    D = s.size
    d = s - z
    au = np.abs(d) / np.sqrt(np.sum(d * d))
    eps_u = 2 * unit + norm_rel_err(D + 2, unit)
    dd = abs(float(np.dot(au * np.sign(d), z1) - np.dot(au * np.sign(d), z2)))
    ddd = (eps_u + gamma(D + 2, unit)) * float(np.sum(au * (np.abs(z1) + np.abs(z2)))) + unit * dd
    return gs * (au * ddd + dd * au * (eps_u + 2 * unit)) + unit * np.abs(q)


def abs_err(dev, ref):
    """|dev - ref| for a double and an mpf, at the references' precision."""
    with mpmath.workdps(MP_DPS):
        return float(abs(mpmath.mpf(float(dev)) - ref))


def norm_exact(a, b):
    """|a - b| at 45 digits."""
    with mpmath.workdps(MP_DPS):
        return mpmath.sqrt(_sumsq_exact(a, b))


def q_error(q_dev, q_ref):
    """|q_dev - q_ref| per element for a reference in mpf (object array) or longdouble."""
    if q_ref.dtype == object:
        with mpmath.workdps(MP_DPS):
            return np.array([float(abs(mpmath.mpf(float(a)) - b)) for a, b in zip(q_dev, q_ref)])
    return np.abs(q_dev.astype(np.longdouble) - q_ref).astype(np.float64)
