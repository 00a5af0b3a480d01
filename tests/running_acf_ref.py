"""numpy statement of the running autocorrelation function (``emcee_b200/csrc/running_acf.h``): the blocked lag sums
of every (walker, parameter) series, their double-double accumulation, the final combination and the walker
reduction, operation for operation, so that it equals the device's ``rho`` and the g++ probe of the header with
``==``.  numpy has no fused multiply-add, so :func:`fma` emulates a correctly rounded one (Boldo & Melquiond 2008).

:func:`rounding_bound` is the bound DESIGN §5.7 derives for ``|rho - exact|``, the exact walker-averaged function of
the recorded states."""
import numpy as np

B = 64  # RACF_B
WCHUNK = 64  # RACF_WCHUNK
U = 2.0 ** -53


def gamma(n):
    return n * U / (1.0 - n * U)


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    """p + e == a b exactly (Dekker; no fma needed, |a|, |b| far below overflow)"""
    f = 134217729.0  # 2^27 + 1
    ca, cb = f * a, f * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    p = a * b
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _round_odd_sum(a, b):
    """a + b rounded to odd: the neighbour with an odd last bit when a + b is not a double"""
    s, e = _two_sum(a, b)
    s = np.array(s, dtype=np.float64, copy=True)
    e = np.asarray(e, dtype=np.float64)
    even = (s.view(np.int64) & 1) == 0
    fix = (e != 0) & even
    if np.any(fix):
        s[fix] = np.nextafter(s[fix], np.where(e[fix] > 0, np.inf, -np.inf))
    return s


def fma(a, b, c):
    """round(a b + c) once, elementwise (Boldo & Melquiond, "Emulation of FMA and correctly rounded sums", 2008)"""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, dtype=np.float64) for v in (a, b, c)))
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    v = _round_odd_sum(tl, ul)
    with np.errstate(invalid="ignore"):
        r = th + v
    exact0 = (uh == 0) & (ul == 0)  # a b == 0: a b + c is c, or +-0 by IEEE's rule for a zero sum
    return np.where(exact0, (a * b) + c, r)


# ---- double-double, as running_acf.h -------------------------------------------------------------------------------
def _fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def dd_add_d(a, b):
    s, e = _two_sum(a[0], b)
    return _fast_two_sum(s, e + a[1])


def dd_add(a, b):
    s, e = _two_sum(a[0], b[0])
    t, f = _two_sum(a[1], b[1])
    s, e = _fast_two_sum(s, e + t)
    return _fast_two_sum(s, e + f)


def dd_sub(a, b):
    return dd_add(a, (-b[0], -b[1]))


def dd_mul(a, b):
    p = a[0] * b[0]
    e = fma(a[0], b[0], -p)
    e = fma(a[0], b[1], e)
    e = fma(a[1], b[0], e)
    return _fast_two_sum(p, e)


def dd_mul_d(a, b):
    p = a[0] * b
    e = fma(a[1], b, fma(a[0], b, -p))
    return _fast_two_sum(p, e)


def dd_div_d(a, b):
    q1 = a[0] / b
    p = q1 * b
    pe = fma(q1, b, -p)
    r = (a[0] - p) + (a[1] - pe)
    return _fast_two_sum(q1, r / b)


def cov(s, y, head, tail, n, tau):
    ybar = dd_div_d(y, float(n))
    t = dd_add(dd_sub(y, head), dd_sub(y, tail))
    c = dd_sub(s, dd_mul(ybar, t))
    c = dd_add(c, dd_mul_d(dd_mul(ybar, ybar), float(n - tau)))
    return c[0]


class RunningAcf(object):
    """The running sums of series x[nwalkers, ndim]; :meth:`record` one state, :meth:`read` rho at any time."""

    def __init__(self, max_lag, nwalkers, ndim):
        self.max_lag, self.N, self.D = int(max_lag), int(nwalkers), int(ndim)
        S = self.N * self.D
        self.y = []  # every shifted value (the device keeps a ring of the last max_lag + B, and the first max_lag)
        self.x0 = None
        self.s = (np.zeros((self.max_lag + 1, S)), np.zeros((self.max_lag + 1, S)))
        self.Y = (np.zeros(S), np.zeros(S))

    @property
    def n(self):
        return len(self.y)

    def _yat(self, t):
        return self.y[t] if t >= 0 else np.zeros(self.N * self.D)

    def _chain(self, base, m, tau, p=None):
        p = np.zeros(self.N * self.D) if p is None else p
        for k in range(m):
            p = fma(self.y[base + k], self._yat(base + k - tau), p)
        return p

    def record(self, x):
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        if self.x0 is None:
            self.x0 = x.copy()
            self.y.append(np.zeros_like(x))
        else:
            self.y.append(x - self.x0)
        n = self.n
        if n % B == 0:  # block (n / B - 1) is complete
            base = n - B
            for k in range(B):
                self.Y = dd_add_d(self.Y, self.y[base + k])
            hi, lo = self.s[0].copy(), self.s[1].copy()
            for tau in range(self.max_lag + 1):
                hi[tau], lo[tau] = dd_add_d((hi[tau], lo[tau]), self._chain(base, B, tau))
            self.s = (hi, lo)

    def read(self):
        n = self.n
        L = min(n, self.max_lag + 1)
        S = self.N * self.D
        base, m = n // B * B, n % B
        Y = self.Y
        for k in range(m):
            Y = dd_add_d(Y, self.y[base + k])
        hd = tl = (np.zeros(S), np.zeros(S))
        r = np.empty((L, S))
        c0 = None
        for tau in range(L):
            if tau > 0:
                hd = dd_add_d(hd, self.y[tau - 1])
                tl = dd_add_d(tl, self.y[n - tau])
            s = (self.s[0][tau], self.s[1][tau])
            if m:
                s = dd_add_d(s, self._chain(base, m, tau))
            c = cov(s, Y, hd, tl, n, tau)
            if tau == 0:
                c0 = c
            with np.errstate(invalid="ignore", divide="ignore"):
                r[tau] = c / c0
        return walker_mean(r.reshape(L, self.N, self.D))


def walker_mean(r):
    """rho[L, D] of the per-walker ratios r[L, N, D] in running_acf.h's order"""
    N = r.shape[1]
    parts = []
    for c0 in range(0, N, WCHUNK):
        a = r[:, c0].copy()
        for w in range(c0 + 1, min(N, c0 + WCHUNK)):
            a = a + r[:, w]
        parts.append(a)
    a = parts[0]
    for p in parts[1:]:
        a = a + p
    return a / float(N)


def running_acf(x, max_lag, cuts=None):
    """rho of the states x[n, nwalkers, ndim] recorded one after the other (``cuts``: indices after which a read is
    made and thrown away, as a mid-block read of the device is)"""
    n, N, D = x.shape
    acc = RunningAcf(max_lag, N, D)
    cuts = set(cuts or ())
    for t in range(n):
        acc.record(x[t])
        if t in cuts:
            acc.read()
    return acc.read()


# ---- the rounding bound (DESIGN §5.7) ------------------------------------------------------------------------------
def exact_parts(x, max_lag):
    """High-precision (longdouble, two-pass) ratios r[L, N, D] and autocovariances c[L, N, D] of x[n, N, D]; only
    the bound's magnitudes and the comparison's reference in the random tests come from here."""
    n = x.shape[0]
    L = min(n, max_lag + 1)
    xl = x.astype(np.longdouble)
    d = xl - xl.mean(axis=0)
    c = np.empty((L,) + x.shape[1:], dtype=np.longdouble)
    for tau in range(L):
        c[tau] = np.sum(d[tau:] * d[: n - tau], axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = c / c[0]
    return r.astype(np.float64), c.astype(np.float64)


def rounding_bound(x, max_lag):
    """Bound[L, D] on |rho - exact| for the recorded states x[n, N, D] (DESIGN §5.7):

    per series, with y_t = x_t - x_0, A(tau) = sum |y_t y_{t-tau}|, ybar the mean of y and M(tau) = A(tau) +
    2 |ybar| sum |y| + (n - tau) ybar^2:
      e_c(tau) = gamma_B A(tau)                       the fma chain of a block, at most B terms
               + eps2 M(tau)                          the lag sums' double-double additions, head, tail and the
                                                      combination, eps2 = 16 (n/B + 2 max_lag + 16) u^2
               + 3 n u^2 sum|y| (4 |ybar| + 2 ymax)   Y: n double-double additions of one value each (at most
                                                      2 u^2 of the running sum), times |dc/dY| <= 4 |ybar| + 2 ymax
               + 4 u ymax sum|d| + 4 n u^2 ymax^2     the shift x_t - x_0 rounded once (|delta_t| <= u |y_t|)
               + u |c(tau)|                           the combination rounded to a double
      beta(tau) = (e_c(tau) + |r| e_c(0)) / (c(0) - e_c(0)) (1 + u) + u |r|       the ratio
    and over the walkers, depth = WCHUNK - 1 + nchunks - 1 additions:
      |rho - exact| <= (sum beta + gamma_depth sum(|r| + beta)) / N (1 + u) + u |rho|."""
    n, N, D = x.shape
    L = min(n, max_lag + 1)
    r, c = exact_parts(x, max_lag)
    y = np.abs(x - x[0])
    ymax = y.max(axis=0)
    ybar = np.abs((x - x[0]).mean(axis=0))
    ysum = y.sum(axis=0)
    dsum = np.abs(x - x.mean(axis=0)).sum(axis=0)
    eps2 = 16.0 * (n / B + 2 * max_lag + 16) * U * U
    e = np.empty((L, N, D))
    for tau in range(L):
        A = np.sum(y[tau:] * y[: n - tau], axis=0)
        M = A + 2 * ybar * ysum + (n - tau) * ybar ** 2
        e[tau] = (gamma(B) * A + eps2 * M + 3 * n * U * U * ysum * (4 * ybar + 2 * ymax)
                  + 4 * U * ymax * dsum + 4 * n * U * U * ymax ** 2 + U * np.abs(c[tau]))
    ar = np.abs(r)
    with np.errstate(invalid="ignore", divide="ignore"):
        beta = (e + ar * e[0][None]) / (c[0][None] - e[0][None]) * (1 + U) + U * ar
    nchunks = (N + WCHUNK - 1) // WCHUNK
    depth = min(N, WCHUNK) - 1 + nchunks - 1
    rho = np.abs(r.mean(axis=1))
    return (beta.sum(axis=1) + gamma(depth) * (ar + beta).sum(axis=1)) / N * (1 + U) + U * rho


def fft_bound(x):
    """Bound[n, D] on |np.mean(autocorr._acf(x), axis=1) - exact|: numpy's transforms (tests/acf_exact.py) and its
    mean over the walkers"""
    import acf_exact

    n, N, D = x.shape
    M = acf_exact.fft_length(n)
    xs = x.reshape(n, N * D)
    d = xs - xs.mean(axis=0)
    a0 = np.sum(d * d, axis=0)
    norm = acf_exact.acf_norm(d, M)
    rho_s = acf_exact.series_bound(M, norm, extra=acf_exact.mean_rounding(xs, a0)).reshape(N, D)
    r, _ = exact_parts(x, n)
    dev = acf_exact.walker_mean_bound(rho_s, r, reference_rounding=False)
    return dev + gamma(N) * np.abs(r).sum(axis=1) / N
