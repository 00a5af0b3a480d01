"""High-precision references and first-order rounding bounds for the WalkMove / GaussianMove proposals and the
chain moment sums (``test_gpu_proposals_exact.py`` holds the derivation of the bounds and the table of cases;
``test_proposals_exact_host.py`` checks this module against the numpy oracle on the CPU).

Arithmetic of the references: standard normals with ``mpmath`` at 45 digits; covariances exactly, from integer
images of the coordinates; the thresholded Cholesky factor ``chol_psd`` with ``mpmath`` up to ``MP_MAX_D``
columns and in ``np.longdouble`` above, whose own roundings (unit ``ULD``) are added to the bounds."""
import mpmath
import numpy as np
from scipy.linalg import solve_triangular

from oracle import philox as px

U = 2.0 ** -53
ULD = float(np.finfo(np.longdouble).eps) / 2  # unit roundoff of the longdouble references
UMP = 1e-44  # unit roundoff of the 45-digit mpmath references
MP_DPS = 45
MP_MAX_D = 32
TWO_PI = 6.283185307179586  # the double constant of normal_pair (moves_extra.cu) and oracle.philox.normals
NORMAL_ERR = 7 * U  # |fl(normal) - normal| / |normal|: log 2u/2 + sqrt u + sincos 4u + product u (module docstring)


def gamma(n, u=U):
    return n * u / (1.0 - n * u)


def longdouble_ok():
    return float(np.finfo(np.longdouble).eps) < 1e-18


# ---- standard normals -------------------------------------------------------------------------------------------
def normals_mp(seed, step, split, index, count):
    """``[len(index), count]`` object array of mpf: the normals of ``oracle.philox.normals`` with
    ``r = sqrt(-2 ln(1 - u1))`` and ``cos`` / ``sin`` of the double ``fl(TWO_PI * u2)`` at 45 digits."""
    index = np.atleast_1d(np.asarray(index, dtype=np.uint64))
    out = np.empty((len(index), int(count)), dtype=object)
    with mpmath.workdps(MP_DPS):
        for k in range((int(count) + 1) // 2):
            w0, w1, w2, w3 = px.draw_words(seed, step, px.sub_split(split, k), px.TAG_NORMAL, index)
            u1 = px.u53(w0, w1)
            th = TWO_PI * px.u53(w2, w3)  # rounded once, as on the device
            for row in range(len(index)):
                r = mpmath.sqrt(-2 * mpmath.log(1 - mpmath.mpf(float(u1[row]))))
                c, s = mpmath.cos_sin(mpmath.mpf(float(th[row])))
                out[row, 2 * k] = r * c
                if 2 * k + 1 < count:
                    out[row, 2 * k + 1] = r * s
    return out


def mp_to_ld(a):
    """object array of mpf -> np.longdouble (within ULD relative)."""
    flat = [np.longdouble(mpmath.nstr(v, 25, min_fixed=1, max_fixed=0)) if v != 0 else np.longdouble(0)
            for v in np.ravel(a)]
    return np.array(flat, dtype=np.longdouble).reshape(np.shape(a))


def mp_to_f64(a):
    return np.array([float(v) for v in np.ravel(a)], dtype=np.float64).reshape(np.shape(a))


# ---- exact covariances ------------------------------------------------------------------------------------------
def int_image(x):
    """``(ints, e)``: object array of Python ints and one exponent with ``x == ints * 2**e`` exactly."""
    x = np.asarray(x, dtype=np.float64)
    m, ex = np.frexp(x)
    mi = (m * 2.0 ** 53).astype(np.int64)
    ex = ex.astype(np.int64) - 53
    nz = mi != 0
    e = int(ex[nz].min()) if nz.any() else 0
    shift = np.where(nz, ex - e, 0)
    out = np.array([int(v) << int(s) for v, s in zip(mi.ravel().tolist(), shift.ravel().tolist())], dtype=object)
    return out.reshape(x.shape), e


class ExactCov(object):
    """``np.cov(X, rowvar=0)`` of ``n`` rows held exactly: ``num * 2**(2 e) / (n (n - 1))`` with ``num = n X^T X -
    S S^T`` in integers.  Integer-valued ``X`` small enough that ``n^2 max|x|^2 < 2^62`` stays in int64 (every
    entry then converts to longdouble exactly); anything else goes through Python integers."""

    def __init__(self, X):
        X = np.asarray(X, dtype=np.float64)
        self.n, self.D = X.shape
        n = self.n
        assert n >= 2
        amax = float(np.max(np.abs(X))) if X.size else 0.0
        if np.all(X == np.round(X)) and float(n) ** 2 * amax * amax < 2.0 ** 62:
            Xi = X.astype(np.int64)
            self.e = 0
            self.num = n * (Xi.T @ Xi) - np.outer(Xi.sum(0), Xi.sum(0))
            self.small = True
        else:
            Xi, self.e = int_image(X)
            S = Xi.sum(axis=0)
            self.num = n * Xi.T.dot(Xi) - np.outer(S, S)
            self.small = False
        self.den = n * (n - 1)

    def ld(self):
        assert self.small and self.e == 0
        return self.num.astype(np.longdouble) / np.longdouble(self.den)

    def mp(self):
        with mpmath.workdps(MP_DPS):
            sc = mpmath.mpf(2) ** (2 * self.e) / self.den
            return [[mpmath.mpf(int(self.num[i, j])) * sc for j in range(self.D)] for i in range(self.D)]

    def f64(self):
        if self.small:
            return self.num.astype(np.float64) / float(self.den)
        return np.array([[float(int(self.num[i, j])) for j in range(self.D)] for i in range(self.D)]) * (
            2.0 ** (2 * self.e) / self.den)


def rankcap_rows(D, rng):
    """D integer rows whose covariance has rank D - 1 with a well-conditioned leading block: 64 e_i plus small
    noise in the first D - 1 columns, an independent last column.  Its last pivot is exactly zero, so only the
    rank cap (not the threshold, once the one-pass sums are noisy) keeps it out of the factor."""
    X = np.zeros((D, D))
    X[:D - 1, :D - 1] = 64.0 * np.eye(D - 1)
    X += np.round(rng.standard_normal((D, D)) * 2)
    X[:, D - 1] = np.round(rng.standard_normal(D) * 64)
    return X


# ---- thresholded Cholesky (oracle.philox.chol_psd) at high precision ---------------------------------------------
def chol_psd_mp(A, max_rank=None):
    """``A``: list of lists of mpf.  Same rule as ``oracle.philox.chol_psd``.  Returns (L as list of lists, pivots)."""
    D = len(A)
    with mpmath.workdps(MP_DPS):
        L = [[mpmath.mpf(0)] * D for _ in range(D)]
        tol = mpmath.mpf(1e-12) * max(max(A[j][j] for j in range(D)), mpmath.mpf(0))
        left = D if max_rank is None else int(max_rank)
        piv = []
        for j in range(D):
            if left <= 0:
                break
            d = A[j][j] - mpmath.fsum(L[j][k] * L[j][k] for k in range(j))
            if not d > tol:
                continue
            left -= 1
            piv.append(j)
            L[j][j] = mpmath.sqrt(d)
            for i in range(j + 1, D):
                L[i][j] = (A[i][j] - mpmath.fsum(L[i][k] * L[j][k] for k in range(j))) / L[j][j]
    return L, piv


def chol_psd_ld(A, max_rank=None):
    """``np.longdouble`` version of the same rule.  Returns (L, pivots)."""
    A = np.asarray(A, dtype=np.longdouble)
    D = A.shape[0]
    L = np.zeros_like(A)
    tol = np.longdouble(1e-12) * max(np.max(np.diag(A)), np.longdouble(0))
    left = D if max_rank is None else int(max_rank)
    piv = []
    for j in range(D):
        if left <= 0:
            break
        d = A[j, j] - np.dot(L[j, :j], L[j, :j])
        if not d > tol:
            continue
        left -= 1
        piv.append(j)
        L[j, j] = np.sqrt(d)
        if j + 1 < D:
            L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L, piv


def chol_reference(A_exact, max_rank=None):
    """(L as float64, L in reference arithmetic, pivots, unit roundoff of the reference) for an ExactCov or a
    float64 matrix (taken as exact)."""
    D = A_exact.D if isinstance(A_exact, ExactCov) else A_exact.shape[0]
    if D <= MP_MAX_D:
        if isinstance(A_exact, ExactCov):
            A = A_exact.mp()
        else:
            A = [[mpmath.mpf(float(v)) for v in row] for row in A_exact]
        L, piv = chol_psd_mp(A, max_rank)
        Lo = np.empty((D, D), dtype=object)
        for i in range(D):
            for j in range(D):
                Lo[i, j] = L[i][j]
        return mp_to_f64(Lo), Lo, piv, UMP
    A = A_exact.ld() if isinstance(A_exact, ExactCov) else np.asarray(A_exact, dtype=np.longdouble)
    L, piv = chol_psd_ld(A, max_rank)
    return L.astype(np.float64), L, piv, ULD


def check_pivot_prefix(L, piv, r, A_diag_max, margin=1e3):
    """The factor the bounds assume: the first ``r`` pivots kept, each well above the threshold, the rest
    zero columns."""
    assert list(piv) == list(range(r)), (piv[:8], r)
    d = np.diag(L)[:r]
    assert np.all(d * d > margin * 1e-12 * A_diag_max), "a kept pivot is near the threshold"


# ---- bounds -----------------------------------------------------------------------------------------------------
def chol_perturbation(L, M, r):
    """First-order componentwise bound on |dL| for the leading-``r`` lower factor ``L`` (float64) of a symmetric
    matrix perturbed by at most ``M`` elementwise: ``dL11 = L11 Phi(L11^-1 dA11 L11^-T)``, ``Phi`` the lower
    triangle with a halved diagonal, and ``dL21 = (dA21 - L21 dL11^T) L11^-T``; columns past ``r`` are zero."""
    D = L.shape[0]
    out = np.zeros((D, D))
    if r == 0:
        return out
    L11 = L[:r, :r]
    Li = np.abs(solve_triangular(L11, np.eye(r), lower=True))
    X = Li @ M[:r, :r] @ Li.T
    Phi = np.tril(X)
    Phi[np.diag_indices(r)] *= 0.5
    dL11 = np.abs(L11) @ Phi
    out[:r, :r] = np.tril(dL11)
    if r < D:
        out[r:, :r] = (M[r:, :r] + np.abs(L[r:, :r]) @ out[:r, :r].T) @ Li.T
    return out


def backward_error(L, u=U):
    """Higham Thm 10.3: the computed factor of A is the exact one of A + E, |E| <= gamma_{D+1} |L| |L^T|."""
    D = L.shape[0]
    aL = np.abs(L)
    return gamma(D + 1, u) * (aL @ aL.T)


def cov_error_one_pass(Y, n, depth, A):
    """|fl(cov) - cov| for cov = (S2 - S1 S1^T / n) / (n - 1) formed from moment sums about a shift:
    ``Y`` the rows minus the shift (float64), ``depth`` the longest chain of additions into one sum.
    y = fl(x - shift) is off by u|y|; every sum by gamma_depth of its absolute sum; the product S1 S1^T / n
    takes two roundings, the subtraction and the division one each."""
    aY = np.abs(Y)
    P = aY.T @ aY
    S1 = np.abs(Y.sum(axis=0))
    dS1 = (U + gamma(depth)) * aY.sum(axis=0)
    C = np.outer(S1, S1) / n
    M = ((2 * U + gamma(depth)) * P + (np.outer(dS1, S1) + np.outer(S1, dS1)) / n + 2 * U * C) / (n - 1)
    return M + 2 * U * np.abs(A)


def cov_error_two_pass(X, A):
    """The helper-subset kernel: mean = (sum x) / s, then sum fma(x_r - m_r, x_c - m_c) / (s - 1).  The mean is
    off by dm <= (gamma_s + u) mean|x|; Y = fl(x - m~) by u|y|; sum(x - m~)(x - m~)^T = sum (x - m)(x - m)^T +
    s dm dm^T exactly; the fma chain adds gamma_s."""
    s = X.shape[0]
    m = X.mean(axis=0)
    dm = (gamma(s) + U) * np.abs(X).mean(axis=0) + U * np.abs(m)
    aY = np.abs(X - m) + dm
    P = aY.T @ aY
    M = ((2 * U + gamma(s)) * P + s * np.outer(dm, dm)) / (s - 1)
    return M + U * np.abs(A)


def mvn_bound(L, Mcov, r, z_abs, q_abs, u_ref):
    """Per-element bound on |fl(s + L z) - (s + L z)| with L the factor of a covariance that the device formed
    with error <= ``Mcov`` and then factorised (``walk_*_propose_kernel``): covariance and Cholesky rounding
    carried to L, the normals' own error, the fma chain of L z and the final addition; plus the reference's own
    roundings with unit ``u_ref``.  ``z_abs``: [rows, D]."""
    D = L.shape[0]
    aL = np.abs(L)
    M = Mcov + backward_error(L) + backward_error(L, u_ref) + u_ref * (aL @ aL.T)
    dL = chol_perturbation(L, M, r)
    Lz = z_abs @ aL.T
    return (z_abs @ dL.T + (NORMAL_ERR + gamma(D + 1) + gamma(D + 2, u_ref)) * Lz
            + (U + u_ref) * q_abs)


def factor_f(p1, seed, step):
    """GaussianMove's per-step scale (gaussian.py:88-91) on the host: exact value (mpf) and the relative error
    bound of the double the engine computes, exp(-lf + (lf - -lf) u) with lf = log(p1): log and exp within
    1 ulp (2u relative), lf - -lf exact, the product and the sum one rounding each."""
    if p1 is None:
        return mpmath.mpf(1), 0.0
    w0, w1, _, _ = px.draw_words(seed, step, 0, px.TAG_MOVE, np.array([1]))
    ud = float(px.u53(w0, w1)[0])
    with mpmath.workdps(MP_DPS):
        lf = mpmath.log(mpmath.mpf(p1))
        arg = -lf + 2 * lf * mpmath.mpf(ud)
        f = mpmath.exp(arg)
    lf, arg = float(lf), float(arg)
    darg = 2 * U * abs(lf) * abs(2 * ud - 1) + U * abs(2 * lf * ud) + U * abs(arg)
    return f, darg + 2 * U


def colmean_device_order(X):
    """colmean_kernel (analysis.cu) in double, in its summation order: eight strided partial sums per column,
    added in order, then divided by the row count."""
    X = np.asarray(X, dtype=np.float64)
    part = np.zeros((8, X.shape[1]))
    for y in range(8):
        for r in range(y, X.shape[0], 8):
            part[y] = part[y] + X[r]
    s = np.zeros(X.shape[1])
    for y in range(8):
        s = s + part[y]
    return s / float(X.shape[0])


def moments_depth(nrows, D, sm_count, ncalls):
    """Longest chain of additions into one moment sum: the rows one CTA of moments_partial_kernel stages (CH per
    chunk, every grid-th chunk), the CTA partials moments_reduce_kernel adds, and one += per accumulation call."""
    nblk = (D + 7) // 8
    Dp = 8 * nblk
    RS = Dp
    while RS % 32 != 8:
        RS += 8
    CH = min(64, max(4, ((96 * 1024) // (RS * 8)) & ~3))
    per = (Dp + Dp * Dp) * 8
    grid = max(1, min((64 << 20) // per, sm_count))
    nchunks = (nrows + CH - 1) // CH
    grid = min(grid, nchunks)
    per_cta = ((nchunks + grid - 1) // grid) * CH
    return per_cta + grid + ncalls, grid, CH
