"""The walker Gram matrix of ``eb_walkers_gram`` in reference arithmetic, its first-order rounding bound, and a
double-precision emulation of the independence decision as the engine took it before sums of squares were
range-checked (``test_gpu_walkers_independent.py`` holds the derivation; ``test_walkers_independent_host.py``
checks this module on the CPU).

What the device computes for ``x[N, D]``: the shift ``m = colmean(x)`` in ``colmean_kernel``'s order
(``proposals_exact.colmean_device_order``, bit for bit), ``y = fl(x - m)``, the uncorrected sums
``M = y^T y`` on the DMMA pipe (``launch_moments``, one accumulation), and on the host
``G_jk = M_jk / (sqrt(M_jj) sqrt(M_kk))``.  The reference takes the same double ``m`` as exact."""
import numpy as np

import proposals_exact as PX

U = PX.U
ULD = PX.ULD


def pairs(D, rng, full_max=16, extra=512):
    """(i, j) of the compared Gram entries: all of them up to ``full_max`` columns, else the diagonal, rows 0 and
    D - 1, and ``extra`` more."""
    if D <= full_max:
        i, j = np.meshgrid(np.arange(D), np.arange(D), indexing="ij")
        return i.ravel(), j.ravel()
    i = np.r_[np.arange(D), np.zeros(D, np.int64), np.full(D, D - 1), rng.integers(0, D, extra)]
    j = np.r_[np.arange(D), np.arange(D), np.arange(D), rng.integers(0, D, extra)]
    return i, j


def gram_reference(X, shift, i, j, depth):
    """``(G_ref[i, j] as longdouble, bound[i, j])`` for the device's Gram matrix of ``X`` about ``shift``.

    Reference: y = x - shift and every product and sum in np.longdouble (``|dy| <= ULD |y|``, one rounding per
    product, ``gamma_N(ULD)`` per sum), normalised in longdouble (two square roots, a product and a division).
    Bound, per entry, with e = 2u + gamma_depth (device sums) and e' = 3 ULD + gamma_N(ULD) (reference sums):
    (e + e') P_ij / sqrt(M_ii M_jj) + (e + e' + 4u + 4 ULD) |G_ij|, P = |Y|^T |Y| (module docstring of
    ``test_gpu_walkers_independent.py``)."""
    X = np.asarray(X, dtype=np.float64)
    N = X.shape[0]
    Y = X.astype(np.longdouble) - np.asarray(shift, dtype=np.float64).astype(np.longdouble)
    aY = np.abs(X - shift)
    diag = np.sum(Y * Y, axis=0)
    M = np.empty(len(i), dtype=np.longdouble)
    P = np.empty(len(i))
    for a in range(0, len(i), 64):
        sl = slice(a, a + 64)
        M[sl] = np.sum(Y[:, i[sl]] * Y[:, j[sl]], axis=0)
        P[sl] = np.sum(aY[:, i[sl]] * aY[:, j[sl]], axis=0)
    den = np.sqrt(diag[i]) * np.sqrt(diag[j])
    G = M / den
    e = 2 * U + PX.gamma(depth)
    e_ref = 3 * ULD + PX.gamma(N, ULD)
    bound = (e + e_ref) * (P / den.astype(np.float64)) + (e + e_ref + 4 * U + 4 * ULD) * np.abs(G.astype(np.float64))
    return G, bound


def parent_gram(X):
    """The parent's ``eb_walkers_gram`` in double: colmean_kernel's shift, the uncorrected sums (a plain matmul in
    place of the DMMA order; none of the failures below depends on that order), ``den = sqrt(M_jj M_kk)``, flag 2
    where ``M_jj`` is not > 0, flag 1 for non-finite input."""
    X = np.asarray(X, dtype=np.float64)
    with np.errstate(all="ignore"):
        Y = X - PX.colmean_device_order(X)
        M = Y.T @ Y
        d = np.diag(M)
        flags = (0 if np.all(np.isfinite(X)) else 1) | (0 if np.all(d > 0) else 2)
        den = np.sqrt(np.outer(d, d))
        G = np.where(den > 0, M / np.where(den > 0, den, 1.0), 0.0)
    return G, flags


def device_gram(X):
    """``eb_walkers_gram`` as it is now, in double (the DMMA order again a plain matmul): ``den = sqrt(M_jj)
    sqrt(M_kk)``, flag 4 and zero entries where ``M_jj`` is not a positive normal double."""
    _, flags = parent_gram(X)  # bits 0 and 1 are unchanged
    with np.errstate(all="ignore"):
        Y = X - PX.colmean_device_order(X)
        M = Y.T @ Y
        d = np.diag(M)
        ok = np.isfinite(d) & (d >= np.finfo(np.float64).tiny)
        rt = np.where(ok, np.sqrt(np.where(ok, d, 1.0)), 0.0)
        den = np.outer(rt, rt)
        G = np.where(den > 0, M / np.where(den > 0, den, 1.0), 0.0)
    bad = ~np.isfinite(G)
    return np.where(bad, 0.0, G), flags | (4 if (not ok.all() or bad.any()) else 0)


def parent_decision(X, host):
    """The parent's ``_walkers_independent``: False on any flag, True when cond <= 1e6 by the Gram matrix, else
    ``host(X)``.  Raises ``LinAlgError`` where its eigen-solve does (a NaN in the Gram matrix)."""
    G, flags = parent_gram(X)
    if flags:
        return False
    ev = np.linalg.eigvalsh(G)
    if ev[0] > 0 and np.sqrt(ev[-1] / ev[0]) <= 1e6:
        return True
    return bool(host(X))
