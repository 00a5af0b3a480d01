"""Exact log-probabilities of the device models and the first-order rounding-error bound of each kernel's
operation sequence (``test_gpu_logprob_exact.py`` holds the derivation; ``test_gpu_accept_exact.py`` uses the same
references and bounds for the log-probability inside the accept test).

Every double is an integer times a power of two, so the references are exact in Python integers (``Fraction``),
except the ring's square root, which ``decimal`` takes at 60 digits."""
import decimal
from fractions import Fraction

import numpy as np

U = 2.0 ** -53
ETA = 2.0 ** -1074


def gamma(n):
    return n * U / (1.0 - n * U)


def _ints(*arrays):
    """Python-int images of float64 arrays at one common exponent e <= 0: value = int * 2**e exactly."""
    parts = []
    for a in arrays:
        m, ex = np.frexp(np.asarray(a, dtype=np.float64))
        parts.append(((m * 2.0 ** 53).astype(np.int64), ex.astype(np.int64) - 53))
    nz = [ex[mi != 0] for mi, ex in parts if np.any(mi != 0)]
    e = min(0, min(int(x.min()) for x in nz)) if nz else 0
    out = []
    for mi, ex in parts:
        shift = np.where(mi == 0, 0, ex - e)  # (frexp gives zeros the exponent 0)
        flat = [int(v) << int(s) for v, s in zip(mi.ravel().tolist(), shift.ravel().tolist())]
        out.append(np.array(flat, dtype=object).reshape(mi.shape))
    return out, e


def _frac(n, e):
    return Fraction(n) * (Fraction(2) ** e)


def _to_float(q):
    try:
        return float(q)
    except OverflowError:
        return -np.inf if q < 0 else np.inf


def exact_iso(x):
    (n,), e = _ints(x)
    s = sum(v * v for v in n)
    return -_frac(s, 2 * e) / 2


def bound_iso(x):
    D = x.size
    with np.errstate(over="ignore"):
        return gamma(D) * 0.5 * float(np.sum(np.abs(x) ** 2)) + (D + 2) * ETA


def exact_ring(x, R, sigma):
    (n,), e = _ints(x)
    s = sum(v * v for v in n)
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        S = decimal.Decimal(s) * decimal.Decimal(2) ** (2 * e)
        d = S.sqrt() - decimal.Decimal(R)
        lp = -(d * d) / (2 * decimal.Decimal(sigma) ** 2)
        if abs(lp) > decimal.Decimal(np.finfo(np.float64).max):
            return -np.inf, float(d)
        return lp, float(d)


def bound_ring(x, R, sigma, d, lp):
    D = x.size
    with np.errstate(over="ignore"):
        S = float(np.sum(x * x)) + (D + 2) * ETA
    r = np.sqrt(S)
    dd = r * (0.5 * gamma(D) + U) + U * abs(d)
    return (2 * abs(d) * dd + dd * dd) / (2 * sigma * sigma) + gamma(3) * abs(lp) + 8 * ETA


def exact_rosen(x, a, b):
    (n, na, nb), e = _ints(x, np.float64(a), np.float64(b))
    na, nb = int(na), int(nb)
    sh = -e  # e <= 0
    tot = 0
    for i in range(len(n) - 1):
        t = (int(n[i + 1]) << sh) - int(n[i]) * int(n[i])  # (x1 - x0^2) * 2**(-2e)
        uu = na - int(n[i])  # (a - x0) * 2**(-e)
        tot += nb * t * t + ((uu * uu) << (3 * sh))  # * 2**(-5e)
    return -_frac(tot, 5 * e)


def bound_rosen(x, a, b):
    x0, x1 = x[:-1], x[1:]
    D = x.size
    with np.errstate(over="ignore", invalid="ignore"):
        t = x1 - x0 * x0
        u = a - x0
        dt = 2 * U * (x0 * x0 + np.abs(x1))
        per = b * (2 * np.abs(t) * dt + 2 * U * t * t) + 3 * U * u * u
        terms = b * t * t + u * u
        return float(np.sum(per) + gamma(D) * np.sum(terms)) + 6 * D * ETA


def exact_dense(x, mu, A):
    """A: the matrix, or its _ints image (converting it once per matrix saves most of the time)."""
    (nA,), eA = _ints(A) if isinstance(A, np.ndarray) else A
    (nx, nm), e = _ints(x, mu)
    xc = nx - nm
    q = int(xc.dot(nA.dot(xc)))  # xc^T A xc * 2**(-2e - eA)
    return -_frac(q, 2 * e + eA) / 2


def bound_dense_generic(x, mu, A):
    D = x.size
    xc = np.abs(x - mu)
    return gamma(2 * D + 2) * 0.5 * float(xc @ np.abs(A) @ xc) + (D * D + 4 * D + 8) * ETA


def bound_dense_dmma(x, mu, L):
    D = x.size
    z = np.abs(L).T @ np.abs(x - mu)
    return gamma(4 * D + 4) * 0.5 * float(z @ z) + (D * D + 4 * D + 8) * ETA
