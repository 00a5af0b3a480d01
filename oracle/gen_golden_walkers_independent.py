#!/usr/bin/env python
"""Generate ``tests/golden/walkers_independent/reference.npz`` from the UNMODIFIED reference (TEST INFRASTRUCTURE).

    python -m oracle.gen_golden_walkers_independent   # needs oracle/_ref/emcee_reference.zip (make_ref.py)

The rows are initial ensembles for the independence check of ``sample()`` (reference ``ensemble.py:653-663``):
conditioning sweeps, exact and rounded linear dependence, scales from 1e-310 to 1e300, constant and near-constant
columns, non-finite input and fewer walkers than dimensions.  Every row is built from a seed by ``build(row)``.
Rows of at most ``STORE_MAX_N`` walkers and ``STORE_MAX_D`` dimensions are stored with the reference's decision
and ``kappa``, the condition number of the exactly centred, column-normalised matrix (exact integer sums, the
normalisation and eigenvalues in mpmath at 50 digits; ``inf`` where a column is constant or the columns are
exactly dependent, ``nan`` for non-finite input).  Larger rows are rebuilt from their seeds by the tests, which
decide them with the host restatement ``emcee_b200.ensemble.walkers_independent``.  Importing this module does not
import the reference."""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ZIP = os.path.join(HERE, "_ref", "emcee_reference.zip")
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "walkers_independent", "reference.npz")
STORE_MAX_N, STORE_MAX_D = 400, 8
RAISES = -1  # stored decision of a row on which the reference raises LinAlgError (its SVD sees NaN)

KAPPAS = (1e1, 1e4, 9e5, 1.1e6, 1e7, 5e7, 2e8, 1e9, 1e12)
# coordinate scales: the 1e-80 band is where the product M_jj M_kk of two sums of squares turns subnormal
SCALES = ((1e-310, 64), (1e-300, 64), (1e-200, 64), (1e-160, 64), (1e-155, 64)) + tuple(
    (10.0 ** (-e / 2.0), 64) for e in range(152, 169)) + ((1e-20, 64), (1e20, 64)) + tuple(
    (10.0 ** (e / 2.0), 64) for e in range(152, 169)) + ((1e150, 64), (1e155, 1001), (1e160, 64), (1e300, 64))
CONSTANTS = (0.3, 1.1, 7.7, 1.5, 0.0)
CONST_N = tuple(range(16, 401))


def _row(name, cls, N, D, **kw):
    r = dict(name=name, cls=cls, N=int(N), D=int(D))
    r.update(kw)
    return r


def rows():
    """Every row of the table, in a fixed order (dicts: name, cls, N, D and the builder's parameters)."""
    out = []
    for kappa in KAPPAS:
        for D in (2, 8, 33, 128):
            for N in sorted({2 * D + 1, 64, 1001}):
                if N <= D + 1:
                    continue
                for off in (0.0, 1e6):
                    out.append(_row("cond-k%.1e-D%d-N%d-off%g" % (kappa, D, N, off), "cond", N, D, kappa=kappa,
                                    offset=off))
    for D, N in ((4, 64), (8, 200)):
        for off in (0.0, 7.0, 1e6, 2.0 ** 40):
            out.append(_row("dep-int-D%d-N%d-off%g" % (D, N, off), "dep_int", N, D, offset=off))
    for off in (0.0, 1e3):
        out.append(_row("dep-times3-off%g" % off, "dep_times3", 64, 4, offset=off))
    for scale, N in SCALES:
        reps = 3 if 3e-85 < scale < 3e-76 else 1  # three draws across the 1e-80 band
        for dep in (False, True):
            for rep in range(reps):
                out.append(_row("scale%.3g-N%d-%s%s" % (scale, N, "dep" if dep else "ind", "-r%d" % rep if reps > 1
                                                         else ""), "scale", N, 4, scale=scale, dep=dep, rep=rep))
    out.append(_row("scale-mixed-1e-200-1e200", "mixed", 64, 4))
    for c in CONSTANTS:
        for N in CONST_N:
            out.append(_row("const%g-N%d" % (c, N), "const", N, 4, value=c))
    for N in (16, 17, 100, 399):
        for where in ("first", "middle", "last"):
            out.append(_row("nearconst-N%d-%s" % (N, where), "nearconst", N, 4, where=where))
    for v in (np.inf, -np.inf, np.nan):
        for r, c in ((0, 0), (0, 3), (31, 0), (31, 3)):
            out.append(_row("nonfinite-%s-r%d-c%d" % (v, r, c), "nonfinite", 32, 4, value=v, at=(r, c)))
    for kind in ("halves", "one"):
        out.append(_row("overflow-centring-%s" % kind, "overflow", 32, 4, kind=kind))
    for D, N in ((4, 4), (4, 3), (4, 2), (8, 8), (8, 7), (8, 2), (1, 2), (1, 3), (1, 1001), (1025, 1030)):
        out.append(_row("smalln-D%d-N%d" % (D, N), "smalln", N, D))
    return out


def stored(row):
    return row["N"] <= STORE_MAX_N and row["D"] <= STORE_MAX_D


def kappa_target(row):
    """The condition number a row is built to have: the cond sweep's construction, ``inf`` for exact dependence,
    constant columns and fewer walkers than dimensions, ``nan`` for non-finite input, None where it is not set."""
    cls = row["cls"]
    if cls == "cond":
        return row["kappa"]
    if cls in ("dep_int", "const"):
        return np.inf
    if cls == "smalln":
        return np.inf if row["N"] <= row["D"] else None
    if cls == "nonfinite":
        return np.nan
    return None


def _rng(row):
    return np.random.default_rng(zlib.crc32(row["name"].encode()))


def build(row):
    """The coordinates ``[N, D]`` of a row."""
    rng = _rng(row)
    N, D, cls = row["N"], row["D"], row["cls"]
    if cls == "cond":
        # X = Q B: Q has orthonormal columns orthogonal to the ones vector (exactly centred), B = I except its
        # last column (cos t, 0, ..., sin t) with t = 2 atan(1 / kappa).  The columns of X have unit norm,
        # X^T X = B^T B has eigenvalues 1 +- cos t and 1, so cond(X) = cot(t / 2) = kappa.
        Z = rng.standard_normal((N, D))
        Q = np.linalg.qr(Z - Z.mean(0))[0]
        t = 2.0 * np.arctan(1.0 / row["kappa"])
        B = np.eye(D)
        B[0, D - 1], B[D - 1, D - 1] = np.cos(t), np.sin(t)
        return row["offset"] + Q @ B
    if cls == "dep_int":
        X = rng.integers(-50, 51, (N, D)).astype(np.float64)
        X[:, 3] = X[:, 0] + X[:, 1]
        if D > 5:
            X[:, 5] = X[:, 2] - X[:, 4]
        return X + row["offset"]
    if cls == "dep_times3":
        X = row["offset"] + rng.standard_normal((N, D))
        X[:, 3] = 3.0 * X[:, 0]
        return X
    if cls == "scale":
        X = row["scale"] * rng.standard_normal((N, D))
        if row["dep"]:
            X[:, 3] = 3.0 * X[:, 0]
        return X
    if cls == "mixed":
        X = rng.standard_normal((N, D))
        X[:, 0] *= 1e-200
        X[:, 1] *= 1e200
        return X
    if cls == "const":
        X = rng.standard_normal((N, D))
        X[:, 2] = row["value"]
        return X
    if cls == "nearconst":
        X = rng.standard_normal((N, D))
        X[:, 2] = 1.1
        r = {"first": 0, "middle": N // 2, "last": N - 1}[row["where"]]
        X[r, 2] = np.nextafter(1.1, 2.0)
        return X
    if cls == "nonfinite":
        X = rng.standard_normal((N, D))
        X[row["at"]] = row["value"]
        return X
    if cls == "overflow":
        X = rng.standard_normal((N, D))
        if row["kind"] == "halves":  # the mean itself overflows (inf - inf)
            X[: N // 2, 0] = 1.5e308
            X[N // 2:, 0] = -1.5e308
        else:  # the mean is finite, x - mean is not
            X[:, 0] = -1.5e308
            X[0, 0] = 1.5e308
        return X
    if cls == "smalln":
        return rng.standard_normal((N, D))
    raise ValueError(cls)


# ---- exact condition number ----------------------------------------------------------------------------------
def _int_image(x):
    """Object array of Python ints ``n`` and one exponent ``e`` with ``x == n * 2**e`` exactly."""
    m, ex = np.frexp(x)
    mi = (m * 2.0 ** 53).astype(np.int64)
    ex = ex.astype(np.int64) - 53
    nz = mi != 0
    e = int(ex[nz].min()) if nz.any() else 0
    sh = np.where(nz, ex - e, 0)
    return np.array([int(v) << int(s) for v, s in zip(mi.ravel().tolist(), sh.ravel().tolist())],
                    dtype=object).reshape(x.shape), e


def kappa_exact(X, dps=50):
    """cond of the exactly centred, column-normalised ``X``: the exact scaled covariance ``N X^T X - S S^T`` in
    integers, its correlation matrix and eigenvalues in mpmath.  ``inf`` for a zero column or an eigenvalue
    below 1e-40 of the largest (exact dependence), ``nan`` for non-finite input."""
    import mpmath

    X = np.asarray(X, dtype=np.float64)
    if not np.all(np.isfinite(X)):
        return np.nan
    N, D = X.shape
    Xi, _ = _int_image(X)
    S = Xi.sum(axis=0)
    A = N * Xi.T.dot(Xi) - np.outer(S, S)
    if any(A[j, j] == 0 for j in range(D)):
        return np.inf
    with mpmath.workdps(dps):
        r = [mpmath.sqrt(mpmath.mpf(int(A[j, j]))) for j in range(D)]
        R = mpmath.matrix(D, D)
        for j in range(D):
            for k in range(D):
                R[j, k] = mpmath.mpf(int(A[j, k])) / (r[j] * r[k])
        ev = sorted(mpmath.eigsy(R, eigvals_only=True))
        if ev[0] <= ev[-1] * mpmath.mpf(10) ** -40:
            return np.inf
        return float(mpmath.sqrt(ev[-1] / ev[0]))


# ---- the reference side ---------------------------------------------------------------------------------------
def import_reference():
    if REF_ZIP not in sys.path:
        sys.path.insert(0, REF_ZIP)
    import emcee

    assert REF_ZIP in emcee.__file__, emcee.__file__
    return emcee


def selected(table, decide):
    """The stored rows: every small row except the constant-column sweep, of which a few rows of each reference
    outcome per value are kept (the full sweep is rebuilt from seeds by the GPU test)."""
    keep, per = [], {}
    for row in table:
        if not stored(row):
            continue
        if row["cls"] == "const":
            d = decide(row)
            k = (row["value"], d)
            if per.get(k, 0) >= 3:
                continue
            per[k] = per.get(k, 0) + 1
        keep.append(row)
    return keep


def generate(out=OUT):
    import warnings

    emcee = import_reference()

    def decide(row):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                return int(bool(emcee.ensemble.walkers_independent(build(row))))
            except np.linalg.LinAlgError:
                return RAISES

    keep = selected(rows(), decide)
    arrays = dict(names=np.array([r["name"] for r in keep]), decision=np.array([decide(r) for r in keep], dtype=np.int8),
                  kappa=np.array([kappa_exact(build(r)) for r in keep]))
    for i, r in enumerate(keep):
        arrays["x%d" % i] = build(r)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print("%d rows stored: %d True, %d False, %d raise" % tuple([len(keep)] + [int(np.sum(arrays["decision"] == v))
                                                                 for v in (1, 0, RAISES)]))


if __name__ == "__main__":
    generate()
