"""``kde_exact.py`` on the CPU: its reference against the oracle and mpmath, a double emulation of ``kde.cu``'s
kernels in their operation order within the factor bound, mutants of that emulation far outside it, and the
restated ``kde_plan``.

The emulation (``emulate``) follows ``kde_factor_kernel`` (column-wise forward substitution with fl(bw * L_ik)),
``kde_prepare_kernel`` (q = c + bw (L z), y = X (x - mean) summed in column order) and ``kde_lse_kernel`` /
``kde_merge_kernel``: 64 x 64 tiles, dimensions in chunks of 32 summed in order, each thread's 4 points x 4
centres (centre lanes tc + 16 c), the per-tile rescale of the running (max, sum), the 16-lane xor fold and the fold
of the ``gridDim.y`` chunks.  numpy has no fused multiply-add: every fma is a product then a sum, two roundings
where the device has one, which the same gamma_n counts cover (a chain of n terms sees at most n roundings either
way).  Its factor is the numpy Cholesky of the correctly rounded covariance (within the one-pass bound)."""
import numpy as np
import pytest

import kde_exact as KX
import proposals_exact as PX
from oracle import kde as ok
from oracle import philox as px

SM = 132


def _fold(m, s, mo, so, rescale=True):
    M = np.maximum(m, mo)
    with np.errstate(invalid="ignore"):
        if rescale:
            ns = s * np.exp(m - M) + so * np.exp(mo - M)
        else:
            ns = s + so
    keep = M == -np.inf
    return np.where(keep, m, M), np.where(keep, s, ns)


def emulate(X_all, act, comp, seed, step, split, bw_method, sm_count=SM, mutant=None):
    """(f, Q): the device's factors and proposals of one split, in double, in the kernels' order."""
    C = X_all[comp]
    S = X_all[act]
    nc, D = C.shape
    ns = len(act)
    shift = PX.colmean_device_order(X_all)
    mean = shift + (C - shift).sum(axis=0) / nc
    L = np.linalg.cholesky(PX.ExactCov(C).f64())
    bw = KX.bandwidth(bw_method, nc, D)[0]
    bwx = 1.0 if mutant == "whiten_L" else bw
    # kde_factor_kernel: columns j by forward substitution (zero products before k = j add nothing)
    X = np.zeros((D, D))
    for i in range(D):
        v = np.zeros(D)
        for k in range(i):
            v = v + (bwx * L[i, k]) * X[k]
        X[i, :i] = -v[:i] / (bwx * L[i, i])
        X[i, i] = 1.0 / (bwx * L[i, i])
    # kde_prepare_kernel
    j = KX.centre_ranks(seed, step, split, ns, nc)
    z = px.normals(seed, step, split, np.arange(ns), D)
    Lz = np.zeros((ns, D))
    for k in range(D):
        Lz = Lz + z[:, k:k + 1] * L[:, k][None, :]
    Q = C[j] + bw * Lz

    def whiten(R):
        V = R - mean
        y = np.zeros_like(V)
        for k in range(D):
            y = y + X[:, k][None, :] * V[:, k:k + 1]
        return y

    yp = whiten(np.concatenate([S, Q]))
    yc = whiten(C)
    # kde_lse_kernel
    plan = KX.kde_plan(ns, nc, sm_count)
    P, ctiles, tpc, nch = plan["P"], plan["ctiles"], plan["tpc"], plan["nchunks"]
    ycp = np.zeros((ctiles * KX.KT, D))
    ycp[:nc] = yc
    dims = D
    if mutant == "drop_last_dchunk":
        dims = ((D - 1) // KX.KD) * KX.KD
    lanes = np.arange(16)
    part_m = np.empty((nch, P))
    part_s = np.empty((nch, P))
    for y in range(nch):
        lo = y * tpc
        hi = min(lo + tpc + (1 if mutant == "tile_twice" and y < nch - 1 else 0), ctiles)
        if mutant == "skip_last_ctile" and hi == ctiles:
            hi -= 1
        m = np.full((P, 16), -np.inf)
        s = np.zeros((P, 16))
        for ct in range(lo, hi):
            c0 = ct * KX.KT
            acc = np.zeros((P, KX.KT))
            for d in range(dims):
                diff = yp[:, d:d + 1] - ycp[c0:c0 + KX.KT, d][None, :]
                acc = acc + diff * diff
            col = np.arange(KX.KT)
            t = np.where((c0 + col < nc)[None, :], -0.5 * acc, -np.inf).reshape(P, 4, 16)
            tmax = t.max(axis=1)
            up = tmax > m
            with np.errstate(invalid="ignore"):
                s = np.where(up, s * np.exp(m - tmax), s)
            m = np.where(up, tmax, m)
            for c in range(4):
                with np.errstate(invalid="ignore"):
                    s = np.where(m > -np.inf, s + np.exp(t[:, c, :] - m), s)
        for off in (8, 4, 2, 1):
            m, s = _fold(m, s, m[:, lanes ^ off], s[:, lanes ^ off])
        part_m[y], part_s[y] = m[:, 0], s[:, 0]
    # kde_merge_kernel
    m = np.full(P, -np.inf)
    s = np.zeros(P)
    for y in range(nch):
        m, s = _fold(m, s, part_m[y], part_s[y], rescale=mutant != "merge_no_rescale")
    lse = m + np.log(s)
    return lse[:ns] - lse[ns:], Q


def _setup(name, seed=0x5EED, step=0):
    _, N, D, nsplits, bw, kind = KX.ROW[name]
    rng = np.random.default_rng(seed ^ (N * 1315423911 + D))
    X0 = KX.state(kind, N, D, rng)
    inds = px.split_assignment(seed, step, N, nsplits, True)
    sets = [np.flatnonzero(inds == j) for j in range(nsplits)]
    act, comp = sets[-1], np.concatenate(sets[:-1])
    return X0, act, comp, seed, step, nsplits - 1, bw


_CACHE = {}


def _checked(name):
    """(f_emulated, reference, bound, ranks) of a row at 132 SMs."""
    if name not in _CACHE:
        X0, act, comp, seed, step, split, bw = _setup(name)
        f, Q = emulate(X0, act, comp, seed, step, split, bw)
        case = KX.Case(X0[comp], X0, bw, SM)
        case.pivots_ok()
        plan = KX.kde_plan(len(act), len(comp), SM)
        ranks = KX.checked_ranks(len(act), plan, 32)
        S = X0[act][ranks]
        ref = KX.factor_reference(case, S, Q[ranks])
        if ref is None:
            pytest.skip("np.longdouble is not wider than double here")
        bound = KX.factor_bounds(case, ref, S, Q[ranks], plan)
        _CACHE[name] = (f, ref, bound, ranks, (X0, act, comp, seed, step, split, bw, case, Q))
    return _CACHE[name]


EMU_ROWS = ["d1", "d33", "d64", "d100", "ragged", "bench4096", "ns3", "far", "cond"]


@pytest.mark.parametrize("name", EMU_ROWS)
def test_emulation_within_factor_bound(name):
    f, ref, bound, ranks, _ = _checked(name)
    ratio = KX.factor_error(f[ranks], ref["f"]) / bound
    print("%s: emulation largest error / bound = %.3g" % (name, ratio.max()))
    assert ratio.max() < 1.0


MUTANTS = [
    ("skip_last_ctile", "d1"), ("skip_last_ctile", "d33"),
    ("drop_last_dchunk", "d33"), ("drop_last_dchunk", "d100"),
    ("merge_no_rescale", "ragged"), ("merge_no_rescale", "bench4096"),
    ("tile_twice", "ragged"),
    ("whiten_L", "d64"),
]


@pytest.mark.parametrize("mutant,name", MUTANTS)
def test_mutant_exceeds_factor_bound(mutant, name):
    _, ref, bound, ranks, (X0, act, comp, seed, step, split, bw, case, Q) = _checked(name)
    f, _ = emulate(X0, act, comp, seed, step, split, bw, mutant=mutant)
    ratio = KX.factor_error(f[ranks], ref["f"]) / bound
    print("%s at %s: largest error / bound = %.3g" % (mutant, name, ratio.max()))
    assert ratio.max() >= 1e3


@pytest.mark.parametrize("name", ["d1", "d33", "far"])
def test_reference_against_oracle(name):
    """The oracle's ``kde_logpdf`` (numpy / LAPACK arithmetic) agrees with the reference within the factor bound,
    and at ndim 1 the longdouble reference agrees with mpmath within its own bound.  The oracle whitens the rows
    without centring them, so its bound takes |x| where the device's takes |x - mean|: at ``far`` (rows near 1e4,
    unit spread) that is the cancellation the device's centring removes."""
    _, ref, bound, ranks, (X0, act, comp, seed, step, split, bw, case, Q) = _checked(name)
    C = X0[comp]
    S = X0[act][ranks]
    L = np.linalg.cholesky(np.cov(C, rowvar=0).reshape(case.D, case.D)) * case.bw
    f_or = ok.kde_logpdf(C, L, S) - ok.kde_logpdf(C, L, Q[ranks])
    plan = KX.kde_plan(len(act), len(comp), SM)
    bound_or = KX.factor_bounds(case, ref, S, Q[ranks], plan, shift=np.zeros(case.D))
    ratio = KX.factor_error(f_or, ref["f"]) / bound_or
    print("%s: device bound / oracle bound = %.3g" % (name, float(np.max(bound / bound_or))))
    print("%s: oracle largest error / bound = %.3g" % (name, ratio.max()))
    assert ratio.max() < 1.0
    if ref["f"].dtype == object and PX.longdouble_ok():
        old = KX.MP_MAX_WORK
        KX.MP_MAX_WORK = 0
        try:
            ld = KX.factor_reference(case, S, Q[ranks])
        finally:
            KX.MP_MAX_WORK = old
        err = KX.factor_error(np.asarray(ld["f"], dtype=np.float64), ref["f"])
        # the longdouble result rounded to double adds u |f|
        b = KX.factor_bounds(case, ld, S, Q[ranks], KX.kde_plan(len(act), len(comp), SM))
        assert np.all(err <= b), float(np.max(err / b))


# kde_plan at 132 and 114 SMs: (tpc, nchunks, last chunk tiles) of the table's rows
PLAN_132 = {"d1": (1, 2, 1), "d33": (1, 2, 1), "d64": (1, 3, 1), "ragged": (5, 7, 4), "bench4096": (4, 8, 4),
            "n16384": (43, 3, 42), "n65536": (512, 1, 512), "d257": (1, 5, 1), "d1024": (2, 9, 1),
            "ns3": (1, 11, 1), "ns32": (1, 32, 1)}
PLAN_114 = dict(PLAN_132, n16384=(64, 2, 64))


@pytest.mark.parametrize("sm,table", [(132, PLAN_132), (114, PLAN_114)])
def test_kde_plan_geometries(sm, table):
    for name, want in sorted(table.items()):
        _, N, D, nsplits, _, _ = KX.ROW[name]
        plan, ns, nc = KX.last_split_plan(N, nsplits, sm)
        assert (plan["tpc"], plan["nchunks"], plan["last_chunk"]) == want, (name, plan)
    assert KX.REQUIRED_REGIMES <= KX.coverage(sm), KX.REQUIRED_REGIMES - KX.coverage(sm)
    # the edges the table names
    p, ns, nc = KX.last_split_plan(130, 2, sm)
    assert (nc, p["last_ctile"], p["P"], p["last_ptile"]) == (65, 1, 130, 2)
    p, ns, nc = KX.last_split_plan(600, 2, sm)
    assert p["last_ctile"] == 44
    p, ns, nc = KX.last_split_plan(2080, 32, sm)
    assert (ns, nc, p["ptiles"], p["tpc"]) == (65, 2015, 3, 1)
