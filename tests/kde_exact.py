r"""High-precision references and first-order rounding bounds for KDEMove (``kde.cu``): its proposals and its
Hastings factors, and ``kde_plan`` restated (``test_gpu_kde_exact.py`` runs them against the device,
``test_kde_exact_host.py`` against the oracle and a double emulation of the log-sum-exp kernels).

Notation: u = 2^-53, gamma_n = n u / (1 - n u), L the exact lower Cholesky factor of the complement covariance
(``proposals_exact.ExactCov``), bw the exact bandwidth, M = bw L, X = M^-1.  Bounds are first order in u.

Bandwidth.  The host forms bw with C ``pow`` (``step.cu`` kde_bandwidth): the exponent -1.0 / (D + 4) is rounded
once (relative u, so bw^(1 + u) = bw (1 + u |ln bw|)) and pow is within one ulp (2u):
delta_bw = u (2 + |ln bw|).  A scalar bandwidth is the double itself: delta_bw = 0.

Proposals (``kde_prepare_kernel``): q_i = fl(c[j_i] + fl(bw * fl(L^ z_i))) with L^ the device factor.  The fma
chain and the factor's error are ``mvn_bound``'s terms (covariance and Cholesky rounding carried to L, normals,
gamma_{D+1}); ``__dmul_rn(bw, acc)`` adds u |bw L z|, the host's bw delta_bw |bw L z|, ``__dadd_rn`` u |q|.  The
longdouble reference (u_ld) converts L, z and bw once each and sums D products: gamma_{D+2}(u_ld) |L||z| (in
``mvn_bound``), 2 u_ld |bw L z| and u_ld |q|.

Hastings factors.  The device computes, for a point p (an active row s_i or its proposal q_i) and a centre c,
t_c = -|y_p - y_c|^2 / 2 with y = X^ fl(x - mean), and f_i = LSE_c t_c(s_i) - LSE_c t_c(q_i).

 1. Factor.  The moment sums about the whole-ensemble column mean (``step.cu`` launch_step_kde) are off by
    ``cov_error_one_pass`` with the complement-gather ``moments_depth``; ``cov_chol_kernel``'s backward error is
    gamma_{D+1} |L||L^T| (Higham Thm 10.3); both carried to L by ``chol_perturbation``: |dL|.  With the host's
    bandwidth: |dM| <= bw |dL| + delta_bw bw |L|, and X changes by -X dM X.
 2. ``kde_factor_kernel`` forms X^ column by column by forward substitution with the products fl(bw * L_ik)
    (one rounding), an fma chain (at most D) and a division (one): the residual |M X^ - I| <= gamma_{D+2} |M||X^|
    (Higham §14.2), so X^ - X = X (M X^ - I) adds gamma_{D+2} |X||M||X|.  With 1: |X^ - X| <= B' and, acting on
    a difference dx = x_p - x_c, |dX dx| <= B |dx| with B = |X| (|dM| + gamma_{D+2} |M|) |X|.
 3. v = fl(x - mean): u |v|.  The error of mean itself is one shift common to every row: it cancels in v_p - v_c.
 4. ``whiten_row``'s fma chain of at most D terms: gamma_D |X^||v|.
    1-4: |d(y_p - y_c)| <= B |dx| + (u + gamma_D) |X| (|v_p| + |v_c|) =: e_pc.
 5. The distance: one rounded difference per dimension, squared, and an fma chain of D terms
    (``kde_lse_kernel``): gamma_{D+2} |t_c|; the factor -0.5 is exact.
    So |dt_c| <= |y_p - y_c|^T e_pc + gamma_{D+2} |t_c|.  Componentwise where a point costs at most ``COMP_MAX``
    products; otherwise by Cauchy-Schwarz |dy|^T e <= ||dy|| (||B||_2 ||dx|| + (u + gamma_D) || |X| (|v_p| +
    |v_c|) ||), with ||B||_2 computed once per case.

The log-sum-exp (``kde_lse_kernel`` per thread, its 16-lane xor fold, ``kde_merge_kernel``'s fold of the chunks):

 * the input errors: |dLSE| <= sum_c w_c |dt_c|, w the exact softmax weights of t;
 * every exponent is a difference of t_c and a running maximum, each rounded once; along one term's path (its own
   exp(t_c - m), every rescale exp(m_old - m_new), every fold exp(m - M)) the maxima only grow, so the arguments
   telescope to m - t_c with m = max t: u (m - t_c) relative, i.e. u sum_c w_c (m - t_c);
 * CUDA's ``exp`` and ``log`` are within 1 ulp (CUDA C++ Programming Guide, "Mathematical Functions", double
   precision), i.e. 2u relative; a product or a sum one rounding u.  One term's path: its own exp (2u); per tile
   of its chunk a rescale (exp and product, 3u) and four additions (4u); four lane-fold levels and ``nchunks``
   chunk folds of (exp, product, sum: 4u) each: chain = (2 + 7 tpc + 16 + 4 nchunks) u relative to the sum;
 * log(s): 2u |log s|; m + log s: u |LSE|.
Then |df_i| <= dLSE(s_i) + dLSE(q_i) + u |f_i|.

References.  The factors are recomputed from the device's own stored rows (s, q and the complement, taken as
exact) in mpmath at 45 digits where a case has at most ``MP_MAX_WORK`` point x centre x dim products and ndim
<= 32, in ``np.longdouble`` otherwise, by the same algorithm (explicit inverse by forward substitution, a common
shift, direct differences, log-sum-exp): its own roundings are the bound above with u -> u_ref, the exact
covariance instead of the moment sums (u_ref |A| and the u_ref Cholesky backward error; a converted mpmath factor
adds u_ref |L|), and a sequential chain of nc + 4 for the sum.
"""
import math

import mpmath
import numpy as np
from scipy.linalg import solve_triangular

import proposals_exact as PX
from oracle import philox as px

U = PX.U
KT = 64  # points and centres per tile (kde.cu)
KD = 32  # dimensions per staged chunk
MP_MAX_WORK = 1e6
COMP_MAX = 2e7  # products per point above which the |dt| bound goes normwise


def gamma(n, u=U):
    return PX.gamma(n, u)


# ---- kde_plan (kde.cu:251-263) -----------------------------------------------------------------------------------
def kde_plan(ns, nc, sm_count):
    """The launch geometry of ``kde_lse_kernel`` for ``ns`` active rows and ``nc`` centres, and its ragged edges."""
    P = 2 * ns
    ptiles = -(-P // KT)
    ctiles = -(-nc // KT)
    want = -(-(4 * sm_count) // ptiles)
    want = max(1, min(want, ctiles))
    tpc = -(-ctiles // want)
    nchunks = -(-ctiles // tpc)
    return dict(P=P, ptiles=ptiles, ctiles=ctiles, tpc=tpc, nchunks=nchunks,
                last_ptile=P - (ptiles - 1) * KT, last_ctile=nc - (ctiles - 1) * KT,
                last_chunk=ctiles - (nchunks - 1) * tpc)


def variant(plan):
    return "kde tpc=%d nchunks=%d" % (plan["tpc"], plan["nchunks"])


def split_sizes(N, nsplits):
    """Walkers per split (``red_blue.py:77``: arange(N) % nsplits; a shuffle keeps the counts)."""
    return [len(range(j, N, nsplits)) for j in range(nsplits)]


def last_split_plan(N, nsplits, sm_count):
    ns = split_sizes(N, nsplits)[-1]
    return kde_plan(ns, N - ns, sm_count), ns, N - ns


def regimes(plan, ns, nc, D):
    """The set of regime names one geometry exercises."""
    out = set()
    if plan["nchunks"] == 1 and plan["tpc"] > 1:
        out.add("one chunk, many tiles")
    if plan["nchunks"] > 1 and plan["tpc"] == 1:
        out.add("chunks of one tile")
    if plan["nchunks"] > 1 and plan["tpc"] > 1 and plan["last_chunk"] < plan["tpc"]:
        out.add("chunks of many tiles, short last chunk")
    if D > KD and D % KD != 0:
        out.add("ragged last dim chunk")
    if plan["last_ptile"] < KT:
        out.add("ragged last point tile")
    if plan["last_ctile"] < KT and plan["ctiles"] > 1:
        out.add("ragged last centre tile")
    return out


REQUIRED_REGIMES = {"one chunk, many tiles", "chunks of one tile", "chunks of many tiles, short last chunk",
                    "ragged last dim chunk", "ragged last point tile", "ragged last centre tile"}


# ---- bandwidth ----------------------------------------------------------------------------------------------------
def bandwidth(bw_method, n, D):
    """(the host's double, the exact value as mpf, delta_bw): scipy's factor of ``n`` uniformly weighted points."""
    if bw_method is not None and not isinstance(bw_method, str):
        return float(bw_method), mpmath.mpf(float(bw_method)), 0.0
    with mpmath.workdps(PX.MP_DPS):
        base = mpmath.mpf(n * (D + 2)) / 4 if bw_method == "silverman" else mpmath.mpf(n)
        exact = base ** (-mpmath.mpf(1) / (D + 4))
    host = math.pow(n * (D + 2.0) / 4.0 if bw_method == "silverman" else float(n), -1.0 / (D + 4))
    return host, exact, U * (2.0 + abs(math.log(host)))


def centre_ranks(seed, step, split, ns, nc):
    """Complement rank of the kernel centre of every active rank (block (i, TAG_PROP_A), kde_centre_rank)."""
    w0, w1, _, _ = px.draw_words(seed, step, split, px.TAG_PROP_A, np.arange(ns))
    return px.bounded64(w0, w1, nc)


# ---- the factor of a case -----------------------------------------------------------------------------------------
class Case(object):
    """The exact covariance of the complement ``C`` (integer-valued rows), its reference factor and the device
    factor's error |dL|.  ``X_all``: the whole ensemble at the half-step (the moment sums' shift)."""

    def __init__(self, C, X_all, bw_method, sm_count, max_rank=None):
        self.C = np.asarray(C, dtype=np.float64)
        self.nc, self.D = self.C.shape
        self.A = PX.ExactCov(self.C)
        self.L, self.Lref, self.piv, self.uref = PX.chol_reference(self.A, max_rank)
        self.Af = self.A.f64()
        self.bw, self.bw_mp, self.dbw = bandwidth(bw_method, self.nc, self.D)
        self.shift = PX.colmean_device_order(X_all)
        self.depth = PX.moments_depth(self.nc, self.D, sm_count, 1)[0]
        self.Mcov = PX.cov_error_one_pass(self.C - self.shift, self.nc, self.depth, self.Af)
        aL = np.abs(self.L)
        # the device's covariance, its Cholesky rounding and the reference's own (as mvn_bound takes them)
        Mdev = self.Mcov + PX.backward_error(self.L)
        self.dL = PX.chol_perturbation(self.L, Mdev, self.D)
        Mref = PX.backward_error(self.L, self.uref) + self.uref * (aL @ aL.T)
        self.dL_ref = PX.chol_perturbation(self.L, Mref, self.D)
        self.mean = self.shift + (self.C - self.shift).sum(axis=0) / self.nc

    def pivots_ok(self):
        PX.check_pivot_prefix(self.L, self.piv, self.D, float(np.max(np.diag(self.Af))))

    def Lref_ld(self):
        return PX.mp_to_ld(self.Lref) if self.Lref.dtype == object else self.Lref

    def bw_ld(self):
        return np.longdouble(mpmath.nstr(self.bw_mp, 25, min_fixed=1, max_fixed=0))


# ---- proposals ----------------------------------------------------------------------------------------------------
def proposal_reference(case, j, z):
    """c[j] + bw L z in longdouble: ``z`` [rows, D] mpf normals, ``j`` complement ranks."""
    zl = PX.mp_to_ld(z)
    return case.C[j].astype(np.longdouble) + case.bw_ld() * (zl @ case.Lref_ld().T)


def proposal_bound(case, zabs, qabs):
    """Per-element bound on |q_device - q_reference| (module docstring)."""
    D = case.D
    uref = PX.ULD
    Lz = zabs @ np.abs(case.L).T
    base = PX.mvn_bound(case.L, case.Mcov, D, zabs, np.zeros_like(qabs), uref)
    if case.Lref.dtype == object:
        base = base + uref * Lz  # the mpmath factor converted to longdouble
    return case.bw * base + (case.dbw + U + 2 * uref) * case.bw * Lz + (U + uref) * qabs


# ---- factor references --------------------------------------------------------------------------------------------
def _inverse_ld(M):
    """M^-1 of a lower-triangular longdouble matrix by forward substitution (row by row, every column at once)."""
    D = M.shape[0]
    X = np.zeros_like(M)
    for i in range(D):
        r = -(M[i, :i] @ X[:i, :]) if i else np.zeros(D, dtype=M.dtype)
        r[i] += 1
        X[i, :] = r / M[i, i]
    return X


def factor_reference(case, S, Q):
    """LSE over the complement of t_c = -|(bw L)^-1 (x - c)|^2 / 2 for the rows ``S`` and ``Q`` (float64, taken as
    exact).  Returns dict(f, lse_s, lse_q: float64; t_s, t_q, w_s, w_q: float64 [rows, nc]; u: unit roundoff of
    the reference)."""
    C = case.C
    nc, D = C.shape
    rows = np.concatenate([S, Q])
    use_mp = rows.shape[0] * nc * D <= MP_MAX_WORK and case.Lref.dtype == object
    if use_mp:
        return _factor_reference_mp(case, rows, len(S))
    if not PX.longdouble_ok():
        return None
    M = case.bw_ld() * case.Lref_ld()
    X = _inverse_ld(M)
    sh = case.mean.astype(np.longdouble)
    yc = (C.astype(np.longdouble) - sh) @ X.T
    yp = (rows.astype(np.longdouble) - sh) @ X.T
    t = np.empty((len(rows), nc), dtype=np.longdouble)
    for p in range(len(rows)):
        d = yc - yp[p]
        t[p] = -0.5 * np.sum(d * d, axis=1)
    m = t.max(axis=1)
    e = np.exp(t - m[:, None])
    ssum = e.sum(axis=1)
    lse = m + np.log(ssum)
    w = (e / ssum[:, None]).astype(np.float64)
    return _pack(lse, t.astype(np.float64), w, len(S), PX.ULD)


def _factor_reference_mp(case, rows, ns):
    nc, D = case.C.shape
    with mpmath.workdps(PX.MP_DPS):
        bw = case.bw_mp
        Lm = [[case.Lref[i, k] * bw for k in range(D)] for i in range(D)]

        def whiten(x):
            y = []
            for i in range(D):
                y.append((mpmath.mpf(float(x[i])) - mpmath.fsum(Lm[i][k] * y[k] for k in range(i))) / Lm[i][i])
            return y

        yc = [whiten(c) for c in case.C]
        yp = [whiten(x) for x in rows]
        lse = np.empty(len(rows), dtype=object)
        t64 = np.empty((len(rows), nc))
        w64 = np.empty((len(rows), nc))
        for p in range(len(rows)):
            t = [-mpmath.fsum((a - b) ** 2 for a, b in zip(yp[p], yc[c])) / 2 for c in range(nc)]
            m = max(t)
            e = [mpmath.exp(v - m) for v in t]
            ssum = mpmath.fsum(e)
            lse[p] = m + mpmath.log(ssum)
            t64[p] = [float(v) for v in t]
            w64[p] = [float(v / ssum) for v in e]
        return _pack(lse, t64, w64, ns, PX.UMP)


def _pack(lse, t, w, ns, u):
    f = lse[:ns] - lse[ns:]
    return dict(f=f, lse_s=lse[:ns], lse_q=lse[ns:], t_s=t[:ns], t_q=t[ns:], w_s=w[:ns], w_q=w[ns:], u=u)


def factor_error(f_dev, f_ref):
    if f_ref.dtype == object:
        with mpmath.workdps(PX.MP_DPS):
            return np.array([float(abs(mpmath.mpf(float(a)) - b)) for a, b in zip(f_dev, f_ref)])
    return np.abs(np.asarray(f_dev).astype(np.longdouble) - f_ref).astype(np.float64)


# ---- factor bound -------------------------------------------------------------------------------------------------
class FactorBound(object):
    """|dt_c| and |dLSE| bounds of one arithmetic (unit ``u``): ``dL`` the error of its factor, ``dbw`` of its
    bandwidth, ``chain`` its log-sum-exp path length in units of u (module docstring)."""

    def __init__(self, case, dL, dbw, chain, u, shift=None):
        D = case.D
        self.case, self.u, self.chain = case, u, chain
        self.shift = case.mean if shift is None else shift
        M = case.bw * case.L
        self.X = solve_triangular(M, np.eye(D), lower=True)
        aX = np.abs(self.X)
        dM = case.bw * dL + dbw * case.bw * np.abs(case.L)
        self.B = aX @ (dM + gamma(D + 2, u) * np.abs(M)) @ aX
        self.aX = aX
        self.comp = case.nc * D * D <= COMP_MAX
        self.nB = float(np.linalg.norm(self.B, 2))
        self.aXvc = np.abs(case.C - self.shift) @ aX.T  # |X| |v_c|, [nc, D]

    def dt(self, x, t):
        """Bound on |dt_c| for the point ``x`` against every centre; ``t`` its exact t_c (float64)."""
        case, D, u = self.case, self.case.D, self.u
        dx = x - case.C
        aXv = self.aXvc + self.aX @ np.abs(x - self.shift)
        rnd = u + gamma(D, u)
        if self.comp:
            dy = np.abs(dx @ self.X.T)
            e = np.abs(dx) @ self.B.T + rnd * aXv
            lin = np.sum(dy * e, axis=1)
        else:
            ndy = np.sqrt(np.abs(2 * t))
            lin = ndy * (self.nB * np.linalg.norm(dx, axis=1) + rnd * np.linalg.norm(aXv, axis=1))
        return lin + gamma(D + 2, u) * np.abs(t)

    def lse(self, x, t, w, lse):
        """Bound on |dLSE| of the point ``x``."""
        u = self.u
        dt = self.dt(x, t)
        m = float(np.max(t))
        lse = float(lse)
        return float(np.sum(w * (dt + u * (m - t)))) + self.chain * u + 2 * u * abs(lse - m) + u * abs(lse)


def lse_chain(plan):
    return 2 + 7 * plan["tpc"] + 16 + 4 * plan["nchunks"]


def factor_bounds(case, ref, S, Q, plan, shift=None):
    """Bound on |f_device - f_reference| per row of ``S`` / ``Q``: the device's arithmetic and the reference's.
    ``shift``: the rows' common shift before whitening, if not the complement mean (the oracle whitens x itself:
    zero)."""
    dev = FactorBound(case, case.dL, case.dbw, lse_chain(plan), U, shift)
    uref = ref["u"]
    dLr = case.dL_ref + (uref * np.abs(case.L) if case.Lref.dtype == object else 0.0)
    rb = FactorBound(case, dLr, uref, case.nc + 4, uref)
    out = np.empty(len(S))
    for i in range(len(S)):
        f = float(ref["lse_s"][i] - ref["lse_q"][i])
        b = 0.0
        for fb in (dev, rb):
            b += fb.lse(S[i], ref["t_s"][i], ref["w_s"][i], ref["lse_s"][i])
            b += fb.lse(Q[i], ref["t_q"][i], ref["w_q"][i], ref["lse_q"][i])
        out[i] = b + (U + uref) * abs(f)
    return out


# ---- the cases ----------------------------------------------------------------------------------------------------
# id, nwalkers, ndim, nsplits, bw_method, state kind (geometries for 132 SMs; the last split is the one observed)
ROWS = [
    ("d1", 130, 1, 2, None, "int"),
    ("d33", 129, 33, 2, None, "int"),
    ("d64", 258, 64, 2, "silverman", "int"),
    ("d100", 450, 100, 2, 0.05, "int"),
    ("ragged", 4225, 40, 2, None, "int"),
    ("bench4096", 4096, 16, 2, None, "int"),
    ("n16384", 16384, 32, 2, None, "int"),
    ("n65536", 65536, 8, 2, None, "int"),
    ("d257", 600, 257, 2, "silverman", "int"),
    ("d1024", 2112, 1024, 2, None, "int"),
    ("ns3", 1001, 24, 3, 1.5, "int"),
    ("ns32", 2080, 8, 32, None, "int"),
    ("far", 258, 12, 2, None, "far"),
    ("cond", 450, 24, 2, "silverman", "cond"),
]
ROW = {r[0]: r for r in ROWS}


def state(kind, N, D, rng):
    """Integer-valued ensembles (their covariances are exact in int64)."""
    if kind == "far":
        return 1.0e4 + np.round(rng.standard_normal((N, D)))
    if kind == "cond":
        q, _ = np.linalg.qr(rng.standard_normal((D, D)))
        return np.round((rng.standard_normal((N, D)) * np.logspace(0, 4, D)) @ q.T)
    return np.round(rng.standard_normal((N, D)) * 16.0)


def coverage(sm_count):
    """Regimes the rows exercise at ``sm_count`` SMs."""
    seen = set()
    for _, N, D, nsplits, _, _ in ROWS:
        plan, ns, nc = last_split_plan(N, nsplits, sm_count)
        seen |= regimes(plan, ns, nc, D)
    return seen


def checked_ranks(ns, plan, spread):
    """Active ranks whose factors are checked: both ends, the ranks of the last point tile's points (s or q
    half), and ``spread`` more."""
    P = plan["P"]
    last = np.arange((plan["ptiles"] - 1) * KT, P)
    r = np.r_[0, ns - 1, last[last < ns], last[last >= ns] - ns, np.linspace(0, ns - 1, spread).astype(np.int64)]
    return np.unique(r)
