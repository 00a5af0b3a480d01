"""The initial-state independence check (``EnsembleSampler._walkers_independent``, reference
``ensemble.py:653-663``): the device Gram matrix against an exact reference under a first-order bound, every
decision against the unmodified reference, the fast path, and ``run_mcmc`` end to end.

Gram matrix (``eb_walkers_gram``).  For ``x[N, D]`` the device forms the shift ``m`` (``colmean_kernel``; its
order is reproduced bit for bit), ``y = fl(x - m)``, the uncorrected sums ``M = y^T y`` on the DMMA pipe
(``launch_moments``, one accumulation), and on the host ``G_jk = M_jk / (sqrt(M_jj) sqrt(M_kk))``.  The reference
(``gram_exact.gram_reference``) takes the same double ``m`` as exact and works in np.longdouble.  Bound, per entry,
with u = 2^-53, gamma_n = n u / (1 - n u):

* centring: ``|fl(x - m) - (x - m)| <= u |y|``, so every product ``y_j y_k`` carries 2u;
* sums: each of ``M`` runs through at most ``depth`` additions (the rows one CTA stages, the CTA partials, the
  final +=; ``proposals_exact.moments_depth``), so ``|dM| <= (2u + gamma_depth) P`` with ``P = |Y|^T |Y|``;
  write e = 2u + gamma_depth;
* normalisation: ``dG / G = dM_jk / M_jk - dM_jj / (2 M_jj) - dM_kk / (2 M_kk)`` to first order, and
  ``P_jj = M_jj``, so the sums contribute ``e P_jk / sqrt(M_jj M_kk) + e |G_jk|``; two square roots, their product
  and the division add 4u |G_jk|;
* reference: ``ULD |y|`` for its own subtraction, one rounding per product and ``gamma_N(ULD)`` per sum (e' =
  3 ULD + gamma_N(ULD)), and 4 ULD |G| for its normalisation.

Total: ``(e + e') P_jk / sqrt(M_jj M_kk) + (e + e' + 4u + 4 ULD) |G_jk|``; since ``P_jk <= sqrt(M_jj M_kk)`` by
Cauchy-Schwarz this is at most ``2 e + ...``, a few hundred u.  The bound holds while ``M_jj`` and the denominator
are normal doubles: from ``|x| ~ 1e-154`` down the squares are subnormal, from ``1e154`` up they overflow, and the
device then sets flag bit 2 and returns 0 for the column's entries (never a NaN).  At ``|x| ~ 1e-80`` the sums are
normal while ``M_jj M_kk`` is not: the former ``sqrt(M_jj M_kk)`` lost digits there, the bound catches it.

Decisions.  ``tests/golden/walkers_independent/reference.npz`` holds the small rows of
``oracle/gen_golden_walkers_independent.py`` with the reference's decision (1, 0, or -1 where it raises
LinAlgError); larger rows are rebuilt from their seeds and decided by the host restatement
``emcee_b200.ensemble.walkers_independent``.  Which rows aim at which failure of the former engine:

=====================================  ==========================================================================
scale1e-200-*, scale1e-300-*           every square underflows: a healthy ensemble was refused
scale1e+160-*, scale1e+300-*           the sums overflow to inf, inf / inf = NaN: eigvalsh raised LinAlgError
scale*e-7[6-9]* ... scale*e-84-*-dep   M_jj M_kk subnormal: G's diagonal off by ~1e-7, a dependent ensemble
                                       (3 x_0 in column 3) accepted
const*                                 the zero-span test about the device's column mean instead of numpy's
=====================================  ==========================================================================
"""
import warnings

import numpy as np
import pytest

import gram_exact as GX
import proposals_exact as PX
from oracle import gen_golden_walkers_independent as W

import emcee_b200
from emcee_b200 import ensemble as ens
from emcee_b200 import models

pytestmark = pytest.mark.gpu

U = PX.U
FIXTURE = W.OUT
_SAMPLERS = {}


def sampler(D):
    if D not in _SAMPLERS:
        _SAMPLERS[D] = emcee_b200.EnsembleSampler(2 * D + 2, D, models.GaussianIso(), seed=1)
    return _SAMPLERS[D]


def sm_count():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


class Tracker(object):
    """Largest |device - reference| / bound of one class."""

    def __init__(self, name):
        self.name, self.worst, self.where = name, 0.0, None

    def check(self, err, bound, what):
        r = float(np.max(err / bound))
        if r > self.worst:
            self.worst, self.where = r, what
        assert r < 1.0, (self.name, what, r)

    def report(self):
        print("%-34s largest error / bound = %.3g (%s)" % (self.name, self.worst, self.where))


# ---- (a) the Gram matrix at every moments geometry -----------------------------------------------------------
GRAM_D = [1, 5, 8, 9, 17, 64, 128, 129, 255, 520, 1023, 1024]


def _row_counts(D):
    """N = D + 1, 2, a partial last chunk, and every CTA striding at least 4 chunks."""
    _, grid, CH = PX.moments_depth(10 ** 9, D, sm_count(), 1)
    return [D + 1, 2, 3 * CH + 5, 4 * grid * CH + 3]


def _inputs(N, D, rng):
    base = rng.standard_normal((N, D))
    yield "mixture+3", base @ (rng.standard_normal((D, D)) / np.sqrt(D)) + 3.0
    yield "1e6+1e-3", 1e6 + 1e-3 * base
    yield "spans1e-100..1e100", base * 10.0 ** np.linspace(-100.0, 100.0, D)


@pytest.mark.parametrize("D", GRAM_D)
def test_gram_matrix_exact(D):
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here")
    rng = np.random.default_rng(D)
    s = sampler(D)
    trackers = {}
    for N in _row_counts(D):
        depth = PX.moments_depth(N, D, sm_count(), 1)[0]
        for kind, X in _inputs(N, D, rng):
            gram, flags = s._engine.walkers_gram(X)
            assert flags == 0, (kind, N, flags)
            i, j = GX.pairs(D, rng)
            ref, bound = GX.gram_reference(X, PX.colmean_device_order(X), i, j, depth)
            err = np.abs(gram[i, j].astype(np.longdouble) - ref).astype(np.float64)
            trackers.setdefault(kind, Tracker("gram %s D=%d" % (kind, D))).check(err, bound, "N=%d" % N)
    for t in trackers.values():
        t.report()


def test_gram_matrix_out_of_range_is_flagged():
    """Raw calls whose sums of squares leave the normal range set bit 2 and return no NaN; at 1e-80 the sums are
    normal (only the product M_jj M_kk is not) and the bound holds."""
    rng = np.random.default_rng(80)
    N, D = 64, 4
    s = sampler(D)
    base = rng.standard_normal((N, D))
    for scale in (1e-160, 1e-200, 1e160):
        gram, flags = s._engine.walkers_gram(scale * base)
        assert flags & 4, (scale, flags)
        assert np.all(np.isfinite(gram)), scale
    t = Tracker("gram scale 1e-80")
    for X in (1e-80 * base, 1e-80 * np.c_[base[:, :3], 3.0 * base[:, 0]]):
        gram, flags = s._engine.walkers_gram(X)
        assert flags == 0
        i, j = GX.pairs(D, rng)
        ref, bound = GX.gram_reference(X, PX.colmean_device_order(X), i, j, PX.moments_depth(N, D, sm_count(), 1)[0])
        t.check(np.abs(gram[i, j].astype(np.longdouble) - ref).astype(np.float64), bound, "N=64")
    t.report()


# ---- (b) decisions --------------------------------------------------------------------------------------------
def _decide(fn, x):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return int(bool(fn(x)))
        except np.linalg.LinAlgError:
            return W.RAISES


def _stored():
    f = np.load(FIXTURE)
    return [(str(n), int(d), f["x%d" % k]) for k, (n, d) in enumerate(zip(f["names"], f["decision"]))]


STORED = _stored()
GENERATED = [r for r in W.rows() if not W.stored(r) and r["cls"] != "const"]


@pytest.mark.parametrize("name,decision,x", STORED, ids=[r[0] for r in STORED])
def test_decision_stored(name, decision, x):
    assert _decide(sampler(x.shape[1])._walkers_independent, x) == decision


@pytest.mark.parametrize("row", GENERATED, ids=[r["name"] for r in GENERATED])
def test_decision_generated(row):
    x = W.build(row)
    assert _decide(sampler(row["D"])._walkers_independent, x) == _decide(ens.walkers_independent, x)


@pytest.mark.parametrize("value", W.CONSTANTS)
def test_decision_constant_column_sweep(value):
    """One column held at ``value``, N = 16 ... 400: the decision follows numpy's mean of the column."""
    s = sampler(4)
    bad, seen = [], set()
    for row in W.rows():
        if row["cls"] == "const" and row["value"] == value:
            x = W.build(row)
            want = _decide(ens.walkers_independent, x)
            seen.add(want)
            if _decide(s._walkers_independent, x) != want:
                bad.append((row["N"], want))
    print("constant %g: reference outcomes %s" % (value, sorted(seen)))
    assert not bad, bad


# ---- (c) the fast path survives ------------------------------------------------------------------------------
def _count_host(monkeypatch):
    calls = []
    orig = ens.walkers_independent

    def counting(coords):
        calls.append(np.shape(coords))
        return orig(coords)

    monkeypatch.setattr(ens, "walkers_independent", counting)
    return calls


def test_fast_path_keeps_well_conditioned_ensembles_on_the_device(monkeypatch):
    calls = _count_host(monkeypatch)
    rows = [r for r in W.rows() if (r["cls"] == "cond" and r["kappa"] <= 1e5)
            or (r["cls"] == "scale" and not r["dep"] and 1e-100 <= r["scale"] <= 1e100)
            or r["name"] == "scale-mixed-1e-200-1e200"]
    for r in rows:
        assert sampler(r["D"])._walkers_independent(W.build(r)), r["name"]
    x = 3.0 + np.random.default_rng(128).standard_normal((65536, 128))
    assert sampler(128)._walkers_independent(x)
    assert calls == [], calls
    print("%d well-conditioned rows and 65536 x 128 decided on the device" % (len(rows) + 1))


def test_borderline_ensembles_go_to_the_host(monkeypatch):
    calls = _count_host(monkeypatch)
    rows = [r for r in W.rows() if r["cls"] == "cond" and 1e6 < r["kappa"] < 1e8 and r["offset"] == 0]
    for r in rows:
        n = len(calls)
        assert sampler(r["D"])._walkers_independent(W.build(r)), r["name"]
        assert len(calls) == n + 1, r["name"]


# ---- (d) end to end --------------------------------------------------------------------------------------------
MESSAGE = "Initial state has a large condition number. Make sure that your walkers are linearly independent"


def _stored_row(name):
    (row,) = [r for r in STORED if r[0] == name]
    return row


def test_run_mcmc_initial_state_check():
    _, d, x = _stored_row("scale1e-200-N64-ind")
    assert d == 1
    s = emcee_b200.EnsembleSampler(64, 4, models.GaussianIso(), seed=3)
    s.run_mcmc(x, 2, store=False)
    _, d, x = _stored_row("scale1e-80-N64-dep-r0")
    assert d == 0
    with pytest.raises(ValueError, match=MESSAGE):
        s.run_mcmc(x, 2, store=False)
    n = 0
    for name, d, x in STORED:
        if not name.startswith("const"):
            continue
        s = emcee_b200.EnsembleSampler(x.shape[0], 4, models.GaussianIso(), seed=3)
        if d:
            s.run_mcmc(x, 1, store=False)
        else:
            with pytest.raises(ValueError, match=MESSAGE):
                s.run_mcmc(x, 1, store=False)
        n += 1
    assert n >= 10
