"""The independence-check fixture (``tests/golden/walkers_independent/reference.npz``, made by
``oracle/gen_golden_walkers_independent.py`` from the unmodified reference) and the helpers of
``test_gpu_walkers_independent.py``, on the CPU: every stored kappa is what its row was built to have, the host
restatement of ``walkers_independent`` takes every stored reference decision, the Gram bound holds against an
emulation of the device arithmetic and fails against a planted error, and an emulation of the engine's former
decision fails on the rows the GPU test names for each of its four failures."""
import os
import warnings

import numpy as np
import pytest

import gram_exact as GX
import proposals_exact as PX
from oracle import gen_golden_walkers_independent as W

from emcee_b200.ensemble import walkers_independent

FIXTURE = W.OUT
TABLE = {r["name"]: r for r in W.rows()}


def _fixture():
    f = np.load(FIXTURE)
    names = [str(n) for n in f["names"]]
    return names, f["decision"], f["kappa"], [f["x%d" % k] for k in range(len(names))]


def _host(x):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return int(bool(walkers_independent(x)))
        except np.linalg.LinAlgError:
            return W.RAISES


def test_fixture_rows_are_the_table():
    names, _, _, xs = _fixture()
    for name, x in zip(names, xs):
        row = TABLE[name]
        assert W.stored(row)
        assert np.array_equal(x, W.build(row), equal_nan=True), name
    classes = {TABLE[n]["cls"] for n in names}
    assert classes == {"cond", "dep_int", "dep_times3", "scale", "mixed", "const", "nearconst", "nonfinite",
                       "overflow", "smalln"}


def test_fixture_kappa_matches_construction():
    """kappa of a cond row is its construction's up to what the rounding of the coordinates can move it (relative
    kappa u (1 + offset), checked where that is below 1/2); exact dependence, constant columns and N <= D are
    infinite; non-finite rows are NaN; the rounded dependence of ``3 x_0`` sits far above the reference's 1e8."""
    names, _, kappa, _ = _fixture()
    for name, k in zip(names, kappa):
        row = TABLE[name]
        t = W.kappa_target(row)
        if row["cls"] == "cond":
            tol = 1e-8 + t * (1.0 + row["offset"]) * PX.U
            if tol < 0.5:  # else the rounding to the offset's grid has replaced the construction
                assert abs(k / t - 1.0) <= tol, (name, k)
        elif t is not None and np.isnan(t):
            assert np.isnan(k), name
        elif t is not None:
            assert k == np.inf, (name, k)
        elif row["cls"] in ("dep_times3",) or (row["cls"] == "scale" and row["dep"]):
            assert k > 1e12, (name, k)
        elif row["cls"] in ("scale", "mixed", "nearconst", "overflow", "smalln"):
            assert k < 10.0, (name, k)


def test_host_restatement_takes_every_reference_decision():
    names, decision, _, xs = _fixture()
    got = np.array([_host(x) for x in xs])
    bad = [n for n, g, d in zip(names, got, decision) if g != d]
    assert not bad, bad


def test_constant_columns_take_both_outcomes():
    """Whether numpy's mean of a constant column is the constant decides the reference's zero-span test: the
    fixture holds both outcomes for 0.3, 1.1 and 7.7 and only False for 0 and 1.5."""
    names, decision, _, _ = _fixture()
    out = {}
    for n, d in zip(names, decision):
        if TABLE[n]["cls"] == "const":
            out.setdefault(TABLE[n]["value"], set()).add(int(d))
    assert out == {0.3: {0, 1}, 1.1: {0, 1}, 7.7: {0, 1}, 1.5: {0}, 0.0: {0}}


@pytest.mark.skipif(not PX.longdouble_ok(), reason="np.longdouble is not wider than double here")
def test_gram_bound_holds_for_an_emulation_and_catches_a_planted_error():
    """The bound against the device's arithmetic done in double (shift, y = fl(x - m), sums in row order,
    sqrt(M_jj) sqrt(M_kk)); and a Gram matrix normalised by sqrt(M_jj M_kk) taken from sums one relative 1e-13
    off fails it."""
    rng = np.random.default_rng(3)
    N, D = 300, 9
    X = 3.0 + rng.standard_normal((N, D)) @ rng.standard_normal((D, D))
    m = PX.colmean_device_order(X)
    Y = X - m
    M = np.zeros((D, D))
    for r in range(N):
        M += np.outer(Y[r], Y[r])
    rt = np.sqrt(np.diag(M))
    G = M / np.outer(rt, rt)
    i, j = GX.pairs(D, rng)
    ref, bound = GX.gram_reference(X, m, i, j, N)
    err = np.abs(G[i, j].astype(np.longdouble) - ref).astype(np.float64)
    assert np.max(err / bound) < 1.0
    bad = G * (1.0 + 1e-13 * (np.arange(D)[:, None] != np.arange(D)[None, :]))
    err = np.abs(bad[i, j].astype(np.longdouble) - ref).astype(np.float64)
    assert np.max(err / bound) > 1.0


def _rows(prefix):
    names, decision, _, xs = _fixture()
    return [(n, d, x) for n, d, x in zip(names, decision, xs) if n.startswith(prefix)]


def test_former_decision_fails_where_the_gpu_test_aims():
    """The engine's decision before the range check, emulated in double, on the stored rows: (1) the 1e-200
    ensemble is refused, (2) the 1e160 ensemble raises LinAlgError, (3) some dependent row of the 1e-80 band is
    accepted, (4) constant-column rows are decided against the reference in both directions.  The new decision
    puts a scaled copy of the host-centred coordinates on the device; its emulation agrees on every row."""
    ((_, d, x),) = _rows("scale1e-200-N64-ind")
    assert d == 1 and GX.parent_decision(x, walkers_independent) is False
    ((_, d, x),) = _rows("scale1e+160-N64-ind")
    assert d == 1
    with pytest.raises(np.linalg.LinAlgError):
        GX.parent_decision(x, walkers_independent)
    band = [(n, d, x) for n, d, x in _rows("scale")
            if TABLE[n]["cls"] == "scale" and TABLE[n]["dep"] and 3e-85 < TABLE[n]["scale"] < 3e-76]
    assert len(band) == 51 and all(d == 0 for _, d, _ in band)
    accepted = [n for n, _, x in band if GX.parent_decision(x, walkers_independent)]
    assert accepted, "no false acceptance in the 1e-80 band"
    wrong = {(int(d), GX.parent_decision(x, walkers_independent)) for n, d, x in _rows("const")
             if TABLE[n]["value"] in (0.3, 1.1, 7.7)}
    assert (1, False) in wrong and (0, True) in wrong, wrong
    names, decision, _, xs = _fixture()
    got = [_new_decision(x) for x in xs]
    bad = [n for n, g, d in zip(names, got, decision) if g != d]
    assert not bad, bad


def _new_decision(x):
    """``EnsembleSampler._walkers_independent`` itself, with ``device_gram`` in place of the engine."""
    from types import SimpleNamespace

    from emcee_b200.ensemble import EnsembleSampler

    fake = SimpleNamespace(ndim=x.shape[1], _engine=SimpleNamespace(walkers_gram=GX.device_gram))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return int(bool(EnsembleSampler._walkers_independent(fake, x)))
        except np.linalg.LinAlgError:
            return W.RAISES


def test_decision_path_on_the_constant_column_sweep():
    """The whole constant-column sweep (N = 16 ... 400), decided by ``_walkers_independent`` over the emulated
    device Gram matrix, against the host restatement."""
    bad = []
    for row in W.rows():
        if row["cls"] == "const":
            x = W.build(row)
            if _new_decision(x) != _host(x):
                bad.append(row["name"])
    assert not bad, bad
