"""The reference machinery of ``test_gpu_proposals_exact.py`` checked on the CPU: high-precision normals and the
thresholded Cholesky factor against the numpy oracle, exact covariances against ``np.cov``, and that each bound
rejects a deliberately wrong proposal (a factor off by 1e-10, ``ddof = 0``, a dropped rank cap)."""
import numpy as np
import pytest

import proposals_exact as PX
from oracle import philox as px

U = PX.U

needs_ld = pytest.mark.skipif(not PX.longdouble_ok(), reason="np.longdouble is not wider than double here")


def test_normals_match_the_oracle_to_a_few_ulps():
    for seed, step, split, count in ((1, 0, 0, 7), (0xB200, 99, 1, 64), (5, 2 ** 40, 31, 3)):
        idx = np.arange(0, 4000, 37)
        z = PX.mp_to_f64(PX.normals_mp(seed, step, split, idx, count))
        o = px.normals(seed, step, split, idx, count)
        assert np.all(np.abs(o - z) <= PX.NORMAL_ERR * np.abs(z) + 1e-300)
        assert np.max(np.abs(o - z) / np.maximum(np.abs(z), 1e-300)) > 0  # the reference is not the oracle itself


def _oracle_bound_check(A, max_rank, r):
    """chol_psd of the oracle (double) within the Cholesky bound of the high-precision factor."""
    L, Lref, piv, uref = PX.chol_reference(A, max_rank)
    Af = A.f64() if isinstance(A, PX.ExactCov) else A
    Lo = px.chol_psd(Af, max_rank=max_rank)
    PX.check_pivot_prefix(L, piv, r, float(np.max(np.diag(Af))))
    aL = np.abs(L)
    M = PX.backward_error(L) + PX.backward_error(L, uref) + (U + uref) * (aL @ aL.T)
    dL = PX.chol_perturbation(L, M, r)
    assert np.all(np.abs(Lo - L) <= dL + U * aL), np.max(np.abs(Lo - L) - dL)
    assert np.all(Lo[:, r:] == 0)
    return L


@pytest.mark.parametrize("D", [5, 24, pytest.param(40, marks=needs_ld), pytest.param(96, marks=needs_ld)])
def test_chol_psd_full_rank_and_rank_capped(D):
    rng = np.random.default_rng(D)
    X = np.round(rng.standard_normal((3 * D, D)) * 20)
    _oracle_bound_check(PX.ExactCov(X), 3 * D - 1, D)
    # n = D rows: rank D - 1, the cap stops after D - 1 pivots
    _oracle_bound_check(PX.ExactCov(X[:D]), D - 1, D - 1)
    # s = 5 helpers: rank 4
    _oracle_bound_check(PX.ExactCov(X[:5]), 4, 4)


def test_chol_psd_threshold_drops_exactly_zero_pivots():
    """A PSD matrix of rank D - 2 (last two columns in the span of the others): no cap, the threshold drops the
    two pivots that are zero in exact arithmetic."""
    D = 16
    B = np.round(np.random.default_rng(3).standard_normal((D - 2, D - 2)) * 8)
    W = np.vstack([np.eye(D - 2), np.round(np.random.default_rng(4).standard_normal((2, D - 2)) * 2)])
    Xi = (np.round(np.random.default_rng(5).standard_normal((40, D - 2)) * 4) @ B.T) @ W.T
    A = PX.ExactCov(Xi)
    L, _, piv, _ = PX.chol_reference(A, None)
    assert piv == list(range(D - 2))
    _oracle_bound_check(A, None, D - 2)


def test_exact_cov_matches_numpy():
    rng = np.random.default_rng(11)
    for X in (np.round(rng.standard_normal((50, 6)) * 100), 1e6 + np.round(rng.standard_normal((20, 3))),
              rng.standard_normal((30, 4)) * 1e-3 + 0.5):
        A = PX.ExactCov(X).f64()
        C = np.cov(X, rowvar=0)
        sc = np.sqrt(np.outer(np.diag(C), np.diag(C)))
        assert np.all(np.abs(A - C) <= 1e-9 * sc)
    # non-integer rows take the Python-integer path and agree with the integer path on integer rows
    X = np.round(rng.standard_normal((9, 3)) * 7)
    a, b = PX.ExactCov(X), PX.ExactCov(X + 0.5)
    assert a.small and not b.small
    np.testing.assert_allclose(a.f64(), b.f64(), rtol=4 * U, atol=0)


def _simulated_walk(X, shift, z, cov_scale=1.0, ddof=1, cap=True, factor_scale=1.0):
    """q = s + L z as cov_chol_kernel and walk_shared_propose compute it, in double on the CPU, with optional
    defects: ddof, no rank cap, a scaled factor."""
    n, D = X.shape
    Y = X - shift
    S1 = Y.sum(0)
    A = (Y.T @ Y - np.outer(S1, S1) / n) / (n - ddof) * cov_scale
    L = np.zeros((D, D))
    tol = 1e-12 * np.max(np.diag(A))
    left = n - 1 if cap else D
    for j in range(D):
        d = A[j, j] - np.dot(L[j, :j], L[j, :j])
        piv = np.sqrt(d) if (left > 0 and d > tol) else 0.0
        if piv > 0:
            left -= 1
            L[j, j] = piv
            L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / piv
    return (L * factor_scale) @ z


def _walk_case(X, zseed, all_X):
    n, D = X.shape
    A = PX.ExactCov(X)
    L, Lref, piv, uref = PX.chol_reference(A, n - 1)
    r = min(D, n - 1)
    z_mp = PX.normals_mp(zseed, 0, 0, [0], D)
    z = PX.mp_to_f64(z_mp)[0]
    Lz_ref = np.array([float(sum(Lref[e, k] * z_mp[0, k] for k in range(e + 1))) for e in range(D)])
    shift = PX.colmean_device_order(all_X)
    depth = PX.moments_depth(n, D, 132, 1)[0]
    Mcov = PX.cov_error_one_pass(X - shift, n, depth, A.f64())
    bound = PX.mvn_bound(L, Mcov, r, np.abs(z)[None, :], np.abs(Lz_ref)[None, :], uref)[0]
    return shift, z, Lz_ref, bound


def test_bounds_reject_wrong_proposals():
    rng = np.random.default_rng(21)
    D, n = 12, 40
    all_X = np.round(rng.standard_normal((2 * n, D)) * 16)
    X = all_X[:n]
    shift, z, Lz_ref, bound = _walk_case(X, 9, all_X)
    good = _simulated_walk(X, shift, z)
    assert np.all(np.abs(good - Lz_ref) < bound)
    assert np.any(np.abs(_simulated_walk(X, shift, z, factor_scale=1 + 1e-10) - Lz_ref) > bound)
    assert np.any(np.abs(_simulated_walk(X, shift, z, ddof=0) - Lz_ref) > bound)
    # a shift of zero for an ensemble at 1e6: the one-pass sums lose digits the bound does not allow
    Xo = X + 1.0e6
    shift_o, z, Lz_ref, bound = _walk_case(Xo, 9, all_X + 1.0e6)
    assert np.all(np.abs(_simulated_walk(Xo, shift_o, z) - Lz_ref) < bound)
    assert np.any(np.abs(_simulated_walk(Xo, 0.0, z) - Lz_ref) > bound)


def test_bound_rejects_a_dropped_rank_cap():
    """n = D rows with the shift far from them (the mean of an ensemble whose other D + 1 walkers sit 4096 away):
    the pivot the cap drops is rounding noise above the threshold, which an uncapped factorisation turns into a
    column."""
    D = 16
    caught = 0
    for seed in range(8):
        rng = np.random.default_rng(seed)
        X = PX.rankcap_rows(D, rng)
        all_X = np.vstack([X, np.round(rng.standard_normal((D + 1, D)) * 4) + 4096.0])
        shift, z, Lz_ref, bound = _walk_case(X, seed, all_X)
        assert np.all(np.abs(_simulated_walk(X, shift, z) - Lz_ref) < bound)
        caught += bool(np.any(np.abs(_simulated_walk(X, shift, z, cap=False) - Lz_ref) > bound))
    assert caught >= 3, caught
