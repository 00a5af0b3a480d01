"""CPU checks behind ``test_gpu_autocorr_exact.py``: the exact autocorrelation reference (``acf_exact.py``) against
numpy's ACF (``autocorr._acf``), so that a wrong reference cannot let the GPU test pass; and the launch geometry of
the autocorrelation kernels (``emcee_b200/csrc/acf_grid.h``, compiled for the host) against the device limits for
every FFT length and the walker slabs ``acf_slabs`` can allocate."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import acf_exact as X
from emcee_b200 import autocorr

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- exact reference -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_t,nw,nd", [(2, 3, 2), (3, 1, 1), (100, 7, 3), (257, 2, 2), (4097, 2, 1), (5000, 3, 2)])
def test_exact_reference_matches_numpy(n_t, nw, nd):
    rng = np.random.default_rng(n_t)
    x = X.int_series(rng, n_t, nw, nd)
    assert np.all(np.abs(x) <= X.AMP) and np.all(np.sum(x, axis=0) % n_t == 0)
    lags = X.lag_set(n_t, rng)
    assert len(lags) == (n_t if n_t <= 4097 else 192) and lags[0] == 0 and lags[-1] == n_t - 1
    ref, r, a0 = X.exact_acf(x, lags)
    assert np.all(a0 > 0)
    want = autocorr._acf(x)[lags]  # [L, nw, nd]
    np.testing.assert_allclose(r, want, rtol=0, atol=1e-13)
    np.testing.assert_allclose(ref, want.mean(axis=1), rtol=0, atol=1e-13)
    assert np.all(r[0] == 1.0) and np.all(ref[0] == 1.0)
    # numpy's own float64 ACF stays inside the bound the GPU test applies
    M = X.fft_length(n_t)
    d = (x - x.mean(axis=0)).reshape(n_t, -1)
    rho = X.series_bound(M, X.acf_norm(d, M)).reshape(nw, nd)
    assert np.all(np.abs(want.mean(axis=1) - ref) <= X.walker_mean_bound(rho, r))


def test_exact_reference_lag_sums_by_hand():
    x = np.array([[1.0], [4.0], [-2.0], [5.0]])  # mean 2: d = -1, 2, -4, 3
    a, d = X.lag_sums(x, [0, 1, 2, 3])
    assert d.ravel().tolist() == [-1, 2, -4, 3]
    assert a.ravel().tolist() == [30, -2 - 8 - 12, 4 + 6, -3]
    ref, r, a0 = X.exact_acf(x[:, :, None], [0, 1, 2, 3])
    assert r.ravel().tolist() == [1.0, -22 / 30, 10 / 30, -3 / 30] and a0.item() == 30


def test_exact_reference_two_samples_and_stuck_series():
    x = np.zeros((2, 3, 2))
    x[:, :, 0] = [[3, 8, -1], [5, 2, 1]]
    x[:, :, 1] = 7.0  # never moves: a_0 = 0
    ref, r, a0 = X.exact_acf(x, [0, 1])
    assert np.array_equal(ref[:, 0], [1.0, -0.5])
    assert np.all(np.isnan(ref[:, 1])) and np.all(a0[:, 1] == 0)
    with np.errstate(invalid="ignore"):
        assert np.all(np.isnan(autocorr._acf(x)[:, :, 1]))


def test_reference_detects_a_wrong_acf():
    """The comparison has teeth: numpy's ACF with the first walker's lag 0 as the normaliser fails the bound."""
    rng = np.random.default_rng(9)
    n_t, nw, nd = 300, 4, 2
    x = X.int_series(rng, n_t, nw, nd)
    lags = X.lag_set(n_t, rng)
    ref, r, a0 = X.exact_acf(x, lags)
    d = x - x.mean(axis=0)
    f = np.fft.rfft(d, n=X.fft_length(n_t), axis=0)
    acf = np.fft.irfft(f.real ** 2 + f.imag ** 2, n=X.fft_length(n_t), axis=0)[:n_t]
    wrong = (acf / acf[0, 0][None, None, :]).mean(axis=1)
    rho = X.series_bound(X.fft_length(n_t), X.acf_norm(d.reshape(n_t, -1), X.fft_length(n_t))).reshape(nw, nd)
    assert np.any(np.abs(wrong - ref) > X.walker_mean_bound(rho, r))


def test_bound_is_tight_at_long_lengths():
    """The per-lag bound of one AR(1) series at M = 2^18 stays below 1e-12 relative to a_0."""
    rng = np.random.default_rng(3)
    x = X.int_series(rng, 65537, 1, 1)
    M = X.fft_length(65537)
    assert M == 2 ** 18
    d = (x - x.mean(axis=0)).reshape(65537, 1)
    rho = X.series_bound(M, X.acf_norm(d, M))
    assert rho.max() < 1e-12


# ---- launch geometry -------------------------------------------------------------------------------------------
GRID_X_MAX = 2 ** 31 - 1
HBM = 80 << 30  # an H100's memory: a slab whose scratch exceeds it is refused by cudaMalloc before any launch
FIELDS = ["M", "wb", "bytes", "B", "threads", "local", "mean", "load_t", "load", "global", "lag_tiles", "accumulate"]


@pytest.fixture(scope="module")
def grid_probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("acfgrid") / "libacf_grid_probe.so")
    subprocess.run(
        ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", "acf_grid_host.cpp")],
        check=True,
    )
    lib = C.CDLL(out)
    lib.probe_acf_grid.restype = None
    lib.probe_acf_grid.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64)]

    def probe(n_t, nw, nd):
        v = np.zeros(len(FIELDS), dtype=np.uint64)
        lib.probe_acf_grid(n_t, nw, nd, v.ctypes.data_as(C.POINTER(C.c_uint64)))
        return dict(zip(FIELDS, (int(a) for a in v)))

    return probe


def _check_slab(g, n_t, wn, nd):
    """Every grid dimension of launch_acf_slab for a slab of wn walkers within the device limits, and covering the
    slab's work (g: the grid of a full slab, recomputed here for wn)."""
    S, M, B = wn * nd, g["M"], g["B"]
    local = S * (M // B)
    mean = (S + 127) // 128
    load = g["load_t"] * ((S + 31) // 32)
    glob = (S * (M // 2) + 255) // 256
    acc = g["lag_tiles"] * nd
    for blocks in (local, mean, load, glob, acc):
        assert 1 <= blocks <= GRID_X_MAX, (n_t, wn, nd, g)
    assert local * B == S * M and g["load_t"] * 32 >= M and g["lag_tiles"] * 256 >= n_t
    assert B * 16 <= 128 * 1024 and g["threads"] <= 1024 and (g["threads"] == 512) == (B >= 1024)


def test_launch_grids_within_device_limits(grid_probe):
    nds = [1, 2, 3, 8, 15, 64, 128, 1000, 65535, 65536, 65537, 2 ** 20, 2 ** 24]
    nws = [1, 2, 7, 4369, 8192, 60000, 65537, 2 ** 20, 2 ** 24]
    checked = 0
    for j in range(1, 28):
        M = 2 ** j
        for n_t in sorted({M // 4 + 1, M // 2} if M > 2 else {1}):
            if n_t > 2 ** 26:
                continue
            for nd in nds:
                for nw in nws + [max(1, 2 ** 31 // nd)]:
                    if nw * nd > 2 ** 31:  # acf_slabs refuses these
                        continue
                    g = grid_probe(n_t, nw, nd)
                    assert g["M"] == M and g["bytes"] == 16 * M + 8 * n_t
                    wb = g["wb"]
                    assert 1 <= wb <= nw
                    assert wb == nw or wb == 1 or wb * nd * g["bytes"] <= 1 << 30 < (wb + 1) * nd * g["bytes"]
                    if wb * nd * g["bytes"] > HBM:
                        continue
                    assert g["local"] == wb * nd * M // g["B"] and g["accumulate"] == g["lag_tiles"] * nd
                    _check_slab(g, n_t, wb, nd)
                    if nw % wb:
                        _check_slab(g, n_t, nw % wb, nd)  # the partial last slab
                    checked += 1
    assert checked > 2000


def test_launch_grids_of_the_shapes_that_needed_grid_y(grid_probe):
    """The shapes whose slabs put more than 65 535 on grid y before the grids were 1-D."""
    g = grid_probe(100, 8192, 8)  # 100 stored steps of 8 192 x 8: one slab of 65 536 series
    assert g["wb"] == 8192 and g["local"] == 65536
    g = grid_probe(4, 65536, 64)  # 4.2 M series: ceil(S / 32) > 65 535 tiles of acf_load_kernel
    assert g["wb"] == 65536 and (65536 * 64 + 31) // 32 > 65535 and g["load"] == g["load_t"] * 131072
    g = grid_probe(5, 1, 65536)  # 65 536 parameters of one walker
    assert g["accumulate"] == 65536
    g = grid_probe(100, 64000, 8)  # three slabs, each of more than 65 535 series
    assert g["wb"] == 27413 and 64000 % 27413 * 8 > 65535
