"""The per-ensemble summaries of a stored device chain (``eb_chain_select_segments``, ``eb_chain_moments_segments``,
``eb_chain_autocorr_segments``, ``eb_chain_histogram{,2d}_segments``, ``eb_chain_read_segments_to``) on the paths
that large ensembles and large batches take, against plain references of each ensemble's own slice.

Chains are crafted and uploaded with ``DeviceBackend.reset / grow / save_step`` (walkers ``[k N, (k + 1) N)`` are
ensemble / segment ``k``), and read through ``backend._ch`` with ``nseg`` and through a ``BatchSampler`` built over
the same backend.  Each row asserts the path it is there for:

=====================  =====================================================  =======================================
row                    shape (segments x walkers x D, stored steps)           path, and how the row shows it
=====================  =====================================================  =======================================
select many values     {2, 3, 7} x 64 x {1, 5, 33}, 80 (5 120 per column)     more than SEL_CAP = 4 096 values: a
                                                                              histogram pass first, ``passes >= 2``;
                                                                              D = 5 puts several segments in one
                                                                              32-column task, D = 33 splits one
select 48 shared bits  3 x 64 x 2, 80; one segment column shares its top      ``passes == 8``; the same chain without
                       48 bits                                                that column takes at most 4
select specials        3 x 64 x 3, 80; constant, +-0, +-inf, subnormals in    the constant column resolves all 64
                       segment 0                                              bits: ``passes == 8``
select > SEL_HMAX      2 x 2 048 x 1, 512; log-uniform 1e-300 .. 1e300 in     the host plan (select_host.cpp) gives
                       segment 1, 1 001 ranks                                 that column several CTA tasks
candidate budget       8 192 x 32 x 5, 100 (1 GB)                             every column fits SEL_CAP but a batch's
                                                                              5 461 x 3 200 keys exceed 2^23:
                                                                              ``passes`` > the pair batches
pair-batch NaN         the 8 192 chain, NaN in column 5 461 (ranks 1, 2 in    every ``out`` entry of a flagged column
                       batch 2), in the percentile plan's straddling column   is NaN, ``out`` pre-filled with a
                       and wholly inside batch 4; nseg = 1 at D = 7 with      sentinel; ``get_percentile`` equals
                       3 000 ranks, NaN in columns 5 and 6                    ``np.percentile``
moments chunks         8 192 x 32 x 5, 100                                    3 chunks of 34 / 34 / 32 steps
moments cs = 4         2 x 256 x 64, 200                                      50 chunks of 4 steps
moments ndim 1 024     2 x 16 x 1 024, 4                                      one chunk
moments one walker     64 x 1 x 3, 60; far: 3 x 32 x 4, 300, one segment      (chunk counts by ``_seg_chunks``, a
                       1e4 sigma out and drifting; outlier: 4 x 32 x 3, 50    restatement of ``moments_seg_chunks``)
autocorr slabs         512 x 32 x 5, n_t = 1 000                              slabs of 5 248 x 3 + 640 walkers; the
                                                                              unrounded slab (5 267) is not a
                                                                              multiple of 32
autocorr split         3 x 32 768 x 128, n_t = 8                              each segment in slabs of 26 214 + 6 554
histograms             {2, 3, 7} x 4 096 x 3, 200; values on edges, outside   many CTA rows per segment column
=====================  =====================================================  =======================================

Selection is compared with ``==`` against ``np.sort`` of each segment's flat slice (and ``has_nan``),
``get_percentile`` with ``==`` against ``np.percentile``.  Moments meet the long-double bound of
``proposals_exact.segment_moments_ratios`` with depth ``cs * N + nchunks`` and repeat bit for bit.  Autocorrelation
rows use exact integer series (``acf_exact``): each checked segment meets ``walker_mean_bound`` and equals, with
``==``, the function of that segment stored alone; ``BatchSampler.get_autocorr_time`` agrees with the host route
within ``rtol = 1e-8``.  Histograms of a ``DeviceBackend`` batch equal those of a host-``Backend`` batch.  The last
test stores a large ``BatchSampler`` run (2 x 2 048 x 4) and runs every summary on it against the host batch.
"""
import ctypes as C

import numpy as np
import pytest

import acf_exact as X
import proposals_exact as PX
from test_batch_device_backend_host import acf_probe, sel_probe  # noqa: F401 -- fixtures
from test_gpu_batch import MODELS, MOVES, _p0, _seeds
from test_gpu_batch_histogram import _assert_same
from test_gpu_chain_summary import SPECIAL

import emcee_b200
from emcee_b200 import Backend, DeviceBackend, State, _lib, models
from emcee_b200.summary import percentile_ranks

pytestmark = pytest.mark.gpu

SELECT_PAIR_BATCH = 16384  # engine.cuh
SELECT_CAND_MAX = 1 << 23
QS = [[16, 50, 84], 0, 100, 50, [[5, 50], [95, 99.5]], np.linspace(0, 100, 21)]


def _upload(x, lp, host=True, split=None):
    """x[steps, W, D], lp[steps, W] into a DeviceBackend (and a host Backend) through save_step; with ``split``
    both grow in two calls, so the device chain holds two storage blocks."""
    steps, W, D = x.shape
    cuts = [0, split, steps] if split else [0, steps]
    out = []
    for cls in (DeviceBackend, Backend) if host else (DeviceBackend,):
        b = cls()
        b.reset(W, D)
        for a, c in zip(cuts[:-1], cuts[1:]):
            b.grow(c - a, None)
            for s in range(a, c):
                b.save_step(State(x[s], log_prob=lp[s], random_state=None), np.zeros(W, dtype=bool))
        out.append(b)
    return out if host else out[0]


def _flat(x, K):
    """[steps, K N, ...] -> each segment's flat slice [K, steps N, ...]"""
    steps, W = x.shape[:2]
    return np.swapaxes(x.reshape((steps, K, W // K) + x.shape[2:]), 0, 1).reshape((K, steps * (W // K)) + x.shape[2:])


def _batch(b, K, N, D):
    return emcee_b200.BatchSampler(K, N, D, models.GaussianIso(), seeds=1, backend=b)


def _check_select(ch, flat, ranks, name="chain"):
    """select of every segment against np.sort of its flat slice (``flat[K, n, D]``); returns passes"""
    K, n = flat.shape[:2]
    ranks = np.asarray(ranks, dtype=np.uint64)
    v, has_nan, passes = ch.select(name, 0, 1, n // (ch.nwalkers // K), ranks, nseg=K)
    D = flat.shape[2] if flat.ndim == 3 else 1
    v, has_nan = v.reshape(K, ranks.size, D), has_nan.reshape(K, D)
    f = flat.reshape(K, n, D)
    want_nan = np.isnan(f).any(axis=1)
    assert np.array_equal(has_nan, want_nan)
    want = np.sort(f, axis=1)[:, ranks.astype(np.intp)] + 0.0  # -0.0 selects as +0.0
    want = np.where(want_nan[:, None, :], np.nan, want)
    assert np.array_equal(v, want, equal_nan=True)
    return passes


def _check_percentiles(s, flat, name="chain", qs=QS):
    for q in qs:
        want = np.array([np.percentile(flat[k], q, axis=0) for k in range(flat.shape[0])])
        got = s.get_percentile(q, name=name)
        assert got.shape == want.shape and np.array_equal(got, want, equal_nan=True)


# ---- selection ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 5, 33])
@pytest.mark.parametrize("K", [2, 3, 7])
def test_select_many_values(K, D):
    N, steps = 64, 80
    n = steps * N
    rng = np.random.default_rng(100 * K + D)
    x = rng.standard_normal((steps, K * N, D)) * rng.uniform(0.1, 10.0, D) + rng.normal(0, 3, D)
    x[..., 0] = np.round(x[..., 0], 1)  # ties
    lp = rng.standard_normal((steps, K * N)) * 10
    dev, host = _upload(x, lp)
    ranks = [0, 1, 2559, 2560, n - 2, n - 1]
    assert _check_select(dev._ch, _flat(x, K), ranks) >= 2
    assert _check_select(dev._ch, _flat(lp, K), ranks, name="log_prob") >= 2  # one column per segment
    s = _batch(dev, K, N, D)
    _check_percentiles(s, _flat(x, K))
    _check_percentiles(s, _flat(lp, K), name="log_prob")
    _check_percentiles(_batch(host, K, N, D), _flat(x, K), qs=QS[:1])


def test_select_segments_finish_at_different_passes():
    K, N, steps, D = 3, 64, 80, 2
    rng = np.random.default_rng(7)
    x = rng.standard_normal((steps, K * N, D))
    lp = rng.standard_normal((steps, K * N))
    ranks = [0, 77, 2560, 5119]
    plain = _upload(x, lp, host=False)
    assert _check_select(plain._ch, _flat(x, K), ranks) <= 4
    base = np.float64(-1.2345).view(np.uint64) & ~np.uint64(0xFFFF)
    x[:, N:2 * N, 1] = (base | rng.integers(0, 1 << 16, (steps, N)).astype(np.uint64)).view(np.float64)
    dev = _upload(x, lp, host=False)
    assert _check_select(dev._ch, _flat(x, K), ranks) == 8
    _check_percentiles(_batch(dev, K, N, D), _flat(x, K))


def test_select_special_values_in_one_segment():
    K, N, steps, D = 3, 64, 80, 3
    rng = np.random.default_rng(8)
    x = rng.standard_normal((steps, K * N, D))
    x[:, :N, 0] = 2.0
    x[:, :N, 1] = rng.choice(SPECIAL, (steps, N))
    x[:, :N, 2] = rng.standard_normal((steps, N)) * 1e-310
    lp = rng.standard_normal((steps, K * N))
    lp[0, :N:5] = -np.inf
    dev = _upload(x, lp, host=False)
    assert _check_select(dev._ch, _flat(x, K), [0, 1, 2559, 2560, 5118, 5119]) == 8
    _check_select(dev._ch, _flat(lp, K), [0, 1, 5119], name="log_prob")
    s = _batch(dev, K, N, D)
    _check_percentiles(s, _flat(x, K))
    _check_percentiles(s, _flat(lp, K), name="log_prob")


def test_select_column_split_over_tasks(sel_probe):
    """A column with more live histogram groups than SEL_HMAX = 40: about 125 first-digit groups of more than
    SEL_CAP values each (1e6 log-uniform values), each holding ranks.  The host run of the same plan shows the column
    split over several one-column tasks, and gives the same values and passes."""
    K, N, steps, D = 2, 2048, 512, 1
    n = steps * N
    rng = np.random.default_rng(9)
    x = rng.standard_normal((steps, K * N, D))
    x[:, N:, 0] = 10.0 ** rng.uniform(-300, 300, (steps, N))
    lp = np.zeros((steps, K * N))
    dev = _upload(x, lp, host=False)
    ranks = np.unique(np.linspace(0, n - 1, 1001).astype(np.uint64))
    assert ranks.size == 1001
    passes = _check_select(dev._ch, _flat(x, K), ranks)
    out = np.empty((K, ranks.size, D))
    has_nan = np.zeros((K, D), dtype=np.uint8)
    xs = np.ascontiguousarray(x.reshape(steps, K, N, D))
    budget = min(min(K * D * ranks.size, SELECT_PAIR_BATCH) * 4096, SELECT_CAND_MAX)
    host_passes = sel_probe.probe_select_segments(
        xs.ctypes.data_as(C.POINTER(C.c_double)), steps, K, N, D, ranks.ctypes.data_as(C.POINTER(C.c_uint64)),
        ranks.size, budget, out.ctypes.data_as(C.POINTER(C.c_double)), has_nan.ctypes.data_as(C.POINTER(C.c_uint8)))
    assert host_passes == passes
    assert sel_probe.probe_select_max_column_tasks() > 1
    v, _, _ = dev._ch.select("chain", 0, 1, steps, ranks, nseg=K)
    assert np.array_equal(v, out)
    _check_percentiles(_batch(dev, K, N, D), _flat(x, K), qs=[np.linspace(0, 100, 501)])


# ---- 8 192 ensembles of 32 x 5 over 100 stored steps --------------------------------------------------------------
BK, BN, BD, BSTEPS = 8192, 32, 5, 100


@pytest.fixture(scope="module")
def big():
    rng = np.random.default_rng(10)
    x = rng.standard_normal((BSTEPS, BK * BN, BD))
    x += rng.normal(0, 2, (BK * BN, BD))[None]  # every walker and ensemble its own centre
    lp = rng.standard_normal((BSTEPS, BK * BN))
    b = _upload(x, lp, host=False)
    srt = _flat(x, BK)
    srt.sort(axis=1)
    yield x, lp, b, srt
    b.close()


def _select_into(ch, count, ranks, nseg, D, fill):
    """eb_chain_select_segments into ``out`` pre-filled with ``fill``: an entry the call leaves unwritten shows"""
    ranks = np.ascontiguousarray(ranks, dtype=np.uint64)
    out = np.full((nseg, ranks.size, D), fill)
    has_nan = np.zeros((nseg, D), dtype=np.uint8)
    passes = C.c_uint32()
    rc = _lib.lib().eb_chain_select_segments(
        ch._h, nseg, _lib.EB_CHAIN_COORDS, 0, 1, count, ranks.ctypes.data_as(C.POINTER(C.c_uint64)), ranks.size,
        out.ctypes.data_as(C.POINTER(C.c_double)), has_nan.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(passes))
    assert rc == _lib.EB_OK
    return out, has_nan.astype(bool), passes.value


def test_candidate_budget_overflow(big):
    x, lp, b, srt = big
    ranks = np.array([0, 1600, 3199], dtype=np.uint64)
    v, has_nan, passes = b._ch.select("chain", 0, 1, BSTEPS, ranks, nseg=BK)
    batches = -(-BK * BD * ranks.size // SELECT_PAIR_BATCH)
    # a batch holds 5 461 columns of 3 200 values, 17.5e6 keys > 2^23: part of it is refined by histogram first
    assert (SELECT_PAIR_BATCH // ranks.size) * BSTEPS * BN > SELECT_CAND_MAX
    assert passes > batches, (passes, batches)
    assert not has_nan.any() and np.array_equal(v, srt[:, ranks.astype(np.intp)])


def test_pair_batch_nan(big):
    """(column, rank) pairs are planned in batches of 16 384.  Column 5 461 (ensemble 1 092, parameter 1) has its
    rank 0 in the first batch and ranks 1, 2 in the second; column c_q is the one the percentile plan's ranks split
    the same way; column 20 003 (ensemble 4 000, parameter 3) lies wholly inside the fourth batch.  Each holds one
    NaN; every entry of a flagged column is NaN, whatever ``out`` held before."""
    x, lp, b, srt = big
    q = [16, 50, 84]
    plan = percentile_ranks(q, BSTEPS * BN)
    r = plan.ranks.size
    assert SELECT_PAIR_BATCH % 3 and SELECT_PAIR_BATCH % r
    cols = [SELECT_PAIR_BATCH // 3, SELECT_PAIR_BATCH // r, 20003]
    assert (cols[2] * 3) // SELECT_PAIR_BATCH == ((cols[2] + 1) * 3 - 1) // SELECT_PAIR_BATCH == 3
    slots = [37, 81, 5]
    for (col, s) in zip(cols, slots):
        k, d = divmod(col, BD)
        xs = x[s].copy()
        xs[k * BN + 7, d] = np.nan
        b._ch.write(s, xs, lp[s])
    try:
        nan = np.zeros((BK, BD), dtype=bool)
        for col in cols:
            nan[col // BD, col % BD] = True
        for ranks in (np.array([511, 1600, 2688], dtype=np.uint64), plan.ranks):
            out, has_nan, _ = _select_into(b._ch, BSTEPS, ranks, BK, BD, -7.25)
            assert np.array_equal(has_nan, nan)
            assert np.all(np.isnan(out[np.broadcast_to(nan[:, None, :], out.shape)]))
            ok = ~np.broadcast_to(nan[:, None, :], out.shape)
            assert np.array_equal(out[ok], srt[:, ranks.astype(np.intp)][ok])
        got = _batch(b, BK, BN, BD).get_percentile(q)
        flat = srt.copy()
        flat[nan.nonzero()[0], 0, nan.nonzero()[1]] = np.nan
        want = np.array([np.percentile(flat[k], q, axis=0) for k in range(BK)])
        assert np.array_equal(got, want, equal_nan=True)
    finally:
        for s in slots:
            b._ch.write(s, x[s], lp[s])


def test_pair_batch_nan_one_segment():
    """nseg = 1, ndim 7, 3 000 ranks: column 5's pairs 15 000 .. 17 999 straddle the first batch boundary, column 6's
    lie wholly inside the second batch."""
    N, steps, D = 64, 100, 7
    rng = np.random.default_rng(11)
    x = rng.standard_normal((steps, N, D))
    x[40, 3, 5] = np.nan
    x[90, 60, 6] = np.nan
    lp = rng.standard_normal((steps, N))
    dev, host = _upload(x, lp)
    ranks = np.arange(0, 6000, 2, dtype=np.uint64)
    out, has_nan, _ = _select_into(dev._ch, steps, ranks, 1, D, 123.5)
    assert has_nan[0].tolist() == [False] * 5 + [True, True]
    assert np.all(np.isnan(out[0, :, 5:]))
    assert np.array_equal(out[0, :, :5], np.sort(x.reshape(-1, D), axis=0)[ranks.astype(np.intp), :5])
    for q in (np.linspace(0, 100, 1500), [16, 50, 84]):
        want = np.percentile(x.reshape(-1, D), q, axis=0)
        assert np.array_equal(dev.get_percentile(q), want, equal_nan=True)
        assert np.array_equal(host.get_percentile(q), want, equal_nan=True)


# ---- moments ------------------------------------------------------------------------------------------------------
def _seg_chunks(count, nseg, D):
    """moments_seg_chunks (analysis.cu), restated: the chunks of stored steps eb_chain_moments_segments sums apart,
    as their lengths"""
    per = nseg * (D + D * D)
    c = -(-(1 << 19) // per)
    c = min(c, 65535, (1 << 25) // per)
    nchunks = max(1, min(c, count))
    cs = -(-count // nchunks)
    ny = -(-count // cs)
    return [cs] * (ny - 1) + [count - cs * (ny - 1)]


def _check_moments(moments, x, K, segs=None):
    """``moments()`` (mean[K, D], cov[K, D, D], n) of x[steps, K N, D]: the segments ``segs`` (all by default)
    under the long-double bound; a repeat call is bit-identical"""
    if not PX.longdouble_ok():
        pytest.skip("np.longdouble is not wider than double here")
    steps, W, D = x.shape
    N = W // K
    mean_d, cov_d, m = moments()
    assert m == steps * N
    again = moments()
    assert np.array_equal(again[0], mean_d) and np.array_equal(again[1], cov_d)
    chunks = _seg_chunks(steps, K, D)
    depth = chunks[0] * N + len(chunks)
    worst = [0.0, 0.0]
    for k in range(K) if segs is None else segs:
        Xk = x[:, k * N:(k + 1) * N].reshape(-1, D)
        shift = np.cumsum(x[0, k * N:(k + 1) * N], axis=0)[-1] / N  # walkers ascending, as the device adds them
        rm, rc = PX.segment_moments_ratios(Xk, shift, mean_d[k], cov_d[k], depth)
        worst = [max(worst[0], rm), max(worst[1], rc)]
    print("moments %d x %d x %d, %d steps, chunks %s: largest error / bound mean %.3g, cov %.3g"
          % (K, N, D, steps, chunks[:3], worst[0], worst[1]))
    assert worst[0] <= 1.0 and worst[1] <= 1.0
    return chunks, mean_d, cov_d


def test_moments_8192_three_chunks(big):
    x, lp, b, srt = big
    chunks, mean_d, cov_d = _check_moments(_batch(b, BK, BN, BD).get_moments, x, BK,
                                           segs=[0, 1, 1092, 4000, BK - 1] + list(range(17, BK, 331)))
    assert chunks == [34, 34, 32]
    # every segment within 1e-10 of numpy's, measured against its spread where an entry is near zero
    flat = _flat(x, BK)
    mean = flat.mean(axis=1)
    flat -= mean[:, None, :]
    cov = np.einsum("kmi,kmj->kij", flat, flat) / (flat.shape[1] - 1)
    scale = np.sqrt(np.einsum("kii->ki", cov))
    assert np.all(np.abs(mean_d - mean) <= 1e-10 * (np.abs(mean) + scale))
    assert np.all(np.abs(cov_d - cov) <= 1e-10 * (np.abs(cov) + scale[:, :, None] * scale[:, None, :]))


def _moments_rows():
    rng = np.random.default_rng(12)
    far = rng.standard_normal((300, 3 * 32, 4))
    far[:, 32:64] += 1.0e4 + np.cumsum(rng.normal(0, 0.3, (300, 1, 4)), axis=0)  # 1e4 sigma out, drifting
    out = rng.standard_normal((50, 4 * 32, 3))
    out[:, 64] += 1.0e3  # segment 2's first walker: the shift is that segment's first stored step
    return {"cs4": (2, lambda: rng.standard_normal((200, 2 * 256, 64)) * 2.0 + 0.5, [4] * 50),
            "ndim1024": (2, lambda: rng.standard_normal((4, 2 * 16, 1024)), [4]),
            "one-walker": (64, lambda: rng.standard_normal((60, 64, 3)) + 5.0, [1] * 60),
            "far-drift": (3, lambda: far, [1] * 300),
            "outlier": (4, lambda: out, [1] * 50)}


MOMENT_ROWS = _moments_rows()


@pytest.mark.parametrize("row", list(MOMENT_ROWS))
def test_moments_rows(row):
    K, make, want_chunks = MOMENT_ROWS[row]
    x = make()
    steps, W, D = x.shape
    dev = _upload(x, np.zeros((steps, W)), host=False)
    chunks, mean_d, cov_d = _check_moments(lambda: dev._ch.moments(0, 1, steps, nseg=K), x, K)
    assert chunks == want_chunks
    if W // K > 1:  # a batch needs two walkers per ensemble
        m, c, _ = _batch(dev, K, W // K, D).get_moments()
        assert np.array_equal(m, mean_d) and np.array_equal(c, cov_d)
    dev.close()


def test_moments_segments_refuse_ndim_1025():
    b = DeviceBackend()
    b.reset(4, 1025)
    b.grow(1, None)
    b.save_step(State(np.ones((4, 1025)), log_prob=np.zeros(4)), np.zeros(4, dtype=bool))
    with pytest.raises(NotImplementedError, match="ndim <= 1024"):
        b._ch.moments(0, 1, 1, nseg=2)
    b.close()


# ---- autocorrelation ------------------------------------------------------------------------------------------------
def _alone(xk):
    """the autocorrelation function of one segment x[n_t, N, D] stored alone in its own chain"""
    n_t, N, D = xk.shape
    ch = _lib.Chain(N, D)
    try:
        ch.grow(n_t)
        for t in range(n_t):
            ch.write(t, xk[t], np.zeros(N))
        return ch.autocorr_function(0, 1, n_t)
    finally:
        ch.close()


def _check_acf_segment(f, xk, rng):
    """f[n_t, D] of one segment against the exact lag sums, and == the segment stored alone; error / bound"""
    n_t, N, D = xk.shape
    assert np.array_equal(f, _alone(xk), equal_nan=True)
    lags = X.lag_set(n_t, rng)
    ref, r, _ = X.exact_acf(xk, lags)
    M = X.fft_length(n_t)
    norm = X.acf_norm((xk - xk.mean(axis=0)).reshape(n_t, N * D), M).reshape(N, D)
    bound = X.walker_mean_bound(X.series_bound(M, norm), r)
    got = f[lags]
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)
    ratio = float(np.max(np.abs(got - ref)[~nan] / bound[~nan]))
    assert ratio < 1.0
    return ratio


@pytest.fixture(scope="module")
def slab_chain():
    """512 ensembles of 32 x 5 integer series, n_t = 1 000, in a DeviceBackend grown in two blocks (600 + 400
    steps) and in a host Backend"""
    K, N, D, n_t = 512, 32, 5, 1000
    rng = np.random.default_rng(13)
    x = X.int_series(rng, n_t, K * N, D)
    dev, host = _upload(x, np.zeros((n_t, K * N)), split=600)
    yield x, dev, host, (K, N, D, n_t)
    dev.close()


def test_autocorr_multi_slab(slab_chain, acf_probe):
    x, dev, host, (K, N, D, n_t) = slab_chain
    w0, wn, _ = acf_probe(n_t, K * N, D, K)
    assert wn.tolist() == [5248, 5248, 5248, 640]
    raw = int(acf_probe(n_t, K * N, D, 1)[1][0])  # acf_slab_walkers(n_t, nw, nd): not a multiple of a segment
    assert raw == 5267 and raw % N
    f = dev._ch.autocorr_function(0, 1, n_t, nseg=K)
    assert f.shape == (K, n_t, D)
    # the first and last segment of every slab, the segments an unrounded slab would split, and a few others
    segs = sorted({int(w) // N for w in w0} | {int(a + b - 1) // N for a, b in zip(w0, wn)}
                  | {j * raw // N for j in (1, 2, 3)} | {3, 200, 400})
    rng = np.random.default_rng(14)
    worst = max(_check_acf_segment(f[k], x[:, k * N:(k + 1) * N], rng) for k in segs)
    print("autocorr multi-slab, %d segments checked: largest error / bound %.3g" % (len(segs), worst))
    tau_d = _batch(dev, K, N, D).get_autocorr_time(tol=0)
    tau_h = _batch(host, K, N, D).get_autocorr_time(tol=0)
    np.testing.assert_allclose(tau_d, tau_h, rtol=1e-8)


def test_read_segments_across_blocks(slab_chain):
    x, dev, host, (K, N, D, n_t) = slab_chain
    sd, sh = _batch(dev, K, N, D), _batch(host, K, N, D)
    for discard, thin in ((0, 1), (550, 7), (599, 2), (999, 1)):
        for name in ("chain", "log_prob"):
            want = sh.get_value(name, flat=True, discard=discard, thin=thin)
            got = sd.get_value(name, flat=True, discard=discard, thin=thin, cuda=True)
            assert got.shape == want.shape and np.array_equal(got.get(), want)


def test_autocorr_segments_split_across_slabs(acf_probe):
    K, N, D, n_t = 3, 32768, 128, 8
    w0, wn, _ = acf_probe(n_t, K * N, D, K)
    assert wn.tolist() == [26214, 6554] * K
    rng = np.random.default_rng(15)
    x = X.int_series(rng, n_t, K * N, D)
    dev = _upload(x, np.zeros((n_t, K * N)), host=False)
    f = dev._ch.autocorr_function(0, 1, n_t, nseg=K)
    dev.close()
    worst = max(_check_acf_segment(f[k], x[:, k * N:(k + 1) * N], rng) for k in range(K))
    print("autocorr split segments: largest error / bound %.3g" % worst)


# ---- histograms -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 3, 7])
def test_histograms_many_rows_per_segment(K):
    N, steps, D = 4096, 200, 3
    rng = np.random.default_rng(16 + K)
    edges = np.linspace(-1.0, 1.0, 21)  # numpy's edges of range (-1, 1) at 20 bins
    x = np.empty((steps, K * N, D))
    x[..., 0] = rng.choice(np.r_[edges, np.linspace(-1.0, 1.0, 4097), -1.5, 1.5, 3.0], (steps, K * N))  # outside too
    x[..., 1] = rng.standard_normal((steps, K * N))
    x[..., 2] = rng.integers(-3, 4, (steps, K * N)) * 0.25  # ties on the autodetected edges
    lp = rng.standard_normal((steps, K * N))
    dev, host = (_batch(b, K, N, D) for b in _upload(x, lp))
    shared = [(-1.0, 1.0)] * D
    per = np.moveaxis(host.get_percentile([1, 99]), 1, 2).copy()
    for rng_ in (None, shared, per):
        for bins in (20, 4096):
            kw = dict(bins=bins, range=rng_)
            _assert_same(lambda: dev.get_histogram(**kw), lambda: host.get_histogram(**kw))
    _assert_same(lambda: dev.get_histogram(bins=20, name="log_prob"),
                 lambda: host.get_histogram(bins=20, name="log_prob"))
    for rng_ in (None, shared):
        kw = dict(bins=128, range=rng_)
        _assert_same(lambda: dev.get_histogram2d(**kw), lambda: host.get_histogram2d(**kw))


# ---- a large batch run stored on the device -------------------------------------------------------------------------
def test_large_batch_run_summaries():
    """2 ensembles of 2 048 x 4 (test_gpu_batch.LARGE_CASES: the split table's second chunk) stored into a
    DeviceBackend and a host Backend: every summary of the device batch against the host batch."""
    K, N, D, steps = 2, 2048, 4, 60
    out = []
    for backend in (DeviceBackend(), None):
        s = emcee_b200.BatchSampler(K, N, D, MODELS["ring"](D), moves=MOVES["de"](3, True), seeds=_seeds(K, 21),
                                    backend=backend)
        s.run_mcmc(_p0(K, N, D, 21), steps, skip_initial_state_check=True)
        out.append(s)
    dev, host = out
    assert np.array_equal(dev.get_chain(), host.get_chain())
    x = dev.get_chain().reshape(steps, K * N, D)
    assert _check_select(dev.backend._ch, _flat(x, K), [0, 1, 61439, 61440, steps * N - 1]) >= 2
    _check_percentiles(dev, _flat(x, K))
    _check_percentiles(dev, dev.get_log_prob(flat=True), name="log_prob", qs=QS[:2])
    _check_moments(dev.get_moments, x, K)
    np.testing.assert_allclose(dev.get_autocorr_time(tol=0), host.get_autocorr_time(tol=0), rtol=1e-8)
    f = dev.backend._ch.autocorr_function(0, 1, steps, nseg=K)
    for k in range(K):
        assert np.array_equal(f[k], _alone(x[:, k * N:(k + 1) * N]), equal_nan=True)
    for kw in (dict(bins=20), dict(bins=4096, discard=10, thin=3), dict(bins=20, name="log_prob")):
        _assert_same(lambda: dev.get_histogram(**kw), lambda: host.get_histogram(**kw))
    _assert_same(lambda: dev.get_histogram2d(bins=128), lambda: host.get_histogram2d(bins=128))
    got = dev.get_value("chain", flat=True, discard=5, thin=4, cuda=True)
    assert np.array_equal(got.get(), host.get_value("chain", flat=True, discard=5, thin=4))
