"""Every production cell of dense_dmma at multi-tile shapes, against exact arithmetic.

``launch_t<KB>`` (dense_dmma.cu) picks one of 16 factor widths (KB = D / 8) and, inside it, ``HAS_MEAN x BOUNDED``
(64 production cells) times ``TIMELINE`` (64 instrumented ones).  What differs between cells: the zero-padded last
column pair of odd KB (``col_pairs``, ``tile_sumsq``), the register rebalance (``dmma_rebalance``), the box test of
the producer, and the two-tile-deep producer -> consumer pipeline, which only runs when a consumer warp gets
several tiles.

* ``test_cell_table`` (CPU): ``STEP_ROWS`` covers all 64 cells, every rebalanced cell and every odd KB >= 7 at a
  shape where every consumer warp gets at least ``TILES`` tiles and the last tile is partial; the timeline, stand-alone
  and threshold rows cover what they promise.
* ``test_cell_multi_tile`` (``STEP_ROWS``): N from the SM count, so each consumer warp gets ``TILES`` tiles of a
  half-step and one consumer a fourth, partial one.  A random SPD precision matrix of condition 1e6 (non-symmetric
  at ``ASYM_WIDTHS``, whose symmetric part is exact in doubles), a mean at |mu| ~ 1e3 (q - mu cancels), and a box
  that about a third of the proposals leave, with bounds that are proposal coordinates (rows on a bound are inside).
  Step 1 starts at log_prob = -inf, so the state shows every proposal:
    - coordinates bit-exact against the stretch proposals of ``oracle/redblue.py``; rows outside the box keep their
      old coordinates and -inf; accept counts equal the oracle's;
    - every stored log-probability ``==`` ``compute_log_prob`` of the stored row (``tile_sumsq``'s bit-identity);
    - at least 256 rows per cell (first and last active ranks, the whole last partial tile) within
      ``bound_dense_dmma`` of ``exact_dense``.
  Step 2 starts from a finite state: per split, in order, the accept mask must be ``fl(fl(F + lp_dev) - lp_old) >
  log u`` with the draw specification's F and u and the device's own ``lp_dev = compute_log_prob(q)``.  Walkers
  whose ``lp_old`` lies within the ``accept_exact`` bound of their exact threshold are skipped and counted.
* ``test_threshold_rows`` (``THRESHOLD_ROWS``): the threshold bisection of ``test_gpu_accept_exact.py`` (its three
  (seed, step) pairs, 64 sampled walkers per split, its bound) at odd KB, rebalanced and boxed cells.
* ``test_timeline_cells`` (``TIMELINE_ROWS``): ``dmma_timeline`` 1 and 2 give coordinates, log-probabilities,
  accept masks and counts byte-identical to a twin engine without the option; ``debug_timeline`` has the documented
  shape [SM][8 consumers][8 tiles][12 events] and event 0 holds the tiles of the SM-major deal.  No timing is checked.
* ``test_standalone_cells``: ``compute_log_prob`` of every KB x mean x box on 8k +- 1 rows, rows far from the mean,
  rows whose 0.5 |L^T xc|^2 overflows (-inf, no error) and rows on / one ulp outside every 8-column block's bounds.

The largest error / bound of each cell is printed and must stay below 1.
"""
import time
from fractions import Fraction

import numpy as np
import pytest

import accept_exact as AX
import logprob_exact as LX
from oracle import philox as px
from oracle import redblue as rb

import emcee_b200
from emcee_b200 import models, moves

U = 2.0 ** -53
CONSUMERS = 8  # consumer warps per CTA (dense_dmma.cu DMMA_CONSUMERS)
TILE = 8  # walkers per tile
TILES = 3  # tiles every consumer warp gets in a half-step of STEP_ROWS
TIMELINE_TILES = 2  # ... of TIMELINE_ROWS (both in-flight records)
ASYM_WIDTHS = (24, 88, 120)
SEED = 0xCE11
STEP = 41
EXACT_ROWS = 256


def dmma_rebalance(KB, mean, box):
    """dense_dmma.cu's dmma_rebalance: the cells whose producers give registers to the consumers."""
    return not box and (KB >= 15 or (mean and KB >= 11))


CELLS = [(KB, mean, box) for KB in range(1, 17) for mean in (False, True) for box in (False, True)]

# D, mean, box, nsplits: every production cell once, one cell per width at three splits
STEP_ROWS = [
    (8, False, False, 3), (8, True, False, 2), (8, False, True, 2), (8, True, True, 2),
    (16, False, False, 2), (16, True, False, 3), (16, False, True, 2), (16, True, True, 2),
    (24, False, False, 2), (24, True, False, 2), (24, False, True, 3), (24, True, True, 2),
    (32, False, False, 2), (32, True, False, 2), (32, False, True, 2), (32, True, True, 3),
    (40, False, False, 3), (40, True, False, 2), (40, False, True, 2), (40, True, True, 2),
    (48, False, False, 2), (48, True, False, 3), (48, False, True, 2), (48, True, True, 2),
    (56, False, False, 2), (56, True, False, 2), (56, False, True, 3), (56, True, True, 2),
    (64, False, False, 2), (64, True, False, 2), (64, False, True, 2), (64, True, True, 3),
    (72, False, False, 3), (72, True, False, 2), (72, False, True, 2), (72, True, True, 2),
    (80, False, False, 2), (80, True, False, 3), (80, False, True, 2), (80, True, True, 2),
    (88, False, False, 2), (88, True, False, 2), (88, False, True, 3), (88, True, True, 2),
    (96, False, False, 2), (96, True, False, 2), (96, False, True, 2), (96, True, True, 3),
    (104, False, False, 3), (104, True, False, 2), (104, False, True, 2), (104, True, True, 2),
    (112, False, False, 2), (112, True, False, 3), (112, False, True, 2), (112, True, True, 2),
    (120, False, False, 2), (120, True, False, 2), (120, False, True, 3), (120, True, True, 2),
    (128, False, False, 2), (128, True, False, 2), (128, False, True, 2), (128, True, True, 3),
]

# D, mean, box: every width with and without a mean, and a box at every odd KB
TIMELINE_ROWS = [(D, mean, False) for D in range(8, 129, 8) for mean in (False, True)] + [
    (8, True, True), (24, False, True), (40, True, True), (56, False, True),
    (72, True, True), (88, False, True), (104, True, True), (120, False, True),
]

# id, model kind of test_gpu_accept_exact._model, N, D
THRESHOLD_ROWS = [
    ("dmma-D56", "dense", 301, 56), ("dmma-D56-mean", "dense-mean", 301, 56),
    ("dmma-D72", "dense", 517, 72), ("dmma-D72-mean", "dense-mean", 517, 72),
    ("dmma-D80", "dense", 517, 80),
    ("dmma-D88", "dense", 517, 88), ("dmma-D88-mean", "dense-mean", 517, 88),
    ("dmma-D104", "dense", 517, 104), ("dmma-D104-mean", "dense-mean", 517, 104),
    ("dmma-D112-mean", "dense-mean", 1001, 112),
    ("dmma-D120", "dense", 1001, 120), ("dmma-D120-mean", "dense-mean", 1001, 120),
    ("dmma-D120-box", "dense-box", 1001, 120),
]


def _row_id(r):
    return "D%d%s%s%s" % (r[0], "-mean" if r[1] else "", "-box" if r[2] else "", "-s%d" % r[3] if len(r) > 3 else "")


def active_count(sm, tiles, extra):
    """Active walkers of a split such that every consumer warp of ``sm`` CTAs gets ``tiles`` tiles and one warp a
    last, partial tile of ``extra`` walkers."""
    return TILE * tiles * CONSUMERS * sm + extra


def _extra(D, mean, box):
    return 1 + (D // 8 + 2 * mean + 4 * box) % 7  # 1..7: never a multiple of 8


def consumer_tiles(count, grid):
    """Tiles of each consumer warp [CTA, pair] under the SM-major deal (tile0 = CTA + grid * pair, stride
    grid * 8), and the (CTA, pair) that gets the last tile."""
    ntiles = -(-count // TILE)
    out = np.zeros((grid, CONSUMERS), dtype=np.int64)
    for b in range(grid):
        for p in range(CONSUMERS):
            out[b, p] = len(range(b + grid * p, ntiles, grid * CONSUMERS))
    last = ntiles - 1
    return out, (last % grid, (last // grid) % CONSUMERS)


# ---- CPU: the cell table ----------------------------------------------------------------------------------------
def test_cell_table():
    """Deleting a row of STEP_ROWS, TIMELINE_ROWS or THRESHOLD_ROWS fails here."""
    assert len(CELLS) == 64
    rebalanced = {c for c in CELLS if dmma_rebalance(*c)}
    assert sorted(rebalanced) == [(11, True, False), (12, True, False), (13, True, False), (14, True, False),
                                  (15, False, False), (15, True, False), (16, False, False), (16, True, False)]
    padded = {c for c in CELLS if c[0] % 2 == 1}
    assert len(padded) == 32
    covered = {(D // 8, mean, box) for D, mean, box, _ in STEP_ROWS}
    assert covered == set(CELLS), sorted(set(CELLS) - covered)
    assert len(STEP_ROWS) == len(set((D, m, b) for D, m, b, _ in STEP_ROWS)) == 64
    # every row runs at a multi-tile shape: at any SM count every consumer warp gets TILES tiles, the split's
    # active count is not a multiple of 8, and the last, partial tile goes to a warp with several tiles
    for sm in (1, 78, 114, 132, 144):
        for D, mean, box, nsplits in STEP_ROWS:
            count = active_count(sm, TILES, _extra(D, mean, box))
            assert count % TILE != 0
            tiles, (b, p) = consumer_tiles(count, min(-(-count // TILE), sm))
            assert tiles.min() >= TILES and tiles[b, p] == TILES + 1
    assert rebalanced <= covered
    assert {c for c in padded if c[0] >= 7} <= covered
    for KB in range(1, 17):
        assert sum(1 for D, _, _, s in STEP_ROWS if D == 8 * KB and s == 3) == 1, KB
    # timeline: every width with and without a mean, a box at every odd KB
    tl = set(TIMELINE_ROWS)
    for KB in range(1, 17):
        assert (8 * KB, False, False) in tl and (8 * KB, True, False) in tl
        if KB % 2:
            assert any(D == 8 * KB and box for D, _, box in tl), KB
    # threshold bisection: odd KB >= 7 with and without a mean, the rebalanced D = 112 with a mean, D = 120 boxed
    th = {(kind, D) for _, kind, _, D in THRESHOLD_ROWS}
    for D in (56, 72, 88, 104, 120):
        assert ("dense", D) in th and ("dense-mean", D) in th
    assert {("dense-mean", 112), ("dense-box", 120), ("dense", 80)} <= th
    assert dmma_rebalance(14, True, False) and not dmma_rebalance(15, False, True)


def test_precision_symmetric_part_is_exact():
    """The non-symmetric precision's symmetric part, 0.5 (A + A^T) as the host forms it, is the SPD matrix the
    exact reference sees (x^T A x = x^T A_s x)."""
    for D in ASYM_WIDTHS:
        A = precision(D, True)
        S = precision(D, False)
        assert not np.array_equal(A, A.T)
        assert np.array_equal(0.5 * (A + A.T), S)
        assert np.array_equal(A + A.T, 2.0 * S)  # the sum is exact too
        w = np.linalg.eigvalsh(S)
        assert w.min() > 0 and 5e5 < w.max() / w.min() < 2e6


# ---- inputs ------------------------------------------------------------------------------------------------------
def precision(D, asym):
    """SPD, condition 1e6, on a grid of 2^-36 (|A| < 2^10); with ``asym`` plus an antisymmetric matrix on a grid of
    2^-6, so 0.5 (A + A^T) is exact."""
    rng = np.random.default_rng(1000 + D)
    q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    A = (q * np.logspace(-3, 3, D)) @ q.T
    A = np.round(0.5 * (A + A.T) * 2.0 ** 36) / 2.0 ** 36
    if asym:
        K = np.triu(np.round(rng.standard_normal((D, D)) * 64) / 64, 1)
        A = A + (K - K.T)
    return A


def far_mean(D):
    j = np.arange(D)
    return 1e3 * (1.0 + 0.25 * np.sin(j)) * np.where(j % 2, -1.0, 1.0)


def _box(q):
    """Per-coordinate bounds that a third of the rows of ``q`` leave: the i-th smallest and largest proposal
    coordinate of every column, i bisected."""
    qs = np.sort(q, axis=0)
    n = q.shape[0]
    a, b = 0, n // 2 - 1  # outside fraction: 0 at i = 0, most rows at n / 2 - 1
    while b - a > 1:
        i = (a + b) // 2
        if np.mean(~_inside(q, qs[i], qs[n - 1 - i])) < 1.0 / 3.0:
            a = i
        else:
            b = i
    return qs[b], qs[n - 1 - b]


def _inside(x, lo, hi):
    return np.all((lo <= x) & (x <= hi), axis=-1)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _sm():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


class Worst(object):
    """Largest |device - exact| / bound of one cell."""

    def __init__(self, name):
        self.name, self.worst, self.n = name, 0.0, 0

    def check(self, dev, x, mu, Aint, L, what):
        self.n += 1
        exact = LX.exact_dense(x, mu, Aint)
        if np.isinf(LX._to_float(exact)):
            assert dev == -np.inf, (self.name, what, dev)
            return
        assert np.isfinite(dev), (self.name, what, dev, float(exact))
        ratio = float(abs(Fraction(float(dev)) - exact)) / LX.bound_dense_dmma(x, mu, L)
        self.worst = max(self.worst, ratio)
        assert ratio < 1.0, (self.name, what, float(dev), float(exact), ratio)


class Setup(object):
    """Model, engine and initial state of one cell."""

    def __init__(self, D, mean, box, nsplits, N, seed):
        self.D, self.mean, self.box, self.N, self.nsplits = D, mean, box, N, nsplits
        self.A = precision(D, D in ASYM_WIDTHS)
        self.mu = far_mean(D) if mean else np.zeros(D)
        self.Aint = LX._ints(self.A)
        self.L = np.linalg.cholesky(0.5 * (self.A + self.A.T))
        rng = np.random.default_rng(seed ^ (N * 7919 + D))
        self.X0 = self.mu + rng.standard_normal((N, D))
        self.mv = rb.Stretch(nsplits=nsplits)
        self.lo = self.hi = None
        if box:
            # the proposals of split 0 depend only on X0: bound them
            inds = px.split_assignment(SEED, STEP, N, nsplits, True)
            sets = [np.flatnonzero(inds == k) for k in range(nsplits)]
            o = rb.OracleSampler(N, D, None, [(self.mv, 1.0)], seed=SEED)
            o.coords = self.X0
            q0, _ = o._stretch(self.mv, self.X0[sets[0]], sets[1:], STEP, 0)
            self.lo, self.hi = _box(q0)

    def model(self):
        m = models.GaussianDense(self.A, self.mu if self.mean else None)
        return models.Bounded(m, self.lo, self.hi) if self.box else m

    def engine(self, **options):
        eng = emcee_b200.EnsembleSampler(self.N, self.D, self.model(), seed=1)._engine
        for k, v in options.items():
            eng.set_option(k, v)
        return eng

    def desc(self):
        return moves.StretchMove(nsplits=self.nsplits).descriptor()

    def lp_fn(self):
        """The oracle's log-probability for a step from log_prob = -inf: every finite proposal is accepted, one
        outside the box is not (-inf - -inf is NaN)."""
        if not self.box:
            return lambda p: np.zeros(p.shape[0])
        return lambda p: np.where(_inside(p, self.lo, self.hi), 0.0, -np.inf)


def _step(eng, X, lp, desc, seed, step):
    eng.set_state(X, lp)
    eng.set_rng(seed, step)
    return eng.step([(desc, 1.0)], 1)


def _sample_ranks(count, n):
    """First and last ranks, the last partial tile, and ``n`` evenly spread ranks."""
    tail = np.arange(count - count % TILE, count)
    return np.unique(np.r_[0, count - 1, tail, np.linspace(0, count - 1, n).astype(np.int64)])


# ---- GPU: every cell at a multi-tile shape ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D,mean,box,nsplits", STEP_ROWS, ids=[_row_id(r) for r in STEP_ROWS])
def test_cell_multi_tile(D, mean, box, nsplits):
    t0 = time.time()
    sm = _sm()
    count = active_count(sm, TILES, _extra(D, mean, box))
    N = nsplits * count  # every split has `count` active walkers
    s = Setup(D, mean, box, nsplits, N, SEED)
    eng = s.engine()
    desc = s.desc()
    name = "dense_dmma %s N=%d" % (_row_id((D, mean, box, nsplits)), N)

    # ---- step 1 from log_prob = -inf: the state shows every proposal
    minus_inf = np.full(N, -np.inf)
    acc1 = _step(eng, s.X0, minus_inf, desc, SEED, STEP)
    variant = eng.last_kernel_variant()
    assert variant == "dense_dmma nhalf_max=1 grid=%d" % min(-(-count // TILE), sm), variant
    X1, lp1 = eng.get_state()
    o = rb.OracleSampler(N, D, s.lp_fn(), [(s.mv, 1.0)], seed=SEED, step=STEP)
    o.set_state(s.X0, minus_inf)
    o.run(1)
    assert _same(X1, o.coords), "coordinates differ from the stretch proposals of the draw specification"
    assert np.array_equal(acc1, o.naccepted == 1)
    assert np.array_equal(eng.naccepted(), o.naccepted.astype(np.uint64))
    if box:
        out = ~acc1
        frac = out.mean()
        assert 0.2 < frac < 0.5, frac
        assert np.all(lp1[out] == -np.inf) and _same(X1[out], s.X0[out])
        on = np.any((X1 == s.lo) | (X1 == s.hi), axis=1) & acc1
        assert on.any(), "no accepted proposal lies exactly on a bound"
    else:
        assert acc1.all()
    # every stored log-probability is compute_log_prob's value of the stored row, bit for bit
    assert _same(lp1[acc1], eng.compute_log_prob(X1[acc1]))

    # ---- exact log-probabilities of sampled rows, the last partial tile and the first / last ranks included
    inds = px.split_assignment(SEED, STEP, N, nsplits, True)
    sets = [np.flatnonzero(inds == k) for k in range(nsplits)]
    wk = Worst(name)
    for k in range(nsplits):
        inside = np.flatnonzero(acc1[sets[k]])  # (rows outside the box hold -inf: checked above)
        spread = inside[np.linspace(0, inside.size - 1, -(-EXACT_ROWS // nsplits)).astype(np.int64)]
        for r in np.unique(np.r_[_sample_ranks(count, 0), spread]):
            w = sets[k][r]
            if acc1[w]:
                wk.check(lp1[w], X1[w], s.mu, s.Aint, s.L, (k, int(r)))
    assert wk.n >= EXACT_ROWS, wk.n

    # ---- step 2 from a finite state: the accept mask against fl(fl(F + lp_dev) - lp_old) > log u
    X2 = X1.copy()
    if box:
        X2[~acc1] = np.clip(s.X0[~acc1], s.lo, s.hi)
    lp2 = eng.compute_log_prob(X2)
    assert np.all(np.isfinite(lp2))
    nacc0 = eng.naccepted()
    acc2 = _step(eng, X2, lp2, desc, SEED, STEP + 1)
    X3, lp3 = eng.get_state()
    assert np.array_equal(eng.naccepted() - nacc0, acc2.astype(np.uint64))
    inds = px.split_assignment(SEED, STEP + 1, N, nsplits, True)
    sets = [np.flatnonzero(inds == k) for k in range(nsplits)]
    cur, lp_cur = X2.copy(), lp2.copy()
    po = rb.OracleSampler(N, D, None, [(s.mv, 1.0)], seed=SEED)
    skipped = 0
    for k in range(nsplits):
        act = sets[k]
        po.coords = cur
        q, F = po._stretch(s.mv, cur[act], sets[:k] + sets[k + 1:], STEP + 1, k)
        zz = po.taps["zz"]
        lpq = eng.compute_log_prob(q)
        u = AX.accept_u(SEED, STEP + 1, k, np.arange(len(act)))
        lnu = np.log(u)
        old = lp_cur[act]
        with np.errstate(invalid="ignore"):
            pred = ((F + lpq) - old) > lnu
        # near the threshold T = F + lp_dev - ln u: skip |lp_old - T| <= B (accept_exact.threshold, dlp = 0)
        fin = np.isfinite(lpq)
        with np.errstate(invalid="ignore"):
            B = 3 * U * np.abs(F) + U * np.abs(F + lpq) + 3 * U * np.abs(lnu)
            slack = 4 * U * (np.abs(F) + np.abs(lpq) + np.abs(old) + np.abs(lnu))
            cand = fin & (np.abs(old - ((F + lpq) - lnu)) <= 2 * B + slack)
        skip = np.zeros(len(act), dtype=bool)
        for i in np.flatnonzero(cand):
            Fm, dF = AX.stretch_factor(zz[i], D)
            T_, B_ = AX.threshold(Fm, dF, AX.mpf(lpq[i]), 0.0, u[i])
            skip[i] = abs(float(AX.mpf(old[i]) - T_)) <= B_
        skipped += int(skip.sum())
        dev = acc2[act]
        bad = np.flatnonzero((pred != dev) & ~skip)
        assert bad.size == 0, ("accept mask", k, act[bad][:8], pred[bad][:8], dev[bad][:8])
        won = act[dev]
        cur[won] = q[dev]
        lp_cur[won] = lpq[dev]
    assert _same(X3, cur), "second step: coordinates differ"
    assert _same(lp3, lp_cur), "second step: stored log-probabilities are not compute_log_prob's"
    print("%s: %d rows exact, largest error / bound = %.3g; step 2: %d of %d accepted, %d skipped near the "
          "threshold; %.1f s" % (name, wk.n, wk.worst, int(acc2.sum()), N, skipped, time.time() - t0))
    assert skipped <= max(8, N // 1000)


# ---- GPU: exact accept thresholds at the cells that change the arithmetic -----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,D", [r[1:] for r in THRESHOLD_ROWS], ids=[r[0] for r in THRESHOLD_ROWS])
def test_threshold_rows(kind, N, D):
    import test_gpu_accept_exact as AE

    AE.test_accept_threshold_exact(kind, N, D, AE.ST, (), "dmma", "normal")


# ---- GPU: the instrumented cells compute what production computes ----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D,mean,box", TIMELINE_ROWS, ids=[_row_id(r) for r in TIMELINE_ROWS])
def test_timeline_cells(D, mean, box):
    t0 = time.time()
    sm = _sm()
    count = active_count(sm, TIMELINE_TILES, _extra(D, mean, box))
    N = 2 * count
    s = Setup(D, mean, box, 2, N, SEED + 1)
    desc = s.desc()
    ref = s.engine()
    lp0 = ref.compute_log_prob(s.X0)
    ref.set_state(s.X0, lp0)
    ref.set_rng(SEED, STEP)
    acc_ref = ref.step([(desc, 1.0)], 2)
    X_ref, lp_ref = ref.get_state()
    grid = min(-(-count // TILE), sm)
    assert ref.last_kernel_variant() == "dense_dmma nhalf_max=1 grid=%d" % grid
    tiles, _ = consumer_tiles(count, grid)
    assert tiles.min() >= TIMELINE_TILES
    for mode in (1, 2):
        eng = s.engine(dmma_timeline=mode)
        eng.set_state(s.X0, lp0)
        eng.set_rng(SEED, STEP)
        acc = eng.step([(desc, 1.0)], 2)
        X, lp = eng.get_state()
        assert _same(X, X_ref) and _same(lp, lp_ref), ("dmma_timeline", mode)
        assert np.array_equal(acc, acc_ref) and np.array_equal(eng.naccepted(), ref.naccepted())
        assert eng.last_kernel_variant() == ref.last_kernel_variant()
        tl = eng.debug_timeline()
        assert tl.shape == (grid, CONSUMERS, 8, 12), tl.shape
        # event 0: the tile a consumer took, SM-major (every split has `count` walkers, so mode 2's first split
        # deals as mode 1's last)
        b, p, kk = np.meshgrid(np.arange(grid), np.arange(CONSUMERS), np.arange(TIMELINE_TILES), indexing="ij")
        assert np.array_equal(tl[:, :, :TIMELINE_TILES, 0], b + grid * p + kk * grid * CONSUMERS)
    print("dmma_timeline %s N=%d: twins byte-identical; %.1f s" % (_row_id((D, mean, box)), N, time.time() - t0))


# ---- GPU: the stand-alone log-probability kernel, every cell -----------------------------------------------------
def _standalone_rows(D, mu, lo, hi, rng):
    """(label, rows, expect -inf) of one cell."""
    out = [("8k%+d" % d, mu + rng.standard_normal((n, D)), None) for n, d in ((7, -1), (9, 1), (17, 1), (63, -1))]
    out.append(("far", mu + 1e4 * rng.standard_normal((9, D)), None))
    z = rng.standard_normal((9, D))
    out.append(("overflow", mu + np.sign(z + 0.5) * 1e160 * (1.0 + np.abs(z)), True))
    if lo is not None:
        base = np.clip(mu + 0.5 * rng.standard_normal(D), lo, hi)
        cols = sorted(set([8 * b + (3 * b) % 8 for b in range(D // 8)] + list(range(D - 8, D))))
        rows, outside = [], []
        for j in cols:
            for v, o in ((lo[j], False), (hi[j], False), (np.nextafter(lo[j], -np.inf), True),
                         (np.nextafter(hi[j], np.inf), True)):
                x = base.copy()
                x[j] = v
                rows.append(x)
                outside.append(o)
        out.append(("bounds", np.array(rows), np.array(outside)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("D", list(range(8, 129, 8)))
def test_standalone_cells(D):
    for mean in (False, True):
        for box in (False, True):
            A = precision(D, D in ASYM_WIDTHS)
            mu = far_mean(D) if mean else np.zeros(D)
            lo = hi = None
            m = models.GaussianDense(A, mu if mean else None)
            if box:
                lo, hi = mu - 2.5, mu + 2.5
                m = models.Bounded(m, lo, hi)
            eng = emcee_b200.EnsembleSampler(max(2, 2 * D), D, m, seed=1)._engine
            Aint, L = LX._ints(A), np.linalg.cholesky(0.5 * (A + A.T))
            t0 = time.time()
            wk = Worst("compute_log_prob %s" % _row_id((D, mean, box)))
            rng = np.random.default_rng(D * 4 + 2 * mean + box)
            for label, x, minus_inf in _standalone_rows(D, mu, lo, hi, rng):
                dev = eng.compute_log_prob(x)
                if minus_inf is True:
                    assert np.all(dev == -np.inf), (wk.name, label)
                    continue
                if lo is not None and minus_inf is None:
                    minus_inf = ~_inside(x, lo, hi)
                for r in range(x.shape[0]):
                    if minus_inf is not None and minus_inf[r]:
                        assert dev[r] == -np.inf, (wk.name, label, r)
                    else:
                        assert lo is None or _inside(x[r], lo, hi)
                        wk.check(dev[r], x[r], mu, Aint, L, (label, r))
            print("%s: %d rows, largest error / bound = %.3g; %.1f s" % (wk.name, wk.n, wk.worst, time.time() - t0))
            assert wk.n > 0
