"""Red-blue half-steps at split counts above 5: every kernel that reads the split table, at 6 to 32 splits, at
splits of one walker and at fixed splits, against the oracle and the existing high-precision harnesses.

``nsplits`` is a user parameter of every red-blue move (``[2, min(32, nwalkers)]``).  The split table has one warp
per set, the per-walker draws carry the split index in their counter (``draw_words``) and the Walk subsets and
captured proposals draw per split (``sub_split``), so a split index >= 8 or a set smaller than a kernel's tile is an
edge of its own.  The golden chains of the unmodified reference at 6 to 32 splits are in ``tests/golden`` (the
``*nsplits*`` cases) and run through test_gpu_parity, test_gpu_callback and test_gpu_device_backend.

==============================  =====================================================  =========================
row                             cell and edge                                          check
==============================  =====================================================  =========================
test_stretch_cell[tma16-*]      tma_rows R=16 (D 16): P 7 sets of 16-17 (straddling    oracle, bit for bit
                                R), P 32 sets of 10-11 (below R), P 32 fixed
test_stretch_cell[tma2-*]       tma_rows R=2 (D 128): P 7, P 32 with sets of 1-2
                                (below and straddling R, live_dangerously)
test_stretch_cell[tma1-*]       tma_rows R=1 (D 256): P 32, P 7 fixed
test_stretch_cell[generic-*]    generic kernel at D 37, nsplits == nwalkers == 32
test_stretch_cell[dmma-*]       dense_dmma one half-step per launch at P 32 with       oracle, bit for bit
                                splits of 1-2, 3-4 and 6-7 walkers (under one
                                8-walker tile), pdl 1 and 0; P 7 and 32 fixed
test_de_walk_cell               DE on tma_rows at P 9 and 32; Walk whole complement    test_gpu_parity's
                                at P 9, Walk s = smallest complement at P 32 (both     tolerances
                                Walk kernels in one step)
test_grouped_dense_dmma         dmma_group 2 / 5 / 64 at P 7 and 32: groups span       dmma_group 1 and the
                                step boundaries                                        oracle, launch counts
test_mixed_schedule_610_steps   stretch at P 2 / 7 fixed / 32, 610 steps through two   oracle, bit for bit
                                run_mcmc calls (a 512-step chunk) and a sample loop
test_table_cache_schedule_      one engine steps schedule A, rewinds with set_rng and  a fresh engine and the
  switch                        steps schedule B over the same steps; B differs in     oracle, bit for bit
                                nsplits or in randomize_split
test_accept_exact               test_gpu_accept_exact's threshold bisection at P 7     exact thresholds
                                (stretch on tma_rows R=16, DE on R=8)
test_walk_proposals_exact       test_gpu_proposals_exact's 45-digit Walk rows: whole   high-precision bound
                                complement and subset at P 9 and 32 (split >= 8 in
                                the subset draws)
test_numpy_user_move            a numpy RedBlueMove at 32 ragged splits                UserOracle, bit for bit
test_captured_proposal          CudaGraphRedBlueMove at 32 ragged splits, record=True  draws bit for bit, s / c
                                                                                       equal the mask gathers
test_one_row_calls              HostFunction and CudaGraphFunction at nsplits ==       the device model / the
                                nwalkers: every call has one row                       CUDA-array twin
test_blobs_at_32_splits         HostFunction with blobs, stretch / DE / Walk at P 32   blobs follow their walker
test_nsplits_refused            nsplits 33 and nsplits > nwalkers                      error, state untouched
==============================  =====================================================  =========================

Sharded ensembles at more than 2 splits are not tested here (they need two GPUs).
"""
import numpy as np
import pytest

from oracle import redblue as rb
from oracle import targets as T

from gpu_util import device_model, device_moves, move_rows_from_oracle

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _tma(R, epl, own_reg, warps=16):
    return "tma_rows R=%d epl=%d own_reg=%d warps=%d" % (R, epl, own_reg, warps)


def _dmma(N, P):
    """One half-step per launch; the grid of the last launch covers the last split (the smallest set)."""
    return "dense_dmma nhalf_max=1 grid=%d" % ((N // P + 7) // 8)


def _oracle_and_sampler(model, N, D, omoves, seed, live=False, options=()):
    target, p0 = T.make_config(model, N, D)
    o = rb.OracleSampler(N, D, target, omoves, seed=seed)
    o.set_state(p0)
    dm = device_moves(move_rows_from_oracle(omoves))
    for m, _ in dm:
        m.live_dangerously = live
    s = emcee_b200.EnsembleSampler(N, D, device_model(model, target=target), moves=dm, seed=seed)
    for k, v in options:
        s._engine.set_option(k, v)
    return o, s, p0, target


def _check(s, o, last, target, exact):
    if exact:
        assert np.array_equal(last.coords, o.coords)
        np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-11, atol=1e-11)
    else:  # test_gpu_parity's DE / Walk tolerances
        np.testing.assert_allclose(last.coords, o.coords, rtol=1e-9, atol=1e-11)
        np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-9, atol=1e-10)
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    np.testing.assert_allclose(last.log_prob, target(last.coords), rtol=1e-11, atol=1e-11)


# id, model, N, D, nsplits, randomize_split, live_dangerously, options, expected variant
STRETCH_CELLS = [
    ("tma16-p7-straddle", "gauss_iso", 7 * 16 + 3, 16, 7, True, False, (), _tma(16, 8, 1)),
    ("tma16-p32-below", "gauss_iso", 32 * 10 + 5, 16, 32, True, False, (), _tma(16, 8, 1)),
    ("tma16-p32-fixed", "rosenbrock", 32 * 16 + 9, 16, 32, False, False, (), _tma(16, 8, 1)),
    ("tma2-p7", "ring", 7 * 40 + 3, 128, 7, True, False, (), _tma(2, 8, 0)),
    ("tma2-p32-sets1-2", "ring", 33, 128, 32, True, True, (), _tma(2, 8, 0)),
    ("tma1-p32", "ring", 32 * 16 + 3, 256, 32, True, False, (), _tma(1, 8, 0)),
    ("tma1-p7-fixed", "ring", 7 * 74 + 1, 256, 7, False, False, (), _tma(1, 8, 0)),
    ("generic-d37-p32-one-walker-sets", "gauss_iso", 32, 37, 32, True, True, (), "generic G=16"),
    ("dmma-d16-p32-sets1-2", "gauss_dense", 40, 16, 32, True, False, (), _dmma(40, 32)),
    ("dmma-d16-p32-sets3-4", "gauss_dense", 100, 16, 32, True, False, (), _dmma(100, 32)),
    ("dmma-d24-p32-sets6-7", "gauss_dense", 215, 24, 32, True, False, (), _dmma(215, 32)),
    ("dmma-d24-p32-sets6-7-pdl0", "gauss_dense", 215, 24, 32, True, False, (("pdl", 0),), _dmma(215, 32)),
    ("dmma-d64-p32-sets4-5-pdl0", "gauss_dense", 128 + 3, 64, 32, True, False, (("pdl", 0),), _dmma(131, 32)),
    ("dmma-d32-p7-fixed", "gauss_dense", 7 * 20 + 5, 32, 7, False, False, (), _dmma(145, 7)),
    ("dmma-d16-p32-fixed", "gauss_dense", 100, 16, 32, False, False, (), _dmma(100, 32)),
]


@pytest.mark.parametrize("model,N,D,P,rand,live,options,variant", [c[1:] for c in STRETCH_CELLS],
                         ids=[c[0] for c in STRETCH_CELLS])
def test_stretch_cell(model, N, D, P, rand, live, options, variant):
    om = [(rb.Stretch(nsplits=P, randomize_split=rand, live_dangerously=live), 1.0)]
    o, s, p0, target = _oracle_and_sampler(model, N, D, om, 0x5911 + N + D, live, options)
    last = s.run_mcmc(p0, 6, store=False, skip_initial_state_check=True)
    o.run(6)
    assert s._engine.last_kernel_variant() == variant
    _check(s, o, last, target, True)


# id, model, N, D, oracle moves, expected kernel variant or name
DE_WALK_CELLS = [
    ("de-tma8-p9", "gauss_iso", 9 * 34 + 4, 24, [(rb.DE(nsplits=9), 1.0)], _tma(8, 0, 0)),
    ("de-tma4-p32", "rosenbrock", 32 * 11 + 7, 32, [(rb.DE(nsplits=32), 1.0)], _tma(4, 0, 0)),
    ("walk-all-p9", "ring", 9 * 7 + 2, 6, [(rb.Walk(nsplits=9), 1.0)], "walk"),
    ("walk-s-p32", "gauss_iso", 32 * 3 + 5, 4, [(rb.Walk(s=97, nsplits=32), 1.0)], "walk"),
]


@pytest.mark.parametrize("model,N,D,omoves,variant", [c[1:] for c in DE_WALK_CELLS], ids=[c[0] for c in DE_WALK_CELLS])
def test_de_walk_cell(model, N, D, omoves, variant):
    o, s, p0, target = _oracle_and_sampler(model, N, D, omoves, 0x5D1 + N + D)
    last = s.run_mcmc(p0, 6, store=False, skip_initial_state_check=True)
    o.run(6)
    if variant == "walk":
        assert s._engine.last_kernel_name() == "walk"
    else:
        assert s._engine.last_kernel_variant() == variant
    _check(s, o, last, target, False)


# id, D, N as (SM multiple, offset), nsplits, mean, the dmma_group of each call
GROUPED = [
    ("D32-p7", 32, (8, -3), 7, False, (2, 5, 64, 2)),
    ("D16-p32", 16, (8, 5), 32, True, (5, 64, 2, 5)),
    ("D64-p32-small", 64, (1, 3), 32, False, (64, 2, 5, 64)),
]


@pytest.mark.parametrize("D,nm,P,mean,groups", [c[1:] for c in GROUPED], ids=[c[0] for c in GROUPED])
def test_grouped_dense_dmma(D, nm, P, mean, groups):
    """test_gpu_variants' grouped script (run_mcmc store=False, thinned storage, one step per call) at 7 and 32
    splits: bit-identical to dmma_group = 1 and to the oracle, with the launch count of the flush rule."""
    import test_gpu_variants as tv

    tv.test_grouped_dense_dmma(D, nm, P, mean, groups)


MIXED = [(rb.Stretch(), 0.3), (rb.Stretch(nsplits=7, randomize_split=False), 0.3), (rb.Stretch(nsplits=32), 0.4)]


@pytest.mark.parametrize("model,N,D,kernel", [("gauss_dense", 203, 16, "dense_dmma"), ("ring", 150, 16, _tma(16, 8, 1))],
                         ids=["dmma", "tma"])
def test_mixed_schedule_610_steps(model, N, D, kernel):
    """A schedule of stretch moves at 2, 7 (fixed) and 32 splits over 610 steps: run_mcmc(530) crosses the 512-step
    table chunk, run_mcmc(20) and a 60-step sample loop use the 64-step look-ahead build."""
    o, s, p0, target = _oracle_and_sampler(model, N, D, MIXED, 0x3170 + N)
    st = s.run_mcmc(p0, 530, store=False, skip_initial_state_check=True)
    o.run(530)
    _check(s, o, st, target, True)
    st = s.run_mcmc(st, 20, store=False, skip_initial_state_check=True)
    o.run(20)
    _check(s, o, st, target, True)
    for k, st in enumerate(s.sample(st, iterations=60, store=False, skip_initial_state_check=True)):
        o.run(1)
        assert np.array_equal(st.coords, o.coords), k
    _check(s, o, st, target, True)
    assert s.random_state[2] == 610
    assert s._engine.last_kernel_variant().startswith(kernel)


SWITCH = [
    ("nsplits-7-to-32", rb.Stretch(nsplits=7), rb.Stretch(nsplits=32)),
    ("nsplits-32-to-2", rb.Stretch(nsplits=32), rb.Stretch()),
    ("random-to-fixed-p7", rb.Stretch(nsplits=7), rb.Stretch(nsplits=7, randomize_split=False)),
    ("fixed-to-random-p32", rb.Stretch(nsplits=32, randomize_split=False), rb.Stretch(nsplits=32)),
]


@pytest.mark.parametrize("model,N,D,kernel", [("gauss_dense", 203, 16, "dense_dmma"), ("gauss_iso", 150, 5, "generic")],
                         ids=["dmma", "generic"])
@pytest.mark.parametrize("a,b", [c[1:] for c in SWITCH], ids=[c[0] for c in SWITCH])
def test_table_cache_schedule_switch(a, b, model, N, D, kernel):
    """The engine keeps the split tables of the steps it has tabulated and reuses them only for the same nsplits
    and randomize_split.  Stepping schedule A, rewinding the counter with set_rng and stepping schedule B over the
    same steps must give what a fresh engine gives for B (a caller of the C ABI may do this)."""
    seed, n = 0x5C4E + N, 12
    ob, s, p0, target = _oracle_and_sampler(model, N, D, [(b, 1.0)], seed)
    ob.run(n)
    eng = s._engine
    da = device_moves(move_rows_from_oracle([(a, 1.0)]))[0][0].descriptor()
    db = device_moves(move_rows_from_oracle([(b, 1.0)]))[0][0].descriptor()
    eng.set_state(p0)
    lp0 = eng.get_state()[1]
    eng.set_rng(seed, 0)
    eng.step([(da, 1.0)], n)
    eng.set_state(p0, lp0)
    eng.set_rng(seed, 0)
    acc_b = [eng.step([(db, 1.0)], 1) for _ in range(n // 2)]  # one step per call: the cached tables' path
    acc_b.append(eng.step([(db, 1.0)], n - n // 2))
    coords, lp = eng.get_state()
    assert eng.last_kernel_variant().startswith(kernel)
    fresh = emcee_b200.EnsembleSampler(N, D, device_model(model, target=target), seed=seed)._engine
    fresh.set_state(p0, lp0)
    fresh.set_rng(seed, 0)
    fresh.step([(db, 1.0)], n)
    assert np.array_equal(coords, fresh.get_state()[0]) and np.array_equal(lp, fresh.get_state()[1])
    assert np.array_equal(coords, ob.coords)
    np.testing.assert_allclose(lp, ob.log_prob, rtol=1e-11, atol=1e-11)


ACCEPT_ROWS = [
    # model, N, D, mspec, options, variant, state kind, nsplits
    ("st16-iso-p7", "iso", 7 * 16 + 3, 16, ("stretch", 2.0), (), _tma(16, 8, 1), "normal", 7),
    ("de24-iso-p7", "iso", 7 * 40 + 5, 24, ("de", 1e-5, None), (), _tma(8, 0, 0), "normal", 7),
]


@pytest.mark.parametrize("model_kind,N,D,mspec,options,variant,skind,nsplits", [r[1:] for r in ACCEPT_ROWS],
                         ids=[r[0] for r in ACCEPT_ROWS])
def test_accept_exact(model_kind, N, D, mspec, options, variant, skind, nsplits):
    import test_gpu_accept_exact as ax

    ax.test_accept_threshold_exact(model_kind, N, D, mspec, options, variant, skind, nsplits)


WALK_ROWS = [
    # N, D, nsplits, s, state kind
    ("whole-p9", 9 * 6 + 4, 4, 9, None, "int"),
    ("whole-p32", 32 * 2 + 7, 3, 32, None, "int"),
    ("subset-s5-p9", 9 * 6 + 4, 4, 9, 5, "int"),
    ("subset-s5-p32", 32 * 2 + 7, 3, 32, 5, "int"),
]


@pytest.mark.parametrize("N,D,nsplits,s,kind", [r[1:] for r in WALK_ROWS], ids=[r[0] for r in WALK_ROWS])
def test_walk_proposals_exact(N, D, nsplits, s, kind):
    import test_gpu_proposals_exact as pe

    pe.test_walk_proposals_exact(N, D, nsplits, s, kind)


def test_numpy_user_move():
    """A numpy RedBlueMove at 32 ragged splits (70 walkers: sets of 3 and 2) against UserOracle."""
    import test_gpu_user_moves as um

    um.test_splits_and_odd_sizes(70, 4, 32, True)
    um.test_splits_and_odd_sizes(75, 3, 32, False)


def test_captured_proposal():
    """A CudaGraphRedBlueMove at 32 ragged splits: the purpose-9 draws of every split bit for bit (uniform), and
    the s and c its capture saw equal the boolean-mask gathers of the last split of each size."""
    import test_gpu_graph_moves as gm

    gm.test_draws_and_gathers("uniform", 70, 32)


def test_one_row_calls():
    """nsplits == nwalkers: every call of a user log-probability has one row."""
    import test_gpu_callback as cb
    import test_gpu_graph_function as gf

    N, D = 32, 5
    cb._identity_case(moves.StretchMove(nsplits=N), N, D, True)
    cb._identity_case(moves.DEMove(nsplits=N), N, D, True)
    a, g, cap = gf._pair(N, D, lambda: moves.StretchMove(nsplits=N))
    for s in (a, g):
        s.run_mcmc(gf._p0(N, D), 8, thin_by=2, skip_initial_state_check=True)
    gf._assert_same(a, g)
    assert g._engine.last_kernel_variant().endswith("where=graph")


@pytest.mark.parametrize("kind", ["stretch", "de", "walk"])
def test_blobs_at_32_splits(kind):
    import test_gpu_blobs as tb

    make = dict(tb.MOVES)[kind]
    tb.test_blobs_follow_their_walker(kind, make, 32, 5, "host")


@pytest.mark.parametrize("nsplits,N", [(33, 40), (33, 33), (9, 8), (3, 2)])
def test_nsplits_refused(nsplits, N):
    """nsplits outside [2, min(32, nwalkers)]: the engine's error, before the state or the step counter change."""
    D = 1
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianIso(), seed=7)
    eng = s._engine
    p0 = np.random.default_rng(N).standard_normal((N, D))
    eng.set_state(p0)
    eng.set_rng(7, 3)
    before = eng.get_state()
    for mv in (moves.StretchMove(nsplits=nsplits), moves.DEMove(nsplits=nsplits)):
        with pytest.raises(NotImplementedError, match="nsplits must be in"):
            eng.step([(mv.descriptor(), 1.0)], 2)
        after = eng.get_state()
        assert after[0].tobytes() == before[0].tobytes() and after[1].tobytes() == before[1].tobytes()
        assert eng.get_rng() == (7, 3)
