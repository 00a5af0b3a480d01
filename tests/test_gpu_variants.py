"""Every run-time variant of the half-step kernels against the oracle, with the cell it ran asserted through
``eb_last_kernel_variant``.

Which kernel instantiation runs depends on ndim, the move, the model and a few options; the parity suite checks a
fixed list of shapes.  Each row below names the cell its launcher is expected to pick, so a change to the
shared-memory budget heuristic that moves a shape onto another cell fails here instead of silently leaving a
cell untested.

tma_rows cells (``launch_tma_t`` in tma_rows.cu: R walkers per tile, G = 32 / R lanes per walker, EPL = 8 the
register path, 0 the strided one, OWN_REG the own row in registers):

=========  ================  ====================================  ==========================================
move       D                 cell                                  test ids (test_tma_cell[...])
=========  ================  ====================================  ==========================================
stretch    16                R=16 (G=2) EPL=8 OWN_REG              s16-iso-a1, s16-rosen-a15
stretch    32                R=8 (G=4) EPL=8 OWN_REG               s32-ring-a1, s32-rosen-a7
stretch    64                R=4 (G=8) EPL=8 OWN_REG               s64-iso-a1, s64-rosen-a3
stretch    128               R=2 (G=16) EPL=8                      s128-ring-a1, s128-rosen-a1
stretch    22, 44            R=16 / R=8 EPL=0                      s22-ring, s44-iso
stretch    96                R=2 (G=16) EPL=0                      s96-iso
stretch    200, 320          R=1 (G=32) EPL=0, 16 warps            s200-rosen, s320-iso
stretch    256               R=1 (G=32) EPL=8, 16 warps            s256-ring, s256-rosen
stretch    400, 768          R=1 EPL=0, 14 and 8 warps             s400-iso, s768-rosen
DE         24, 32, 64, 128   R=8 / 4 / 2 / 1 (G=4 / 8 / 16 / 32)   de24-iso, de32-rosen, de64-ring, de128-iso
DE         256               R=1 (G=32) EPL=8, 13 warps            de256-ring
snooker    16, 32, 64        R=8 / 4 / 2 (G=4 / 8 / 16) EPL=0      sn16-iso, sn32-ring, sn64-rosen
snooker    96, 200           R=1 (G=32), 16 and 13 warps           sn96-iso, sn200-ring
snooker    256               R=1 (G=32) EPL=8, 10 warps            sn256-iso
any        odd D             generic kernel                        s37-iso-generic
=========  ================  ====================================  ==========================================

The Rosenbrock register path (its cross-lane ``x[e+1]`` shuffle) and the ring / iso register path run at each of
G = 2, 4, 8 and 16 (stretch D = 16, 32, 64, 128) and G = 32 (stretch, DE and snooker D = 256).  The ``-aK`` rows have
an active count of K mod R: partial tiles on the register and OWN_REG paths.  Batch crossings (a warp with more
than G tiles, so the per-lane walker metadata of a new batch is tabulated mid-loop) are in test_batch_crossing at
G = 16 and G = 32, sized from the device's SM count.  test_options_bit_identical runs one shape per path under
tma_rows = 2 / 1 / 0 and tma_own_reg = 1 / 0.

Dense Gaussian under the stretch move (test_dense_cuda_core): the CUDA-core generic kernel at D % 8 != 0, D > 128,
with dense_dmma = 0, and with an indefinite precision matrix (its Cholesky factorisation fails, so dense_dmma must
not run).  Grouped dense_dmma (dmma_group > 1: several half-steps per cooperative launch with a grid barrier
between them) is in test_grouped_dense_dmma*.

Checks: stretch rows bit-exact coordinates and accept counts; DE / snooker rows the tolerances of
test_gpu_parity.test_against_oracle; on every row the device log-probabilities equal a float64 evaluation of the
target at the device's own coordinates to 1e-11 relative.
"""
import numpy as np
import pytest

from oracle import philox as px
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


ST, DE, SN = [(rb.Stretch(), 1.0)], [(rb.DE(), 1.0)], [(rb.Snooker(), 1.0)]

# id, model, N, D, oracle moves, expected variant
CELLS = [
    ("s16-iso-a1", "gauss_iso", 2 * (16 * 8 + 1), 16, ST, _tma(16, 8, 1)),
    ("s16-rosen-a15", "rosenbrock", 2 * (16 * 8 + 15), 16, ST, _tma(16, 8, 1)),
    ("s32-ring-a1", "ring", 2 * (8 * 20 + 1), 32, ST, _tma(8, 8, 1)),
    ("s32-rosen-a7", "rosenbrock", 2 * (8 * 20 + 7), 32, ST, _tma(8, 8, 1)),
    ("s64-iso-a1", "gauss_iso", 2 * (4 * 40 + 1), 64, ST, _tma(4, 8, 1)),
    ("s64-rosen-a3", "rosenbrock", 2 * (4 * 40 + 3), 64, ST, _tma(4, 8, 1)),
    ("s128-ring-a1", "ring", 2 * (2 * 150 + 1), 128, ST, _tma(2, 8, 0)),
    ("s128-rosen-a1", "rosenbrock", 2 * (2 * 150 + 1) + 1, 128, ST, _tma(2, 8, 0)),
    ("s22-ring", "ring", 301, 22, ST, _tma(16, 0, 0)),
    ("s44-iso", "gauss_iso", 307, 44, ST, _tma(8, 0, 0)),
    ("s96-iso", "gauss_iso", 403, 96, ST, _tma(2, 0, 0)),
    ("s200-rosen", "rosenbrock", 611, 200, ST, _tma(1, 0, 0)),
    ("s256-ring", "ring", 1029, 256, ST, _tma(1, 8, 0)),
    ("s256-rosen", "rosenbrock", 1030, 256, ST, _tma(1, 8, 0)),
    ("s320-iso", "gauss_iso", 1001, 320, ST, _tma(1, 0, 0)),
    ("s400-iso", "gauss_iso", 1203, 400, ST, _tma(1, 0, 0, 14)),
    ("s768-rosen", "rosenbrock", 1603, 768, ST, _tma(1, 0, 0, 8)),
    ("de24-iso", "gauss_iso", 301, 24, DE, _tma(8, 0, 0)),
    ("de32-rosen", "rosenbrock", 333, 32, DE, _tma(4, 0, 0)),
    ("de64-ring", "ring", 413, 64, DE, _tma(2, 0, 0)),
    ("de128-iso", "gauss_iso", 517, 128, DE, _tma(1, 0, 0)),
    ("de256-ring", "ring", 1031, 256, DE, _tma(1, 8, 0, 13)),
    ("sn16-iso", "gauss_iso", 301, 16, SN, _tma(8, 0, 0)),
    ("sn32-ring", "ring", 405, 32, SN, _tma(4, 0, 0)),
    ("sn64-rosen", "rosenbrock", 413, 64, SN, _tma(2, 0, 0)),
    ("sn96-iso", "gauss_iso", 517, 96, SN, _tma(1, 0, 0)),
    ("sn200-ring", "ring", 806, 200, SN, _tma(1, 0, 0, 13)),
    ("sn256-iso", "gauss_iso", 1030, 256, SN, _tma(1, 8, 0, 10)),
    ("s37-iso-generic", "gauss_iso", 301, 37, ST, "generic G=16"),
]


def _check_against_oracle(s, o, last, omoves, target):
    stretch_only = all(m.kind == "stretch" for m, _ in omoves)
    snooker = any(m.kind == "snooker" for m, _ in omoves)
    if stretch_only:
        assert np.array_equal(last.coords, o.coords)
        np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=1e-11, atol=1e-11)
    else:
        tol = 1e-6 if snooker else 1e-11  # as test_gpu_parity.test_against_oracle
        np.testing.assert_allclose(last.coords, o.coords, rtol=tol, atol=tol)
        np.testing.assert_allclose(last.log_prob, o.log_prob, rtol=max(tol, 1e-11), atol=max(100 * tol, 1e-11))
    assert np.array_equal(s._engine.naccepted(), o.naccepted.astype(np.uint64))
    # the kernel's log-probability of its own coordinates, independent of any drift between the chains
    np.testing.assert_allclose(last.log_prob, target(last.coords), rtol=1e-11, atol=1e-11)


def _run_row(model, N, D, omoves, nsteps, seed, options=(), target=None, p0=None):
    if target is None:
        target, p0 = T.make_config(model, N, D)
    o = rb.OracleSampler(N, D, target, omoves, seed=seed)
    o.set_state(p0)
    o.run(nsteps)
    s = emcee_b200.EnsembleSampler(
        N, D, device_model(model, target=target), moves=device_moves(move_rows_from_oracle(omoves)), seed=seed
    )
    for k, v in options:
        s._engine.set_option(k, v)
    last = s.run_mcmc(p0, nsteps, store=False, skip_initial_state_check=True)
    _check_against_oracle(s, o, last, omoves, target)
    return s, last


@pytest.mark.parametrize("model,N,D,omoves,variant", [c[1:] for c in CELLS], ids=[c[0] for c in CELLS])
def test_tma_cell(model, N, D, omoves, variant):
    s, _ = _run_row(model, N, D, omoves, 4, seed=0x7A1 + N + D)
    assert s._engine.last_kernel_variant() == variant


def test_batch_crossing():
    """More than G tiles per warp at G = 16 (stretch, register path) and G = 32 (DE, R = 1): every warp
    tabulates the walker metadata of a new batch of G tiles inside its tile loop."""
    sm = _sm_count()
    for model, D, omoves, R, variant in (
        ("gauss_iso", 128, ST, 2, _tma(2, 8, 0)),
        ("rosenbrock", 128, DE, 1, _tma(1, 0, 0)),
    ):
        G = 32 // R
        a_count = R * (G * 16 * sm + 2 * sm) + 1  # > G tiles for every one of the 16 warps of every SM
        N = 2 * a_count
        s, _ = _run_row(model, N, D, omoves, 2, seed=0xC805 + D)
        assert s._engine.last_kernel_variant() == variant


OPTION_SHAPES = [
    # model, N, D, moves, variant at tma_rows = 2 with own_reg = 1 / 0, at tma_rows = 1
    ("rosenbrock", 334, 32, ST, _tma(8, 8, 1), _tma(8, 8, 0), _tma(8, 8, 1)),
    ("ring", 1203, 400, ST, _tma(1, 0, 0, 14), _tma(1, 0, 0, 14), "generic G=32"),
    ("gauss_iso", 517, 96, SN, _tma(1, 0, 0), _tma(1, 0, 0), "generic G=32"),
]


@pytest.mark.parametrize("model,N,D,omoves,v_own,v_noown,v_short", OPTION_SHAPES, ids=["s32-rosen", "s400-ring", "sn96-iso"])
def test_options_bit_identical(model, N, D, omoves, v_own, v_noown, v_short):
    """One shape under tma_rows = 2 / 1 / 0 and tma_own_reg = 1 / 0: the same cell or the generic kernel, the
    same bits (stretch) -- long rows with tma_rows = 1 fall back to the generic kernel."""
    G = 4
    while G < 32 and G * 4 < D:
        G *= 2
    expect = {
        (2, 1): v_own,
        (2, 0): v_noown,
        (1, 1): v_short,
        (1, 0): v_short if v_short.startswith("generic") else v_noown,
        (0, 1): "generic G=%d" % G,
    }
    runs = []
    for (tma, own), variant in expect.items():
        s, last = _run_row(model, N, D, omoves, 3, seed=0x0971 + D, options=(("tma_rows", tma), ("tma_own_reg", own)))
        assert s._engine.last_kernel_variant() == variant, (tma, own)
        runs.append((last.coords.copy(), last.log_prob.copy(), s._engine.naccepted()))
    if all(m.kind == "stretch" for m, _ in omoves):
        for r in runs[1:]:
            assert np.array_equal(r[0], runs[0][0]) and np.array_equal(r[2], runs[0][2])


def _indefinite(D, seed=3):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    ev = np.linspace(1.0, 2.0, D) * np.where(np.arange(D) % 3 == 2, -0.25, 1.0)
    A = (q * ev) @ q.T
    return 0.5 * (A + A.T)


DENSE_CASES = [
    # id, N, D, mean, options, icov kind
    ("D20", 301, 20, False, (), "random"),
    ("D20-mean", 301, 20, True, (), "random"),
    ("D37", 301, 37, False, (), "random"),
    ("D37-mean", 301, 37, True, (), "random"),
    ("D136", 401, 136, False, (), "random"),
    ("D136-mean", 401, 136, True, (), "random"),
    ("D64-dmma-off", 301, 64, True, (("dense_dmma", 0),), "random"),
    ("D16-indefinite", 301, 16, False, (), "indefinite"),
]


@pytest.mark.parametrize("N,D,mean,options,icov", [c[1:] for c in DENSE_CASES], ids=[c[0] for c in DENSE_CASES])
def test_dense_cuda_core(N, D, mean, options, icov):
    """The dense Gaussian on the CUDA-core generic kernel under the stretch move (model_logprob<GAUSS_DENSE>)."""
    base, p0 = T.make_config("gauss_dense", N, D)
    A = base.icov if icov == "random" else _indefinite(D)
    mu = np.linspace(-0.7, 1.3, D) if mean else None
    target = T.GaussDense(A, mu)
    G = 4
    while G < 32 and G * 4 < D:
        G *= 2
    s, last = _run_row("gauss_dense", N, D, ST, 5, seed=0xDE5 + D, options=options, target=target, p0=p0)
    assert s._engine.last_kernel_name() == "generic"
    assert s._engine.last_kernel_variant() == "generic G=%d" % G
    # the stand-alone log-prob kernel takes the same path as the half-step
    np.testing.assert_allclose(s.compute_log_prob(last.coords)[0], last.log_prob, rtol=1e-13, atol=1e-13)


# ---- grouped dense_dmma ----------------------------------------------------------------------------------------
class LaunchModel(object):
    """Host-side mirror of run_steps (step.cu) for one single-GPU engine with a dense-Gaussian model: predicts the
    launch count of a stepping call (eb_last_step_timing) and the largest / last dense_dmma group.  Keeps the
    engine's split-table cache (64-step look-ahead, tables of at most 512 steps) across calls."""

    def __init__(self, N, seed, sm):
        self.N, self.seed, self.sm = N, seed, sm
        self.cap = max(1, min((64 << 20) // (N * 4), 512))
        self.tbl = None  # (step0, [info of each step])
        self.have_shift = False

    def call(self, omoves, weights, step, nsteps, group, sync_every=0, moments_every=0):
        w = np.asarray(weights, dtype=np.float64)
        w = w / w.sum()
        info = lambda k: (omoves[k].nsplits, omoves[k].randomize_split)
        pick = lambda st: px.move_choice(self.seed, st, w) if len(omoves) > 1 else 0
        launches, nhalf_max, last = 0, 0, None
        done = 0
        while done < nsteps:
            chunk = min(nsteps - done, self.cap)
            picks = [pick(step + k) for k in range(chunk)]
            hit = False
            if self.tbl is not None:
                t0, ti = self.tbl
                hit = step >= t0 and step + chunk <= t0 + len(ti)
                hit = hit and all(ti[step - t0 + k] == info(picks[k]) for k in range(chunk))
            if not hit:
                build = min(self.cap, max(chunk, 64))
                self.tbl = (step, [info(pick(step + k)) for k in range(build)])
                launches += 1
            grp_n, grp_max, grp_move = 0, 0, None

            def flush():
                nonlocal grp_n, grp_max, launches, nhalf_max, last
                if grp_n:
                    launches += 1
                    nhalf_max = max(nhalf_max, grp_n)
                    last = ("dmma", grp_max)
                grp_n, grp_max = 0, 0

            for k in range(chunk):
                mi = picks[k]
                mv = omoves[mi]
                P = mv.nsplits
                sizes = [(self.N - j + P - 1) // P for j in range(P)]
                if mv.kind == "stretch":
                    if grp_move is not None and grp_move != mi:
                        flush()
                    grp_move = mi
                    for split in range(P):
                        grp_n += 1
                        grp_max = max(grp_max, sizes[split])
                        if grp_n >= group and split + 1 < P:
                            flush()
                    moments_now = moments_every > 0 and (step + 1) % moments_every == 0
                    host_event = moments_now or (sync_every > 0 and (done + k + 1) % sync_every == 0)
                    if host_event or k + 1 == chunk or grp_n >= group:
                        flush()
                else:
                    if grp_move is not None:
                        flush()
                    launches += P
                    last = ("generic", None)
                step += 1
                if moments_every > 0 and step % moments_every == 0:
                    launches += 2 if self.have_shift else 3
                    self.have_shift = True
            done += chunk
        if last is not None and last[0] == "dmma":
            grid = min((last[1] + 7) // 8, self.sm)
            variant = "dense_dmma nhalf_max=%d grid=%d" % (nhalf_max, grid)
        else:
            variant = None
        return launches, variant


class GroupedRun(object):
    """One device sampler, the oracle and the launch model, driven through the same sequence of calls."""

    def __init__(self, N, D, omoves, seed, sm, mean=False, options=()):
        base, self.p0 = T.make_config("gauss_dense", N, D)
        mu = np.linspace(-1.0, 0.5, D) if mean else None
        self.target = T.GaussDense(base.icov, mu)
        self.omoves = omoves
        self.o = rb.OracleSampler(N, D, self.target, omoves, seed=seed)
        self.o.set_state(self.p0)
        dm = device_moves(move_rows_from_oracle(omoves))
        self.s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(base.icov, mu), moves=dm, seed=seed)
        for k, v in options:
            self.s._engine.set_option(k, v)
        self.model = LaunchModel(N, seed, sm)
        self.state = self.p0
        self.step = 0
        self.moments_every = 0
        self.outputs = []  # everything the device returned, in call order (bitwise comparison between runs)

    def _expect(self, nsteps, group, sync_every=0):
        launches, variant = self.model.call(
            [m for m, _ in self.omoves], [w for _, w in self.omoves], self.step, nsteps, group, sync_every,
            self.moments_every
        )
        self.step += nsteps
        return launches, variant

    def _check(self, launches, variant):
        eng = self.s._engine
        assert eng.last_step_timing()[1] == launches
        if variant is not None:
            assert eng.last_kernel_variant() == variant

    def _compare(self, coords, log_prob):
        if all(m.kind == "stretch" for m, _ in self.omoves):
            assert np.array_equal(coords, self.o.coords)
        else:
            np.testing.assert_allclose(coords, self.o.coords, rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(log_prob, self.o.log_prob, rtol=1e-11, atol=1e-11)

    def run_store_false(self, nsteps, group):
        self.s._engine.set_option("dmma_group", group)
        expect = self._expect(nsteps, group)
        self.state = self.s.run_mcmc(self.state, nsteps, store=False, skip_initial_state_check=True)
        self._check(*expect)
        self.o.run(nsteps)
        self._compare(self.state.coords, self.state.log_prob)
        self.outputs += [self.state.coords.copy(), self.state.log_prob.copy()]

    def run_store_thinned(self, nstored, thin_by, group):
        self.s._engine.set_option("dmma_group", group)
        self.s.reset()
        expect = self._expect(nstored * thin_by, group, sync_every=thin_by)
        self.state = self.s.run_mcmc(self.state, nstored, store=True, thin_by=thin_by, skip_initial_state_check=True)
        self._check(*expect)
        chain, lp = self.s.get_chain(), self.s.get_log_prob()
        for k in range(nstored):
            self.o.run(thin_by)
            self._compare(chain[k], lp[k])
        self.outputs += [chain.copy(), lp.copy()]

    def run_stepwise(self, nsteps, group):
        self.s._engine.set_option("dmma_group", group)
        k = 0
        for st in self.s.sample(self.state, iterations=nsteps, store=False, skip_initial_state_check=True):
            expect = self._expect(1, group)
            self._check(*expect)
            self.o.run(1)
            self._compare(st.coords, st.log_prob)
            self.outputs += [st.coords.copy(), st.log_prob.copy()]
            k += 1
        assert k == nsteps
        self.state = st

    def finish(self):
        eng = self.s._engine
        assert np.array_equal(eng.naccepted(), self.o.naccepted.astype(np.uint64))
        # the stand-alone log-prob kernel runs the same tensor-pipe block as the half-step (a walker last moved by
        # a DE step got its log-prob from the generic kernel: another summation order)
        fresh = self.s.compute_log_prob(self.state.coords)[0]
        if all(m.kind == "stretch" for m, _ in self.omoves):
            assert np.array_equal(fresh, self.state.log_prob)
        else:
            np.testing.assert_allclose(fresh, self.state.log_prob, rtol=1e-12, atol=1e-12)
        self.outputs.append(eng.naccepted())


def _same_bits(a, b):
    assert len(a.outputs) == len(b.outputs)
    for x, y in zip(a.outputs, b.outputs):
        assert np.array_equal(x, y)


GROUPED = [
    # id, D, N as (SM multiple, offset), nsplits, mean, the dmma_group of each call
    ("D64-small-p2", 64, (8, -3), 2, False, (2, 64, 3, 4)),
    ("D40-small-p3", 40, (8, -5), 3, True, (3, 4, 2, 64)),
    ("D128-large-p3", 128, (64, 5), 3, True, (4, 2, 64, 3)),
    ("D16-large-p2", 16, (64, 7), 2, False, (64, 3, 2, 4)),
]


def _grouped_script(r, groups):
    r.run_store_false(5, groups[0])
    r.run_store_thinned(4, 3, groups[1])
    r.run_stepwise(3, groups[2])
    r.run_store_false(7, groups[3])
    r.finish()


@pytest.mark.parametrize("D,nm,P,mean,groups", [c[1:] for c in GROUPED], ids=[c[0] for c in GROUPED])
def test_grouped_dense_dmma(D, nm, P, mean, groups):
    """Several calls with different dmma_group values on one engine (the grid-barrier counter carries over
    between launches), through run_mcmc(store=False), run_mcmc(store=True, thin_by=3) and sample() one step at a
    time: bit-identical to the oracle and to dmma_group = 1, with the launch count of the flush rule."""
    sm = _sm_count()
    N = nm[0] * sm + nm[1]
    assert N % P != 0
    om = [(rb.Stretch(nsplits=P), 1.0)]
    seed = 0x6A0 + D
    ref = GroupedRun(N, D, om, seed, sm, mean)
    _grouped_script(ref, (1, 1, 1, 1))
    runs = [GroupedRun(N, D, om, seed, sm, mean)]
    if D == 64:
        runs.append(GroupedRun(N, D, om, seed, sm, mean, options=(("dmma_stagger", 0),)))
        runs.append(GroupedRun(N, D, om, seed, sm, mean, options=(("pdl", 0),)))
    for r in runs:
        _grouped_script(r, groups)
        _same_bits(r, ref)


def test_grouped_dense_dmma_long_run():
    """A run longer than one 512-step chunk of split tables in grouped launches."""
    sm = _sm_count()
    N, D = 8 * sm - 3, 32
    om = [(rb.Stretch(), 1.0)]
    ref = GroupedRun(N, D, om, 0x10A6, sm)
    ref.run_store_false(530, 1)
    r = GroupedRun(N, D, om, 0x10A6, sm)
    r.run_store_false(530, 64)
    r.run_store_false(3, 4)
    ref.run_store_false(3, 1)
    r.finish()
    ref.finish()
    _same_bits(r, ref)


SCHEDULES = [
    ("stretch-de", lambda P: [(rb.Stretch(nsplits=P), 0.5), (rb.DE(nsplits=P), 0.5)]),
    ("two-stretch", lambda P: [(rb.Stretch(a=2.0, nsplits=P), 0.5), (rb.Stretch(a=1.6, nsplits=P), 0.5)]),
]


@pytest.mark.parametrize("make", [c[1] for c in SCHEDULES], ids=[c[0] for c in SCHEDULES])
@pytest.mark.parametrize("P", [2, 3])
def test_grouped_dense_dmma_mixed_schedule(make, P):
    """A move change flushes the group (a DE step runs on the generic kernel; two StretchMoves with different a
    are different move objects)."""
    sm = _sm_count()
    N, D = 64 * sm + 1, 48
    om = make(P)
    ref = GroupedRun(N, D, om, 0x3C1 + P, sm, mean=True)
    _grouped_script(ref, (1, 1, 1, 1))
    r = GroupedRun(N, D, om, 0x3C1 + P, sm, mean=True)
    _grouped_script(r, (4, 3, 2, 64))
    _same_bits(r, ref)


def test_grouped_dense_dmma_with_moments():
    """enable_moments(2): a moment accumulation after every second step ends the group before it."""
    sm = _sm_count()
    N, D = 8 * sm - 1, 56
    om = [(rb.Stretch(nsplits=3), 1.0)]
    out = []
    for group in (1, 4):
        r = GroupedRun(N, D, om, 0x30E, sm)
        r.s.enable_moments(2)
        r.moments_every = 2
        r.run_store_false(9, group)
        r.run_stepwise(3, group)
        r.run_store_false(4, 1 if group == 1 else 64)
        r.finish()
        mean, cov, n = r.s.moments()
        assert n == N * 8
        out.append((r, mean, cov))
    _same_bits(out[1][0], out[0][0])
    assert np.array_equal(out[1][1], out[0][1]) and np.array_equal(out[1][2], out[0][2])
