"""The Metropolis accept decision of the half-steps whose inputs come from outside the kernel -- a user
log-probability function (``HostFunction``, ``CudaArrayFunction``, ``CudaGraphFunction``), a user proposal
(``RedBlueMove.get_proposal``, ``MHMove(HostProposal / CudaArrayProposal)``) and ``KDEMove`` -- against exact
ladders of ``lp_old`` (``accept_external_exact.py``).

Protocol (that of ``test_gpu_accept_exact.py``, with rungs in place of bisection):

1. observation run: every walker starts at ``log_prob = -inf``, so one step accepts every finite proposal; the state
   then holds each proposal and the ``lp_new`` the device used, bit for bit.  The functions log their inputs and
   outputs; the taps (``debug_taps``) give stretch's zz and the KDE factors;
2. per split k: the walkers of splits below k start at ``-inf`` again, so split k sees the same complement, and every
   walker of split k starts at an ``lp_old`` of its ladder.  Nine runs with the same ``(seed, step)`` rotate the
   rungs, so that every walker meets every rung.  Before anything is checked, split k's proposals must be the
   observation run's: every accepted walker of split k holds the observed proposal and ``lp_new``, and a logging
   function saw the observed rows;
3. the mask ``eng.step`` returns is the decision: a rung the rule of ``accept_external_exact`` decides must go that
   way.

Inputs of the ladders: ``lp_new`` is the observed value (exact: it is the device's own double).  The factor is exact
where the device did not compute it -- a user factor, a tapped KDE factor, 0 for DE, Walk and Gaussian -- and the
band then is the device's log(u) alone, 1 ulp.  Where the device computed it (stretch: ``(D - 1) log zz``, snooker:
the bound of ``accept_exact.snooker_factor``) the band adds its bound, and the rungs are spread over it
(``band_spacing``).

User moves choose their inputs: half the walkers get an order-splitting triple (``|lp_new| ~ 2^41``, a factor whose
low bits one order rounds away) and one extra run at the triple's ``lp_old``, where the red-blue and the MH order
fall on opposite sides of the band; the other half get "fine" inputs under which every double next to ``ln u`` is a
rung, so the decision is pinned to one ulp of ``ln u``.  A kernel that used the other order fails the triple runs.

Rows (three (seed, step) pairs each; ``last_kernel_name`` / ``last_kernel_variant`` asserted on every row):

===========================  =====================================================================================
host-{st,de,sn,walk,gauss}   ``HostFunction`` x stretch, DE, snooker, Walk, Gaussian at ndim 5 and 37 (G = 4, 16)
host-st-nsplits3-odd         stretch, three splits of an odd ensemble: split starts and sizes uneven
cuda-st-strided / -sn-side   ``CudaArrayFunction``: a strided result; a late result on a side stream (v3)
graph-{st,de,kde}            ``CudaGraphFunction`` with a strided x and lp; KDE: the last split (its factors tapped)
user-rb-{numpy,torch}-*      a user ``RedBlueMove`` under a device ``GaussianIso`` (integer rows, exact lp_new) and
                             under a ``HostFunction``: the red-blue order
user-mh-{host,cuda}-*        ``MHMove(HostProposal / CudaArrayProposal)``, the same two models: the MH order
kde-iso                      ``KDEMove`` under ``GaussianIso``: the last split, tapped factors
blobs-host-st                a ``HostFunction`` with blobs: accepted walkers hold their proposal's record, rejected
                             ones their old one
===========================  =====================================================================================

Each path prints how far from ``ln u`` (in its ulps) the device's decisions reach into each side: the largest
``ln u - lnpdiff`` it accepted and the largest ``lnpdiff - ln u`` it rejected.
"""
import time

import numpy as np
import pytest

import accept_exact as AX
import accept_external_exact as EX
from oracle import philox as px
from oracle import redblue as rb

import emcee_b200
from emcee_b200 import models, moves

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SEED_STEPS = [(0x5EED, 0), (0xB200, 17), (7, 123456789)]
REACH = {}  # path -> [largest accepted ln u - lnpdiff, largest rejected lnpdiff - ln u] in ulps of ln u


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for path in sorted(REACH):
        a, r = REACH[path]
        print("%-22s accepted down to %.3g ulps below ln u, rejected up to %.3g ulps above" % (path, a, r))


def _iso(x):
    return -0.5 * np.sum(x * x, axis=1)


# ---- logging functions ---------------------------------------------------------------------------------------
class HostLog(object):
    """A numpy log-probability that logs every call's rows and values.  ``table`` (row bytes -> lp) overrides the
    default -0.5 |x|^2 for the rows it holds; ``blob`` adds a blob per row."""

    def __init__(self, blob=False):
        self.calls, self.table, self.blob = [], {}, blob

    def __call__(self, x):
        lp = _iso(x)
        for j, row in enumerate(x):
            lp[j] = self.table.get(row.tobytes(), lp[j])
        self.calls.append((x.copy(), lp.copy()))
        if self.blob:
            return [(float(v), float(b)) for v, b in zip(lp, blob_of(x))]
        return lp


def blob_of(x):
    return 3.0 * np.asarray(x)[..., 0] + 1.0


class CudaLog(object):
    """A torch log-probability that logs clones of its rows and values; ``how``: "strided" returns a strided view,
    "side" computes on a side stream after a delay and names that stream (interface v3)."""

    def __init__(self, how):
        self.how, self.calls = how, []

    def __call__(self, rows):
        x = torch.as_tensor(rows, device="cuda")
        if self.how == "side":
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(1_000_000)  # late: the engine must wait for it
                lp = -0.5 * (x * x).sum(dim=1)
                self.calls.append((x.clone(), lp.clone()))
            return _V3(lp, side)
        lp = -0.5 * (x * x).sum(dim=1)
        buf = torch.empty(2 * x.shape[0], dtype=torch.float64, device="cuda")
        buf[::2] = lp
        self.calls.append((x.clone(), lp.clone()))
        return buf[::2]

    def logged(self):
        torch.cuda.synchronize()
        return [(a.cpu().numpy(), b.cpu().numpy()) for a, b in self.calls]


class _V3(object):
    def __init__(self, t, stream):
        self.t = t
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, version=3, stream=stream.cuda_stream)


def _graph_capture(D):
    from test_gpu_graph_function import Capture, iso_columns

    return Capture(iso_columns, D, strided=True)


# ---- user moves: inputs chosen per walker ------------------------------------------------------------------------
class Plan(object):
    """The inputs of a user-move row for one (seed, step): per walker its proposal row ``q``, ``lp_new`` (exact),
    factor ``F``, whether it carries an order-splitting triple, and the triple's ``lp_old``."""

    def __init__(self, N, D):
        self.q = np.zeros((N, D))
        self.lp = np.zeros(N)
        self.F = np.zeros(N)
        self.triple = np.zeros(N, dtype=bool)
        self.L = np.zeros(N)
        self.by_row = {}  # X0 row bytes -> walker


def make_plan(X0, sets, seed, step, order, model, rng):
    """Triples on even ranks, fine inputs on odd ones.  ``model`` "iso": integer rows, lp_new = -|q|^2 / 2 exactly
    (a device GaussianIso); "host": random rows, lp_new chosen and returned by the function's table."""
    N, D = X0.shape
    p = Plan(N, D)
    p.by_row = {X0[w].tobytes(): w for w in range(N)}
    for k, act in enumerate(sets):
        ranks = np.arange(len(act))
        lnu = EX.ln_u(AX.accept_u(seed, step, k, ranks))
        tri = ranks % 2 == 0
        t0 = EX.nearest(lnu)
        for j, w in enumerate(act):
            if model == "iso":
                if tri[j]:
                    q0 = int(np.floor(np.sqrt(2.0**42 * rng.uniform(1.05, 1.9))))
                    p.q[w, 0] = q0
                    p.q[w, 1] = w + 1  # rows differ even where q0 repeats
                elif order == "mh":
                    p.q[w] = 0.0  # lp_new = 0: lp_new - lp_old stays small
                else:
                    p.q[w] = rng.integers(-3, 4, D)
                    p.q[w, 1] = w + 1
                p.lp[w] = -0.5 * float(np.sum(p.q[w] * p.q[w]))
            else:
                p.q[w] = rng.standard_normal(D)
                if tri[j]:
                    p.lp[w] = -(2.0**41) * rng.uniform(1.01, 1.99)
                elif order == "mh":
                    p.lp[w] = -1e-3 * abs(t0[j]) * rng.uniform()
                else:
                    p.lp[w] = -0.5 * float(np.sum(p.q[w] ** 2))
        w_t, w_f = act[tri], act[~tri]
        F_t, _, L_t = EX.order_splitting_triples([lnu[j] for j in np.flatnonzero(tri)], p.lp[w_t])
        p.F[w_t], p.L[w_t], p.triple[w_t] = F_t, L_t, True
        p.F[w_f] = EX.fine_factors([lnu[j] for j in np.flatnonzero(~tri)], p.lp[w_f], order, rng)
    return p


class NumpyPlanMove(moves.RedBlueMove):
    """A user red-blue move whose proposals and factors come from a Plan, looked up by the walker's row."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.plan, self.calls = None, []

    def _lookup(self, S):
        w = np.array([self.plan.by_row[row.tobytes()] for row in S], dtype=np.int64)
        self.calls.append(w)
        return self.plan.q[w].copy(), self.plan.F[w].copy()

    def get_proposal(self, s, c, random):
        return self._lookup(s)


class TorchPlanMove(moves.CudaArrayRedBlueMove):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.plan, self.calls = None, []

    def get_proposal(self, s, c, random):
        S = torch.as_tensor(s, device="cuda").cpu().numpy()
        q, F = NumpyPlanMove._lookup(self, S)
        return torch.as_tensor(q, device="cuda"), torch.as_tensor(F, device="cuda")


class MHPlan(object):
    """An MHMove proposal function from a Plan: walker w proposes q[w] with factor F[w]."""

    def __init__(self, cuda):
        self.cuda, self.plan, self.calls = cuda, None, []

    def __call__(self, coords, random):
        self.calls.append(len(coords) if not self.cuda else coords.__cuda_array_interface__["shape"][0])
        if self.cuda:
            return torch.as_tensor(self.plan.q, device="cuda"), torch.as_tensor(self.plan.F, device="cuda")
        return self.plan.q.copy(), self.plan.F.copy()


# ---- rows --------------------------------------------------------------------------------------------------------
def _callback_variant(D, where):
    G = 4
    while G < 32 and G * 4 < D:
        G <<= 1
    return "callback G=%d where=%s" % (G, where)


BUILTIN = {
    "st": (lambda: moves.StretchMove(), "stretch"),
    "de": (lambda: moves.DEMove(), "zero"),
    "sn": (lambda: moves.DESnookerMove(), "snooker"),
    "walk": (lambda: moves.WalkMove(), "zero"),
    "gauss": (lambda: moves.GaussianMove(0.3), "zero"),
    "st3": (lambda: moves.StretchMove(nsplits=3), "stretch"),
    "kde": (lambda: moves.KDEMove(), "kde"),
}


def _rows():
    rows = []
    for D, N in ((5, 66), (37, 83)):
        for mv in ("st", "de", "sn", "walk", "gauss"):
            rows.append(("host-%s-D%d" % (mv, D), dict(N=N, D=D, model="host", move=mv)))
    rows.append(("host-st-nsplits3-odd", dict(N=67, D=5, model="host", move="st3")))
    rows.append(("cuda-st-strided", dict(N=66, D=5, model="cuda-strided", move="st")))
    rows.append(("cuda-sn-side", dict(N=66, D=5, model="cuda-side", move="sn")))
    for mv in ("st", "de", "kde"):
        rows.append(("graph-%s" % mv, dict(N=66, D=5, model="graph", move=mv)))
    for how in ("numpy", "torch"):
        for model in ("iso", "host"):
            rows.append(("user-rb-%s-%s" % (how, model), dict(N=66, D=5, model=model, move="user-" + how)))
    for how in ("host", "cuda"):
        for model in ("iso", "host"):
            rows.append(("user-mh-%s-%s" % (how, model), dict(N=65, D=5, model=model, move="mh-" + how)))
    rows.append(("kde-iso", dict(N=66, D=5, model="iso", move="kde")))
    rows.append(("blobs-host-st", dict(N=66, D=5, model="host-blobs", move="st")))
    return rows


ROWS = [(name, dict(spec, id=name)) for name, spec in _rows()]


def _build(spec):
    """(sampler, logging function or None, user-move object or None, factor kind, order, variant check)."""
    N, D, model, mv = spec["N"], spec["D"], spec["model"], spec["move"]
    fn, umove = None, None
    if mv.startswith("user-"):
        umove = (NumpyPlanMove if mv == "user-numpy" else TorchPlanMove)()
        move, kind, order = umove, "user", "red_blue"
    elif mv.startswith("mh-"):
        umove = MHPlan(mv == "mh-cuda")
        move = moves.MHMove((moves.CudaArrayProposal if umove.cuda else moves.HostProposal)(umove))
        kind, order = "user", "mh"
    else:
        make, kind = BUILTIN[mv]
        move, order = make(), "red_blue"
    if model == "iso":
        lpf = models.GaussianIso()
    elif model in ("host", "host-blobs"):
        fn = HostLog(blob=model == "host-blobs")
        lpf = models.HostFunction(fn, vectorize=True, blobs_dtype=np.float64 if fn.blob else None)
    elif model.startswith("cuda-"):
        fn = CudaLog(model.split("-")[1])
        lpf = models.CudaArrayFunction(fn)
    else:
        lpf = models.CudaGraphFunction(_graph_capture(D))
    s = emcee_b200.EnsembleSampler(N, D, lpf, moves=move, seed=1)
    where = {"iso": None, "host": "host", "host-blobs": "host", "cuda-strided": "device", "cuda-side": "device",
             "graph": "graph"}[model]
    if umove is not None:
        ud = "host" if mv in ("user-numpy", "mh-host") else "device"

        def check(eng):
            assert eng.last_kernel_variant() == "user_move where=%s" % ud, eng.last_kernel_variant()
    elif where is None:  # KDE under a device model
        def check(eng):
            assert eng.last_kernel_name() == "kde" and eng.last_kernel_variant().startswith("kde tpc=")
    else:
        def check(eng):
            assert eng.last_kernel_name() == "callback"
            assert eng.last_kernel_variant() == _callback_variant(D, where), eng.last_kernel_variant()
    return s, fn, umove, kind, order, check


def _sets(desc, seed, step, N):
    if desc["kind"] in ("gaussian", "user_mh"):  # every walker in one set, accept uniform indexed by walker
        return [np.arange(N)]
    inds = px.split_assignment(seed, step, N, desc["nsplits"], desc["randomize_split"])
    return [np.flatnonzero(inds == j) for j in range(desc["nsplits"])]


def _logged(fn):
    if fn is None:
        return None
    return fn.logged() if isinstance(fn, CudaLog) else [(a.copy(), b.copy()) for a, b in fn.calls]


def _factors(kind, D, seed, step, k, act, state, X1, taps, sets, desc, umove):
    """(F doubles, dF) of split k's walkers: dF = 0 where F is the device's own double."""
    n = len(act)
    if kind == "zero":
        return np.zeros(n), np.zeros(n)
    if kind == "user":
        return umove.plan.F[act].copy(), np.zeros(n)
    if kind == "kde":
        assert np.array_equal(taps["active"], act)
        return taps["scalar"].copy(), np.zeros(n)
    F, dF = np.zeros(n), np.zeros(n)
    if kind == "stretch":
        zz = AX.stretch_zz(desc["p0"], seed, step, k, np.arange(n))
        for j in range(n):
            f, df = AX.stretch_factor(zz[j], D)
            F[j], dF[j] = float(f), df
        return F, dF
    omove = rb.Snooker(gammas=desc["p0"])
    o = rb.OracleSampler(state.shape[0], D, None, [(omove, 1.0)], seed=seed)
    o.coords = state
    with np.errstate(all="ignore"):
        o._snooker(omove, state[act], sets[:k] + sets[k + 1:], step, k)
    for j, w in enumerate(act):
        f, df = AX.snooker_factor(state[w], state[o.taps["z"][j]], X1[w], D)
        F[j], dF[j] = float(f), df
    return F, dF


@pytest.mark.parametrize("spec", [r[1] for r in ROWS], ids=[r[0] for r in ROWS])
def test_accept_external_exact(spec):
    t0 = time.time()
    s, fn, umove, kind, order, check = _build(spec)
    N, D = spec["N"], spec["D"]
    eng = s._engine
    sched = s._schedule()
    desc = sched[0][0]
    path = spec["id"]
    if kind in ("stretch", "snooker", "kde"):
        eng.set_option("debug_taps", 1)
    reach = REACH.setdefault(path, [0.0, 0.0])
    blobs = fn is not None and getattr(fn, "blob", False)
    old_blobs = -1e6 - np.arange(N, dtype=np.float64) if blobs else None
    ndec = 0
    for seed, step in SEED_STEPS:
        rng = np.random.default_rng([seed, step, N, D])
        X0 = rng.standard_normal((N, D))
        sets = _sets(desc, seed, step, N)
        if umove is not None:
            umove.plan = make_plan(X0, sets, seed, step, order, spec["model"], rng)
            if fn is not None:
                fn.table = {umove.plan.q[w].tobytes(): umove.plan.lp[w] for w in range(N)}

        def run(lp):
            if fn is not None:
                fn.calls = []
            eng.set_state(X0, lp, old_blobs)
            eng.set_rng(seed, step)
            return eng.step(sched, 1)

        # 1. observation
        minus_inf = np.full(N, -np.inf)
        acc = run(minus_inf)
        check(eng)
        X1, lp1 = eng.get_state()
        assert acc.all() and np.all(np.isfinite(lp1)), "a proposal was not accepted: the state does not show it"
        taps = eng.debug_taps() if kind in ("stretch", "kde") else None
        obs_log = _logged(fn)
        if obs_log is not None:  # the device used what the function returned, for the row it was given
            seen = {x.tobytes(): v for xs, lps in obs_log for x, v in zip(xs, lps)}
            got = np.array([seen[X1[w].tobytes()] for w in range(N)])
            assert got.tobytes() == lp1.tobytes(), "lp_new differs from the function's value for its row"
        if umove is not None:
            assert X1.tobytes() == umove.plan.q.tobytes() and np.array_equal(lp1, umove.plan.lp)
        if kind == "stretch" and taps is not None:
            last = sets[-1]
            zz = AX.stretch_zz(desc["p0"], seed, step, len(sets) - 1, np.arange(len(last)))
            assert np.array_equal(taps["active"], last) and taps["scalar"].tobytes() == zz.tobytes()
        splits = [len(sets) - 1] if kind == "kde" else range(len(sets))
        for k in splits:
            act = sets[k]
            ranks = np.arange(len(act))
            lnu = EX.ln_u(AX.accept_u(seed, step, k, ranks))
            state = X0.copy()
            for j in range(k):
                state[sets[j]] = X1[sets[j]]
            F, dF = _factors(kind, D, seed, step, k, act, state, X1, taps, sets, desc, umove)
            lp_new = lp1[act]
            spacing = EX.band_spacing(F, dF, lp_new, lnu) if dF.any() else 0.0
            L, d = EX.ladder_all(F, lp_new, lnu, order, spacing)
            rule = EX.rule(d, lnu, EX.slack(F, dF, lp_new, L, d))
            runs = [(L[(ranks + r) % 9, ranks], d[(ranks + r) % 9, ranks], rule[(ranks + r) % 9, ranks])
                    for r in range(9)]
            if umove is not None:  # the triples: their own lp_old, decided by the row's order alone
                Lt = np.where(umove.plan.triple[act], umove.plan.L[act], L[4])
                dt = EX.lnpdiff(F, lp_new, Lt, order)
                rt = EX.rule(dt[None], lnu)[0]
                assert np.all(rt[umove.plan.triple[act]] != 0)
                runs.append((Lt, dt, rt))
            lower = np.concatenate(sets[:k]) if k else np.zeros(0, dtype=np.int64)
            for Lr, dr, rr in runs:
                lp_run = minus_inf.copy()
                lp_run[act] = Lr
                acc = run(lp_run)
                X2, lp2 = eng.get_state()
                # the same proposals as observed, before anything else
                assert X2[lower].tobytes() == X1[lower].tobytes(), ("split below moved elsewhere", seed, step, k)
                a = acc[act]
                assert X2[act[a]].tobytes() == X1[act[a]].tobytes(), ("proposal differs", seed, step, k)
                assert lp2[act[a]].tobytes() == lp1[act[a]].tobytes(), ("lp_new differs", seed, step, k)
                assert X2[act[~a]].tobytes() == X0[act[~a]].tobytes()
                log = _logged(fn)
                if log is not None:
                    assert len(log) > k and log[k][0].tobytes() == obs_log[k][0].tobytes(), "the function saw other rows"
                if blobs:
                    b = eng.get_blobs()
                    want = np.where(a, blob_of(X1[act]), old_blobs[act])
                    assert b[act].tobytes() == want.tobytes(), ("blobs", seed, step, k)
                    assert b[lower].tobytes() == blob_of(X1[lower]).tobytes()
                bad = np.flatnonzero(((rr == 1) & ~a) | ((rr == -1) & a))
                assert bad.size == 0, ("decision against the rule", path, seed, step, k, act[bad],
                                       EX.distance_ulps(dr[bad][None], [lnu[j] for j in bad]))
                dist = EX.distance_ulps(dr[None], lnu)[0]
                if (a & (dist < 0)).any():
                    reach[0] = max(reach[0], float(-dist[a & (dist < 0)].min()))
                if (~a & (dist > 0)).any():
                    reach[1] = max(reach[1], float(dist[~a & (dist > 0)].max()))
                ndec += int((rr != 0).sum())
    assert ndec > 0
    print("%s: %d decided rungs, %.1f s" % (path, ndec, time.time() - t0))
