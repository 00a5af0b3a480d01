"""User moves shared by the user-proposal tests, and a numpy driver of the reference's step loop that runs them
(TEST INFRASTRUCTURE ONLY).

``UserOracle`` extends ``oracle.redblue.OracleSampler`` with the two plugin boundaries of the reference:
``RedBlueMove.propose`` calling ``get_proposal(s, c, random)`` (``src/emcee/moves/red_blue.py:52-106``) and
``MHMove.propose`` calling ``proposal_function(coords, random)`` (``src/emcee/moves/mh.py:35-65``), with ``random``
= ``moves.user_random(seed, step, split)`` and the split assignment / accept draws of the draw specification.  The
move classes below are plain numpy (module level, so samplers holding them pickle)."""
import os

import numpy as np

from oracle import gen_golden_user_moves as gen
from oracle import philox as px
from oracle import redblue as rb

from emcee_b200 import moves

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "user_moves")


class NumpyStretch(moves.RedBlueMove):
    """``stretch.py:26-33`` restated with ``random``'s own draws."""

    def __init__(self, a=2.0, **kw):
        self.a = a
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        c = np.concatenate(c, axis=0)
        ns, nc = len(s), len(c)
        ndim = s.shape[1]
        zz = ((self.a - 1.0) * random.rand(ns) + 1) ** 2.0 / self.a
        factors = (ndim - 1.0) * np.log(zz)
        rint = random.randint(nc, size=(ns,))
        return c[rint] - (c[rint] - s) * zz[:, None], factors


class NumpyDE(moves.RedBlueMove):
    """A differential-evolution-like move: two complement walkers drawn with replacement."""

    def __init__(self, gamma=0.7, sigma=1e-3, **kw):
        self.gamma, self.sigma = gamma, sigma
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        c = np.concatenate(c, axis=0)
        ns, nc = len(s), len(c)
        pairs = random.randint(nc, size=(ns, 2))
        g = self.gamma * (1.0 + self.sigma * random.randn(ns, 1))
        return s + g * (c[pairs[:, 0]] - c[pairs[:, 1]]), np.zeros(ns)


class Recording(NumpyStretch):
    """NumpyStretch that keeps every (s, c) it saw and the ensembles its setup saw."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.calls, self.setups = [], []

    def get_proposal(self, s, c, random):
        self.calls.append((s.copy(), [x.copy() for x in c]))
        return super().get_proposal(s, c, random)


class WithSetup(NumpyStretch):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.setups = []

    def setup(self, coords):
        self.setups.append(np.array(coords, copy=True))


def gauss_mh(coords, random):
    """Gaussian random walk with a non-zero (made-up) log factor: exercises mh.py:57's rounding order."""
    q = coords + 0.3 * random.randn(*coords.shape)
    return q, 0.25 * random.randn(len(coords))


def gauss_mh_symmetric(coords, random):
    return coords + 0.5 * random.randn(*coords.shape), np.zeros(len(coords))


class UserOracle(rb.OracleSampler):
    """``OracleSampler`` that also runs user moves: the emcee_b200 move objects themselves, host-side."""

    def _propose(self, mv, step):
        if isinstance(mv, moves.RedBlueMove) and type(mv).get_proposal is not moves.RedBlueMove.get_proposal:
            return self._propose_user(mv, step)
        if isinstance(mv, moves.MHMove) and mv.kind == "user_mh":
            return self._propose_user_mh(mv, step)
        return super()._propose(mv, step)

    def _accept(self, act, q, f, new_lp, step, split, mh):
        u0, u1, _, _ = px.draw_words(self.seed, step, split, px.TAG_ACCEPT, np.arange(len(act)))
        with np.errstate(divide="ignore", invalid="ignore"):
            if mh:
                acc = np.log(px.u53(u0, u1)) < new_lp - self.log_prob[act] + f  # mh.py:57-58
            else:
                acc = f + new_lp - self.log_prob[act] > np.log(px.u53(u0, u1))  # red_blue.py:99-100
        won = act[acc]
        self.coords[won] = q[acc]
        self.log_prob[won] = new_lp[acc]
        return won

    def _propose_user(self, mv, step):
        N = self.nwalkers
        if N < 2 * self.ndim and not mv.live_dangerously:
            raise RuntimeError("It is unadvisable to use a red-blue move "
                               "with fewer walkers than twice the number of dimensions.")
        if type(mv).setup is not moves.RedBlueMove.setup:
            mv.setup(self.coords.copy())  # red_blue.py:73
        accepted = np.zeros(N, dtype=bool)
        inds = px.split_assignment(self.seed, step, N, mv.nsplits, mv.randomize_split)
        for split in range(mv.nsplits):
            sets = [np.flatnonzero(inds == j) for j in range(mv.nsplits)]  # red_blue.py:85
            act = sets[split]
            c = [self.coords[sets[j]] for j in range(mv.nsplits) if j != split]
            q, f = mv.get_proposal(self.coords[act], c, moves.user_random(self.seed, step, split))
            new_lp = self.compute_log_prob(q)
            accepted[self._accept(act, q, f, new_lp, step, split, False)] = True
        return accepted

    def _propose_user_mh(self, mv, step):
        N = self.nwalkers
        q, f = mv.get_proposal(self.coords.copy(), moves.user_random(self.seed, step, 0))
        new_lp = self.compute_log_prob(q)
        accepted = np.zeros(N, dtype=bool)
        accepted[self._accept(np.arange(N), q, f, new_lp, step, 0, True)] = True
        return accepted


# ---- the golden cases of oracle/gen_golden_user_moves.py --------------------------------------------------------
class GoldenUser(moves.RedBlueMove):
    """A user red-blue move calling one of the generator's proposal functions."""

    def __init__(self, fname, **kw):
        self.fname = fname
        super().__init__(**kw)

    def get_proposal(self, s, c, random):
        return gen.FUNCTIONS[self.fname](s, c, random)


def golden_moves(spec):
    """The engine's moves for a case of ``gen.CASES``."""
    out = []
    for kind, fname, w, kw in spec:
        if kind == "user":
            m = GoldenUser(fname, **kw)
        elif kind == "user_mh":
            m = moves.MHMove(moves.HostProposal(gen.FUNCTIONS[fname]))
        elif kind == "stretch":
            m = moves.StretchMove(**kw)
        else:
            m = moves.DEMove(**kw)
        out.append((m, w))
    return out


def oracle_moves(mv):
    """``mv`` with the built-in moves replaced by their ``oracle.redblue`` counterparts."""
    out = []
    for m, w in mv:
        if isinstance(m, moves.StretchMove):
            m = rb.Stretch(a=m.a, nsplits=m.nsplits, randomize_split=m.randomize_split)
        elif isinstance(m, moves.DEMove):
            m = rb.DE(sigma=m.sigma, gamma0=m.gamma0, nsplits=m.nsplits, randomize_split=m.randomize_split)
        out.append((m, w))
    return out


def golden_cases():
    return [c[0] for c in gen.CASES]


def load_case(name):
    case = {c[0]: c for c in gen.CASES}[name]
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    return case, g
