"""KDEMove in the oracle (TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``).

Follows, line by line:

* ``KDEMove.get_proposal`` .................... ``src/emcee/moves/kde.py:39-43`` with
  ``scipy.stats.gaussian_kde`` (``__init__``, ``set_bandwidth``, ``resample``, ``logpdf``; uniform weights)
* the red-blue half-step around it ............ ``src/emcee/moves/red_blue.py:52-106``, as
  ``oracle/redblue.py``'s ``OracleSampler._propose`` restates it

and the shim's two extra draws for ``gaussian_kde.resample`` (``KdePhilox``).  Draw specification (DESIGN.md §2):
the kernel centre of active rank ``i`` is ``mulhi64(w1:w0, Nc)`` of block ``(index=i, TAG_PROP_A)``; its normals are
the ``TAG_NORMAL`` normals of row ``i``, and ``multivariate_normal(0, cov, size=Ns)`` row ``i`` is ``L z_i``.
"""

import numpy as np

from . import philox as px
from . import redblue as rb
from .philox import PhiloxRandom

__all__ = ["KDE", "KdeOracleSampler", "KdePhilox", "kde_bandwidth"]


class KDE(rb._RedBlue):
    kind = "kde"

    def __init__(self, bw_method=None, **kw):
        self.bw_method = bw_method
        super().__init__(**kw)


def kde_bandwidth(bw_method, n, d):
    """``gaussian_kde.factor`` of ``n`` uniformly weighted ``d``-dimensional points (``set_bandwidth``)."""
    neff = 1 / np.vecdot(np.ones(n) / n, np.ones(n) / n)  # gaussian_kde.neff
    if bw_method is None or bw_method == "scott":
        return np.power(neff, -1.0 / (d + 4))  # scotts_factor
    if bw_method == "silverman":
        return np.power(neff * (d + 2.0) / 4.0, -1.0 / (d + 4))  # silverman_factor
    return bw_method  # a scalar is the factor itself


def kde_logpdf(c, L, x):
    """``gaussian_kde.logpdf(x)`` up to the normaliser and log-weight, which cancel in kde.py:42: the log-sum-exp
    over the points ``c`` of ``-|L^-1 (x - c)|^2 / 2`` from direct differences of whitened rows."""
    from scipy.linalg import solve_triangular

    yc = solve_triangular(L, c.T, lower=True).T
    yx = solve_triangular(L, x.T, lower=True).T
    out = np.empty(len(x))
    for i in range(len(x)):
        t = -0.5 * np.sum((yx[i] - yc) ** 2, axis=1)
        m = np.max(t)
        out[i] = m + np.log(np.sum(np.exp(t - m)))
    return out


class KdeOracleSampler(rb.OracleSampler):
    """``OracleSampler`` whose schedule may hold ``KDE`` moves; every other move runs the base class's code.
    ``logpdf`` is ``kde_logpdf`` unless replaced (a test may evaluate the same sums elsewhere at large sizes)."""

    logpdf = staticmethod(kde_logpdf)

    def _kde(self, mv, s, sets_c, step, split):
        import scipy.linalg

        comp = np.concatenate(sets_c)  # kde.py:40
        c = self.coords[comp]
        Ns, Nc = len(s), len(comp)
        if self.ndim > Nc:  # gaussian_kde.__init__
            raise ValueError("Number of dimensions is greater than number of samples.")
        bw = kde_bandwidth(mv.bw_method, Nc, self.ndim)  # kde.py:41
        cov = np.atleast_2d(np.cov(c.T, rowvar=1, bias=False, aweights=np.ones(Nc) / Nc))  # _compute_covariance
        z = px.normals(self.seed, step, split, np.arange(Ns), self.ndim)
        norm = z @ px.chol_psd(cov * bw**2).T  # resample: multivariate_normal(0, covariance, size=Ns)
        w0, w1, _, _ = px.draw_words(self.seed, step, split, px.TAG_PROP_A, np.arange(Ns))
        j = px.bounded64(w0, w1, Nc)  # resample: choice(Nc, size=Ns, p=weights)
        q = c[j] + norm  # resample: means + norm (kde.py:41)
        L = scipy.linalg.cholesky(cov, lower=True) * bw  # gaussian_kde.cho_cov
        factors = self.logpdf(c, L, s) - self.logpdf(c, L, q)  # kde.py:42
        self.taps = dict(rank=j, partner=comp[j], z=z)
        return q, factors

    # -- red_blue.py:52-106 for a KDE move (the base class's _propose for the others) --------------
    def _propose(self, mv, step):
        if mv.kind != "kde":
            return super()._propose(mv, step)
        N, D = self.nwalkers, self.ndim
        if N < 2 * D and not mv.live_dangerously:  # red_blue.py:64-70
            raise RuntimeError(
                "It is unadvisable to use a red-blue move "
                "with fewer walkers than twice the number of "
                "dimensions."
            )
        accepted = np.zeros(N, dtype=bool)
        inds = px.split_assignment(self.seed, step, N, mv.nsplits, mv.randomize_split)  # red_blue.py:77-80
        for split in range(mv.nsplits):
            sets = [np.flatnonzero(inds == j) for j in range(mv.nsplits)]  # red_blue.py:85
            act = sets[split]
            sets_c = sets[:split] + sets[split + 1 :]  # red_blue.py:87
            s = self.coords[act]
            q, factors = self._kde(mv, s, sets_c, step, split)  # red_blue.py:90
            new_lp = self.compute_log_prob(q)  # red_blue.py:93
            u0, u1, _, _ = px.draw_words(self.seed, step, split, px.TAG_ACCEPT, np.arange(len(act)))
            uacc = px.u53(u0, u1)
            with np.errstate(divide="ignore", invalid="ignore"):
                lnpdiff = factors + new_lp - self.log_prob[act]  # red_blue.py:99
                acc = lnpdiff > np.log(uacc)  # red_blue.py:100
            self.taps.update(u_accept=uacc, active=act, q=q, new_lp=new_lp, factors=factors)
            won = act[acc]
            self.coords[won] = q[acc]  # move.py:33
            self.log_prob[won] = new_lp[acc]  # move.py:34
            accepted[won] = True
        return accepted


class KdePhilox(PhiloxRandom, np.random.RandomState):
    """The shim with the two draws ``gaussian_kde.resample`` makes, and a ``RandomState`` as well: ``resample``
    passes its ``random`` through scipy's ``check_random_state``, which takes only a ``RandomState`` or a
    ``Generator``.  Every other call is the base shim's, so the existing golden runs regenerate unchanged."""

    def __init__(self, seed, step=0):
        np.random.RandomState.__init__(self, 0)
        PhiloxRandom.__init__(self, seed, step)

    def choice(self, a, size=None, replace=True, p=None):
        if isinstance(a, (int, np.integer)) and p is not None:
            # resample's ``choice(n, size=ns, p=weights)`` (kde.py:41), uniform weights
            p = np.asarray(p)
            assert replace and np.all(p == p[0])
            self._open_split()
            w0, w1, _, _ = self._words(px.TAG_PROP_A, np.arange(int(size)))
            out = px.bounded64(w0, w1, int(a))
            self._log("kde_choice", out.copy())
            return out
        return PhiloxRandom.choice(self, a, size=size, replace=replace, p=p)

    def multivariate_normal(self, mean, cov, size=None):
        if size is None:
            return PhiloxRandom.multivariate_normal(self, mean, cov)
        # resample's ``multivariate_normal(zeros(d), covariance, size=ns)`` (kde.py:41): row i is L z_i with the
        # normals of active rank i; resample draws it first, so it opens the split
        mean = np.asarray(mean, dtype=np.float64)
        self._open_split()
        z = px.normals(self.seed, self._cur, self._split, np.arange(int(size)), len(mean))
        self._log("kde_z", z.copy())
        return mean + z @ px.chol_psd(cov).T
