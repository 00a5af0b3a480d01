"""``BatchSampler``: many independent ensembles advanced together, one launch per half-step for all of them.

The common emcee workload is many small fits -- one per object, dataset or start point, each a few dozen walkers
in a handful of dimensions.  Run one ``EnsembleSampler`` after another, each pays the launch latency of every
half-step (and a user function its Python round trip) around very little work.  A ``BatchSampler`` holds ``nbatch``
ensembles stacked as the rows of one engine (``eb_create_batch``) and runs each half-step of all of them as one
kernel, and each call of a user function for all of them at once.

Every draw is a pure function of ``(seed, step, split, index, tag)``, and set sizes depend on ``nwalkers`` and the
split count only, so ensemble ``k`` with key ``seeds[k]`` produces exactly the chain of ``EnsembleSampler(nwalkers,
ndim, log_prob_fn, moves=moves, seed=seeds[k])`` started from the same state, whatever else shares the launch."""

import builtins
import itertools
import logging
import operator

import numpy as np

from . import _lib
from .backend import (Backend, DeviceBackend, _check_histogram_name, _check_summary_name, _histogram_params,
                      slice_plan)
from .ensemble import _NOT_INDEPENDENT, _seed_from_numpy
from .models import CallbackFunction, CudaGraphFunction, DeviceModel, HostFunction
from .moves import DEMove, DESnookerMove, StretchMove
from .state import State

__all__ = ["BatchSampler"]

logger = logging.getLogger(__name__)

_MOVES = (StretchMove, DEMove, DESnookerMove)
_ONE_MOVE = (
    "a BatchSampler runs exactly one StretchMove, DEMove or DESnookerMove for every ensemble; a schedule of several "
    "moves would need a move, and with it a split count, per ensemble and step"
)
_MODELS = (
    "a BatchSampler takes a registered device model (optionally models.Bounded), models.CudaArrayFunction(fn) or "
    "models.HostFunction(fn, vectorize=True), where fn maps x[nbatch, m, ndim] to lp[nbatch, m]"
)


def _batch_seeds(seeds, K):
    """``seeds[K]`` (uint64) from ``None`` (derived from numpy's global state without consuming it, as
    ``EnsembleSampler`` does), one integer ``s`` (``s, s + 1, ..., s + K - 1``) or a sequence of ``K`` integers."""
    if seeds is None:
        seeds = _seed_from_numpy()
    if np.ndim(seeds) == 0:
        s = operator.index(seeds)
        return np.array([(s + k) & (2**64 - 1) for k in range(K)], dtype=np.uint64)
    seeds = [operator.index(s) & (2**64 - 1) for s in seeds]
    if len(seeds) != K:
        raise ValueError("seeds must hold one integer per ensemble: expected %d, got %d" % (K, len(seeds)))
    return np.array(seeds, dtype=np.uint64)


def _walkers_independent(coords):
    """The reference's ``walkers_independent`` (``ensemble.py:653-663``) of every ensemble of ``coords[K, N, D]`` in
    one batched pass: ``bool[K]``."""
    finite = np.all(np.isfinite(coords), axis=(1, 2))
    with np.errstate(all="ignore"):
        centred = coords - np.mean(coords, axis=1)[:, None, :]
        span = np.amax(np.abs(centred), axis=1)
        ok = finite & np.all(span != 0, axis=1)
        centred = centred / np.where(span == 0, 1.0, span)[:, None, :]
        centred = centred / np.sqrt(np.sum(centred**2, axis=1))[:, None, :]
    if not np.any(ok):
        return ok
    cond = np.full(len(coords), np.inf)
    cond[ok] = np.linalg.cond(centred[ok])
    return ok & (cond <= 1e8)


class BatchSampler(object):
    """``nbatch`` independent ensembles of ``nwalkers x ndim``, each the twin of ``EnsembleSampler(nwalkers, ndim,
    log_prob_fn, moves=moves, seed=seeds[k])``, advanced together on one H100.

    ``log_prob_fn`` is a registered device model (its parameters shared by every ensemble), or a user function
    ``fn(x[nbatch, m, ndim]) -> lp[nbatch, m]`` wrapped in ``models.CudaArrayFunction`` or
    ``models.HostFunction(fn, vectorize=True)``: it is called once per half-step with the proposals of every
    ensemble, so per-ensemble data broadcasts along the leading axis (``data[nbatch, T]``).  ``moves`` is one
    ``StretchMove``, ``DEMove`` or ``DESnookerMove`` (default ``StretchMove()``), with any of its parameters.

    ``seeds`` is a sequence of ``nbatch`` integers, or one integer ``s`` for ``s, s + 1, ..., s + nbatch - 1``;
    ``None`` derives ``s`` from numpy's global state.  States are ``State(coords[nbatch, nwalkers, ndim],
    log_prob[nbatch, nwalkers])``, chains ``[n, nbatch, nwalkers, ndim]``; the reference's errors apply per ensemble
    with ``EnsembleSampler``'s types and messages.

    ``backend`` stores the chain: ``None`` for a host :class:`~emcee_b200.backends.Backend`, or a
    :class:`~emcee_b200.DeviceBackend` on the sampler's device, which keeps it in GPU memory (a stored step is one
    copy inside HBM) and summarises every ensemble there: :meth:`get_percentile`, :meth:`get_moments`,
    :meth:`get_autocorr_time`, :meth:`get_histogram` and :meth:`get_histogram2d` read the chain where it is.  The
    backend holds the ensembles stacked, ``nbatch * nwalkers`` walkers; an initialised one of that shape with stored
    steps continues its run (``random_state`` and ``run_mcmc(None, ...)`` resume from its last sample)."""

    def __init__(self, nbatch, nwalkers, ndim, log_prob_fn, moves=None, *, seeds=None, device=0, backend=None):
        self.nbatch, self.nwalkers, self.ndim = operator.index(nbatch), operator.index(nwalkers), operator.index(ndim)
        if self.nbatch < 1:
            raise ValueError("nbatch must be >= 1, got {0}".format(self.nbatch))
        if self.nbatch * self.nwalkers > 2**31 - 1:
            raise ValueError("a batch holds at most 2**31 - 1 walkers in all (int32 split tables); got {0} x {1}".format(
                self.nbatch, self.nwalkers))
        if isinstance(log_prob_fn, CudaGraphFunction):
            raise NotImplementedError("CudaGraphFunction is not batched; " + _MODELS)
        if isinstance(log_prob_fn, CallbackFunction):
            if log_prob_fn.blobs_dtype is not None:
                raise NotImplementedError("blobs_dtype is not batched; " + _MODELS)
            if isinstance(log_prob_fn, HostFunction) and not log_prob_fn.vectorize:
                raise NotImplementedError("HostFunction(vectorize=False) is not batched; " + _MODELS)
        elif not isinstance(log_prob_fn, DeviceModel):
            raise TypeError(_MODELS)
        if moves is None:
            moves = StretchMove()
        elif isinstance(moves, (list, tuple)):
            if len(moves) != 1:
                raise NotImplementedError(_ONE_MOVE)
            moves = moves[0][0] if isinstance(moves[0], (list, tuple)) else moves[0]
        if type(moves) not in _MOVES:
            raise NotImplementedError(_ONE_MOVE + "; got {0!r}".format(moves))
        self.move = moves
        self.log_prob_fn = log_prob_fn
        seeds = _batch_seeds(seeds, self.nbatch)
        self._engine = _lib.BatchEngine(self.nbatch, self.nwalkers, self.ndim, seeds, device=device)
        m = log_prob_fn
        if isinstance(m, CallbackFunction):
            self._engine.set_callback(m._call, m.where)
        else:
            self._engine.set_model(m.kind, m.device_params(self.ndim))
            box = m.bounds(self.ndim)
            if box is not None:
                self._engine.set_bounds(*box)
        self.backend = Backend() if backend is None else backend
        self._previous_state = None
        if isinstance(self.backend, DeviceBackend) and self.backend.device != device:
            raise ValueError("the backend keeps its chain on device {0}, the sampler runs on device {1}".format(
                self.backend.device, device))
        if not self.backend.initialized:
            self.reset()
        else:
            shape = (self.nbatch * self.nwalkers, self.ndim)
            if self.backend.shape != shape:
                raise ValueError("the shape of the backend ({0}) is incompatible with the shape of the batch ({1}: "
                                 "nbatch * nwalkers walkers)".format(self.backend.shape, shape))
            self.random_state = self.backend.random_state
            if self.backend.iteration > 0:
                self._previous_state = self.get_last_sample()

    # ------------------------------------------------------------------ state
    @property
    def random_state(self):
        """``("philox4x32-10", seeds[nbatch] uint64, step)``: one step counter for every ensemble."""
        seeds, step = self._engine.get_rng()
        return ("philox4x32-10", seeds, step)

    @random_state.setter
    def random_state(self, state):
        # as EnsembleSampler: try, and stay as we are if it is garbage
        try:
            name, seeds, step = state
            if name == "philox4x32-10":
                self._engine.set_rng(seeds, operator.index(step))
        except Exception:
            pass

    @property
    def iteration(self):
        return self.backend.iteration

    def reset(self):
        self.backend.reset(self.nbatch * self.nwalkers, self.ndim)

    def _state(self, coords, log_prob):
        K, N, D = self.nbatch, self.nwalkers, self.ndim
        return State(coords.reshape(K, N, D), log_prob=log_prob.reshape(K, N), random_state=self.random_state)

    # ------------------------------------------------------------- the driver
    def _stored_before_failure(self, step0, thin_by, k0):
        b = self.backend
        _, step = self._engine.get_rng()
        stored = (step - step0) // thin_by
        b.iteration = k0 + stored
        if stored:
            b.random_state = (self.random_state[0], self.random_state[1], step0 + stored * thin_by)

    def sample(self, initial_state, iterations=1, tune=False, skip_initial_state_check=False, thin_by=1, store=True):
        """Advance every ensemble as a generator (``EnsembleSampler.sample``): yields the live ``State`` of
        ``coords[nbatch, nwalkers, ndim]`` every ``thin_by`` steps.  ``initial_state`` is a ``State`` or a bare
        ``[nbatch, nwalkers, ndim]`` array."""
        return self._sample(initial_state, iterations, skip_initial_state_check, thin_by, store, bulk=False)

    def _sample(self, initial_state, iterations, skip_initial_state_check, thin_by, store, bulk):
        K, N, D = self.nbatch, self.nwalkers, self.ndim
        if iterations is None and store:
            raise ValueError("'store' must be False when 'iterations' is None")
        thin_by = int(thin_by)
        if thin_by <= 0:
            raise ValueError("Invalid thinning argument")
        if N < 2 * D and not self.move.live_dangerously:  # red_blue.py:64-70
            raise RuntimeError(
                "It is unadvisable to use a red-blue move with fewer walkers than twice the number of dimensions.")
        state = State(initial_state)
        coords = np.asarray(state.coords, dtype=np.float64)
        if coords.shape != (K, N, D):
            raise ValueError("incompatible input dimensions {0}".format(coords.shape))
        if not skip_initial_state_check:
            bad = np.flatnonzero(~_walkers_independent(coords))
            if len(bad):
                raise ValueError(_NOT_INDEPENDENT + " (ensemble {0})".format(int(bad[0])))
        self.random_state = state.random_state
        lp = None
        if state.log_prob is not None:
            lp = np.asarray(state.log_prob, dtype=np.float64)
            if lp.shape != (K, N):
                raise ValueError("incompatible input dimensions")
            lp = lp.reshape(K * N)
        eng = self._engine
        eng.set_state(coords.reshape(K * N, D), lp)
        if store:
            self.backend.grow(iterations, None)
        sched = [(self.move.descriptor(), 1.0)]
        return self._steps(sched, iterations, thin_by, store, bulk)

    def _steps(self, sched, iterations, thin_by, store, bulk):
        eng, b = self._engine, self.backend
        device_store = isinstance(b, DeviceBackend)
        if bulk:
            total = iterations * thin_by
            if total > 0:
                if store:
                    k0, k1 = b.iteration, b.iteration + iterations
                    step0 = eng.get_rng()[1]
                    try:
                        if device_store:
                            eng.step_store_chain(sched, total, thin_by, b._ch, k0)
                        else:
                            eng.step_store(sched, total, thin_by, b.chain[k0:k1], b.log_prob[k0:k1], b.accepted)
                    except BaseException:
                        self._stored_before_failure(step0, thin_by, k0)
                        raise
                    b.iteration = k1
                    b.random_state = self.random_state
                else:
                    eng.step(sched, total, want_accepted=False)
            yield self._state(*eng.get_state())
            return
        counter = iter(int, 1) if iterations is None else range(iterations)
        for _ in counter:
            if store:
                k = b.iteration
                if device_store:
                    eng.step_store_chain(sched, thin_by, thin_by, b._ch, k)
                else:
                    eng.step_store(sched, thin_by, thin_by, b.chain[k : k + 1], b.log_prob[k : k + 1], b.accepted)
                b.iteration = k + 1
                b.random_state = self.random_state
            else:
                eng.step(sched, thin_by, want_accepted=False)
            yield self._state(*eng.get_state())

    def run_mcmc(self, initial_state, nsteps, thin_by=1, store=True, skip_initial_state_check=False):
        """Advance every ensemble ``nsteps`` iterations in one call and return the last ``State``
        (``EnsembleSampler.run_mcmc``); ``initial_state=None`` continues the run."""
        if initial_state is None:
            if self._previous_state is None:
                raise ValueError("Cannot have `initial_state=None` if run_mcmc has never been called.")
            initial_state = self._previous_state
        results = None
        for results in self._sample(initial_state, nsteps, skip_initial_state_check, thin_by, store, bulk=True):
            pass
        if nsteps > 0:
            self._previous_state = results
        return results if nsteps > 0 else None

    def compute_log_prob(self, coords):
        """``lp[nbatch, m]`` of ``coords[nbatch, m, ndim]``: the model's kernel, or one call of the function."""
        coords = np.asarray(coords, dtype=np.float64)
        if coords.ndim != 3 or coords.shape[0] != self.nbatch or coords.shape[2] != self.ndim:
            raise ValueError("incompatible input dimensions {0}; expected [{1}, m, {2}]".format(
                coords.shape, self.nbatch, self.ndim))
        K, m, D = coords.shape
        return self._engine.compute_log_prob(coords.reshape(K * m, D)).reshape(K, m)

    # ---------------------------------------------------------------- results
    def get_last_sample(self):
        """The last stored step as a ``State`` of ``coords[nbatch, nwalkers, ndim]``."""
        s = self.backend.get_last_sample()
        K, N, D = self.nbatch, self.nwalkers, self.ndim
        return State(s.coords.reshape(K, N, D), log_prob=s.log_prob.reshape(K, N), random_state=s.random_state)

    @property
    def acceptance_fraction(self):
        """``[nbatch, nwalkers]``."""
        return (self.backend.accepted / float(self.backend.iteration)).reshape(self.nbatch, self.nwalkers)

    def get_value(self, name, flat=False, thin=1, discard=0, cuda=False):
        """``[n, nbatch, nwalkers, ...]``, or with ``flat`` one flat sample per ensemble, ``[nbatch, n * nwalkers,
        ...]``: row ``k`` is what ``get_value(name, flat=True, ...)`` of ensemble ``k``'s twin returns.  ``cuda=True``
        (a :class:`~emcee_b200.DeviceBackend` only): the same values as a :class:`~emcee_b200.DeviceArray`, copied
        inside the GPU's memory."""
        K, N = self.nbatch, self.nwalkers
        if cuda:
            b = self.backend
            if not isinstance(b, DeviceBackend):
                raise TypeError("cuda=True reads a DeviceBackend; this batch stores into {0}".format(type(b).__name__))
            ch, (first, stride, count) = b._plan(discard, thin)
            if name not in ("chain", "log_prob"):
                raise AttributeError(name)
            want_chain = name == "chain"
            if flat:
                x, lp = ch.read_segments_to(K, first, stride, count, coords=want_chain, log_prob=not want_chain)
                return x if want_chain else lp
            shape = (count, K, N) + ((self.ndim,) if want_chain else ())
            x, lp = ch.read_to(first, stride, count, shape if want_chain else None, None if want_chain else shape)
            return x if want_chain else lp
        v = self.backend.get_value(name, thin=thin, discard=discard)
        v = v.reshape((v.shape[0], K, N) + v.shape[2:])
        if flat:
            v = np.swapaxes(v, 0, 1).reshape((K, v.shape[0] * N) + v.shape[3:])
        return v

    def get_chain(self, **kwargs):
        return self.get_value("chain", **kwargs)

    def get_log_prob(self, **kwargs):
        return self.get_value("log_prob", **kwargs)

    def get_percentile(self, q, discard=0, thin=1, name="chain"):
        """``[nbatch] + np.percentile(flat_k, q, axis=0).shape``: row ``k`` is ``np.percentile(get_value(name,
        flat=True, discard=discard, thin=thin)[k], q, axis=0)``, equal with ``==``.  With a ``DeviceBackend`` the
        exact order statistics of every ensemble are selected on the GPU in the same passes
        (``eb_chain_select_segments``) and numpy's interpolation runs on the host; a bad ``q`` raises numpy's
        exception before any device work, an empty slice numpy's error for one."""
        from .summary import percentile_finish, percentile_ranks

        _check_summary_name(name)
        b, K = self.backend, self.nbatch
        if not isinstance(b, DeviceBackend):
            flat = self.get_value(name, flat=True, discard=discard, thin=thin)
            return np.array([np.percentile(flat[k], q, axis=0) for k in range(K)])
        ch, (first, stride, count) = b._plan(discard, thin)
        plan = percentile_ranks(q, count * self.nwalkers)
        shape = (0, self.ndim) if name == "chain" else (0,)
        if count == 0:  # numpy's own result, or error, for an empty slice
            return np.array([np.percentile(np.empty(shape), q, axis=0) for _ in range(K)])
        if plan.ranks.size == 0:
            return np.array([percentile_finish(plan, np.empty(shape)) for _ in range(K)])
        stats, has_nan, _ = ch.select(name, first, stride, count, plan.ranks, nseg=K)
        stats = stats.reshape((K, plan.ranks.size) + (() if name == "log_prob" else (self.ndim,)))
        has_nan = has_nan.reshape((K,) + (() if name == "log_prob" else (self.ndim,)))
        return np.array([percentile_finish(plan, stats[k], has_nan[k]) for k in range(K)])

    def get_moments(self, discard=0, thin=1):
        """``(mean[nbatch, ndim], cov[nbatch, ndim, ndim], n)``: row ``k`` is ``np.mean(axis=0)`` /
        ``np.cov(rowvar=False)`` of ``get_chain(flat=True, discard=discard, thin=thin)[k]``, ``n`` the samples of one
        ensemble; NaN for an empty slice.  With a ``DeviceBackend`` the sums of every ensemble are formed on the GPU
        in one pass (``eb_chain_moments_segments``); ``ndim`` up to 1024."""
        b, K, D = self.backend, self.nbatch, self.ndim
        if isinstance(b, DeviceBackend):
            ch, (first, stride, count) = b._plan(discard, thin)
            mean, cov, n = ch.moments(first, stride, count, nseg=K)
            return mean.reshape(K, D), cov.reshape(K, D, D), n
        flat = self.get_chain(flat=True, discard=discard, thin=thin)
        n = flat.shape[1]
        if n == 0:
            return np.full((K, D), np.nan), np.full((K, D, D), np.nan), 0
        mean = np.array([np.mean(flat[k], axis=0) for k in range(K)])
        cov = np.array([np.cov(flat[k], rowvar=False).reshape(D, D) for k in range(K)])
        return mean, cov, n

    def get_autocorr_time(self, discard=0, thin=1, c=5, tol=50, quiet=False):
        """``tau[nbatch, ndim]``: row ``k`` is ``thin * autocorr.integrated_time(get_chain(discard=discard,
        thin=thin)[:, k], c=c, tol=tol, quiet=quiet)``.  When the chain of any ensemble is shorter than ``tol``
        times its estimate, one :class:`~emcee_b200.autocorr.AutocorrError` (with ``quiet``: one warning) names
        those ensembles, and its ``tau`` holds every row's estimate.  With a ``DeviceBackend`` the autocorrelation
        functions of every ensemble come from one call on the GPU, where the chain is
        (``eb_chain_autocorr_segments``), each bit-identical to that ensemble's own ``DeviceBackend``'s."""
        from . import autocorr

        K = self.nbatch
        if isinstance(self.backend, DeviceBackend):
            ch, (first, stride, count) = self.backend._plan(discard, thin)
            rho = ch.autocorr_function(first, stride, count, nseg=K).reshape(K, count, self.ndim)
            estimate = lambda k: autocorr.integrated_time_from_acf(rho[k], c=c, tol=tol, quiet=False)
        else:
            x = self.get_chain(discard=discard, thin=thin)
            estimate = lambda k: autocorr.integrated_time(x[:, k], c=c, tol=tol, quiet=False)
        taus = np.empty((K, self.ndim))
        failed, first_msg = [], None
        for k in range(K):
            try:
                taus[k] = estimate(k)
            except autocorr.AutocorrError as e:
                taus[k] = e.tau
                failed.append(k)
                first_msg = first_msg or str(e)
        taus *= thin
        if failed:
            msg = "The autocorrelation estimate of ensemble(s) {0} is unreliable. First of them:\n{1}".format(
                failed, first_msg)
            if not quiet:
                raise autocorr.AutocorrError(taus, msg)
            logger.warning(msg)
        return taus

    def _histogram_ranges(self, range, D, log_prob):
        """``range`` of :meth:`get_histogram` / :meth:`get_histogram2d` as ``(r, per)``: ``r(k, d)`` is the range
        numpy gets for parameter ``d`` of ensemble ``k``, ``per`` the array ``[nbatch, D, 2]`` of the per-ensemble
        form (else None).  ``range`` is None, ``D`` pairs or None (one pair for ``log_prob``) shared by every
        ensemble, or an array ``[nbatch, D, 2]`` (``[nbatch, 2]``); ``ValueError`` for any other shape."""
        K = self.nbatch
        if range is None:
            return (lambda k, d: None), None
        try:
            shape = np.shape(range)
        except ValueError:  # a ragged sequence: pairs and Nones
            shape = None
        if shape == ((K, 2) if log_prob else (K, D, 2)):
            per = np.asarray(range)
            if log_prob:
                return (lambda k, d: per[k]), per[:, None]
            return (lambda k, d: per[k, d]), per
        if log_prob:
            if shape != (2,):
                raise ValueError("range of log_prob must be one (lo, hi) pair or an array [nbatch, 2] = [{0}, 2], "
                                 "got shape {1}".format(K, shape))
            return (lambda k, d: range), None
        shared = list(range)
        if len(shared) != D or any(r is not None and np.shape(r) != (2,) for r in shared):
            raise ValueError("range must be one (lo, hi) pair or None per parameter ({0} of them), or an array "
                             "[nbatch, ndim, 2] = [{1}, {0}, 2]".format(D, K))
        return (lambda k, d: shared[d]), None

    def get_histogram(self, bins=10, range=None, discard=0, thin=1, name="chain"):
        """``(hist[nbatch, ndim, bins] int64, edges[nbatch, ndim, bins + 1])``: row ``k`` is what
        ``Backend.get_histogram`` returns for ensemble ``k``'s flat slice ``get_chain(flat=True, discard=discard,
        thin=thin)[k]``; with ``name="log_prob"``, ``(hist[nbatch, bins], edges[nbatch, bins + 1])``.  ``range`` is
        None (each ensemble's own extremes), one ``(lo, hi)`` pair or None per parameter (one pair for
        ``log_prob``) shared by every ensemble, or an array ``[nbatch, ndim, 2]`` (``[nbatch, 2]``) with one range
        per ensemble -- the shape ``get_percentile`` output reshapes into.

        With a ``DeviceBackend`` every ensemble is counted on the GPU in one read of the slice
        (``eb_chain_histogram_segments``), autodetected ranges come from one selection of every ensemble's
        extremes, and numpy's edges are formed on the host for all columns at once; results, dtypes and exceptions
        are the host route's (the first failing ensemble, then parameter, raises).  ``bins`` is an int of at most
        4096 there, and a finite range wider than the largest double raises ``ValueError``, as
        ``DeviceBackend.get_histogram``."""
        from .summary import HIST_BINS_MAX, histogram_bins, uniform_edges

        _check_histogram_name(name)
        b, K = self.backend, self.nbatch
        log_prob = name == "log_prob"
        D = 1 if log_prob else self.ndim
        r, per = self._histogram_ranges(range, D, log_prob)
        if not isinstance(b, DeviceBackend):
            flat = self.get_value(name, flat=True, discard=discard, thin=thin)
            if log_prob:
                out = [np.histogram(flat[k], bins=bins, range=r(k, 0)) for k in builtins.range(K)]
                return np.array([h for h, _ in out]), np.array([e for _, e in out], dtype=np.float64)
            out = [[np.histogram(flat[k][:, d], bins=bins, range=r(k, d)) for d in builtins.range(D)]
                   for k in builtins.range(K)]
            return (np.array([[h for h, _ in row] for row in out]),
                    np.array([[e for _, e in row] for row in out], dtype=np.float64))
        ch, (first, stride, count) = b._plan(discard, thin)
        n = histogram_bins(bins, HIST_BINS_MAX)
        ranges = [r(k, d) for k in builtins.range(K) for d in builtins.range(D)]  # column k * D + d
        if count == 0:  # numpy's empty-input result (edges over [0, 1] without a range), no device work
            out = [np.histogram(np.empty(0), bins=n, range=rr) for rr in ranges]
            hist = np.array([h for h, _ in out]).reshape((K, D, n))
            edges = np.array([e for _, e in out], dtype=np.float64).reshape((K, D, n + 1))
        else:
            lo, hi, has_nan = self._extremes(ch, name, first, stride, count, ranges)
            outer, edges = uniform_edges(n, ranges if per is None else per.reshape(K * D, 2), lo, hi, has_nan)
            hist = ch.histogram(name, first, stride, count, n, outer, edges, nseg=K).reshape((K, D, n))
            edges = edges.reshape((K, D, n + 1))
        return (hist[:, 0], edges[:, 0]) if log_prob else (hist, edges)

    def get_histogram2d(self, params=None, bins=10, range=None, discard=0, thin=1):
        """``(hist[nbatch, npairs, bins, bins] float64, edges[nbatch, len(params), bins + 1], pairs)``: row ``k`` is
        what ``Backend.get_histogram2d`` returns for ensemble ``k``'s flat slice, and ``pairs`` is
        ``list(itertools.combinations(params, 2))``.  ``range`` takes the forms of :meth:`get_histogram`, indexed
        by parameter number.  With a ``DeviceBackend`` every (ensemble, pair) is counted on the GPU in one launch
        (``eb_chain_histogram2d_segments``), as :meth:`get_histogram` does; ``bins`` is an int of at most 128, and
        the counts of every ensemble are held in device memory at once (``nbatch * npairs * bins^2 * 8`` bytes;
        ``MemoryError`` when they do not fit)."""
        from .summary import HIST2_BINS_MAX, histogram_bins, searched_edges

        b, K, D = self.backend, self.nbatch, self.ndim
        params = _histogram_params(params, D)
        r, per = self._histogram_ranges(range, D, False)
        pairs = list(itertools.combinations(params, 2))
        m = len(params)
        if not isinstance(b, DeviceBackend):
            flat = self.get_chain(flat=True, discard=discard, thin=thin)
            hist, edges = [], []
            for k in builtins.range(K):
                hk, ek = [], {}
                for i, j in pairs:
                    h, ei, ej = np.histogram2d(flat[k][:, i], flat[k][:, j], bins=bins,
                                               range=None if range is None else [r(k, i), r(k, j)])
                    hk.append(h)
                    ek.setdefault(i, ei)
                    ek.setdefault(j, ej)
                hist.append(hk)
                edges.append([ek[p] for p in params])
            return np.array(hist), np.array(edges, dtype=np.float64), pairs
        ch, (first, stride, count) = b._plan(discard, thin)
        n = histogram_bins(bins, HIST2_BINS_MAX, two_d=True)
        ranges = [r(k, p) for k in builtins.range(K) for p in params]  # column k * m + position
        if count == 0:  # numpy's empty-input result, no device work
            e = searched_edges(n, ranges, np.zeros(K * m), np.ones(K * m), np.zeros(K * m, dtype=bool))
            return np.zeros((K, len(pairs), n, n)), e.reshape((K, m, n + 1)), pairs
        lo, hi, has_nan = self._extremes(ch, "chain", first, stride, count, ranges)
        at = (np.arange(K)[:, None] * D + np.asarray(params)[None, :]).ravel()
        edges = searched_edges(n, ranges if per is None else per[:, params].reshape(K * m, 2), lo[at], hi[at],
                               has_nan[at])
        hist = ch.histogram2d(first, stride, count, params, n, edges, nseg=K)
        return hist.reshape((K, len(pairs), n, n)).astype(np.float64), edges.reshape((K, m, n + 1)), pairs

    def _extremes(self, ch, name, first, stride, count, ranges):
        """``(lo, hi, has_nan)`` of every column ``k * D + d`` (ranks 0 and n - 1 of every ensemble, one
        ``eb_chain_select_segments`` call), or NaN, unread, when every range the call uses is given"""
        K = self.nbatch
        C = K * (self.ndim if name == "chain" else 1)
        if all(rr is not None for rr in ranges):
            return np.full(C, np.nan), np.full(C, np.nan), np.zeros(C, dtype=bool)
        n = count * self.nwalkers
        stats, has_nan, _ = ch.select(name, first, stride, count, np.array([0, n - 1], dtype=np.uint64), nseg=K)
        stats = stats.reshape(K, 2, -1)
        return stats[:, 0].ravel(), stats[:, 1].ravel(), has_nan.reshape(-1)

