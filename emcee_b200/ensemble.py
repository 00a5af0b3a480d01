"""``EnsembleSampler`` on the H100 engine (reference:
``src/emcee/ensemble.py:32-623``).

Same constructor / ``sample`` / ``run_mcmc`` / ``compute_log_prob`` surface and
the same exceptions, but ``log_prob_fn`` is a registered device model or an
explicitly wrapped user function (``emcee_b200.models``), and every step runs
inside the CUDA library through the C ABI: the walker array stays in HBM
between steps, ``run_mcmc`` is one call for all iterations (a user function is
called back from inside it once per half-step), and stored steps stream back
through pinned buffers.  ``pool`` / ``args`` / ``kwargs`` / ``vectorize``
and ``blobs_dtype`` belong to ``models.HostFunction`` / ``models.CudaArrayFunction``;
named parameters raise ``NotImplementedError``."""

import operator
from collections import namedtuple
from collections.abc import Iterable

import numpy as np

from . import _lib
from .backend import Backend, ChainWindow, DeviceBackend
from .model import Model
from .models import CallbackFunction, CudaGraphFunction, DeviceModel, graph_row_counts
from .moves import StretchMove
from .moves.user import user_move_spec
from .rng import DeviceRandom
from .state import State

__all__ = ["EnsembleSampler", "walkers_independent"]


_NO_SHARDED_DEVICE_CHAIN = (
    "a DeviceBackend cannot store a sharded ensemble: a stored step holds every walker, and the replication "
    "of the other ranks' rows before each stored step is built for host chains only; use Backend()"
)
_NO_DEVICE_CHAIN_BLOBS = "a DeviceBackend does not store blobs; use Backend() with a function that returns blobs"
#: the running statistics other than the moments: the sampler attribute that holds each one's configuration, and the
#: refusal of a sharded ensemble.  The attribute is None until the statistic is enabled, and again after unpickling:
#: what was recorded lives in the engine's memory.  It holds the histograms' configuration of enable_histograms (edges,
#: pairs), the cadence the trace and the reservoir recorded their rows with, and the (max_lag, every) of the
#: autocorrelation and the (size, every) of the window.
_RUNNING = (
    ("_hist", "running histograms are counted on one GPU; they cannot be combined with a sharded ensemble"),
    ("_trace_every", "the running trace is recorded on one GPU; it cannot be combined with a sharded ensemble"),
    ("_reservoir_every", "the running reservoir is kept on one GPU; it cannot be combined with a sharded ensemble"),
    ("_autocorr", "the running autocorrelation is summed on one GPU; it cannot be combined with a sharded ensemble"),
    ("_window", "the running window is kept on one GPU; it cannot be combined with a sharded ensemble"),
)
_NO_HISTOGRAMS = "running histograms are not enabled: call enable_histograms(range, ...) first"
_NO_TRACE = "the running trace is not enabled: call enable_trace() first"
_NO_RESERVOIR = "the running reservoir is not enabled: call enable_reservoir(size) first"
_NO_AUTOCORR = "the running autocorrelation is not enabled: call enable_autocorr(max_lag) first"
_NO_WINDOW = "the running window is not enabled: call enable_window(size) first"
_NO_SHARDED_CUDA_ARRAYS = (
    "CUDA arrays in and out are copied on one GPU; a sharded ensemble takes and returns host arrays"
)
_NO_CUDA_STATE_BLOBS = (
    "a state given as CUDA arrays cannot carry blobs; pass host arrays, or leave log_prob out so that the "
    "function's blobs of the initial evaluation become the state's"
)
_NOT_INDEPENDENT = (
    "Initial state has a large condition number. "
    "Make sure that your walkers are linearly independent for the "
    "best performance"
)

#: what :meth:`EnsembleSampler.trace` returns: one entry per recorded step
Trace = namedtuple("Trace", ["step", "mean", "var", "log_prob_mean", "log_prob_max", "accepted"])
#: what :meth:`EnsembleSampler.reservoir` returns: one entry per kept row
Reservoir = namedtuple("Reservoir", ["coords", "log_prob", "step", "walker"])


def _index_at_least(name, value, least):
    """``operator.index(value)`` (``TypeError`` for what is not an integer), ``ValueError`` below ``least``."""
    value = operator.index(value)
    if value < least:
        raise ValueError("{0} must be >= {1}, got {2}".format(name, least, value))
    return value


def _seed_from_numpy():
    """Like the reference, start from numpy's global generator
    (``ensemble.py:140`` ``state = np.random.get_state()``) without consuming it."""
    keys, pos = np.random.get_state()[1:3]
    a, b = int(keys[pos % 624]), int(keys[(pos + 1) % 624])
    return ((a << 32) | b) ^ (int(pos) * 0x9E3779B97F4A7C15 & (2**64 - 1))


class EnsembleSampler(object):
    """An ensemble MCMC sampler whose walker update runs on one H100.

    Args mirror ``ensemble.py:79-98``.  Extra keyword-only arguments: ``seed``
    (Philox key; default derived from numpy's global state), ``device``, and
    ``pinned_results`` (the yielded / returned ``State`` arrays are views of two
    page-locked buffers owned by the sampler and are overwritten by the next
    step -- full-speed D2H for callers that consume each state before asking for
    the next; default ``False`` = fresh arrays, as the reference returns) and
    ``cuda_results`` (every yielded / returned ``State`` holds fresh
    :class:`~emcee_b200.DeviceArray` coords and log_prob, copied inside the GPU's
    memory; blobs still come back as host arrays; not with ``pinned_results``, and
    not on a sharded ensemble).

    ``sample`` / ``run_mcmc`` and ``compute_log_prob`` also take CUDA arrays
    (anything with the CUDA Array Interface: torch, CuPy, Numba, ``DeviceArray``),
    uploaded inside the GPU's memory after the work of the stream they name."""

    def __init__(
        self,
        nwalkers,
        ndim,
        log_prob_fn,
        pool=None,
        moves=None,
        args=None,
        kwargs=None,
        backend=None,
        vectorize=False,
        blobs_dtype=None,
        parameter_names=None,
        # deprecated in the reference; rejected here
        a=None,
        postargs=None,
        threads=None,
        live_dangerously=None,
        runtime_sortingfn=None,
        *,
        seed=None,
        device=0,
        pinned_results=False,
        cuda_results=False,
    ):
        for name, val in (("a", a), ("postargs", postargs), ("threads", threads),
                          ("live_dangerously", live_dangerously), ("runtime_sortingfn", runtime_sortingfn)):
            if val is not None:
                raise NotImplementedError("the deprecated '%s' argument is not supported; use 'moves'" % name)
        if not isinstance(log_prob_fn, (DeviceModel, CallbackFunction)):
            raise TypeError(
                "log_prob_fn must be a registered device model (emcee_b200.models.GaussianIso, ...) or a "
                "wrapped user function: models.HostFunction(fn, vectorize=...) for a numpy function, "
                "models.CudaArrayFunction(fn) for one on CUDA arrays"
            )
        if pool is not None:
            raise NotImplementedError("pool: pass it to models.HostFunction(fn, pool=pool)")
        if args or kwargs:
            raise NotImplementedError(
                "args/kwargs: put the parameters into the device model, or pass them to "
                "models.HostFunction / models.CudaArrayFunction")
        if parameter_names is not None:
            raise NotImplementedError("parameter_names need a host callable")
        if blobs_dtype is not None:
            raise NotImplementedError(
                "blobs_dtype: pass it to models.HostFunction / models.CudaArrayFunction(fn, blobs_dtype=...)")
        if isinstance(backend, DeviceBackend) and getattr(log_prob_fn, "blobs_dtype", None) is not None:
            raise NotImplementedError(_NO_DEVICE_CHAIN_BLOBS)
        if cuda_results and pinned_results:
            raise ValueError("cuda_results and pinned_results exclude each other: a state is returned in device "
                             "memory or in page-locked host memory")

        # move schedule (ensemble.py:115-129)
        if moves is None:
            self._moves, weights = [StretchMove()], [1.0]
        elif isinstance(moves, Iterable):
            moves = list(moves)
            try:
                self._moves, weights = (list(t) for t in zip(*moves))
            except TypeError:
                self._moves, weights = moves, np.ones(len(moves))
        else:
            self._moves, weights = [moves], [1.0]
        self._raw_weights = np.atleast_1d(weights).astype(float)
        self._weights = self._raw_weights / np.sum(self._raw_weights)
        for m in self._moves:
            # the step loop runs inside the CUDA library: a move must be one of the device moves
            # (it only *describes* itself); a host ``Move`` with its own ``propose`` cannot be called
            # back from a kernel -- say so here, not with an AttributeError in the middle of sample()
            if not callable(getattr(m, "descriptor", None)):
                raise TypeError(
                    "moves must be emcee_b200.moves.* device moves; got {0!r}, which has no device "
                    "descriptor (host-side Move subclasses cannot run inside the fused step kernels)".format(m)
                )

        self.pool = None
        self.vectorize = True  # the device path is always batched
        self.blobs_dtype = getattr(log_prob_fn, "blobs_dtype", None)
        self.ndim = int(ndim)
        self.nwalkers = int(nwalkers)
        self.log_prob_fn = log_prob_fn
        self.params_are_named = False

        self._device = int(device)
        self._engine = _lib.Engine(self.nwalkers, self.ndim, _seed_from_numpy() if seed is None else seed,
                                   device=device)
        self._load_model()
        self._load_moves()
        self._random = DeviceRandom(self._engine)
        self._pinned = None
        if pinned_results:
            self._pinned = (_lib.pinned_empty((self.nwalkers, self.ndim)), _lib.pinned_empty((self.nwalkers,)))
        self._cuda_results = bool(cuda_results)
        self._rdv = None  # multi-GPU: the host rendezvous this sampler is attached to (``attach``)
        for attr, _ in _RUNNING:
            setattr(self, attr, None)
        self._gather_results = True

        self.backend = Backend() if backend is None else backend
        if isinstance(self.backend, DeviceBackend) and self.backend.device != self._device:
            raise ValueError(
                "the backend keeps its chain on device {0}, the sampler runs on device {1}".format(
                    self.backend.device, self._device)
            )
        if not self.backend.initialized:  # ensemble.py:137-141
            self._previous_state = None
            self.reset()
        else:
            if self.backend.shape != (self.nwalkers, self.ndim):
                raise ValueError(
                    "the shape of the backend ({0}) is incompatible with the "
                    "shape of the sampler ({1})".format(self.backend.shape, (self.nwalkers, self.ndim))
                )
            self.random_state = self.backend.random_state  # silently ignored if foreign
            if self.backend.iteration > 0:
                self._previous_state = self.get_last_sample()
            else:
                self._previous_state = None

    def _load_model(self):
        # the registered model, then its prior support (models.Bounded): a box is part of the model,
        # so a rebuilt engine (__setstate__) gets it back too; a user function is registered as the
        # engine's callback
        m = self.log_prob_fn
        if isinstance(m, CudaGraphFunction):
            # one capture per row count the schedule evaluates, all checked before the engine sees any
            rows = graph_row_counts(self.nwalkers, [mv.descriptor() for mv in self._moves])
            captured = [m.captured(r, self.ndim, self._device) for r in rows]
            self._engine.set_graphs([spec for _, spec in captured], [g for g, _ in captured])
            return
        if isinstance(m, CallbackFunction):
            self._engine.set_callback(m.evaluate, m.where, self.blobs_dtype)
            return
        self._engine.set_model(m.kind, m.device_params(self.ndim))
        box = m.bounds(self.ndim)
        if box is not None:
            self._engine.set_bounds(*box)

    def _user_slots(self):
        """``{schedule index: proposal slot}`` of the user moves, slots numbered densely in schedule order."""
        idx = [k for k, m in enumerate(self._moves) if user_move_spec(m) is not None]
        return {k: slot for slot, k in enumerate(idx)}

    def _load_moves(self):
        slots = self._user_slots()
        if len(slots) > _lib.EB_MAX_PROPOSAL_SLOTS:
            raise NotImplementedError("a move schedule holds at most %d user moves (got %d)"
                                      % (_lib.EB_MAX_PROPOSAL_SLOTS, len(slots)))
        specs = {k: user_move_spec(self._moves[k]) for k in slots}
        # captured proposals: every capture of every move checked before the engine sees any
        graphs = {k: sp[2]._graph_specs(self.nwalkers, self.ndim, self._device)
                  for k, sp in specs.items() if sp[1] == "graph"}
        for k, slot in slots.items():
            _, where, propose, setup = specs[k]
            if where == "graph":
                self._engine.set_proposal_graphs(slot, propose.draw, propose.ndraws, *graphs[k])
            else:
                self._engine.set_proposal(slot, propose, where, setup)

    # ------------------------------------------------------------------ state
    @property
    def random_state(self):
        """``("philox4x32-10", seed, step)`` -- the complete random state."""
        return self._random.get_state()

    @random_state.setter
    def random_state(self, state):
        # like ensemble.py:228-238: try, and stay as we are if it is garbage
        try:
            self._random.set_state(state)
        except Exception:
            pass

    @property
    def iteration(self):
        return self.backend.iteration

    def reset(self):
        self.backend.reset(self.nwalkers, self.ndim)

    @property
    def model(self):
        """The 4-tuple the reference hands to ``move.propose`` (``ensemble.py:393-395``),
        for callers that drive a move directly through the plugin boundary."""
        return Model(self.log_prob_fn, self.compute_log_prob, map, self._random)

    def __getstate__(self):
        """Picklable like the reference (``ensemble.py:251-256``, pinned by
        ``tests/unit/test_sampler.py:225-234``): the GPU engine is dropped and
        rebuilt on unpickling from the model, the Philox ``(seed, step)`` and
        the device index; the walker state travels through ``_previous_state``
        / the backend as it does in the reference."""
        d = dict(self.__dict__)
        d["_saved_rng"] = self._engine.get_rng()
        d["_saved_pinned"] = self._pinned is not None
        for k in ("_engine", "_random", "_pinned"):
            d.pop(k, None)
        d["_rdv"] = None  # a communicator does not survive pickling: re-attach after loading
        for attr, _ in _RUNNING:
            d[attr] = None  # the running statistics live in the engine's memory: enable them again after loading
        d["pool"] = None
        return d

    def __setstate__(self, d):
        seed, step = d.pop("_saved_rng")
        pinned = d.pop("_saved_pinned")
        self.__dict__.update(d)
        self._engine = _lib.Engine(self.nwalkers, self.ndim, seed, device=self._device)
        self._load_model()
        self._load_moves()
        self._engine.set_rng(seed, step)
        self._random = DeviceRandom(self._engine)
        self._pinned = None
        if pinned:
            self._pinned = (_lib.pinned_empty((self.nwalkers, self.ndim)), _lib.pinned_empty((self.nwalkers,)))

    # ------------------------------------------------------------ multi-GPU
    def attach(self, rdv, mode="p2p", gather_results=True):
        """Shard the ensemble by row block over the ranks of ``rdv``
        (:class:`emcee_b200.dist.Rendezvous`; one process per GPU, every rank
        builds the same sampler with the same seed and calls the same methods).

        ``gather_results=True``: yielded / returned states hold every walker
        (one collective replication per read-back).  ``False``: only the rows
        this rank owns (``owned_rows``) cross PCIe -- the other rows of the
        returned arrays are not refreshed."""
        from . import dist

        if isinstance(self.backend, DeviceBackend):
            raise NotImplementedError(_NO_SHARDED_DEVICE_CHAIN)
        if getattr(self, "_cuda_results", False):
            raise NotImplementedError("cuda_results=True: " + _NO_SHARDED_CUDA_ARRAYS)
        for attr, refusal in _RUNNING:
            if getattr(self, attr, None) is not None:
                raise NotImplementedError(refusal)
        if isinstance(self.log_prob_fn, CallbackFunction):
            raise NotImplementedError("a user log-probability function runs on one GPU; it cannot be sharded")
        if any(user_move_spec(m) is not None for m in self._moves):
            raise NotImplementedError("a user proposal runs on one GPU; a schedule with user moves cannot be sharded")
        if any(getattr(m, "kind", None) == "kde" for m in self._moves):
            raise NotImplementedError("KDEMove runs on one GPU; a schedule with it cannot be sharded")
        dist.attach(self._engine, rdv, mode)
        self._rdv = rdv
        self._gather_results = bool(gather_results)

    @property
    def owned_rows(self):
        """``slice`` of the walkers this process updates (all of them on one GPU)."""
        r0, n = self._engine.owned_rows()
        return slice(r0, r0 + n)

    def _refuse_sharded(self, attr):
        """Enabling the running statistic held in ``attr`` (``_RUNNING``) on a sharded ensemble raises."""
        if self._rdv is not None:
            raise NotImplementedError(dict(_RUNNING)[attr])

    def enable_moments(self, every=1):
        """Accumulate the chain mean / covariance on the device after every
        ``every``-th step (``0`` disables; calling it resets the accumulators)."""
        self._engine.set_option("moments_every", int(every))

    def moments(self):
        """``(mean[ndim], cov[ndim, ndim], count)`` over the ``(step, walker)``
        samples accumulated since :meth:`enable_moments` -- what
        ``np.mean`` / ``np.cov(rowvar=False)`` of ``get_chain(flat=True)`` give,
        without storing or downloading the chain (``store=False`` runs,
        ``ensemble.py:287-291``).  Collective on a sharded ensemble."""
        from . import dist

        part = self._engine.moments()
        parts = [part] if self._rdv is None else self._rdv.allgather(part)
        mean, cov, n, _ = dist.combine_moments(parts)
        return mean, cov, n

    def enable_histograms(self, range, bins=10, every=1, log_prob_range=None, params2d=None, bins2d=10):
        """Count every walker's coordinates into fixed bins on the device after every ``every``-th step (the
        cadence of :meth:`enable_moments`), for runs that store nothing.  :meth:`histogram` and
        :meth:`histogram2d` then return what ``get_histogram(bins, range, thin=every)`` and
        ``get_histogram2d(params2d, bins2d, range, thin=every)`` of a run that stored those steps return, when the
        step counter (``random_state[2]``) is a multiple of ``every`` at this call.

        ``range`` gives one ``(lo, hi)`` pair per parameter: the edges are fixed before any value is seen.
        ``log_prob_range`` (a pair) adds a histogram of the log-probabilities with ``bins`` bins; ``params2d``
        (distinct parameter numbers, at least two) adds ``np.histogram2d`` counts of every pair of them with
        ``bins2d`` bins per axis.  ``bins <= 4096`` and ``bins2d <= 128`` (``NotImplementedError`` beyond); a bad
        ``bins`` or range raises numpy's exception.  Every call zeroes the counts; ``every=0`` counts nothing.
        The counts are not pickled, and a sharded ensemble is refused."""
        from .summary import running_histogram_plan

        self._refuse_sharded("_hist")
        every = _index_at_least("every", every, 0)
        cfg = running_histogram_plan(self.ndim, range, bins, log_prob_range, params2d, bins2d)
        self._hist = None
        self._engine.histograms_config(every, cfg["bins"], cfg["outer"], cfg["edges"], cfg["log_prob"],
                                       cfg["params2d"], cfg["bins2d"], cfg["edges2d"])
        self._hist = cfg

    def _histogram_counts(self, counts=True):
        if getattr(self, "_hist", None) is None:
            raise RuntimeError(_NO_HISTOGRAMS)
        return self._engine.histograms(counts)

    def histogram(self, name="chain"):
        """``(hist, edges)`` of the running histograms (:meth:`enable_histograms`), as ``get_histogram`` returns
        them: ``hist[ndim, bins]`` (int64) and ``edges[ndim, bins + 1]`` for ``name="chain"``, ``hist[bins]`` and
        ``edges[bins + 1]`` for ``"log_prob"``."""
        if name not in ("chain", "log_prob"):
            raise ValueError("histograms are taken of 'chain' or 'log_prob', not {0!r}".format(name))
        hist, _, _ = self._histogram_counts()
        cfg = self._hist
        if name == "log_prob":
            if not cfg["log_prob"]:
                raise RuntimeError("no running histogram of the log-probabilities: pass log_prob_range to "
                                   "enable_histograms")
            return hist[self.ndim].astype(np.int64), cfg["edges"][self.ndim].copy()
        return hist[: self.ndim].astype(np.int64), cfg["edges"][: self.ndim].copy()

    def histogram2d(self):
        """``(hist[npairs, bins2d, bins2d], edges[len(params2d), bins2d + 1], pairs)`` of the running pair
        histograms (:meth:`enable_histograms` with ``params2d``), as ``get_histogram2d`` returns them."""
        _, hist2, _ = self._histogram_counts()
        cfg = self._hist
        if cfg["params2d"] is None:
            raise RuntimeError("no running pair histograms: pass params2d to enable_histograms")
        return hist2.astype(np.float64), cfg["edges2d"].copy(), list(cfg["pairs"])

    @property
    def histogram_count(self):
        """Samples counted per parameter by the running histograms: counted steps times ``nwalkers``."""
        return self._histogram_counts(counts=False)[2]

    def enable_trace(self, every=1):
        """Record one row of ensemble statistics on the device after every ``every``-th step (the cadence of
        :meth:`enable_histograms`), for runs that store nothing: each parameter's mean and variance over the
        walkers, the mean and maximum log-probability and the number of accepted proposals of that step
        (:meth:`trace`), and the best sample of all recorded steps (:meth:`best_sample`).  A row is about
        ``16 * ndim`` bytes where a stored step is ``8 * nwalkers * ndim``.

        Every call with ``every > 0`` drops the rows and the best sample recorded so far; ``every=0`` records nothing
        more and leaves them readable.  The initial state is never recorded.  The rows are not pickled, and a
        sharded ensemble is refused."""
        self._refuse_sharded("_trace_every")
        every = _index_at_least("every", every, 0)
        self._engine.trace_config(every)
        if every > 0 or self._trace_every is None:
            self._trace_every = every

    def _trace_on(self):
        if getattr(self, "_trace_every", None) is None:
            raise RuntimeError(_NO_TRACE)

    def trace(self, discard=0):
        """The rows recorded since :meth:`enable_trace`, from row ``discard`` on, as a :data:`Trace` of ``n`` rows:
        ``step[n]`` (uint64, the step counter), ``mean[n, ndim]`` and ``var[n, ndim]`` (``np.mean(x, axis=0)`` and
        ``np.var(x, axis=0, ddof=1)`` of that step's ensemble), ``log_prob_mean[n]``, ``log_prob_max[n]`` and
        ``accepted[n]`` (int64: the walkers that accepted their proposal in that step).  The sums are taken in a
        fixed order that depends on ``nwalkers`` alone, so the same steps give the same bytes however they were
        run."""
        self._trace_on()
        discard = _index_at_least("discard", discard, 0)
        step, rows = self._engine.trace_read(discard)
        D = self.ndim
        return Trace(step, rows[:, :D].copy(), rows[:, D:2 * D].copy(), rows[:, 2 * D].copy(),
                     rows[:, 2 * D + 1].copy(), rows[:, 2 * D + 2].astype(np.int64))

    def best_sample(self):
        """``(coords[ndim], log_prob, step, walker)`` of the largest log-probability among the steps the running
        trace recorded (:meth:`enable_trace`); ties go to the earliest step, then the lowest walker, as
        ``np.argmax(get_log_prob(thin=every, flat=True))`` of a run that stored those steps picks."""
        self._trace_on()
        if self._engine.trace_count() == 0:
            raise RuntimeError("the running trace has recorded no step yet")
        return self._engine.trace_best()

    def trace_autocorr_time(self, discard=0, **kwargs):
        """Integrated autocorrelation time, in steps, of each parameter's ensemble mean (Goodman & Weare 2010):
        ``every * autocorr.integrated_time(trace(discard).mean[:, None, :], **kwargs)`` with ``c``, ``tol`` and
        ``quiet`` as there, and its :class:`~emcee_b200.autocorr.AutocorrError` / warning for a short series."""
        from . import autocorr

        mean = self.trace(discard).mean
        return self._trace_every * autocorr.integrated_time(mean[:, None, :], **kwargs)

    def enable_reservoir(self, size, every=1):
        """Keep a uniform random sample, without replacement, of ``size`` of the ``(step, walker)`` rows of every
        ``every``-th step (the cadence of :meth:`enable_trace`) in GPU memory of a fixed size, for runs that store
        nothing: what ``get_chain(flat=True, thin=every)`` of a stored run offers, for percentiles, expectations, corner
        plots or downstream draws.  Each row gets a 64-bit key from the draw specification (tag 10, which no other draw
        uses, so the chain does not change) and the ``size`` rows with the smallest ``(key, step, walker)`` are kept: a
        pure function of the seed and the visited states, whatever the calls the run was cut into.  A row costs
        ``8 * ndim + 32`` bytes and the buffer holds ``size + max(size, nwalkers)`` of them (``MemoryError`` when the
        GPU has no room, or for ``size >= 2**32``, with nothing changed).  Setting ``random_state`` to another seed or
        to an earlier step (as ``run_mcmc`` from an earlier state does) empties the reservoir and keeps it enabled:
        the rows of a step offered again would come back with their old keys.

        Every call with ``every > 0`` drops what was kept; ``every=0`` records nothing more and leaves the contents
        readable.  The initial state is never recorded and blobs are not kept.  The contents are not pickled, and a
        sharded ensemble is refused."""
        self._refuse_sharded("_reservoir_every")
        size = _index_at_least("size", size, 1)
        every = _index_at_least("every", every, 0)
        self._engine.reservoir_config(size, every)
        if every > 0 or getattr(self, "_reservoir_every", None) is None:
            self._reservoir_every = every

    def _reservoir_on(self):
        if getattr(self, "_reservoir_every", None) is None:
            raise RuntimeError(_NO_RESERVOIR)

    def reservoir(self, cuda=False):
        """The rows kept since :meth:`enable_reservoir`, as a :data:`Reservoir` of ``k = min(size,
        reservoir_count())`` rows sorted by ``(key, step, walker)``: ``coords[k, ndim]``, ``log_prob[k]``,
        ``step[k]`` (uint64, the step counter the row was recorded at) and ``walker[k]`` (int64).  Any prefix of
        length ``j`` is a uniform sample of size ``j``, the reservoir of the same run with ``size=j``.
        ``cuda=True`` returns coords and log_prob as :class:`~emcee_b200.DeviceArray` s."""
        self._reservoir_on()
        return Reservoir(*self._engine.reservoir_read(cuda=bool(cuda)))

    def reservoir_count(self):
        """Rows offered to the reservoir since :meth:`enable_reservoir`: ``nwalkers`` times the recorded steps."""
        self._reservoir_on()
        return self._engine.reservoir_count()[0]

    def enable_autocorr(self, max_lag, every=1):
        """Estimate the autocorrelation time while sampling, for runs that store nothing: keep, on the GPU, the lag
        sums up to ``max_lag`` of every (walker, parameter) series of the states recorded after every ``every``-th
        step (the cadence of :meth:`enable_trace`; the initial state is never recorded).  They give the
        walker-averaged autocorrelation function (:meth:`autocorr_function`) and the reference estimator's
        :meth:`autocorr_time`, equal up to rounding to what a stored chain gives, in memory that does not grow with
        the run: about ``8 * nwalkers * ndim * (4 * max_lag + 64)`` bytes, allocated here (``MemoryError`` when the
        GPU has no room, with nothing changed).  Sokal's window reads the function up to about ``5 * tau``, so
        ``max_lag`` a few times larger than that is enough.

        Every call with ``every > 0`` drops what was recorded; ``every=0`` records nothing more and leaves the results
        readable.  The sums cannot forget steps, so there is no ``discard``: to leave burn-in out, enable after it.
        The sums are not pickled, and a sharded ensemble is refused."""
        self._refuse_sharded("_autocorr")
        max_lag = _index_at_least("max_lag", max_lag, 1)
        every = _index_at_least("every", every, 0)
        self._engine.running_acf_config(max_lag, every)
        if every > 0 or getattr(self, "_autocorr", None) is None:  # every=0 keeps the lags and cadence recorded
            self._autocorr = (max_lag, every)

    def _autocorr_on(self):
        if getattr(self, "_autocorr", None) is None:
            raise RuntimeError(_NO_AUTOCORR)
        return self._autocorr

    def autocorr_count(self):
        """Steps recorded since :meth:`enable_autocorr`."""
        self._autocorr_on()
        return self._engine.running_acf_count()

    def autocorr_function(self):
        """``rho[min(n, max_lag + 1), ndim]`` of the ``n`` recorded steps: what
        ``np.mean(autocorr._acf(x), axis=1)[:max_lag + 1]`` gives for the recorded states ``x[n, nwalkers, ndim]``
        (the reference's walker-averaged ``function_1d``), up to rounding.  A walker whose series is constant makes
        its parameter NaN, as numpy's ``0 / 0`` does.  Use :meth:`enable_autocorr` after burn-in to leave it out."""
        max_lag, _ = self._autocorr_on()
        return self._engine.running_acf_read(max_lag)

    def autocorr_time(self, c=5, tol=50, quiet=False):
        """Integrated autocorrelation time, in steps, of each parameter: what ``get_autocorr_time(thin=every, c=c,
        tol=tol, quiet=quiet)`` gives for a run that stored exactly the recorded steps, with its
        :class:`~emcee_b200.autocorr.AutocorrError` / warning for a series shorter than ``tol`` times the estimate.
        That holds when each parameter's window closes within ``max_lag`` or all lags are held (``n - 1 <=
        max_lag``); a window beyond ``max_lag`` raises :class:`~emcee_b200.autocorr.AutocorrError` with ``tau =
        every * taus[max_lag]`` (with ``quiet``: a warning, and that estimate).  There is no ``discard``: enable
        after burn-in."""
        from . import autocorr

        max_lag, every = self._autocorr_on()
        n = self.autocorr_count()
        if n == 0:
            raise RuntimeError("no step has been recorded since enable_autocorr")
        rho = self._engine.running_acf_read(max_lag)
        return every * autocorr.integrated_time_from_acf(rho, c=c, tol=tol, quiet=quiet, n_t=n, thin=every)

    def enable_window(self, size, every=1):
        """Keep the last ``size`` of the states recorded after every ``every``-th step (the cadence of
        :meth:`enable_trace`; the initial state is never recorded) in GPU memory, for runs that store nothing:
        :meth:`window` reads them as an ordered chain, the steps ``get_chain(thin=every)[-size:]`` of a run that
        stored every step returns, so the converged tail of an open-ended run can be thinned and analysed like a
        stored chain.  The ring takes ``size * nwalkers * (ndim + 1) * 8`` bytes of states and ``size * nwalkers``
        bytes of accept masks, allocated here (``MemoryError`` when the GPU has no room, with nothing changed).

        Every call with ``every > 0`` drops what was recorded; ``every=0`` records nothing more and leaves the
        contents readable.  Blobs are not kept.  The contents are not pickled, and a sharded ensemble is refused."""
        self._refuse_sharded("_window")
        size = _index_at_least("size", size, 1)
        every = _index_at_least("every", every, 0)
        self._engine.window_config(size, every)
        if every > 0 or getattr(self, "_window", None) is None:  # every=0 keeps the size and cadence recorded
            self._window = (size, every)

    def window(self):
        """The running window (:meth:`enable_window`) as a :class:`~emcee_b200.backend.ChainWindow`: a read-only
        view with ``DeviceBackend``'s readers and analyses that reads the live ring at each call."""
        if getattr(self, "_window", None) is None:
            raise RuntimeError(_NO_WINDOW)
        return ChainWindow(self)

    # ------------------------------------------------------------- the driver
    def _schedule(self):
        sched, slots = [], self._user_slots()
        for k, (m, w) in enumerate(zip(self._moves, self._raw_weights)):
            d = m.descriptor()
            if d["kind"] in ("user", "user_mh"):
                if d["kind"] == "user_mh" and m.ndim is not None and m.ndim != self.ndim:
                    raise ValueError("Dimension mismatch in proposal")  # mh.py:47-49
                d["p0"] = float(slots[k])  # the proposal slot _load_moves registered
            sched.append((d, w))
        return sched

    def _stored_before_failure(self, step0, thin_by, k0):
        """A bulk run stopped by an exception: the backend keeps the stored steps that completed, blobs
        included (the engine drained them before returning), and the random state of the last of them."""
        b = self.backend
        seed, step = self._engine.get_rng()
        stored = (step - step0) // thin_by
        b.iteration = k0 + stored
        if stored:
            b.random_state = (self.random_state[0], seed, step0 + stored * thin_by)

    def _after_steps(self):
        """Advance the host mirrors of stateful moves by what the engine just ran (``GaussianMove``
        mode ``"sequential"`` keeps a running dimension index, ``gaussian.py:102-103``)."""
        stateful = [m for m in self._moves if hasattr(m, "_advance")]
        if stateful:
            picks = self._engine.move_picks(len(self._moves))
            for m, p in zip(self._moves, picks):
                if hasattr(m, "_advance"):
                    m._advance(int(p), self.ndim)

    def sample(
        self,
        initial_state,
        log_prob0=None,
        rstate0=None,
        blobs0=None,
        iterations=1,
        tune=False,
        skip_initial_state_check=False,
        thin_by=1,
        thin=None,
        store=True,
        progress=False,
        progress_kwargs=None,
        _bulk=False,
    ):
        """Advance the chain as a generator (``ensemble.py:258-424``): yields the
        live :class:`State` every ``thin_by`` steps.

        Device-detected errors (NaN log-probability, non-finite proposal -- the
        reference's ``ValueError`` s, ``ensemble.py:476-479,550-551``) are raised
        when the C-ABI call that contains the offending step returns: per yielded
        state here, after the whole run for :meth:`run_mcmc` (one call)."""
        if log_prob0 is not None or rstate0 is not None or blobs0 is not None:
            raise NotImplementedError("log_prob0/rstate0/blobs0 are deprecated in the reference; pass a State")
        pbar = None
        if progress:
            # the reference wraps tqdm (pbar.py:33-60); one tick per yielded state here
            try:
                import tqdm

                total = None if iterations is None else iterations
                pbar = tqdm.tqdm(total=total, **(progress_kwargs or {}))
            except ImportError:
                pbar = None
        if iterations is None and store:
            raise ValueError("'store' must be False when 'iterations' is None")
        device_store = isinstance(self.backend, DeviceBackend)
        if device_store and self._rdv is not None:
            raise NotImplementedError(_NO_SHARDED_DEVICE_CHAIN)
        has_blobs = self.blobs_dtype is not None
        if device_store and has_blobs:
            raise NotImplementedError(_NO_DEVICE_CHAIN_BLOBS)

        # ``State(initial_state, copy=True)`` in the reference (ensemble.py:312): here the
        # upload to the device IS the copy -- the caller's arrays are only read, and
        # the yielded State gets its own arrays from the first device read-back
        state = State(initial_state)
        state = State(state.coords, log_prob=state.log_prob, blobs=state.blobs, random_state=state.random_state)
        if _lib.is_cuda_array(state.coords) or _lib.is_cuda_array(state.log_prob):
            self._set_cuda_state(state, skip_initial_state_check)
        else:
            state_shape = np.shape(state.coords)
            if state_shape != (self.nwalkers, self.ndim):
                raise ValueError("incompatible input dimensions {0}".format(state_shape))
            if state.blobs is not None and not has_blobs:
                raise NotImplementedError(
                    "the state carries blobs, but the log-probability function declares none "
                    "(models.HostFunction / models.CudaArrayFunction(fn, blobs_dtype=...))")
            if (not skip_initial_state_check) and (not self._walkers_independent(state.coords)):
                raise ValueError(_NOT_INDEPENDENT)
            self.random_state = state.random_state  # ensemble.py:335 (ignored if None/foreign)

            if state.log_prob is not None and np.shape(state.log_prob) != (self.nwalkers,):
                raise ValueError("incompatible input dimensions")
            # upload; a missing log_prob is evaluated on the device (ensemble.py:350-358), and a blob function's
            # records of that evaluation become the state's blobs
            self._engine.set_state(state.coords, state.log_prob, state.blobs if state.log_prob is not None else None)
        eng = self._engine
        if has_blobs:
            state.blobs = eng.get_blobs()

        if thin is not None:  # deprecated form: store every `thin`-th, yield every step
            thin = int(thin)
            if thin <= 0:
                raise ValueError("Invalid thinning argument")
            yield_step, checkpoint_step = 1, thin
            if store:
                self.backend.grow(iterations // checkpoint_step, state.blobs)
        else:
            thin_by = int(thin_by)
            if thin_by <= 0:
                raise ValueError("Invalid thinning argument")
            yield_step = checkpoint_step = thin_by
            if store:
                self.backend.grow(iterations, state.blobs)

        native_store = store and (type(self.backend) is Backend or device_store)
        store_blobs = native_store and state.blobs is not None  # the engine writes them into backend.blobs
        sched = self._schedule()

        def refresh():
            bufs = self._pinned if self._pinned is not None else (
                np.empty((self.nwalkers, self.ndim)), np.empty(self.nwalkers))
            if getattr(self, "_cuda_results", False):
                state.coords, state.log_prob = eng.get_state_to()  # device to device: nothing crosses PCIe
            elif self._rdv is not None and not self._gather_results:
                r0, n = eng.owned_rows()  # sharded: only the owned block crosses PCIe
                state.coords, state.log_prob = eng.get_state_rows(r0, n, *bufs)
            else:
                state.coords, state.log_prob = eng.get_state(*bufs)
            if has_blobs:
                state.blobs = eng.get_blobs()
            state.random_state = self.random_state

        if _bulk and iterations is not None and (not store or (native_store and thin is None)):
            # run_mcmc: the whole run is one C-ABI call
            total = iterations * yield_step
            if total > 0:
                if store:
                    b = self.backend
                    k0, k1 = b.iteration, b.iteration + iterations
                    step0 = eng.get_rng()[1]
                    try:
                        if device_store:
                            eng.step_store_chain(sched, total, checkpoint_step, b._ch, k0)
                        else:
                            eng.step_store(sched, total, checkpoint_step, b.chain[k0:k1], b.log_prob[k0:k1],
                                           b.accepted, b.blobs[k0:k1] if store_blobs else None)
                    except BaseException:
                        # a user function's exception, or a NaN it returned, stops the run inside a step
                        self._after_steps()
                        self._stored_before_failure(step0, checkpoint_step, k0)
                        raise
                    self._after_steps()
                    b.iteration = k1
                    b.random_state = self.random_state
                else:
                    try:
                        eng.step(sched, total, want_accepted=False)
                    finally:
                        self._after_steps()
            refresh()
            if pbar is not None:
                pbar.update(iterations)
                pbar.close()
            if iterations > 0:
                yield state
            return

        i = 0
        counter = iter(int, 1) if iterations is None else range(iterations)
        for _ in counter:
            # the steps of this yield window; at most the last one is stored
            sched = self._schedule()  # stateful moves (GaussianMove "sequential") change between calls
            last_is_checkpoint = store and (i + yield_step) % checkpoint_step == 0
            if last_is_checkpoint and native_store:
                b = self.backend
                k = b.iteration
                try:  # a window that stops early stores nothing: its one stored step is its last
                    if device_store:
                        eng.step_store_chain(sched, yield_step, yield_step, b._ch, k)
                    else:
                        eng.step_store(sched, yield_step, yield_step, b.chain[k : k + 1], b.log_prob[k : k + 1],
                                       b.accepted, b.blobs[k : k + 1] if store_blobs else None)
                finally:
                    self._after_steps()
                b.iteration = k + 1
                b.random_state = self.random_state
                refresh()
            else:
                try:
                    accepted = eng.step(sched, yield_step, want_accepted=last_is_checkpoint)
                finally:
                    self._after_steps()
                refresh()
                if last_is_checkpoint:
                    self.backend.save_step(state, accepted)
            i += yield_step
            if pbar is not None:
                pbar.update(1)
            yield state
        if pbar is not None:
            pbar.close()

    def _set_cuda_state(self, state, skip_initial_state_check):
        """The upload of a state given as CUDA arrays (``eb_set_state_from``), with the host path's checks in its
        order.  With ``skip_initial_state_check=False`` the coordinates are downloaded once for
        :meth:`_walkers_independent`: that check is the reference's numpy on the host, bit for bit.  With ``True``
        nothing crosses PCIe."""
        if self._rdv is not None:
            raise NotImplementedError(_NO_SHARDED_CUDA_ARRAYS)
        if not _lib.is_cuda_array(state.coords) or not (state.log_prob is None or _lib.is_cuda_array(state.log_prob)):
            raise TypeError("the initial coords and log_prob must both be CUDA arrays, or both host arrays")
        coords = _lib.CudaRows(state.coords, (self.nwalkers, self.ndim), self._device, "coords")
        if state.blobs is not None:
            raise NotImplementedError(_NO_CUDA_STATE_BLOBS)
        if (not skip_initial_state_check) and (not self._walkers_independent(coords.download(self._device))):
            raise ValueError(_NOT_INDEPENDENT)
        self.random_state = state.random_state  # ensemble.py:335 (ignored if None/foreign)
        lp = None
        if state.log_prob is not None:
            lp = _lib.CudaRows(state.log_prob, (self.nwalkers,), self._device, "log_prob")
        self._engine.set_state_from(coords, lp)

    def run_mcmc(self, initial_state, nsteps, **kwargs):
        """Iterate :func:`sample` for ``nsteps`` iterations and return the last
        state (``ensemble.py:426-456``); ``initial_state=None`` resumes."""
        if initial_state is None:
            if self._previous_state is None:
                raise ValueError("Cannot have `initial_state=None` if run_mcmc has never been called.")
            initial_state = self._previous_state
        results = None
        for results in self.sample(initial_state, iterations=nsteps, _bulk=True, **kwargs):
            pass
        self._previous_state = results
        return results

    def _walkers_independent(self, coords):
        """``walkers_independent`` (``ensemble.py:653-663``) with the O(N D^2) part on
        the device.  What is decided where:

        * host, the reference's own first statements (O(N D)): a non-finite
          coordinate gives False; ``C = coords - mean`` with numpy's mean and
          ``span = amax(|C|, 0)``; a zero span gives False.  The zero-span test
          is the reference's bit for bit, which a constant column needs: whether
          ``C`` is zero there depends on the order the mean was summed in.
        * device: ``eb_walkers_gram`` returns ``G = C^T C`` of ``C`` with column
          ``j`` scaled by ``2**-frexp(span_j)[1]``, re-centred and
          column-normalised.  The scaling is exact (or changes an entry by less
          than 2**-1074) and puts every column's largest entry in [0.5, 1), so
          the sums of squares neither underflow nor overflow at any scale of the
          coordinates.  The host solves the D x D eigen-problem, ``cond(C) =
          sqrt(l_max / l_min)``; squaring halves the digits, so only a clearly
          well-conditioned ensemble (cond <= 1e6 by the Gram matrix) is accepted
          here.
        * host, the reference's SVD statement: everything else -- cond above 1e6
          by the Gram matrix, a Gram matrix the device flags as unreliable, a
          centring that overflows, ndim above 1024."""
        coords = np.asarray(coords, dtype=np.float64)
        if coords.ndim != 2 or coords.shape[1] != self.ndim or self.ndim > 1024:
            return walkers_independent(coords)
        if not np.all(np.isfinite(coords)):
            return False
        # the same expressions as ensemble.py:656-659, so that the mean is numpy's, summed in its order
        centred = coords - np.mean(coords, axis=0)[None, :]
        span = np.amax(np.abs(centred), axis=0)
        if not np.all(np.isfinite(span)):
            return walkers_independent(coords)  # the centring overflowed
        if np.any(span == 0):
            return False
        centred = np.ldexp(centred, -np.frexp(span)[1][None, :])  # not a product: 2**-k overflows for a subnormal span
        gram, flags = self._engine.walkers_gram(centred)
        if flags:
            return walkers_independent(coords)
        ev = np.linalg.eigvalsh(gram)
        if ev[0] > 0 and np.sqrt(ev[-1] / ev[0]) <= 1e6:
            return True
        return walkers_independent(coords)

    def compute_log_prob(self, coords):
        """``(log_prob, blobs)`` for ``coords[..., ndim]`` evaluated on the device, or by the user
        function in one call (``ensemble.py:458-553``); ``blobs`` is None unless the function declares
        ``blobs_dtype``.  Raises ``ValueError`` for non-finite parameters or a NaN log-probability like
        the reference.

        ``coords`` may be a CUDA array of shape ``[m, ndim]`` (rows contiguous, the first axis may be strided):
        the result is then ``(DeviceArray[m], None)``, and nothing crosses PCIe.  A function declared with
        ``blobs_dtype`` takes host arrays only."""
        if _lib.is_cuda_array(coords):
            if self._rdv is not None:
                raise NotImplementedError(_NO_SHARDED_CUDA_ARRAYS)
            if self.blobs_dtype is not None:
                raise NotImplementedError("compute_log_prob of a function with blobs_dtype takes host arrays: blobs "
                                          "do not come back as CUDA arrays")
            return self._engine.compute_log_prob_from(coords), None
        coords = np.asarray(coords, dtype=np.float64)
        if self.blobs_dtype is not None:
            return self._engine.compute_log_prob_blobs(coords)
        return self._engine.compute_log_prob(coords), None

    # ---------------------------------------------------------------- results
    @property
    def acceptance_fraction(self):
        return self.backend.accepted / float(self.backend.iteration)

    def get_chain(self, **kwargs):
        return self.get_value("chain", **kwargs)

    def get_blobs(self, **kwargs):
        return self.get_value("blobs", **kwargs)

    def get_log_prob(self, **kwargs):
        return self.get_value("log_prob", **kwargs)

    def get_last_sample(self, **kwargs):
        """The backend's last stored ``State``; ``cuda=True`` (a ``DeviceBackend``) returns it as
        :class:`~emcee_b200.DeviceArray` s."""
        if "cuda" in kwargs:
            return self.backend.get_last_sample(cuda=kwargs["cuda"])
        return self.backend.get_last_sample()

    def get_value(self, name, **kwargs):
        return self.backend.get_value(name, **kwargs)

    def get_percentile(self, q, **kwargs):
        """``np.percentile`` of the flat stored slice along the samples (``backend.get_percentile``: on the
        device for a ``DeviceBackend``)."""
        return self.backend.get_percentile(q, **kwargs)

    def get_moments(self, **kwargs):
        """``(mean, cov, count)`` of the flat stored slice (``backend.get_moments``)."""
        return self.backend.get_moments(**kwargs)

    def get_histogram(self, bins=10, range=None, discard=0, thin=1, name="chain"):
        """``np.histogram`` of each parameter (or of the log-probabilities) of the flat stored slice
        (``backend.get_histogram``: counted on the device for a ``DeviceBackend``)."""
        return self.backend.get_histogram(bins, range, discard=discard, thin=thin, name=name)

    def get_histogram2d(self, params=None, bins=10, range=None, discard=0, thin=1):
        """``np.histogram2d`` of every pair of ``params`` of the flat stored slice (``backend.get_histogram2d``)."""
        return self.backend.get_histogram2d(params, bins, range, discard=discard, thin=thin)

    def get_autocorr_time(self, discard=0, thin=1, **kwargs):
        """Integrated autocorrelation time of the stored chain (``ensemble.py:619-623``
        -> ``backends/backend.py:130-150``), the FFTs on the GPU (``eb_autocorr``; a
        ``DeviceBackend`` is read in place by ``eb_chain_autocorr``)."""
        from . import autocorr

        if isinstance(self.backend, DeviceBackend):
            return self.backend.get_autocorr_time(discard=discard, thin=thin, **kwargs)
        x = self.get_chain(discard=discard, thin=thin)
        return thin * autocorr.integrated_time(x, engine=self._engine, **kwargs)


def walkers_independent(coords):
    """Initial-state sanity check (``ensemble.py:653-663``): the centred,
    column-normalised walker matrix must have condition number <= 1e8.  Runs
    once per ``sample`` call on the host."""
    coords = np.asarray(coords, dtype=np.float64)
    if not np.all(np.isfinite(coords)):
        return False
    centred = coords - np.mean(coords, axis=0)[None, :]
    span = np.amax(np.abs(centred), axis=0)
    if np.any(span == 0):
        return False
    centred /= span
    centred /= np.sqrt(np.sum(centred**2, axis=0))
    return np.linalg.cond(centred) <= 1e8
