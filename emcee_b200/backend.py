"""Chain stores with the reference's ``Backend`` protocol
(``src/emcee/backends/backend.py:12-237``): ``reset / grow / save_step /
get_chain / get_log_prob / get_last_sample / shape / iteration / accepted /
random_state``.  ``Backend`` keeps the chain in host memory, with the reference's
blob storage; ``DeviceBackend`` keeps it in the GPU's, without blobs.
``ChainWindow`` reads a sampler's running window, the last steps it recorded,
with ``DeviceBackend``'s readers.

The engine's ``eb_step_store_blobs`` writes stored steps straight into the
``chain`` / ``log_prob`` / ``blobs`` arrays of this class (pinned double-buffered
D2H), so ``store=True`` does not need a host round trip per step."""

import builtins
import itertools
import operator

import numpy as np

from .state import State

__all__ = ["Backend", "ChainWindow", "DeviceBackend", "slice_plan"]


class Backend(object):
    def __init__(self, dtype=None):
        self.initialized = False
        self.dtype = np.float64 if dtype is None else dtype
        if np.dtype(self.dtype) != np.float64:
            raise NotImplementedError("the device path stores float64 chains only")

    def reset(self, nwalkers, ndim):
        self.nwalkers, self.ndim = int(nwalkers), int(ndim)
        self.iteration = 0
        self.accepted = np.zeros(self.nwalkers, dtype=self.dtype)  # backend.py:31
        self.chain = np.empty((0, self.nwalkers, self.ndim), dtype=self.dtype)
        self.log_prob = np.empty((0, self.nwalkers), dtype=self.dtype)
        self.blobs = None
        self.random_state = None
        self.initialized = True

    def has_blobs(self):
        return self.blobs is not None

    @property
    def shape(self):
        return self.nwalkers, self.ndim

    # -- growth / writes ------------------------------------------------------
    def _check_blobs(self, blobs):
        """``backend.py:157-162``."""
        if self.has_blobs() and blobs is None:
            raise ValueError("inconsistent use of blobs")
        if self.iteration > 0 and blobs is not None and not self.has_blobs():
            raise ValueError("inconsistent use of blobs")

    def grow(self, ngrow, blobs):
        """Room for ``ngrow`` more stored steps (``backend.py:164-185``).  ``blobs`` (the state's,
        ``[nwalkers, ...]``, or None) gives the record type of the blob store,
        ``(blobs.dtype, blobs.shape[1:])``; every grow must bring the same one."""
        self._check_blobs(blobs)
        extra = max(int(ngrow) - (len(self.chain) - self.iteration), 0)
        if extra:
            total = len(self.chain) + extra
            chain = np.empty((total, self.nwalkers, self.ndim), dtype=self.dtype)
            chain[: len(self.chain)] = self.chain
            log_prob = np.empty((total, self.nwalkers), dtype=self.dtype)
            log_prob[: len(self.log_prob)] = self.log_prob
            self.chain, self.log_prob = chain, log_prob
        if blobs is None:
            return
        blobs = np.asarray(blobs)
        dt = np.dtype((blobs.dtype, blobs.shape[1:]))
        if self.blobs is None:
            self.blobs = np.empty((len(self.chain), self.nwalkers), dtype=dt)
            return
        # the reference concatenates (backend.py:180-185), which refuses another record shape; the engine
        # writes raw records, so another dtype of the same size is refused too
        if np.dtype((self.blobs.dtype, self.blobs.shape[2:])) != dt:
            raise ValueError("inconsistent blobs: stored as {0}, got {1}".format(
                np.dtype((self.blobs.dtype, self.blobs.shape[2:])), dt))
        if len(self.blobs) < len(self.chain):
            grown = np.empty((len(self.chain), self.nwalkers), dtype=dt)
            grown[: len(self.blobs)] = self.blobs
            self.blobs = grown

    def save_step(self, state, accepted):
        """Append one step (``backend.py:187-231``)."""
        self._check_blobs(state.blobs)
        if state.coords.shape != self.shape:
            raise ValueError("invalid coordinate dimensions; expected {0}".format(self.shape))
        if state.log_prob.shape != (self.nwalkers,):
            raise ValueError("invalid log probability size; expected {0}".format(self.nwalkers))
        if state.blobs is not None and not self.has_blobs():
            raise ValueError("unexpected blobs")
        if state.blobs is None and self.has_blobs():
            raise ValueError("expected blobs, but none were given")
        if state.blobs is not None and len(state.blobs) != self.nwalkers:
            raise ValueError("invalid blobs size; expected {0}".format(self.nwalkers))
        if accepted.shape != (self.nwalkers,):
            raise ValueError("invalid acceptance size; expected {0}".format(self.nwalkers))
        self.chain[self.iteration] = state.coords
        self.log_prob[self.iteration] = state.log_prob
        if state.blobs is not None:
            self.blobs[self.iteration] = state.blobs
        self.accepted += accepted
        self.random_state = state.random_state
        self.iteration += 1

    # -- reads ---------------------------------------------------------------
    def get_value(self, name, flat=False, thin=1, discard=0):
        if self.iteration <= 0:
            raise AttributeError(
                "you must run the sampler with 'store == True' before accessing the results"
            )
        if name == "blobs" and not self.has_blobs():
            return None
        v = getattr(self, name)[discard + thin - 1 : self.iteration : thin]  # backend.py:53
        if flat:
            return v.reshape((v.shape[0] * v.shape[1],) + v.shape[2:])
        return v

    def get_chain(self, **kwargs):
        """``[nsteps, nwalkers, ndim]`` (or flattened over walkers)."""
        return self.get_value("chain", **kwargs)

    def get_log_prob(self, **kwargs):
        return self.get_value("log_prob", **kwargs)

    def get_blobs(self, **kwargs):
        return self.get_value("blobs", **kwargs)

    def get_last_sample(self):
        if (not self.initialized) or self.iteration <= 0:
            raise AttributeError(
                "you must run the sampler with 'store == True' before accessing the results"
            )
        k = self.iteration - 1
        blobs = self.blobs[k] if self.has_blobs() else None
        return State(self.chain[k], log_prob=self.log_prob[k], blobs=blobs, random_state=self.random_state)

    def get_autocorr_time(self, discard=0, thin=1, **kwargs):
        """Integrated autocorrelation time per parameter, in steps
        (``backend.py:130-150``)."""
        from . import autocorr

        x = self.get_chain(discard=discard, thin=thin)
        return thin * autocorr.integrated_time(x, **kwargs)

    def get_percentile(self, q, discard=0, thin=1, name="chain"):
        """``np.percentile(get_value(name, flat=True, discard=discard, thin=thin), q, axis=0)``."""
        _check_summary_name(name)
        return np.percentile(self.get_value(name, flat=True, discard=discard, thin=thin), q, axis=0)

    def get_moments(self, discard=0, thin=1):
        """``(mean[ndim], cov[ndim, ndim], count)`` of ``get_chain(flat=True, discard=discard, thin=thin)``:
        ``np.mean(axis=0)``, ``np.cov(rowvar=False)`` (``ddof = 1``) and the number of samples, as
        ``EnsembleSampler.moments()`` gives them; NaN for an empty slice."""
        flat = self.get_chain(flat=True, discard=discard, thin=thin)
        if len(flat) == 0:
            return np.full(self.ndim, np.nan), np.full((self.ndim, self.ndim), np.nan), 0
        cov = np.cov(flat, rowvar=False).reshape(self.ndim, self.ndim)
        return np.mean(flat, axis=0), cov, len(flat)

    def get_histogram(self, bins=10, range=None, discard=0, thin=1, name="chain"):
        """``np.histogram`` of the flat slice: for ``name="chain"``, ``(hist[ndim, bins], edges[ndim, bins + 1])``
        whose row ``d`` is ``np.histogram(flat[:, d], bins, range=None if range is None else range[d])``; for
        ``"log_prob"``, ``np.histogram`` of the flat log-probabilities with ``range`` one pair."""
        _check_histogram_name(name)
        flat = self.get_value(name, flat=True, discard=discard, thin=thin)
        if name == "log_prob":
            return np.histogram(flat, bins=bins, range=range)
        ranges = _histogram_ranges(range, self.ndim)
        out = [np.histogram(flat[:, d], bins=bins, range=ranges[d]) for d in builtins.range(self.ndim)]
        return np.array([h for h, _ in out]), np.array([e for _, e in out], dtype=np.float64)

    def get_histogram2d(self, params=None, bins=10, range=None, discard=0, thin=1):
        """``(hist[npairs, bins, bins], edges[len(params), bins + 1], pairs)``: ``pairs`` is
        ``list(itertools.combinations(params, 2))`` and ``hist[p]`` is ``np.histogram2d(flat[:, i], flat[:, j], bins,
        range=None if range is None else [range[i], range[j]])[0]`` for ``(i, j) = pairs[p]``; ``edges[k]`` are the
        edges of ``params[k]``.  ``params`` (default: every parameter) are distinct, at least two, in any order;
        ``range`` is indexed by parameter number."""
        params = _histogram_params(params, self.ndim)
        ranges = _histogram_ranges(range, self.ndim)
        flat = self.get_chain(flat=True, discard=discard, thin=thin)
        pairs = list(itertools.combinations(params, 2))
        hist, edges = [], {}
        for i, j in pairs:
            h, ei, ej = np.histogram2d(flat[:, i], flat[:, j], bins=bins, range=None if range is None
                                       else [ranges[i], ranges[j]])
            hist.append(h)
            edges.setdefault(i, ei)
            edges.setdefault(j, ej)
        return np.array(hist), np.array([edges[k] for k in params], dtype=np.float64), pairs

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass


def _check_summary_name(name):
    if name not in ("chain", "log_prob"):
        raise ValueError("percentiles are taken of 'chain' or 'log_prob', not {0!r}".format(name))


def _check_histogram_name(name):
    if name not in ("chain", "log_prob"):
        raise ValueError("histograms are taken of 'chain' or 'log_prob', not {0!r}".format(name))


def _histogram_ranges(range, ndim):
    """``range`` (None, or one ``(lo, hi)`` pair or None per parameter) as a list of ``ndim`` entries"""
    if range is None:
        return [None] * ndim
    ranges = list(range)
    if len(ranges) != ndim:
        raise ValueError("range must hold one (lo, hi) pair per parameter: {0} for ndim = {1}".format(
            len(ranges), ndim))
    return ranges


def _histogram_params(params, ndim):
    """``params`` of ``get_histogram2d`` as a list of ints: distinct, in ``[0, ndim)``, at least two"""
    params = list(builtins.range(ndim)) if params is None else [operator.index(p) for p in params]
    if len(params) < 2:
        raise ValueError("get_histogram2d needs at least two parameters, got {0}".format(params))
    if len(set(params)) != len(params) or min(params) < 0 or max(params) >= ndim:
        raise ValueError("params must be distinct parameter numbers in [0, {0}), got {1}".format(ndim, params))
    return params


def slice_plan(iteration, discard=0, thin=1):
    """``(first, stride, count)`` of the stored steps ``get_value`` returns: the indices of
    ``range(iteration)[discard + thin - 1 : iteration : thin]`` (``backend.py:53``)."""
    thin = int(thin)
    if thin < 1:
        raise ValueError("thin must be >= 1")
    r = range(int(iteration))[int(discard) + thin - 1 : int(iteration) : thin]
    return r.start, r.step, len(r)


class DeviceBackend(object):
    """The ``Backend`` protocol with the chain kept in the GPU's memory (``eb_chain``).

    ``EnsembleSampler`` stores into it on the device: a stored step is one
    copy inside HBM instead of a transfer to the host, ``get_autocorr_time``
    reads the chain where it is, and only the slice a reader asks for
    (``get_chain`` / ``get_log_prob`` / ``get_last_sample`` / ``accepted``)
    crosses PCIe.  Capacity is bounded by device memory, not host RAM: a
    ``grow`` that cannot fit raises ``MemoryError``.

    ``cuda=True`` on ``get_chain`` / ``get_log_prob`` / ``get_value`` /
    ``get_last_sample`` returns the same values as
    :class:`~emcee_b200.DeviceArray` s, copied inside the GPU's memory: a caller
    who keeps working on the device (torch, CuPy) never pays the two PCIe trips.

    Nothing is allocated before ``reset`` (the sampler calls it), so the
    object can be built without a GPU.  ``close()`` frees the device memory;
    pickling downloads the contents, and loading uploads them again.
    Blobs and chains other than float64 are not supported."""

    def __init__(self, dtype=None, device=0):
        self.initialized = False
        self.dtype = np.float64 if dtype is None else dtype
        if np.dtype(self.dtype) != np.float64:
            raise NotImplementedError("the device path stores float64 chains only")
        self.device = int(device)
        self._chain = None
        self._closed = False

    @property
    def _ch(self):
        if self._closed:
            raise ValueError("this DeviceBackend was closed")
        return self._chain

    def reset(self, nwalkers, ndim):
        from . import _lib

        if self._closed:
            raise ValueError("this DeviceBackend was closed")
        self._free()
        self.nwalkers, self.ndim = int(nwalkers), int(ndim)
        self.iteration = 0
        self.random_state = None
        self._chain = _lib.Chain(self.nwalkers, self.ndim, self.device)
        self.initialized = True

    def _free(self):
        if self._chain is not None:
            self._chain.close()
            self._chain = None

    def close(self):
        """Free the device memory; any later use raises ``ValueError``."""
        self._free()
        self._closed = True
        self.initialized = False

    @property
    def nbytes(self):
        """Device bytes the chain holds."""
        return 0 if self._chain is None else self._chain.capacity()[1]

    def has_blobs(self):
        return False

    @property
    def shape(self):
        if self._ch is None:
            raise AttributeError("shape: the backend has not been reset")
        return self.nwalkers, self.ndim

    @property
    def accepted(self):
        """Per-walker accepted proposals of the stored steps (float64, ``backend.py:31``), downloaded."""
        return self._ch.accepted()

    # -- growth / writes ------------------------------------------------------
    def grow(self, ngrow, blobs):
        """Room for ``ngrow`` more stored steps (``backend.py:164-185``): one new device segment for
        exactly the missing slots; stored steps are never copied."""
        if blobs is not None:
            raise NotImplementedError("blobs are not supported on the device path")
        self._ch.grow(self.iteration + int(ngrow))

    def save_step(self, state, accepted):
        """Append one step (``backend.py:214-231``), uploaded to the device."""
        ch = self._ch
        if state.coords.shape != self.shape:
            raise ValueError("invalid coordinate dimensions; expected {0}".format(self.shape))
        if state.log_prob.shape != (self.nwalkers,):
            raise ValueError("invalid log probability size; expected {0}".format(self.nwalkers))
        if accepted.shape != (self.nwalkers,):
            raise ValueError("invalid acceptance size; expected {0}".format(self.nwalkers))
        if state.blobs is not None:
            raise NotImplementedError("blobs are not supported on the device path")
        ch.write(self.iteration, state.coords, state.log_prob, accepted)
        self.random_state = state.random_state
        self.iteration += 1

    # -- reads ---------------------------------------------------------------
    def _plan(self, discard, thin):
        ch = self._ch
        if (not self.initialized) or self.iteration <= 0:
            raise AttributeError(
                "you must run the sampler with 'store == True' before accessing the results"
            )
        return ch, slice_plan(self.iteration, discard, thin)

    def get_value(self, name, flat=False, thin=1, discard=0, cuda=False):
        """``Backend.get_value``; ``cuda=True``: a :class:`~emcee_b200.DeviceArray` of the same shape and values,
        device to device (``eb_chain_read_to``)."""
        ch, (first, stride, count) = self._plan(discard, thin)
        if name == "blobs":
            return None
        if name not in ("chain", "log_prob"):
            raise AttributeError(name)
        want_chain = name == "chain"
        if cuda:
            shape = (count, self.nwalkers, self.ndim) if want_chain else (count, self.nwalkers)
            if flat:
                shape = (shape[0] * shape[1],) + shape[2:]
            x, lp = ch.read_to(first, stride, count, shape if want_chain else None, None if want_chain else shape)
            return x if want_chain else lp
        x, lp = ch.read(first, stride, count, coords=want_chain, log_prob=not want_chain)
        v = x if want_chain else lp
        if flat:
            return v.reshape((v.shape[0] * v.shape[1],) + v.shape[2:])
        return v

    def get_chain(self, **kwargs):
        """``[nsteps, nwalkers, ndim]`` (or flattened over walkers), downloaded (``cuda=True``: in device memory)."""
        return self.get_value("chain", **kwargs)

    def get_log_prob(self, **kwargs):
        return self.get_value("log_prob", **kwargs)

    def get_blobs(self, **kwargs):
        return self.get_value("blobs", **kwargs)

    def get_last_sample(self, cuda=False):
        """The last stored step as a ``State``: host arrays, or :class:`~emcee_b200.DeviceArray` s with
        ``cuda=True``."""
        ch, _ = self._plan(0, 1)
        if cuda:
            x, lp = ch.read_to(self.iteration - 1, 1, 1, (self.nwalkers, self.ndim), (self.nwalkers,))
            return State(x, log_prob=lp, blobs=None, random_state=self.random_state)
        x, lp = ch.read(self.iteration - 1, 1, 1)
        return State(x[0], log_prob=lp[0], blobs=None, random_state=self.random_state)

    def get_autocorr_time(self, discard=0, thin=1, **kwargs):
        """Integrated autocorrelation time per parameter, in steps (``backend.py:130-150``): the
        FFTs read the stored slice in device memory (``eb_chain_autocorr``)."""
        from . import autocorr

        ch, (first, stride, count) = self._plan(discard, thin)
        rho = ch.autocorr_function(first, stride, count)
        return thin * autocorr.integrated_time_from_acf(rho, **kwargs)

    def get_percentile(self, q, discard=0, thin=1, name="chain"):
        """``Backend.get_percentile``: ``np.percentile`` of the flat slice along the samples, equal with ``==``
        (a zero comes back as +0.0).  The exact order statistics are selected on the device, where the chain is
        (``eb_chain_select``); only they cross PCIe, and numpy's interpolation runs on the host."""
        from .summary import percentile_finish, percentile_ranks

        _check_summary_name(name)
        ch, (first, stride, count) = self._plan(discard, thin)
        plan = percentile_ranks(q, count * self.nwalkers)
        shape = (0, self.ndim) if name == "chain" else (0,)
        if count == 0:
            return np.percentile(np.empty(shape), q, axis=0)  # numpy's own error for an empty slice
        if plan.ranks.size == 0:
            return percentile_finish(plan, np.empty(shape))
        stats, has_nan, _ = ch.select(name, first, stride, count, plan.ranks)
        if name == "log_prob":
            stats, has_nan = stats[:, 0], has_nan[0]
        return percentile_finish(plan, stats, has_nan)

    def get_moments(self, discard=0, thin=1):
        """``Backend.get_moments`` computed where the chain is (``eb_chain_moments``, the moment sums of
        ``EnsembleSampler.moments()``); ``ndim`` up to 1024."""
        ch, (first, stride, count) = self._plan(discard, thin)
        return ch.moments(first, stride, count)

    def _column_extremes(self, ch, name, first, stride, count, ranges):
        """``(lo, hi, has_nan)`` per column of the slice (ranks 0 and n - 1 of ``eb_chain_select``, one call for
        every column); NaN extremes, unread, when every column has a given range"""
        D = self.ndim if name == "chain" else 1
        if all(r is not None for r in ranges):
            return np.full(D, np.nan), np.full(D, np.nan), np.zeros(D, dtype=bool)
        n = count * self.nwalkers
        stats, has_nan, _ = ch.select(name, first, stride, count, np.array([0, n - 1], dtype=np.uint64))
        return stats[0], stats[1], has_nan

    def get_histogram(self, bins=10, range=None, discard=0, thin=1, name="chain"):
        """``Backend.get_histogram``, equal with ``==``, counted where the chain is (``eb_chain_histogram``, one read
        of the slice).  An autodetected range takes each column's minimum and maximum from ``eb_chain_select``;
        numpy forms the edges from them on the host (``summary.uniform_edges``), so a bad ``bins`` or range raises
        numpy's exception.  ``bins`` is an int of at most 4096; a finite range wider than the largest double
        raises ``ValueError`` (numpy's own result there is not meaningful)."""
        from .summary import HIST_BINS_MAX, histogram_bins, uniform_edges

        _check_histogram_name(name)
        ch, (first, stride, count) = self._plan(discard, thin)
        D = self.ndim if name == "chain" else 1
        ranges = [range] if name == "log_prob" else _histogram_ranges(range, D)
        n = histogram_bins(bins, HIST_BINS_MAX)
        if count == 0:  # numpy's empty-input result (edges over [0, 1] without a range), no device work
            out = [np.histogram(np.empty(0), bins=n, range=r) for r in ranges]
            hist, edges = np.array([h for h, _ in out]), np.array([e for _, e in out], dtype=np.float64)
            return (hist[0], edges[0]) if name == "log_prob" else (hist, edges)
        lo, hi, has_nan = self._column_extremes(ch, name, first, stride, count, ranges)
        outer, edges = uniform_edges(n, ranges, lo, hi, has_nan)
        hist = ch.histogram(name, first, stride, count, n, outer, edges)
        if name == "log_prob":
            return hist[0], edges[0]
        return hist, edges

    def get_histogram2d(self, params=None, bins=10, range=None, discard=0, thin=1):
        """``Backend.get_histogram2d``, equal with ``==``, counted where the chain is (``eb_chain_histogram2d``,
        one read of the slice for every pair of a tile).  Edges come from numpy on each column's ``[min; max]``
        (``summary.searched_edges``).  ``bins`` is an int of at most 128; a finite range wider than the largest
        double raises ``ValueError``.  The counts of all pairs are held in device memory at once
        (``npairs * bins^2 * 8`` bytes; ``MemoryError`` when they do not fit)."""
        from .summary import HIST2_BINS_MAX, histogram_bins, searched_edges

        ch, (first, stride, count) = self._plan(discard, thin)
        params = _histogram_params(params, self.ndim)
        ranges = _histogram_ranges(range, self.ndim)
        n = histogram_bins(bins, HIST2_BINS_MAX, two_d=True)
        pairs = list(itertools.combinations(params, 2))
        col_ranges = [ranges[p] for p in params]
        m = len(params)
        if count == 0:  # numpy's empty-input result, no device work
            e = searched_edges(n, col_ranges, np.zeros(m), np.ones(m), np.zeros(m, dtype=bool))
            return np.zeros((len(pairs), n, n)), e, pairs
        lo, hi, has_nan = self._column_extremes(ch, "chain", first, stride, count, col_ranges)
        edges = searched_edges(n, col_ranges, lo[params], hi[params], has_nan[params])
        hist = ch.histogram2d(first, stride, count, params, n, edges)
        return hist.astype(np.float64), edges, pairs

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    # -- pickling: the contents travel through the host ---------------------------
    def __getstate__(self):
        d = dict(dtype=self.dtype, device=self.device, closed=self._closed, initialized=self.initialized)
        if self.initialized:
            d.update(nwalkers=self.nwalkers, ndim=self.ndim, iteration=self.iteration,
                     random_state=self.random_state, accepted=self.accepted)
            x, lp = self._chain.read(0, 1, self.iteration) if self.iteration else (None, None)
            d.update(chain=x, log_prob=lp)
        return d

    def __setstate__(self, d):
        self.__init__(d["dtype"], d["device"])
        if d["initialized"]:
            self.reset(d["nwalkers"], d["ndim"])
            it = d["iteration"]
            self.grow(it, None)
            acc = d["accepted"]
            if not np.all((acc == np.floor(acc)) & (acc >= 0) & (acc <= it)):
                raise ValueError("accept counts must be integers in [0, iteration]")
            # the chain only adds accept masks: slot k adds (count > k), which sums to count over the slots
            for k in range(it):
                self._chain.write(k, d["chain"][k], d["log_prob"][k], acc > k)
            self.iteration = it
            self.random_state = d["random_state"]
        if d["closed"]:
            self.close()


_WINDOW_READ_ONLY = "a ChainWindow is a read-only view of the sampler's running window; {0} is refused"


class ChainWindow(DeviceBackend):
    """The last ``size`` steps a sampler recorded (``EnsembleSampler.enable_window``), read like a
    :class:`DeviceBackend` that stored them: every reader and analysis of ``DeviceBackend`` (``get_chain``,
    ``get_log_prob``, ``get_value``, ``get_last_sample``, ``cuda=True``, ``get_autocorr_time``, ``get_percentile``,
    ``get_moments``, ``get_histogram``, ``get_histogram2d``), with ``discard`` / ``thin`` taken over the window's own
    slots, oldest first.  Each call reads the ring as it is then, in GPU memory (``eb_window_chain``).

    ``iteration`` is the number of slots filled, ``recorded`` the steps recorded since ``enable_window``, ``steps``
    the step counter of each slot.  ``accepted`` counts each walker's accepted proposals at the steps in the window,
    and ``get_autocorr_time`` is in sampler steps (``every * thin * tau``).  The view writes nothing: ``reset``,
    ``grow``, ``save_step`` and ``close`` raise ``TypeError``, and it cannot be pickled."""

    def __init__(self, sampler):
        self._sampler = sampler
        self.dtype = np.float64
        self.device = sampler._device
        self.nwalkers, self.ndim = sampler.nwalkers, sampler.ndim
        self.initialized = True
        self._closed = False

    @property
    def _engine(self):
        return self._sampler._engine

    @property
    def _ch(self):
        return self._engine.window_chain()

    _chain = _ch

    @property
    def every(self):
        """The cadence the window's steps were recorded with."""
        return self._sampler._window[1]

    @property
    def iteration(self):
        """Slots filled: ``min(recorded, size)``."""
        return self._engine.window_count()[1]

    @property
    def recorded(self):
        """Steps recorded since ``enable_window``."""
        return self._engine.window_count()[0]

    @property
    def steps(self):
        """``uint64[iteration]``: the sampler's step counter after each slot's step, oldest first."""
        return self._engine.window_steps()[0]

    @property
    def random_state(self):
        """``("philox4x32-10", seed, step)`` after the newest slot's step (None when the window is empty): with that
        slot's state it resumes the run exactly."""
        from .rng import STATE_TAG

        steps, seeds = self._engine.window_steps()
        if len(steps) == 0:
            return None
        return (STATE_TAG, int(seeds[-1]), int(steps[-1]))

    @property
    def acceptance_fraction(self):
        """``accepted / iteration``."""
        return self.accepted / float(self.iteration)

    def get_autocorr_time(self, discard=0, thin=1, **kwargs):
        """``DeviceBackend.get_autocorr_time`` of the window, in sampler steps: ``every * thin * tau``, what
        ``get_autocorr_time`` of a run that stored every step gives for the same states."""
        return self.every * super().get_autocorr_time(discard=discard, thin=thin, **kwargs)

    def reset(self, nwalkers, ndim):
        raise TypeError(_WINDOW_READ_ONLY.format("reset"))

    def grow(self, ngrow, blobs):
        raise TypeError(_WINDOW_READ_ONLY.format("grow"))

    def save_step(self, state, accepted):
        raise TypeError(_WINDOW_READ_ONLY.format("save_step"))

    def close(self):
        raise TypeError(_WINDOW_READ_ONLY.format("close"))

    def __getstate__(self):
        raise TypeError("a ChainWindow reads the sampler's GPU memory and cannot be pickled; pickle "
                        "get_chain() / get_log_prob() instead")
