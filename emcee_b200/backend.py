"""Chain stores with the reference's ``Backend`` protocol
(``src/emcee/backends/backend.py:12-237``): ``reset / grow / save_step /
get_chain / get_log_prob / get_last_sample / shape / iteration / accepted /
random_state``.  ``Backend`` keeps the chain in host memory, with the reference's
blob storage; ``DeviceBackend`` keeps it in the GPU's, without blobs.

The engine's ``eb_step_store_blobs`` writes stored steps straight into the
``chain`` / ``log_prob`` / ``blobs`` arrays of this class (pinned double-buffered
D2H), so ``store=True`` does not need a host round trip per step."""

import numpy as np

from .state import State

__all__ = ["Backend", "DeviceBackend", "slice_plan"]


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

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass


def _check_summary_name(name):
    if name not in ("chain", "log_prob"):
        raise ValueError("percentiles are taken of 'chain' or 'log_prob', not {0!r}".format(name))


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

    def get_value(self, name, flat=False, thin=1, discard=0):
        ch, (first, stride, count) = self._plan(discard, thin)
        if name == "blobs":
            return None
        if name not in ("chain", "log_prob"):
            raise AttributeError(name)
        want_chain = name == "chain"
        x, lp = ch.read(first, stride, count, coords=want_chain, log_prob=not want_chain)
        v = x if want_chain else lp
        if flat:
            return v.reshape((v.shape[0] * v.shape[1],) + v.shape[2:])
        return v

    def get_chain(self, **kwargs):
        """``[nsteps, nwalkers, ndim]`` (or flattened over walkers), downloaded."""
        return self.get_value("chain", **kwargs)

    def get_log_prob(self, **kwargs):
        return self.get_value("log_prob", **kwargs)

    def get_blobs(self, **kwargs):
        return self.get_value("blobs", **kwargs)

    def get_last_sample(self):
        ch, _ = self._plan(0, 1)
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
