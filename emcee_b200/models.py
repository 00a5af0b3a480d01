"""Log-probability models: registered device models and user functions.

The reference takes an arbitrary Python callable ``log_prob_fn``
(``src/emcee/ensemble.py:79-83``) and evaluates it row by row or through
``pool.map`` (``ensemble.py:486-496``).  The drop-in takes one of two things:

* a *registered model* (``GaussianIso``, ``GaussianDense``, ``Rosenbrock``,
  ``Ring``, optionally ``Bounded``): a small object naming one of the
  log-probabilities compiled into the CUDA library plus its parameters.  The
  whole half-step -- proposal, log-probability, accept -- is one kernel.
  These classes only carry parameters and are deliberately not callable.
* a *user function*, wrapped explicitly in ``HostFunction`` (numpy on the
  host), ``CudaArrayFunction`` (any CUDA-array library) or
  ``CudaGraphFunction`` (the function captured as CUDA graphs).  The engine calls
  it once per half-step with the whole ``[M, ndim]`` block of proposals of
  one split, never once per walker; split assignment, proposals, the accept
  decision and the update stay on the GPU.  The explicit wrapper keeps the
  rule that nothing is evaluated on the host unless the caller asked for it.
"""

import numpy as np

from . import _lib
from ._lib import FIXED_WIDTH as _FIXED_WIDTH
from ._lib import fixed_width_dtype

__all__ = [
    "DeviceModel", "GaussianIso", "GaussianDense", "Rosenbrock", "Ring", "Bounded",
    "CallbackFunction", "HostFunction", "CudaArrayFunction", "CapturedGraph", "CudaGraphFunction",
]


class DeviceModel(object):
    kind = None

    def device_params(self, ndim):
        """flat float64 parameter vector for ``eb_model_set``"""
        raise NotImplementedError

    def bounds(self, ndim):
        """``(lower, upper)`` of the prior's support for ``eb_model_set_bounds``, or None
        (unbounded)"""
        return None

    def __call__(self, *a, **k):
        raise TypeError(
            "device models are evaluated by the CUDA engine "
            "(EnsembleSampler.compute_log_prob); they cannot be called on the host"
        )


class GaussianIso(DeviceModel):
    """``-0.5 * sum(x**2)`` (the target of the reference's move tests,
    ``tests/integration/test_proposal.py:21-22``)."""

    kind = "gauss_iso"

    def device_params(self, ndim):
        return np.zeros(0)


class GaussianDense(DeviceModel):
    """``-0.5 * (x - mean)^T icov (x - mean)`` with a dense precision matrix
    (``document/plots/oned.py:17-18``)."""

    kind = "gauss_dense"

    def __init__(self, icov, mean=None):
        self.icov = np.ascontiguousarray(icov, dtype=np.float64)
        if self.icov.ndim != 2 or self.icov.shape[0] != self.icov.shape[1]:
            raise ValueError("icov must be a square matrix")
        d = self.icov.shape[0]
        self.mean = np.zeros(d) if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        if self.mean.shape != (d,):
            raise ValueError("mean must have shape (ndim,)")

    def device_params(self, ndim):
        if self.icov.shape[0] != ndim:
            raise ValueError("icov is %dx%d but ndim = %d" % (self.icov.shape + (ndim,)))
        return np.concatenate([self.mean, self.icov.ravel()])


class Rosenbrock(DeviceModel):
    """``-sum_i [ b (x[i+1] - x[i]^2)^2 + (a - x[i])^2 ]``"""

    kind = "rosenbrock"

    def __init__(self, a=1.0, b=100.0):
        self.a, self.b = float(a), float(b)

    def device_params(self, ndim):
        return np.array([self.a, self.b])


class Ring(DeviceModel):
    """``-(|x| - radius)^2 / (2 sigma^2)``"""

    kind = "ring"

    def __init__(self, radius=5.0, sigma=0.5):
        self.radius, self.sigma = float(radius), float(sigma)

    def device_params(self, ndim):
        return np.array([self.radius, self.sigma])


class Bounded(DeviceModel):
    """``model`` restricted to the closed box ``lower <= x <= upper``: the log-probability
    is the model's value inside the box and exactly ``-inf`` outside, which is what the
    usual emcee prior ::

        def log_prior(theta):
            if not ((lower <= theta) & (theta <= upper)).all():
                return -np.inf
            return 0.0

    adds to a log-likelihood.  The bounds are the prior's support, not a
    reparametrisation: walkers move in the same coordinates, proposals outside the
    box are rejected (``red_blue.py:96-101`` with ``lp = -inf``), and walkers that
    start outside have ``log_prob = -inf`` until they accept a proposal inside.

    ``lower`` / ``upper`` are scalars (broadcast to every parameter) or vectors of
    length ``ndim``; ``-inf`` / ``+inf`` give one-sided bounds.  NaN bounds and
    ``lower >= upper`` are refused with ValueError.  Every kernel that evaluates
    the model applies the box, and inside it the values are bit-identical to the
    unbounded model."""

    def __init__(self, model, lower, upper):
        if not isinstance(model, DeviceModel) or isinstance(model, Bounded):
            raise TypeError(
                "Bounded wraps one of the registered device models (not another Bounded, nor a user function: "
                "a HostFunction / CudaArrayFunction applies its prior itself)"
            )
        self.model = model
        self.kind = model.kind
        lo = np.array(lower, dtype=np.float64)
        hi = np.array(upper, dtype=np.float64)
        for name, v in (("lower", lo), ("upper", hi)):
            if v.ndim > 1:
                raise ValueError("%s must be a scalar or a vector of length ndim" % name)
            if np.isnan(v).any():
                raise ValueError("%s bound must not be NaN" % name)
        if lo.ndim == 1 and hi.ndim == 1 and lo.shape != hi.shape:
            raise ValueError("lower and upper have different lengths (%d, %d)" % (lo.size, hi.size))
        if not (lo < hi).all():
            raise ValueError("every lower bound must be below its upper bound")
        self.lower, self.upper = lo, hi

    def device_params(self, ndim):
        return self.model.device_params(ndim)

    def bounds(self, ndim):
        out = []
        for name, v in (("lower", self.lower), ("upper", self.upper)):
            if v.ndim == 1 and v.shape != (ndim,):
                raise ValueError("%s bound has length %d but ndim = %d" % (name, v.size, ndim))
            out.append(np.ascontiguousarray(np.broadcast_to(v, (ndim,)), dtype=np.float64))
        return out[0], out[1]


def _scalar(fx):
    """The reference's ``_scalar`` (``ensemble.py:703-713``): 1.0, np.float64(1.0), np.array([1.0]) and
    np.array(1.0) are all the float 1.0; anything with more than one element is an error."""
    if not np.isscalar(fx):
        try:
            fx = np.asarray(fx).item()
        except (TypeError, ValueError) as e:
            raise ValueError("log_prob_fn should return scalar") from e
        return float(fx)
    else:
        return float(fx)


def blobs_dtype_of(blobs_dtype):
    """``np.dtype(blobs_dtype)``, or ``NotImplementedError`` for a dtype whose records are not fixed-width bytes."""
    return None if blobs_dtype is None else fixed_width_dtype(blobs_dtype)


def log_prob_and_blobs(results, blobs_dtype):
    """``(log_prob[M], blobs[M, ...] or None)`` of a batch of results, by the reference's rules
    (``ensemble.py:498-547``): a result is a scalar (``_scalar``), or a sequence whose first entry is the
    log-probability and whose rest is the blob, ``blob = [r[1:] for r in results if len(r) > 1]``; the blobs
    become ``np.array(blob, dtype=blobs_dtype)`` with the size-1 axes after the first squeezed
    (``ensemble.py:541-545``).  Blobs that do not convert to the fixed-width dtype (strings, objects, ragged
    rows) raise ``NotImplementedError``."""
    try:
        blob = [r[1:] for r in results if len(r) > 1]
        if not len(blob):
            raise IndexError
        log_prob = np.array([_scalar(r[0]) for r in results], dtype=np.float64)
    except (IndexError, TypeError):
        return np.array([_scalar(r) for r in results], dtype=np.float64), None
    if len(blob) != len(log_prob):
        raise ValueError("%d of %d results carry blobs; every result must" % (len(blob), len(log_prob)))
    try:
        blob = np.array(blob, dtype=blobs_dtype)
    except (TypeError, ValueError) as e:
        raise NotImplementedError(_FIXED_WIDTH) from e
    shape = blob.shape[1:]
    if len(shape):
        axes = np.arange(len(shape))[np.array(shape) == 1] + 1
        if len(axes):
            blob = np.squeeze(blob, tuple(axes))
    return log_prob, blob


def log_prob_values(results):
    """The log-probability vector of a batch of results, by the reference's rules
    (``ensemble.py:498-512``): each result is a scalar (``_scalar``), or a sequence whose first entry
    is the log-probability and the rest blobs -- which a function without ``blobs_dtype`` may not
    return, so they raise ``NotImplementedError``."""
    if isinstance(results, np.ndarray) and results.ndim == 1 and results.dtype == np.float64:
        return results  # what the rules below give element by element, without the Python loop
    try:
        blob = [r[1:] for r in results if len(r) > 1]
        if not len(blob):
            raise IndexError
        np.array([_scalar(r[0]) for r in results])
    except (IndexError, TypeError):
        return np.array([_scalar(r) for r in results], dtype=np.float64)
    raise NotImplementedError(
        "the log-probability function returned blobs (a sequence per walker); declare them with "
        "blobs_dtype=... on the wrapper, or return the log-probability alone"
    )


class CallbackFunction(object):
    """A user log-probability function the engine calls back once per half-step
    (``HostFunction`` / ``CudaArrayFunction``).

    ``blobs_dtype`` (default None: the function returns no blobs, and blobs raise ``NotImplementedError``)
    declares that it returns blobs of that fixed-width dtype: the engine carries each walker's record with it
    through the accept step on the GPU and stores it with the chain (``State.blobs``, ``get_blobs``,
    ``compute_log_prob``), as the reference sampler's ``blobs_dtype`` does (``ensemble.py:92-95``)."""

    where = None

    def __init__(self, fn, args=None, kwargs=None, blobs_dtype=None):
        if not callable(fn):
            raise TypeError("fn must be callable, got {0!r}".format(fn))
        self.fn = fn
        self.args = list(args or [])
        self.kwargs = dict(kwargs or {})
        self.blobs_dtype = blobs_dtype_of(blobs_dtype)

    def _call(self, x):
        return self.fn(x, *self.args, **self.kwargs)


class HostFunction(CallbackFunction):
    """A numpy log-probability function, with the reference sampler's arguments and semantics
    (``ensemble.py:79-98, 486-496, 626-650``).

    ``vectorize=True``: one call ``fn(x, *args, **kwargs)`` per half-step with ``x[M, ndim]``, returning
    ``M`` values.  Otherwise one call per row through ``pool.map`` (``pool`` given) or the built-in
    ``map``.  Each row's result goes through the reference's ``_scalar`` rule; blobs raise
    ``NotImplementedError`` unless ``blobs_dtype`` is given, and then follow the reference's blob rules
    (``log_prob_and_blobs``): per-row ``(lp, blob...)`` tuples, ``(lp, array)`` and ``[M, 1 + k]`` arrays
    all work.  ``x`` is a fresh array that the function owns.  Rows reach the function
    only when every parameter is finite; a NaN result stops the run with ``ValueError`` at that
    half-step.  Pickling drops ``pool``, as the sampler does (``ensemble.py:251-256``)."""

    where = "host"

    def __init__(self, fn, vectorize=False, pool=None, args=None, kwargs=None, blobs_dtype=None):
        super().__init__(fn, args, kwargs, blobs_dtype)
        self.vectorize = bool(vectorize)
        self.pool = pool
        if pool is not None and not callable(getattr(pool, "map", None)):
            raise TypeError("pool must have a map() method")

    def evaluate(self, x):
        """``float64[M]`` for ``x[M, ndim]``; ``(float64[M], blobs[M, ...] or None)`` with ``blobs_dtype``."""
        if self.vectorize:
            results = self._call(x)
        else:
            map_func = self.pool.map if self.pool is not None else map
            results = list(map_func(self._call, x))
        if self.blobs_dtype is not None:
            return log_prob_and_blobs(results, self.blobs_dtype)
        return log_prob_values(results)

    def __getstate__(self):
        d = dict(self.__dict__)
        d["pool"] = None
        return d


class CudaArrayFunction(CallbackFunction):
    """A log-probability function on device arrays, for any library that speaks the CUDA Array
    Interface (torch, CuPy, Numba, ...; this package imports none of them).

    ``fn(x, *args, **kwargs)`` receives an immutable object with ``__cuda_array_interface__`` (v3):
    shape ``(M, ndim)``, ``<f8``, and ``stream`` set to the engine's stream.  It points to a scratch
    copy of the proposals in the engine's memory, complete when ``fn`` is called, which ``fn`` may
    overwrite (the proposals the update reads are elsewhere); it is valid only during the call -- copy
    it to keep it.  ``fn`` returns ``M`` float64 values: any CUDA-array-interface object of shape
    ``(M,)``, strided or not, or a numpy array (copied).  A result whose interface has a ``stream``
    entry (v3) is read after the work on that stream; one without (v2, which torch exports) after all
    work on the device, so a result still being computed on any stream is never read early.  ``M`` is
    the size of one split, ``nwalkers`` for ``GaussianMove`` and for the initial state.

    With ``blobs_dtype``, ``fn`` returns ``(lp, blobs)``: ``blobs`` is a CUDA-array-interface object (first
    axis strided or not, each record contiguous) or a numpy array of shape ``(M, *shape)`` and dtype
    ``blobs_dtype``, read under the same stream rules as ``lp``."""

    where = "device"

    def evaluate(self, x):
        return self._call(x)


class CapturedGraph(object):
    """One captured evaluation of ``m`` rows, what ``CudaGraphFunction``'s ``capture(m)`` returns.

    * ``exec``: the executable graph, a ``cudaGraphExec_t`` as an int (torch:
      ``torch.cuda.CUDAGraph().raw_cuda_graph_exec()``), instantiated on the sampler's device;
    * ``x``: its static input, a CUDA-array-interface object of shape ``(m, ndim)`` and dtype ``<f8`` whose rows
      are contiguous (the first axis may be strided);
    * ``lp``: its static output, shape ``(m,)``, ``<f8``, strided or not;
    * ``owner``: anything that must stay alive while the graph is used (torch: the ``CUDAGraph``, which owns the
      executable graph and its memory pool).

    The sampler keeps the object, and so ``x``, ``lp`` and ``owner``, alive while the model is loaded."""

    __slots__ = ("exec", "x", "lp", "owner")

    def __init__(self, exec, x, lp, owner=None):
        self.exec = exec
        self.x = x
        self.lp = lp
        self.owner = owner

    def __repr__(self):
        return "CapturedGraph(exec=%r, x=%r, lp=%r)" % (self.exec, self.x, self.lp)


class CudaGraphFunction(CallbackFunction):
    """A log-probability function that the engine runs as CUDA graphs, without the host.

    ``capture(m)`` returns a :class:`CapturedGraph` that evaluates ``m`` rows: launched, it reads the rows from
    its static ``x`` and writes their log-probabilities to its static ``lp``.  The sampler calls ``capture`` once
    per row count it needs when it loads the model -- in its constructor, and again after unpickling, since graphs
    do not travel: ``nwalkers``, and the split sizes ``ceil((nwalkers - j) / nsplits)`` of every red-blue move of
    the schedule.  From then on every log-probability the sampler evaluates comes from these graphs: each
    half-step copies its proposals into ``x``, launches the graph and reads ``lp`` on the engine's stream, with no
    Python call and no host synchronisation in between; the initial state and ``compute_log_prob`` run the
    ``nwalkers``-row graph in chunks, the last padded with copies of its last row.  Non-finite proposals and NaN
    log-probabilities raise the same exceptions as under :class:`CudaArrayFunction`, and leave the chain, the
    state and the random state where it leaves them; a stepping call reports them where it synchronises anyway, so
    a run with ``store=False`` and no running statistics synchronises once per chunk of up to 512 steps.

    The contract:

    * the graph must be deterministic and draw no random numbers: the engine launches it as captured, and torch's
      ``replay()`` bookkeeping (the random generator's offsets) does not run;
    * the graph may overwrite ``x``, so ``x`` must be writable; it never sees a non-finite row from the caller or a
      move.  After an error the engine copies no more rows into ``x``, and the launches that follow read what ``x``
      last held, possibly the graph's own writes, and their output is discarded;
    * one executable graph must not be shared by two samplers that run at the same time, since both would write
      the same ``x``;
    * no blobs (``blobs_dtype`` raises ``NotImplementedError``), and one GPU only (``attach`` is refused).

    The torch recipe (this package imports no torch)::

        def capture(m):
            x = torch.zeros(m, ndim, dtype=torch.float64, device="cuda")
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):  # warm up outside the capture
                for _ in range(3):
                    f(x)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                lp = f(x)
            return models.CapturedGraph(g.raw_cuda_graph_exec(), x, lp, owner=g)

        sampler = EnsembleSampler(nwalkers, ndim, models.CudaGraphFunction(capture))

    ``capture`` is pickled with the sampler, so for a picklable sampler it must be a module-level function."""

    where = "graph"

    def __init__(self, capture, blobs_dtype=None):
        if blobs_dtype is not None:
            raise NotImplementedError("CudaGraphFunction returns no blobs: a captured graph writes log-probabilities "
                                      "only; use CudaArrayFunction(fn, blobs_dtype=...) for blobs")
        super().__init__(capture)
        self.capture = capture

    def evaluate(self, x):
        raise TypeError("a CudaGraphFunction is evaluated by launching its captured graphs "
                        "(EnsembleSampler.compute_log_prob)")

    def captured(self, m, ndim, device):
        """``(graph, (m, exec, x_ptr, x_row_stride, lp_ptr, lp_stride))``: ``capture(m)`` and its checked
        description.  A result of the wrong type, shape, dtype or strides, or with ``exec = 0``, raises here."""
        g = self.capture(m)
        what = "capture(%d) returned" % m
        if not isinstance(g, CapturedGraph):
            raise TypeError("%s %r; it must return a models.CapturedGraph" % (what, type(g).__name__))
        ex = g.exec
        if isinstance(ex, bool) or not isinstance(ex, (int, np.integer)) or not 0 < int(ex) < 2**64:
            raise ValueError("%s a graph whose exec is %r; it must be a non-zero cudaGraphExec_t handle as an int "
                             "(torch: CUDAGraph.raw_cuda_graph_exec())" % (what, ex))
        bufs = []
        for name, obj, shape in (("x", g.x, (m, ndim)), ("lp", g.lp, (m,))):
            if not _lib.is_cuda_array(obj):
                raise TypeError("%s a graph whose %s is not a CUDA array (it has no __cuda_array_interface__)"
                                % (what, name))
            cai = obj.__cuda_array_interface__
            got = tuple(int(n) for n in cai["shape"])
            if got != shape:
                raise ValueError("%s a graph whose %s has shape %s; it must be %s" % (what, name, got, shape))
            if name == "x" and cai["data"][1]:
                raise ValueError("%s a graph whose x is exported read-only; the engine writes the rows into x, so "
                                 "it must be writable" % what)
            rows = _lib.CudaRows(obj, shape, device, "the graph's " + name)
            if rows.ptr == 0:
                raise ValueError("%s a graph whose %s has a null data pointer" % (what, name))
            bufs.append(rows)
        x, lp = bufs
        return g, (m, int(ex), x.ptr, x.stride, lp.ptr, lp.stride)


def graph_row_counts(nwalkers, descriptors):
    """The row counts a ``CudaGraphFunction`` is captured for: ``nwalkers`` (the initial state, compute_log_prob,
    and the moves that propose every walker at once) and each split size ``ceil((nwalkers - j) / nsplits)`` of the
    moves' descriptors, in ascending order."""
    n = int(nwalkers)
    rows = {n}
    for d in descriptors:
        p = int(d["nsplits"])
        rows.update((n - j + p - 1) // p for j in range(p))
    return sorted(rows)
