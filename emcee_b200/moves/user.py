"""User-written proposals (reference plugin boundary: ``RedBlueMove.get_proposal(s, c, random)``,
``src/emcee/moves/red_blue.py:47,90``, and ``MHMove(proposal_function)``, ``src/emcee/moves/mh.py:31-33,52``).

The engine keeps the split assignment, the gathers, the log-probability of a device model, the accept loop and the
update on the GPU; only the proposal function runs outside it, once per half-step (DESIGN.md §5.9).

``random``: every call gets ``user_random(seed, step, split)``, a fresh legacy ``RandomState`` on numpy's own
Philox4x64 stream keyed by the engine seed (purpose 8 of the draw specification).  It is a pure function of
``(seed, step, split)``, so a resumed chain and one run in a single call see the same draws.  The counter starts at
``(0, step, split, 8)``: the generator advances word 0, so the streams of different ``(step, split)`` are disjoint."""

import numpy as np

from .. import _lib
from .red_blue import RedBlueMove

__all__ = ["HostProposal", "CudaArrayProposal", "CudaArrayRedBlueMove", "user_random", "CapturedProposal",
           "CudaGraphRedBlueMove", "CudaGraphProposal"]

PURPOSE_USER = 8


def user_random(seed, step, split):
    """The ``random`` argument of the user proposal call ``(step, split)`` of an engine keyed ``seed``."""
    key = int(seed) & (2**64 - 1)
    # Philox4x64 advances counter word 0 (carrying into word 1) once per 4-draw block: step and split live in the
    # words above it, so the streams of different calls never share a block
    return np.random.RandomState(np.random.Philox(key=key, counter=[0, int(step), int(split), PURPOSE_USER]))


class _UserProposal(object):
    where = None

    def __init__(self, fn):
        if not callable(fn):
            raise TypeError("the proposal function must be callable")
        self.fn = fn

    def __call__(self, coords, random):
        return self.fn(coords, random)


class HostProposal(_UserProposal):
    """``MHMove(HostProposal(fn))``: ``fn(coords, random) -> (q[N, ndim], factors[N])`` on numpy arrays
    (``mh.py:52``).  ``coords`` is a fresh copy of the whole ensemble in walker order; ``q`` and ``factors`` must be
    float64."""

    where = "host"


class CudaArrayProposal(_UserProposal):
    """``MHMove(CudaArrayProposal(fn))``: as :class:`HostProposal`, but ``coords`` is a read-only object with a v3
    ``__cuda_array_interface__`` (``<f8``, ``stream`` = the engine's stream) pointing at engine scratch that is valid
    only during the call.  ``fn`` returns ``q`` and ``factors`` as CUDA-array-interface objects (read after the stream
    they name, or after the whole device when they name none, as torch's v2 tensors do) or numpy arrays.  For device
    draws, seed a generator of your own from ``random``, e.g.
    ``torch.Generator(device="cuda").manual_seed(int(random.randint(2**62)))``."""

    where = "device"


class CudaArrayRedBlueMove(RedBlueMove):
    """A red-blue move whose ``get_proposal(s, c, random)`` works on CUDA arrays.

    ``s`` (the split's walkers, ascending walker order) and each ``c[j]`` (the other sets, in set order) are read-only
    objects with a v3 ``__cuda_array_interface__`` (``<f8``, ``stream`` = the engine's stream) pointing at engine
    scratch, valid only during the call.  Return ``(q[Ns, ndim], factors[Ns])`` as CUDA-array-interface objects or
    numpy arrays; they are read after the stream they name, or after the whole device when they name none (torch).
    An overridden ``setup(coords)`` receives the ensemble the same way.  ``random`` is the same numpy ``RandomState``
    host moves get; for device draws, seed a generator of your own from it, e.g.
    ``torch.Generator(device="cuda").manual_seed(int(random.randint(2**62)))``."""

    _where = "device"


class CapturedProposal(object):
    """One captured proposal, what the ``capture`` of :class:`CudaGraphRedBlueMove` and :class:`CudaGraphProposal`
    returns.

    * ``exec``: the executable graph, a ``cudaGraphExec_t`` as an int (torch:
      ``torch.cuda.CUDAGraph().raw_cuda_graph_exec()``), instantiated on the sampler's device;
    * static inputs, which the engine fills before every launch: ``s[ns, ndim]``, the active set; ``c[nc, ndim]``,
      the other sets back to back in set order (``None`` for an MHMove); ``draws[ns, ndraws]`` (``None`` when
      ``ndraws == 0``);
    * static outputs, which the engine reads after every launch: ``q[ns, ndim]`` and ``factors[ns]``;
    * ``owner``: anything that must stay alive while the graph is used (torch: the ``CUDAGraph``).

    Every buffer is a CUDA-array-interface object of dtype ``<f8`` whose rows are contiguous (the first axis may be
    strided); ``s``, ``c`` and ``draws`` must be writable.  The sampler keeps the object alive while its move is
    loaded."""

    __slots__ = ("exec", "s", "c", "draws", "q", "factors", "owner")

    def __init__(self, exec, s, c, draws, q, factors, owner=None):
        self.exec = exec
        self.s = s
        self.c = c
        self.draws = draws
        self.q = q
        self.factors = factors
        self.owner = owner

    def __repr__(self):
        return "CapturedProposal(exec=%r, s=%r, c=%r, draws=%r, q=%r, factors=%r)" % (
            self.exec, self.s, self.c, self.draws, self.q, self.factors)


def _draw_args(ndraws, draw):
    if isinstance(ndraws, bool) or not isinstance(ndraws, (int, np.integer)):
        raise TypeError("ndraws must be an int, got %r" % (ndraws,))
    ndraws = int(ndraws)
    if ndraws < 0:
        raise ValueError("ndraws must be >= 0, got %d" % ndraws)
    if ndraws > _lib.EB_MAX_GRAPH_DRAWS:
        raise NotImplementedError("a captured proposal takes at most %d draws per row (got %d)"
                                  % (_lib.EB_MAX_GRAPH_DRAWS, ndraws))
    if draw not in _lib.EB_DRAW_KINDS:
        raise ValueError("draw must be 'uniform' or 'normal', got %r" % (draw,))
    return ndraws, draw


def _checked(p, what, ns, nc, ndim, ndraws, device):
    """The pointers and byte strides ``(exec, s, s_stride, c, c_stride, draws, draws_stride, q, q_stride, factors,
    factors_stride)`` of a captured proposal, or the ``TypeError`` / ``ValueError`` of the first thing wrong with it."""
    if not isinstance(p, CapturedProposal):
        raise TypeError("%s %r; it must return a moves.CapturedProposal" % (what, type(p).__name__))
    ex = p.exec
    if isinstance(ex, bool) or not isinstance(ex, (int, np.integer)) or not 0 < int(ex) < 2**64:
        raise ValueError("%s a proposal whose exec is %r; it must be a non-zero cudaGraphExec_t handle as an int "
                         "(torch: CUDAGraph.raw_cuda_graph_exec())" % (what, ex))
    out = [int(ex)]
    for name, obj, shape, writable in (("s", p.s, (ns, ndim), True), ("c", p.c, (nc, ndim), True),
                                       ("draws", p.draws, (ns, ndraws), True), ("q", p.q, (ns, ndim), False),
                                       ("factors", p.factors, (ns,), False)):
        if (name == "c" and nc == 0) or (name == "draws" and ndraws == 0):
            if obj is not None:
                raise ValueError("%s a proposal with %s; it must be None %s" % (
                    what, name, "for an MHMove" if name == "c" else "when ndraws == 0"))
            out += [0, 0]
            continue
        if not _lib.is_cuda_array(obj):
            raise TypeError("%s a proposal whose %s is not a CUDA array (it has no __cuda_array_interface__)"
                            % (what, name))
        cai = obj.__cuda_array_interface__
        got = tuple(int(n) for n in cai["shape"])
        if got != shape:
            raise ValueError("%s a proposal whose %s has shape %s; it must be %s" % (what, name, got, shape))
        if writable and cai["data"][1]:
            raise ValueError("%s a proposal whose %s is exported read-only; the engine writes it before every "
                             "launch, so it must be writable" % (what, name))
        rows = _lib.CudaRows(obj, shape, device, "the proposal's " + name)
        if rows.ptr == 0:
            raise ValueError("%s a proposal whose %s has a null data pointer" % (what, name))
        out += [rows.ptr, rows.stride]
    return tuple(out)


class _Captured(object):
    """What the two captured-proposal classes share: ``ndraws``, ``draw`` and the capture of every split."""

    def _graph_specs(self, nwalkers, ndim, device):
        """``(specs, owners)`` for ``Engine.set_proposal_graphs``: one spec per split, ``capture`` called once per
        distinct argument tuple, every result checked before any reaches the engine."""
        cache, specs = {}, []
        for split, args in self._capture_args(int(nwalkers)):
            if args not in cache:
                ns = args[0]
                nc = int(nwalkers) - ns if len(args) > 1 else 0
                what = "capture%r returned" % (args,)
                p = self.capture(*args)
                cache[args] = (p, _checked(p, what, ns, nc, int(ndim), self.ndraws, device))
            p, chk = cache[args]
            specs.append((split, args[0]) + chk)
        return specs, [p for p, _ in cache.values()]


class CudaGraphRedBlueMove(_Captured, RedBlueMove):
    """A red-blue move whose proposal runs as captured CUDA graphs inside the engine's step loop.

    ``capture(ns, counts)`` returns a :class:`CapturedProposal` for an active set of ``ns`` rows whose other sets
    have the sizes ``counts`` (a tuple, in set order): launched, the graph reads ``s``, ``c`` and ``draws`` and
    writes the proposals ``q`` and their log Hastings factors ``factors``, as ``get_proposal(s, c, random)`` would
    return them.  The sampler calls ``capture`` once per distinct ``(ns, counts)`` of the move's splits, in its
    constructor and again after unpickling.  From then on every half-step gathers the split's walkers into ``s`` and
    ``c``, fills ``draws``, launches the graph and reads ``q`` and ``factors`` on the engine's stream, with no Python
    call and no host synchronisation.

    ``draws[i, :]`` holds ``ndraws`` values for row ``i``: ``draw="uniform"`` on ``[0, 1)`` or ``"normal"``
    standard normals, counter-addressed by ``(seed, step, split, i)`` like every draw of the engine (purpose 9 of
    the draw specification), so a resumed chain sees the draws of an uninterrupted one.  The graph itself must draw
    nothing: the engine launches it as captured, and torch's ``replay()`` bookkeeping of the generator does not run.

    Non-finite proposals raise the same exceptions as under :class:`CudaArrayRedBlueMove` and leave the chain, the
    state and the random state where it leaves them; a stepping call reports them where it synchronises anyway.
    No ``setup`` hook, ``ndraws <= 2**19``, and one GPU only (``attach`` is refused)."""

    _where = "graph"

    def __init__(self, capture, ndraws=0, draw="uniform", nsplits=2, randomize_split=True, live_dangerously=False):
        if not callable(capture):
            raise TypeError("capture must be callable")
        if type(self).setup is not RedBlueMove.setup:
            raise NotImplementedError("a captured proposal has no setup hook: the engine calls nothing per step")
        super().__init__(nsplits, randomize_split, live_dangerously)
        self.capture = capture
        self.ndraws, self.draw = _draw_args(ndraws, draw)

    def get_proposal(self, sample, complement, random):
        raise NotImplementedError("a captured proposal runs as a CUDA graph inside EnsembleSampler.sample / run_mcmc")

    def descriptor(self):
        return dict(kind="user", nsplits=self.nsplits, randomize_split=bool(self.randomize_split),
                    live_dangerously=bool(self.live_dangerously), p0=float("nan"), p1=float("nan"), mode=0)

    def _capture_args(self, nwalkers):
        """``(split, (ns, counts))`` of every split: sizes ``ceil((nwalkers - j) / nsplits)``, the others' in set
        order."""
        P = self.nsplits
        sizes = [(nwalkers - j + P - 1) // P for j in range(P)]
        return [(j, (sizes[j], tuple(sizes[:j] + sizes[j + 1:]))) for j in range(P)]


class CudaGraphProposal(_Captured, _UserProposal):
    """``MHMove(CudaGraphProposal(capture, ndraws=0, draw="uniform"))``: an MHMove proposal that runs as a captured
    CUDA graph.  ``capture(nwalkers)`` returns a :class:`CapturedProposal` with ``c=None`` whose ``s`` receives the
    whole ensemble in walker order; draws, errors and the rest are those of :class:`CudaGraphRedBlueMove`, with
    split 0."""

    where = "graph"

    def __init__(self, capture, ndraws=0, draw="uniform"):
        super().__init__(capture)
        self.capture = capture
        self.ndraws, self.draw = _draw_args(ndraws, draw)

    def __call__(self, coords, random):
        raise NotImplementedError("a captured proposal runs as a CUDA graph inside EnsembleSampler.sample / run_mcmc")

    def _capture_args(self, nwalkers):
        return [(0, (nwalkers,))]


def user_move_spec(move):
    """``(kind, where, propose(s, c, random), setup or None)`` of a user move, None for a built-in one.  A captured
    proposal has ``where = "graph"`` and its move or proposal object in place of ``propose``."""
    if isinstance(move, CudaGraphRedBlueMove):
        return "user", "graph", move, None
    if isinstance(move, RedBlueMove) and type(move).get_proposal is not RedBlueMove.get_proposal:
        setup = move.setup if type(move).setup is not RedBlueMove.setup else None
        return "user", move._where, move.get_proposal, setup
    fn = getattr(move, "get_proposal", None)
    if isinstance(fn, CudaGraphProposal):
        return "user_mh", "graph", fn, None
    if isinstance(fn, _UserProposal):
        return "user_mh", fn.where, (lambda s, c, random: fn(s, random)), None
    return None
