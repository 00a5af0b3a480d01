"""User-written proposals (reference plugin boundary: ``RedBlueMove.get_proposal(s, c, random)``,
``src/emcee/moves/red_blue.py:47,90``, and ``MHMove(proposal_function)``, ``src/emcee/moves/mh.py:31-33,52``).

The engine keeps the split assignment, the gathers, the log-probability of a device model, the accept loop and the
update on the GPU; only the proposal function runs outside it, once per half-step (DESIGN.md §5.9).

``random``: every call gets ``user_random(seed, step, split)``, a fresh legacy ``RandomState`` on numpy's own
Philox4x64 stream keyed by the engine seed (purpose 8 of the draw specification).  It is a pure function of
``(seed, step, split)``, so a resumed chain and one run in a single call see the same draws.  The counter starts at
``(0, step, split, 8)``: the generator advances word 0, so the streams of different ``(step, split)`` are disjoint."""

import numpy as np

from .red_blue import RedBlueMove

__all__ = ["HostProposal", "CudaArrayProposal", "CudaArrayRedBlueMove", "user_random"]

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


def user_move_spec(move):
    """``(kind, where, propose(s, c, random), setup or None)`` of a user move, None for a built-in one."""
    if isinstance(move, RedBlueMove) and type(move).get_proposal is not RedBlueMove.get_proposal:
        setup = move.setup if type(move).setup is not RedBlueMove.setup else None
        return "user", move._where, move.get_proposal, setup
    fn = getattr(move, "get_proposal", None)
    if isinstance(fn, _UserProposal):
        return "user_mh", fn.where, (lambda s, c, random: fn(s, random)), None
    return None
