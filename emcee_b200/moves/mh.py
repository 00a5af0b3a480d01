"""Metropolis-Hastings move of the device path (reference: ``src/emcee/moves/mh.py:11-65``).

The reference's ``MHMove`` takes an arbitrary host ``proposal_function(coords, rng)``.  The device path runs
the Gaussian family of :class:`emcee_b200.moves.GaussianMove` in its own kernels, and a user function wrapped
as ``moves.HostProposal(fn)`` or ``moves.CudaArrayProposal(fn)`` once per step between the GPU's gather and its
accept (DESIGN.md §5.9).  A bare callable is refused: the wrapper is the explicit opt-in."""

import numpy as np

from .move import Move
from .user import _UserProposal

__all__ = ["MHMove"]


class MHMove(Move):
    """``MHMove(proposal_function, ndim=None)`` (``mh.py:31-33``).  ``proposal_function`` must be a
    device proposal descriptor (``GaussianMove`` builds one); ``propose`` runs one Metropolis step of the
    whole ensemble on the GPU: proposal kernel, batched log-probability, accept ``log u < lnpdiff``
    (``mh.py:57-58``) and in-place update."""

    kind = "gaussian"

    def __init__(self, proposal_function, ndim=None):
        if isinstance(proposal_function, _UserProposal):
            self.kind = "user_mh"
        elif not isinstance(proposal_function, dict) or proposal_function.get("family") != "gaussian":
            raise NotImplementedError(
                "MHMove on the device path needs a device proposal (GaussianMove) or a wrapped user function: "
                "MHMove(moves.HostProposal(fn)) for numpy arrays, MHMove(moves.CudaArrayProposal(fn)) for CUDA arrays"
            )
        self.ndim = ndim
        self.get_proposal = proposal_function
        self.index = 0  # gaussian.py:64 (mode "sequential")

    # the RedBlueMove constructor arguments do not exist for this family; the engine ignores them
    nsplits, randomize_split, live_dangerously = 1, False, True

    def descriptor(self):
        p = self.get_proposal
        if self.kind == "user_mh":  # the sampler fills in p0 = its proposal slot
            return dict(kind=self.kind, nsplits=1, randomize_split=False, live_dangerously=True,
                        p0=float("nan"), p1=float("nan"))
        return dict(kind=self.kind, nsplits=1, randomize_split=False, live_dangerously=True,
                    p0=float("nan"), p1=float("nan") if p["factor"] is None else float(p["factor"]),
                    mode=p["mode"], cov=p["cov"], seq_index=int(self.index))

    def _advance(self, picks, ndim):
        """The engine ran ``picks`` steps with this move: what ``gaussian.py:103`` does to ``index``."""
        if self.kind == "gaussian" and self.get_proposal["mode"] == 2:  # "sequential"
            self.index = (self.index + int(picks)) % int(ndim)

    def propose(self, model, state):
        """One Metropolis step of the ensemble through the plugin boundary (``mh.py:35-65``)."""
        engine = getattr(model.random, "engine", None)
        if engine is None:
            raise TypeError("model.random must be an emcee_b200 DeviceRandom")
        nwalkers, ndim = state.coords.shape
        if self.ndim is not None and self.ndim != ndim:
            raise ValueError("Dimension mismatch in proposal")  # mh.py:47-48
        if self.kind == "user_mh":
            raise NotImplementedError("a user proposal_function runs inside EnsembleSampler.sample / run_mcmc")
        engine.set_state(state.coords, state.log_prob)
        accepted = engine.step([(self.descriptor(), 1.0)], 1)
        self._advance(1, ndim)
        state.coords, state.log_prob = engine.get_state()
        return state, np.asarray(accepted, dtype=bool)
