"""Red-blue split move on the device (reference:
``src/emcee/moves/red_blue.py:11-106``).

The reference's ``propose`` loops over the splits on the host, calling
``get_proposal`` -> ``compute_log_prob_fn`` -> a per-walker Python accept loop
-> ``update``.  Here one C-ABI call (``eb_step``) runs the whole split cycle in
fused CUDA kernels; a subclass only describes itself (``descriptor``).

A subclass that overrides ``get_proposal`` is a user move: the engine calls its ``get_proposal(s, c, random)`` once
per half-step with the split's walkers and the other sets, as ``red_blue.py:85-90`` does, and keeps everything else
on the GPU (DESIGN.md §5.9)."""

import numpy as np

from .move import Move

__all__ = ["RedBlueMove"]


class RedBlueMove(Move):
    """Args mirror ``red_blue.py:37-42``: ``nsplits`` (default 2),
    ``randomize_split`` (default True), ``live_dangerously`` (default False).

    Override ``get_proposal(s, c, random) -> (q, factors)`` to write a move of your own: ``s`` is
    ``float64[Ns, ndim]``, the split's walkers in ascending walker order; ``c`` is the list of the ``nsplits - 1``
    other sets, in set order, each in ascending walker order; ``random`` is a numpy ``RandomState``
    (``moves.user_random``).  Return ``q`` (float64 ``[Ns, ndim]``) and ``factors`` (float64 ``[Ns]``, the log
    Hastings ratios).  An overridden ``setup(coords)`` is called once per step with a copy of the whole ensemble
    before the splits (``red_blue.py:73``), which costs one download of the state per step; without an override
    nothing is downloaded."""

    kind = None
    _where = "host"  # where a user get_proposal runs (moves.CudaArrayRedBlueMove: on CUDA arrays)

    def __init__(self, nsplits=2, randomize_split=True, live_dangerously=False):
        self.nsplits = int(nsplits)
        self.live_dangerously = live_dangerously
        self.randomize_split = randomize_split

    def setup(self, coords):
        pass

    def get_proposal(self, sample, complement, random):
        raise NotImplementedError(
            "proposals are generated inside the fused CUDA half-step kernel; "
            "there is no host-side get_proposal on the device path"
        )

    def _params(self):
        raise NotImplementedError("The proposal must be implemented by subclasses")

    def descriptor(self):
        if type(self).get_proposal is not RedBlueMove.get_proposal:
            # a user move: the sampler fills in p0 = its proposal slot; mode 1 = EB_USER_SETUP
            return dict(kind="user", nsplits=self.nsplits, randomize_split=bool(self.randomize_split),
                        live_dangerously=bool(self.live_dangerously), p0=float("nan"), p1=float("nan"),
                        mode=int(type(self).setup is not RedBlueMove.setup))
        p0, p1 = self._params()
        return dict(
            kind=self.kind,
            nsplits=self.nsplits,
            randomize_split=bool(self.randomize_split),
            live_dangerously=bool(self.live_dangerously),
            p0=p0,
            p1=p1,
        )

    def propose(self, model, state):
        """One ensemble step of this move on ``state`` (``red_blue.py:52-106``).

        ``model.random`` must be the sampler's ``DeviceRandom`` (it carries the
        engine).  The state is uploaded, stepped once on the GPU and read
        back; ``EnsembleSampler.sample`` avoids these copies by keeping the
        state resident and stepping many iterations per call."""
        engine = getattr(model.random, "engine", None)
        if engine is None:
            raise TypeError(
                "model.random must be an emcee_b200 DeviceRandom (the device "
                "path cannot consume a host RandomState)"
            )
        if type(self).get_proposal is not RedBlueMove.get_proposal:
            raise NotImplementedError("a user get_proposal runs inside EnsembleSampler.sample / run_mcmc")
        nwalkers, ndim = state.coords.shape
        if nwalkers < 2 * ndim and not self.live_dangerously:  # red_blue.py:64-70
            raise RuntimeError(
                "It is unadvisable to use a red-blue move "
                "with fewer walkers than twice the number of "
                "dimensions."
            )
        engine.set_state(state.coords, state.log_prob)
        accepted = engine.step([(self.descriptor(), 1.0)], 1)
        coords, log_prob = engine.get_state()
        state.coords = coords
        state.log_prob = log_prob
        return state, np.asarray(accepted, dtype=bool)
