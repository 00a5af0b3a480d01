"""Moves of the device path (reference: ``src/emcee/moves/__init__.py``).

The red-blue family (``StretchMove``, ``DEMove``, ``DESnookerMove``, ``WalkMove``) and the
Metropolis family with Gaussian proposals (``MHMove``, ``GaussianMove``), and user-written proposals:
``RedBlueMove`` subclasses that override ``get_proposal`` (``CudaArrayRedBlueMove`` for CUDA arrays) and
``MHMove(HostProposal(fn))`` / ``MHMove(CudaArrayProposal(fn))``, their captured-graph forms
``CudaGraphRedBlueMove`` / ``MHMove(CudaGraphProposal(capture))``, and ``KDEMove`` (the reference's SciPy
kernel-density proposals, built on the device)."""

from .de import DEMove
from .de_snooker import DESnookerMove
from .gaussian import GaussianMove
from .kde import KDEMove
from .mh import MHMove
from .move import Move
from .red_blue import RedBlueMove
from .stretch import StretchMove
from .user import (CapturedProposal, CudaArrayProposal, CudaArrayRedBlueMove, CudaGraphProposal, CudaGraphRedBlueMove,
                   HostProposal, user_random)
from .walk import WalkMove

__all__ = ["Move", "RedBlueMove", "StretchMove", "DEMove", "DESnookerMove", "WalkMove", "KDEMove", "MHMove",
           "GaussianMove", "HostProposal", "CudaArrayProposal", "CudaArrayRedBlueMove", "user_random",
           "CapturedProposal", "CudaGraphRedBlueMove", "CudaGraphProposal"]
