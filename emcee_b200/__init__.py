"""emcee_b200 -- the walker-update hot path of dfm/emcee on NVIDIA H100.

Exports mirror ``src/emcee/__init__.py:24-36`` for the part of the package
that the hot path covers."""

__version__ = "0.1.0"

from . import autocorr, models, moves
from ._lib import DeviceArray
from .backend import Backend, DeviceBackend
from .batch import BatchSampler
from .ensemble import EnsembleSampler, walkers_independent
from .model import Model
from .state import State

__all__ = ["EnsembleSampler", "BatchSampler", "walkers_independent", "State", "Model", "Backend", "DeviceBackend", "DeviceArray", "moves", "models", "autocorr", "__version__"]
