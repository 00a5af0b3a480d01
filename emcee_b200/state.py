"""Host mirror of the ensemble state (reference: ``src/emcee/state.py:10-75``).

The live walker positions and log-probabilities stay in HBM inside the engine;
a ``State`` is the snapshot handed to / received from the user, with the
reference's attribute names, copy semantics and tuple-unpacking back-compat.
Its arrays are host arrays, or CUDA arrays (anything with the CUDA Array
Interface, such as ``emcee_b200.DeviceArray`` or a torch tensor on the GPU)
for callers that keep their data on the device."""

import copy as _copy

import numpy as np

__all__ = ["State"]


class State(object):
    """Snapshot of the ensemble: ``coords[nwalkers, ndim]``, ``log_prob[nwalkers]``,
    ``blobs`` (``[nwalkers, ...]`` records of a user function declared with ``blobs_dtype``, else ``None``)
    and ``random_state``.  ``coords`` and ``log_prob`` may be CUDA arrays: they are kept as they are (the
    reference's ``np.atleast_2d`` would copy them to the host).

    Iterating yields ``coords, log_prob, random_state`` (plus ``blobs`` when
    present), as the reference does for pre-3.0 callers (``state.py:47-75``)."""

    __slots__ = ("coords", "log_prob", "blobs", "random_state")

    def __init__(self, coords, log_prob=None, blobs=None, random_state=None, copy=False):
        other = coords if hasattr(coords, "coords") else None  # state.py:35-40
        if other is not None:
            fields = (other.coords, other.log_prob, other.blobs, other.random_state)
        else:
            if not hasattr(coords, "__cuda_array_interface__"):
                coords = np.atleast_2d(coords)  # state.py:42
            fields = (coords, log_prob, blobs, random_state)
        if copy:
            fields = tuple(_copy.deepcopy(f) for f in fields)
        self.coords, self.log_prob, self.blobs, self.random_state = fields

    def _as_tuple(self):
        head = (self.coords, self.log_prob, self.random_state)
        return head if self.blobs is None else head + (self.blobs,)

    def __len__(self):
        return len(self._as_tuple())

    def __iter__(self):
        return iter(self._as_tuple())

    def __getitem__(self, index):
        items = self._as_tuple()
        if not -len(items) <= index < len(items):
            raise IndexError("Invalid index '{0}'".format(index))
        return items[index]

    def __repr__(self):
        return "State({0}, log_prob={1}, blobs={2}, random_state={3})".format(
            self.coords, self.log_prob, self.blobs, self.random_state
        )
