"""The numpy statement of the running reservoir (``EnsembleSampler.enable_reservoir``): the tag-10 key of a recorded
row, on ``oracle/philox.py``'s ``draw_words``, and the reservoir of a set of rows as ``np.lexsort`` orders them."""
import numpy as np

from oracle import philox as px

TAG_RESERVOIR = 10


def reservoir_keys(seed, step, walker):
    """uint64 keys ``(w1 << 32) | w0`` of draw block ``(seed, step, split 0, tag 10, index = walker)`` for one step
    counter and an array of walkers"""
    w0, w1, _, _ = px.draw_words(seed, step, 0, TAG_RESERVOIR, np.asarray(walker, dtype=np.uint64))
    return (w1.astype(np.uint64) << np.uint64(32)) | w0.astype(np.uint64)


def reservoir_order(key, step, walker):
    """the indices of the rows in the order (key, step, walker)"""
    return np.lexsort((np.asarray(walker), np.asarray(step), np.asarray(key)))
