"""The numpy statement of purpose 9 of the draw specification (DESIGN.md §2): the draws the engine hands a captured
proposal (``moves.CudaGraphRedBlueMove``, ``moves.CudaGraphProposal``), built on ``oracle.philox``'s primitives.

Row ``i`` (the active rank of a red-blue split, the walker of an MHMove, whose split is 0) gets its draws ``2k`` and
``2k + 1`` from block ``(index=i, sub-index=k, TAG_GRAPH)`` of ``(seed, step, split)``: ``u53(w0, w1)`` and
``u53(w2, w3)`` for ``"uniform"``, the Box-Muller pair of purpose 6 on these words for ``"normal"``."""
import numpy as np

from oracle import philox as px

TAG_GRAPH = 9
MAX_DRAWS = 2 ** 19  # the 18-bit sub-index field holds k < 2**18


def graph_draws(seed, step, split, rows, draw, ndraws):
    """``[rows, ndraws]`` draws of ``(seed, step, split)``; ``rows`` is a row count or an array of row indices."""
    index = np.arange(int(rows), dtype=np.uint64) if np.ndim(rows) == 0 else np.asarray(rows, dtype=np.uint64)
    if draw not in ("uniform", "normal"):
        raise ValueError(draw)
    if not 0 <= int(ndraws) <= MAX_DRAWS:
        raise ValueError(ndraws)
    out = np.empty((len(index), int(ndraws)), dtype=np.float64)
    for k in range((int(ndraws) + 1) // 2):
        w0, w1, w2, w3 = px.draw_words(seed, step, px.sub_split(split, k), TAG_GRAPH, index)
        if draw == "uniform":
            a, b = px.u53(w0, w1), px.u53(w2, w3)
        else:
            r = np.sqrt(-2.0 * np.log(1.0 - px.u53(w0, w1)))
            th = 6.283185307179586 * px.u53(w2, w3)
            a, b = r * np.cos(th), r * np.sin(th)
        out[:, 2 * k] = a
        if 2 * k + 1 < ndraws:
            out[:, 2 * k + 1] = b
    return out
