"""Host-side parts of ``DeviceBackend``: the ``discard`` / ``thin`` slice arithmetic against numpy's
``[discard + thin - 1 : iteration : thin]`` (``backend.py:53``), the segment map of the device chain
(``emcee_b200/csrc/chain_map.h``, compiled for the host), and the contracts that need no GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emcee_b200
from emcee_b200.backend import slice_plan

HERE = os.path.dirname(os.path.abspath(__file__))

LAYOUTS = [[20], [1] * 20, [7, 13], [3, 5, 4, 8], [1, 19], [19, 1], [2, 2, 2, 2, 2, 10]]


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("chainmap") / "libchain_map_probe.so")
    subprocess.run(
        ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "helpers", "chain_map_host.cpp")],
        check=True,
    )
    lib = C.CDLL(out)
    lib.probe_chain_runs.restype = C.c_longlong
    lib.probe_chain_runs.argtypes = [C.POINTER(C.c_uint64), C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64,
                                     C.POINTER(C.c_uint64), C.c_size_t]
    return lib


def _runs(probe, sizes, first, stride, count):
    start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    out = np.zeros((max(count, 1), 4), dtype=np.uint64)
    p = C.POINTER(C.c_uint64)
    n = probe.probe_chain_runs(start.ctypes.data_as(p), len(sizes), first, stride, count, out.ctypes.data_as(p),
                               out.shape[0])
    return None if n < 0 else out[:n].astype(np.int64), start.astype(np.int64)


def test_slice_plan_matches_numpy():
    for it in range(21):
        steps = np.arange(it)
        for discard in range(26):
            for thin in range(1, 8):
                first, stride, count = slice_plan(it, discard, thin)
                want = steps[discard + thin - 1 : it : thin]
                assert count == len(want), (it, discard, thin)
                assert np.array_equal(first + stride * np.arange(count), want), (it, discard, thin)


def test_slice_plan_refuses_bad_thin():
    with pytest.raises(ValueError):
        slice_plan(10, 0, 0)


def test_segment_map(probe):
    """Every (iteration, discard, thin) slice over several segment layouts of a 20-slot chain: the runs
    visit the slice in order, each inside one segment, at the slots the slice names."""
    for sizes in LAYOUTS:
        for it in range(21):
            for discard in range(26):
                for thin in range(1, 8):
                    first, stride, count = slice_plan(it, discard, thin)
                    runs, start = _runs(probe, sizes, first, stride, count)
                    assert runs is not None
                    slots = []
                    k = 0
                    for seg, off, k0, n in runs:
                        assert k0 == k and n >= 1
                        s = start[seg] + off + stride * np.arange(n)
                        assert s[-1] < start[seg + 1], (sizes, it, discard, thin)
                        slots.extend(s)
                        k += n
                    assert k == count
                    assert np.array_equal(slots, first + stride * np.arange(count))
                    # a run ends only where the next slot falls into a later segment
                    for (seg, off, k0, n), nxt in zip(runs[:-1], runs[1:]):
                        assert nxt[0] > seg


def test_segment_map_refusals(probe):
    assert _runs(probe, [3, 4], 0, 1, 8)[0] is None  # past the capacity
    assert _runs(probe, [3, 4], 6, 1, 1)[0] is not None
    assert _runs(probe, [3, 4], 7, 1, 1)[0] is None
    assert _runs(probe, [3, 4], 0, 0, 2)[0] is None  # stride 0
    assert _runs(probe, [3, 4], 1, 2**63, 3)[0] is None  # overflow
    assert len(_runs(probe, [3, 4], 5, 1, 0)[0]) == 0


def test_float32_refused():
    with pytest.raises(NotImplementedError):
        emcee_b200.DeviceBackend(dtype=np.float32)


def test_constructs_without_gpu():
    b = emcee_b200.DeviceBackend(device=3)
    assert not b.initialized and b.nbytes == 0 and b.device == 3 and not b.has_blobs()
    with pytest.raises(AttributeError):
        b.get_chain()
    with pytest.raises(AttributeError):
        b.get_last_sample()
