"""The running reservoir's compaction when the buffer holds two entries of the same (step, walker), no GPU needed.

The engine never offers a step twice -- ``eb_set_rng`` empties the reservoir when it moves the step counter back or
changes the seed -- but the compaction keeps exactly K entries whatever the buffer holds: ties on the key fall to
(step, walker), then to the buffer index (``res_entry_before`` in ``emcee_b200/csrc/reservoir_plan.h``).  The host
statement of the kernels (``tests/helpers/reservoir_host.cpp``) is built with libstdc++'s bounds checks and run on
streams whose steps go back."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from reservoir_ref import reservoir_keys, reservoir_order

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = C.POINTER(C.c_uint64)
U32 = C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("reservoir_rewind") / "libreservoir_checked.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-D_GLIBCXX_ASSERTIONS", "-shared", "-fPIC", "-o", out,
                    os.path.join(HERE, "helpers", "reservoir_host.cpp")], check=True)
    lib = C.CDLL(out)
    lib.probe_reservoir_cap.restype = C.c_uint64
    lib.probe_reservoir_cap.argtypes = [C.c_uint64, C.c_uint64]
    lib.probe_reservoir_stream.restype = C.c_uint64
    lib.probe_reservoir_stream.argtypes = [U64, U64, C.c_uint64, C.c_uint64, C.c_uint64, U64, U64, U32, U64]
    return lib


def _p(a, t):
    return a.ctypes.data_as(t)


def _stream(probe, keys, steps, K):
    R, N = keys.shape
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    steps = np.ascontiguousarray(steps, dtype=np.uint64)
    cap = probe.probe_reservoir_cap(K, N)
    ok, os_, ow = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
    stats = np.zeros(5, np.uint64)
    n = probe.probe_reservoir_stream(_p(keys, U64), _p(steps, U64), R, N, K, _p(ok, U64), _p(os_, U64), _p(ow, U32),
                                     _p(stats, U64))
    assert n != 2**64 - 1, "the live entries overflowed the buffer, passed their bound or missed K"
    return ok[:n], os_[:n], ow[:n]


@pytest.mark.parametrize("N,K", [(16, 10), (16, 1), (16, 16), (16, 17), (7, 30), (33, 5)])
def test_steps_offered_twice(probe, N, K):
    # steps 1 .. 10, then 6 .. 10 again with the same seed: the same keys come back
    steps = np.concatenate([np.arange(1, 11), np.arange(6, 11)]).astype(np.uint64)
    keys = np.stack([reservoir_keys(99, int(t), np.arange(N)) for t in steps])
    k, s, w = _stream(probe, keys, steps, K)
    assert k.size == min(K, steps.size * N)
    # every kept entry is an offered row, and no more copies of a row are kept than were offered
    offered = {}
    for t in steps:
        for v in range(N):
            offered[(int(t), v)] = offered.get((int(t), v), 0) + 1
    kept = {}
    for t, v in zip(s.tolist(), w.tolist()):
        kept[(t, v)] = kept.get((t, v), 0) + 1
    assert all(kept[r] <= offered.get(r, 0) for r in kept)
    for key, t, v in zip(k, s, w):
        assert key == reservoir_keys(99, int(t), [v])[0]
    # with no step offered twice the same stream keeps the first K by (key, step, walker)
    k1, s1, w1 = _stream(probe, keys[:10], steps[:10], K)
    o = reservoir_order(keys[:10].reshape(-1), np.repeat(steps[:10], N), np.tile(np.arange(N), 10))[:K]
    mine = reservoir_order(k1, s1, w1)
    assert np.array_equal(k1[mine], keys[:10].reshape(-1)[o])


@pytest.mark.parametrize("dup", [2, 3, 5])
def test_whole_buffer_of_one_key(probe, dup):
    # every row has the same key and every (step, walker) comes `dup` times: the tie order alone decides
    N, K = 8, 11
    steps = np.tile(np.arange(1, 5, dtype=np.uint64), dup)
    keys = np.full((steps.size, N), 12345, dtype=np.uint64)
    k, s, w = _stream(probe, keys, steps, K)
    assert k.size == K and np.all(k == 12345)
    rows = list(zip(s.tolist(), w.tolist()))
    assert all(rows.count(r) <= dup for r in set(rows))
