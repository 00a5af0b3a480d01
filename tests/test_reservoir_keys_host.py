"""The running reservoir's key and plan built for the host, no GPU needed:

* the tag-10 key of ``emcee_b200/csrc/philox.cuh`` (``reservoir_key``), compiled with g++, against the numpy statement
  (``tests/reservoir_ref.py``) for random seeds, step counters above 2**32 and walkers near 2**31;
* the compaction and schedule of ``emcee_b200/csrc/reservoir_plan.h``, run by ``tests/helpers/reservoir_host.cpp`` in
  the order of the kernels of ``reservoir.cu``, against ``np.lexsort`` of every offered row: on random keys and on
  keys drawn from a handful of values (ties broken by step, then walker), with K below, equal to and above the rows
  offered; the schedule never lets the live entries exceed the buffer."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import philox as px
from reservoir_ref import reservoir_keys, reservoir_order

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = C.POINTER(C.c_uint64)
U32 = C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("reservoir") / "libreservoir_probe.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out,
                    os.path.join(HERE, "helpers", "reservoir_host.cpp")], check=True)
    lib = C.CDLL(out)
    lib.probe_reservoir_keys.restype = None
    lib.probe_reservoir_keys.argtypes = [C.c_uint64, U64, U32, C.c_int, U64]
    lib.probe_reservoir_cap.restype = C.c_uint64
    lib.probe_reservoir_cap.argtypes = [C.c_uint64, C.c_uint64]
    lib.probe_reservoir_compact.restype = None
    lib.probe_reservoir_compact.argtypes = [U64, U64, U32, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint8)]
    lib.probe_reservoir_stream.restype = C.c_uint64
    lib.probe_reservoir_stream.argtypes = [U64, U64, C.c_uint64, C.c_uint64, C.c_uint64, U64, U64, U32, U64]
    return lib


def _p(a, t):
    return a.ctypes.data_as(t)


def host_keys(probe, seed, step, walker):
    step = np.ascontiguousarray(step, dtype=np.uint64)
    walker = np.ascontiguousarray(walker, dtype=np.uint32)
    out = np.zeros(step.size, dtype=np.uint64)
    probe.probe_reservoir_keys(C.c_uint64(seed), _p(step, U64), _p(walker, U32), step.size, _p(out, U64))
    return out


@pytest.mark.parametrize("seed", [0, 1, 0x7ACE, 2**63 + 12345, 2**64 - 1] + [int(s) for s in
                                  np.random.default_rng(10).integers(0, 2**63, 4, dtype=np.uint64)])
def test_key_matches_numpy(probe, seed):
    rng = np.random.default_rng(seed % 2**32)
    steps = [1, 2, 977, 2**32 - 1, 2**32, 2**32 + 1, 2**40 + 3, 2**63 + 5, 2**64 - 1]
    walkers = np.concatenate([np.arange(5), rng.integers(0, 2**31, 40), 2**31 - 1 - np.arange(3), 2**31 + np.arange(3),
                              [2**32 - 1]]).astype(np.uint32)
    for step in steps:
        ref = reservoir_keys(seed, step, walkers)
        got = host_keys(probe, seed, np.full(walkers.size, step, dtype=np.uint64), walkers)
        assert got.dtype == np.uint64 and np.array_equal(got, ref)
    # a purpose of its own: not the first words of the accept draws (tag 5) of the same counter
    w0, w1, _, _ = px.draw_words(seed, 3, 0, px.TAG_ACCEPT, walkers)
    accept = (w1.astype(np.uint64) << np.uint64(32)) | w0.astype(np.uint64)
    assert not np.any(reservoir_keys(seed, 3, walkers) == accept)


def test_cap(probe):
    for K, N in [(1, 1), (1, 64), (7, 64), (64, 64), (200, 64), (10**6, 65536), (10**4, 65536)]:
        assert probe.probe_reservoir_cap(K, N) == K + max(K, N)


def _compact(probe, key, step, walker, K):
    key, step = np.ascontiguousarray(key, np.uint64), np.ascontiguousarray(step, np.uint64)
    walker = np.ascontiguousarray(walker, np.uint32)
    keep = np.zeros(key.size, dtype=np.uint8)
    probe.probe_reservoir_compact(_p(key, U64), _p(step, U64), _p(walker, U32), key.size, K,
                                  keep.ctypes.data_as(C.POINTER(C.c_uint8)))
    return keep.astype(bool)


@pytest.mark.parametrize("values", [None, 1, 3, 40])
@pytest.mark.parametrize("count", [1, 2, 37, 300])
def test_one_compaction_is_lexsort(probe, values, count):
    rng = np.random.default_rng(count * 7 + (values or 0))
    key = (rng.integers(0, 2**64, count, dtype=np.uint64) if values is None
           else rng.integers(0, values, count).astype(np.uint64) << np.uint64(rng.integers(0, 60)))
    step = rng.integers(1, 6, count).astype(np.uint64)
    walker = rng.permutation(count).astype(np.uint32)  # (step, walker) distinct
    order = reservoir_order(key, step, walker)
    for K in sorted({1, 2, count // 2 + 1, count - 1, count, count + 1, 3 * count}):
        if K < 1:
            continue
        keep = _compact(probe, key, step, walker, K)
        want = np.zeros(count, dtype=bool)
        want[order[:K]] = True
        assert np.array_equal(keep, want), K


def _stream(probe, keys, steps, K):
    R, N = keys.shape
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    steps = np.ascontiguousarray(steps, dtype=np.uint64)
    cap = probe.probe_reservoir_cap(K, N)
    ok, os_, ow = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
    stats = np.zeros(5, np.uint64)
    n = probe.probe_reservoir_stream(_p(keys, U64), _p(steps, U64), R, N, K, _p(ok, U64), _p(os_, U64), _p(ow, U32),
                                     _p(stats, U64))
    assert n != 2**64 - 1, "the live entries overflowed the buffer or their bound"
    return ok[:n], os_[:n], ow[:n], stats


@pytest.mark.parametrize("N", [1, 2, 7, 64, 65])
@pytest.mark.parametrize("ties", [False, True])
def test_stream_keeps_the_first_k(probe, N, ties):
    R = 23
    rng = np.random.default_rng(N + 100 * ties)
    if ties:  # a handful of key values: most rows tie with the K-th key, and the order falls to (step, walker)
        keys = rng.integers(0, 5, (R, N)).astype(np.uint64) * np.uint64(2**61)
    else:
        keys = np.stack([reservoir_keys(99, 3 * (r + 1), np.arange(N)) for r in range(R)])
    steps = 3 * np.arange(1, R + 1, dtype=np.uint64)
    all_key = keys.reshape(-1)
    all_step = np.repeat(steps, N)
    all_walker = np.tile(np.arange(N), R)
    order = reservoir_order(all_key, all_step, all_walker)
    total = R * N
    for K in sorted({1, 7, max(N - 1, 1), N, 3 * N + 5, total - 1, total, total + 9}):
        k, s, w, stats = _stream(probe, keys, steps, K)
        cap = K + max(K, N)
        assert stats[3] == cap and stats[4] == total
        assert stats[1] <= cap and stats[2] <= stats[1]
        assert k.size == min(K, total)
        mine = reservoir_order(k, s, w)
        want = order[:K]
        assert np.array_equal(k[mine], all_key[want]) and np.array_equal(s[mine], all_step[want])
        assert np.array_equal(w[mine].astype(np.int64), all_walker[want])
        # at most one compaction every max(1, K / N) records, and one before the read
        assert stats[0] <= R // max(1, K // N) + 1


def test_schedule_bound_never_passes_cap(probe):
    # long runs with the filter rejecting nothing (equal keys lose to the kept ones, so use increasing keys) or
    # everything: the bound grows by N per record and is cut back to min(K, offered)
    for K, N in [(1, 5), (3, 5), (5, 5), (12, 5), (100, 7)]:
        R = 60
        up = np.arange(R * N, dtype=np.uint64)[::-1].reshape(R, N).copy()  # every new row beats the kept ones
        k, s, w, stats = _stream(probe, up, np.arange(1, R + 1, dtype=np.uint64), K)
        assert stats[1] <= K + max(K, N) and stats[2] <= stats[1]
        assert np.array_equal(np.sort(k), np.arange(min(K, R * N), dtype=np.uint64))
