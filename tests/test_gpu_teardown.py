"""Closing engines and device chains while every optional buffer they allocate on demand is live.

* Four engines that between them hold: debug taps, the dense_dmma timeline, the L2-flush buffer and its per-step
  events, running moments, running 1-D and 2-D histograms, a running trace, WalkMove / GaussianMove scratch, the
  log-probability and autocorrelation scratch, a host-mode callback with blobs (after ``compute_log_prob_blobs``),
  pinned store staging with blobs, a host-mode and a device-mode user proposal, and a prior box.
* One device chain grown in two segments, after ``select``, ``moments``, ``histogram``, ``histogram2d`` and the
  autocorrelation of a slice that spans both segments.
* Every destroy call returns ``EB_OK``, and a fresh engine on the same device and seed then reproduces, bit for
  bit, a short run made before any of them was created.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from emcee_b200 import _lib
from emcee_b200.summary import searched_edges, uniform_edges

pytestmark = pytest.mark.gpu

N, D, SEED = 64, 4, 0x7EA4D
NAN = float("nan")


def move(kind, nsplits=2, p0=2.0, p1=NAN, **kw):
    return dict(kind=kind, nsplits=nsplits, randomize_split=False, live_dangerously=False, p0=p0, p1=p1, **kw)


STRETCH = [(move("stretch"), 1.0)]
MIXED = [(move("stretch"), 0.4), (move("walk", p0=NAN), 0.3), (move("gaussian", p0=0, cov=np.full(D, 0.1)), 0.3)]
ICOV = np.eye(D) + 0.1 * np.ones((D, D))


def start():
    return np.random.default_rng(SEED).normal(size=(N, D))


def gauss_dense(e):
    e.set_model("gauss_dense", np.concatenate([np.zeros(D), ICOV.ravel()]))


def gauss_lp(x):
    return -0.5 * np.einsum("ij,jk,ik->i", x, ICOV, x)


def reference_run():
    """(coords, log_prob, naccepted) after 20 stretch steps of a fresh engine."""
    e = _lib.Engine(N, D, SEED)
    gauss_dense(e)
    e.set_state(start())
    e.step(STRETCH, 20)
    x, lp = e.get_state()
    out = (x, lp, e.naccepted())
    close(e)
    return out


def close(obj):
    """Destroy through the C ABI, so that its return code is checked (close() ignores it)."""
    destroy = _lib.lib().eb_chain_destroy if isinstance(obj, _lib.Chain) else _lib.lib().eb_destroy
    assert destroy(obj._h) == _lib.EB_OK
    obj._h = C.c_void_p()


def taps_timeline_flush():
    e = _lib.Engine(N, D, SEED)
    gauss_dense(e)
    e.set_state(start())
    e.set_option("dmma_timeline", 1)
    e.step(STRETCH, 3)
    e.set_option("debug_taps", 1)
    e.set_option("l2_flush", 1)
    e.step([(move("stretch"), 0.5), (move("de", p0=1e-5), 0.5)], 4)
    assert e.debug_taps()["active"].size > 0
    assert e.debug_timeline().size > 0
    return e


def running_statistics():
    e = _lib.Engine(N, D, SEED)
    gauss_dense(e)
    e.set_state(start())
    e.set_option("moments_every", 1)
    bins, bins2 = 16, 8
    rows = [(-6.0, 6.0)] * D + [(-60.0, 1.0)]
    outer, edges = zip(*(uniform_edges(bins, r) for r in rows))
    params2d = [0, 1, 3]
    edges2d = [searched_edges(bins2, rows[p]) for p in params2d]
    e.histograms_config(1, bins, np.array(outer), np.array(edges), log_prob=True, params2d=params2d, bins2d=bins2,
                        edges2d=np.array(edges2d))
    e.trace_config(1)
    e.step(MIXED, 12)
    assert e.moments()[2] == 12 * N
    assert e.histograms(counts=False)[2] == 12 * N
    assert e.trace_count() == 12
    e.compute_log_prob(start()[:7])
    e.walkers_gram(start())
    e.autocorr_function(np.random.default_rng(1).normal(size=(32, N, D)))
    return e


def host_callback_with_blobs():
    e = _lib.Engine(N, D, SEED)
    e.set_callback(lambda x: (gauss_lp(x), x[:, :2].copy()), "host", blobs_dtype=np.float64)
    e.set_state(start())
    e.set_proposal(0, lambda s, c, random: (s + 0.3 * random.randn(*s.shape), np.zeros(len(s))), "host")
    e.step(STRETCH + [(move("user_mh", p0=0), 1.0)], 4)
    lp, blobs = e.compute_log_prob_blobs(start()[:5])
    assert blobs.shape == (5, 2)
    nstore = 3
    chain, log_prob = np.zeros((nstore, N, D)), np.zeros((nstore, N))
    stored = np.zeros((nstore, N, 2))
    e.step_store(STRETCH, nstore, 1, chain, log_prob, np.zeros(N), blobs=stored)
    np.testing.assert_array_equal(stored, chain[:, :, :2])
    return e


def device_proposal():
    def propose(s, c, random):
        x = torch.as_tensor(s, device="cuda")
        q = x + torch.as_tensor(0.3 * random.randn(*x.shape), device="cuda")
        return q, torch.zeros(x.shape[0], dtype=torch.float64, device="cuda")

    e = _lib.Engine(N, D, SEED)
    gauss_dense(e)
    e.set_bounds(np.full(D, -50.0), np.full(D, 50.0))
    e.set_state(start())
    e.set_proposal(1, propose, "device")
    e.step([(move("user_mh", p0=1), 1.0)], 4)
    torch.cuda.synchronize()
    return e


def grown_chain():
    e = _lib.Engine(N, D, SEED)
    gauss_dense(e)
    e.set_state(start())
    ch = _lib.Chain(N, D)
    ch.grow(10)
    e.step_store_chain(STRETCH, 10, 1, ch, 0)
    ch.grow(25)
    e.step_store_chain(STRETCH, 15, 1, ch, 10)
    close(e)
    assert ch.capacity()[0] == 25
    ch.select("chain", 2, 1, 20, [0, 5 * N, 20 * N - 1])
    ch.moments(0, 1, 25)
    bins = 12
    outer, edges = zip(*(uniform_edges(bins, (-6.0, 6.0)) for _ in range(D)))
    ch.histogram("chain", 0, 1, 25, bins, np.array(outer), np.array(edges))
    ch.histogram2d(0, 1, 25, [0, 2], bins, np.array([searched_edges(bins, (-6.0, 6.0))] * 2))
    ch.autocorr_function(0, 1, 25)
    return ch


def test_close_with_every_optional_buffer_live():
    before = reference_run()
    live = [taps_timeline_flush(), running_statistics(), host_callback_with_blobs(), device_proposal(), grown_chain()]
    for obj in live:
        close(obj)
    after = reference_run()
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
