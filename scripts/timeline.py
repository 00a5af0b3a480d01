#!/usr/bin/env python
"""Consumer-warp timeline of the dense_dmma kernel (cycles), headline workload."""
import sys
sys.path.insert(0, ".")
import bench
import emcee_b200
from emcee_b200 import models

w = bench.make_workload("gauss_dense", 65536, 128)
s = emcee_b200.EnsembleSampler(65536, 128, models.GaussianDense(w["icov"]), seed=1)
eng = s._engine
eng.set_state(w["p0"])
sched = s._schedule()
eng.step(sched, 20, want_accepted=False)
eng.set_option("dmma_timeline", 1)
eng.step(sched, 3, want_accepted=False)
tl = eng.debug_timeline()  # [SM, consumer, tile, event]
nsm, ncons = tl.shape[0], tl.shape[1]
ntile = (tl[..., 5] > 0).sum(-1)
print("SMs %d, consumers per SM %d" % (nsm, ncons))
print("tiles per consumer (SM0):", ntile[0], " total per SM min/max:", ntile.sum(1).min(), ntile.sum(1).max())
for sm in sorted({0, nsm // 2, nsm - 1}):
    print("SM", sm)
    for c in range(ncons):
        rows = []
        for k in range(int(ntile[sm, c])):
            e = tl[sm, c, k]
            rows.append("t%d[%5d w%5d q%5d m%6d e%6d]" % (k, e[1], e[2] - e[1], e[3] - e[2], e[4] - e[3], e[5] - e[4]))
        print("  c%d %s" % (c, " ".join(rows)))
valid = tl[..., 5] > 0
wait = (tl[..., 2] - tl[..., 1])[valid]
qld = (tl[..., 3] - tl[..., 2])[valid]
mma = (tl[..., 4] - tl[..., 3])[valid]
epi = (tl[..., 5] - tl[..., 4])[valid]
end = tl[..., 5].max(axis=(1, 2))
print("mean wait %.0f  qload %.0f  mma %.0f  epilogue %.0f  | kernel end per SM: mean %.0f max %.0f" % (
    wait.mean(), qld.mean(), mma.mean(), epi.mean(), end.mean(), end.max()))
# share of each consumer's time from its first wait to its last tile's end spent in each segment
busy = (tl[..., 5].max(-1) - tl[..., 0, 1])[ntile > 0]
print("per consumer, share of first-wait..last-end: wait %.2f  qload %.2f  mma %.2f  epilogue %.2f" % tuple(
    x.sum() / busy.sum() for x in (wait, qld, mma, epi)))
first = tl[:, :, 0, 2]
print("first proposal ready at: mean %.0f min %.0f max %.0f cycles" % (first.mean(), first.min(), first.max()))
for k in range(4):
    v = valid[:, :, k]
    print("tile %d: wait %.0f mma %.0f" % (k, (tl[..., k, 2] - tl[..., k, 1])[v].mean(), (tl[..., k, 4] - tl[..., k, 3])[v].mean()))
