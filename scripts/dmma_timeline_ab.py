#!/usr/bin/env python
"""Where a dense_dmma consumer's cycles go, as medians per segment, on the headline workload
(65 536 x 128 dense Gaussian, StretchMove, L2 flushed before every step).

    python scripts/dmma_timeline_ab.py [--lib PATH] [--label NAME] [--steps K]

`--lib` loads another build of the library (EMCEE_B200_LIB), so two builds can be compared from the same
tree: run the script once per build.  Both launches of the step are reported.  Option "dmma_timeline" = 1
keeps the stamps of the last launch of a call, the second split, which with the flush is the programmatic
dependent of the first; = 2 keeps those of the first split, the launch after the flush that pulls the state
from HBM.  Each of K one-step calls contributes one launch to each.  Segments, in cycles of a consumer warp:
first-tile wait (wait for the first proposal, counted from the warp's entry into the kernel, so it includes
griddepcontrol.wait), later waits, q-load (proposal into registers + slot release), DMMA block, epilogue
(reduction, accept test, stores).  One JSON line goes to stdout."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="path of the libemcee_b200.so to load (default: the in-tree build)")
    ap.add_argument("--label", default=None)
    ap.add_argument("--steps", type=int, default=20, help="one-step calls recorded (one launch each)")
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if args.lib:
        os.environ["EMCEE_B200_LIB"] = os.path.abspath(args.lib)
    sys.path.insert(0, ROOT)
    import numpy as np

    import bench
    import emcee_b200
    from emcee_b200 import models

    N, D = 65536, 128
    w = bench.make_workload("gauss_dense", N, D)
    s = emcee_b200.EnsembleSampler(N, D, models.GaussianDense(w["icov"]), seed=1)
    eng = s._engine
    eng.set_option("l2_flush", 1)
    eng.set_state(w["p0"])
    sched = s._schedule()
    eng.step(sched, args.warmup, want_accepted=False)
    out = {"label": args.label or (args.lib or "in-tree"), "calls": args.steps, "launches": {}}
    for mode, launch in ((2, "first split (after the L2 flush)"), (1, "second split (PDL dependent of the first)")):
        eng.set_option("dmma_timeline", mode)
        seg = {k: [] for k in ("first_wait", "later_wait", "qload", "dmma", "epilogue")}
        end = []
        for _ in range(args.steps):
            eng.step(sched, 1, want_accepted=False)
            tl = eng.debug_timeline()  # [SM, consumer, tile, event]
            valid = tl[..., 5] > 0
            wait = tl[..., 2] - tl[..., 1]
            seg["first_wait"].append(tl[:, :, 0, 2][valid[:, :, 0]])  # from the warp's entry
            seg["later_wait"].append(wait[:, :, 1:][valid[:, :, 1:]])
            seg["qload"].append((tl[..., 3] - tl[..., 2])[valid])
            seg["dmma"].append((tl[..., 4] - tl[..., 3])[valid])
            seg["epilogue"].append((tl[..., 5] - tl[..., 4])[valid])
            end.append(tl[..., 5].max(axis=(1, 2)))
        eng.set_option("dmma_timeline", 0)
        med = {k: float(np.median(np.concatenate(v))) for k, v in seg.items()}
        r = {"median_cycles": med, "kernel_end_per_sm_median": float(np.median(np.concatenate(end))),
             "kernel_end_per_sm_max_median": float(np.median([e.max() for e in end]))}
        out["launches"][launch] = r
        print("%-10s %-6s first-wait %6.0f  later-wait %6.0f  q-load %5.0f  dmma %5.0f  epilogue %5.0f  | end/SM %6.0f"
              % (out["label"], launch.split()[0], med["first_wait"], med["later_wait"], med["qload"], med["dmma"],
                 med["epilogue"], r["kernel_end_per_sm_median"]), file=sys.stderr)
    out["kernel"] = eng.last_kernel_name()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
