#!/usr/bin/env python
"""Where a dense_dmma consumer's cycles go, as medians per segment, on the headline workload
(65 536 x 128 dense Gaussian, StretchMove, L2 flushed before every step).

    python scripts/dmma_timeline_ab.py [--lib PATH] [--label NAME] [--steps K] [--no-stagger]

`--lib` loads another build of the library (EMCEE_B200_LIB), so two builds can be compared from the same
tree: run the script once per build.  Both launches of the step are reported.  Option "dmma_timeline" = 1
keeps the stamps of the last launch of a call, the second split, which with the flush is the programmatic
dependent of the first; = 2 keeps those of the first split, the launch after the flush that pulls the state
from HBM.  Each of K one-step calls contributes one launch to each.

All stamps of one CTA count cycles from the CTA barrier at the end of the kernel's prologue, so a producer's
stamps and its consumer's compare directly.  Segments of a consumer warp, over all tiles: first-tile wait (from
that barrier to the first proposal, so it includes griddepcontrol.wait), later waits, q-load (proposal into
registers + slot release), DMMA block, epilogue (reduction, accept test, stores).

The fill, i.e. the first tile of every pair, split by pair index (0-3 and 4-7: with the stagger, pairs 4-7
request their first rows only after pairs 0-3's have landed): predecessor done (griddepcontrol.wait returned in
the producer; ~0 for a launch that is not a programmatic dependent), own rows requested, partner rows requested,
rows landed (the producer's wait for them returned), proposal published, consumer sees it; factor landed (the
consumer's wait on the packed factor returned).  Reported both as times since the barrier and as the segments
entry -> request, request -> landed, landed -> published, published -> seen.  One JSON line goes to stdout."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# event indices of a tile record (dense_dmma.cu): consumer 1 wait start, 2 proposal ready, 3 in registers,
# 4 DMMA done, 5 tile done, 9 factor landed (first record); producer 6 rows requested (own rows when they are
# requested early), 7 rows landed, 8 proposal published, 10 griddepcontrol.wait returned, 11 partner rows
# requested (first record)
GROUPS = (("pairs 0-3", slice(0, 4)), ("pairs 4-7", slice(4, 8)))


def fill_table(tl, np):
    """Medians over SMs and calls of the first tile's stamps, per pair group."""
    out = {}
    for name, sl in GROUPS:
        t = tl[:, :, sl, 0, :].reshape(-1, tl.shape[-1])  # [calls*SM*pairs, event]
        t = t[t[:, 5] > 0]
        med = lambda x: float(np.median(x))  # noqa: E731
        out[name] = {
            "at": {"pred_done": med(t[:, 10]), "own_request": med(t[:, 6]), "partner_request": med(t[:, 11]),
                   "landed": med(t[:, 7]), "published": med(t[:, 8]), "seen": med(t[:, 2]),
                   "factor_landed": med(t[:, 9])},
            "seg": {"entry_to_request": med(t[:, 11]), "request_to_landed": med(t[:, 7] - t[:, 11]),
                    "landed_to_published": med(t[:, 8] - t[:, 7]), "published_to_seen": med(t[:, 2] - t[:, 8]),
                    "factor_after_seen": med(t[:, 9] - t[:, 2])},
        }
        later = tl[:, :, sl, 1:, :].reshape(-1, tl.shape[-1])
        later = later[later[:, 5] > 0]
        out[name]["later"] = {"request_to_landed": med(later[:, 7] - later[:, 6]),
                              "landed_to_published": med(later[:, 8] - later[:, 7]),
                              "consumer_wait": med(later[:, 2] - later[:, 1])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="path of the libemcee_b200.so to load (default: the in-tree build)")
    ap.add_argument("--label", default=None)
    ap.add_argument("--steps", type=int, default=20, help="one-step calls recorded (one launch each)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--no-stagger", action="store_true", help='option "dmma_stagger" = 0')
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
    if args.no_stagger:
        eng.set_option("dmma_stagger", 0)
    eng.set_state(w["p0"])
    sched = s._schedule()
    eng.step(sched, args.warmup, want_accepted=False)
    out = {"label": args.label or (args.lib or "in-tree"), "calls": args.steps, "stagger": not args.no_stagger,
           "launches": {}}
    for mode, launch in ((2, "first split (after the L2 flush)"), (1, "second split (PDL dependent of the first)")):
        eng.set_option("dmma_timeline", mode)
        seg = {k: [] for k in ("first_wait", "later_wait", "qload", "dmma", "epilogue")}
        end, raw = [], []
        for _ in range(args.steps):
            eng.step(sched, 1, want_accepted=False)
            tl = eng.debug_timeline()  # [SM, consumer, tile, event]
            raw.append(tl)
            valid = tl[..., 5] > 0
            wait = tl[..., 2] - tl[..., 1]
            seg["first_wait"].append(tl[:, :, 0, 2][valid[:, :, 0]])  # from the prologue's barrier
            seg["later_wait"].append(wait[:, :, 1:][valid[:, :, 1:]])
            seg["qload"].append((tl[..., 3] - tl[..., 2])[valid])
            seg["dmma"].append((tl[..., 4] - tl[..., 3])[valid])
            seg["epilogue"].append((tl[..., 5] - tl[..., 4])[valid])
            end.append(tl[..., 5].max(axis=(1, 2)))
        eng.set_option("dmma_timeline", 0)
        med = {k: float(np.median(np.concatenate(v))) for k, v in seg.items()}
        r = {"median_cycles": med, "kernel_end_per_sm_median": float(np.median(np.concatenate(end))),
             "kernel_end_per_sm_max_median": float(np.median([e.max() for e in end])),
             "fill": fill_table(np.stack(raw), np)}
        out["launches"][launch] = r
        print("%-10s %-6s first-wait %6.0f  later-wait %6.0f  q-load %5.0f  dmma %5.0f  epilogue %5.0f  | end/SM %6.0f"
              % (out["label"], launch.split()[0], med["first_wait"], med["later_wait"], med["qload"], med["dmma"],
                 med["epilogue"], r["kernel_end_per_sm_median"]), file=sys.stderr)
        for name, f in r["fill"].items():
            a, s_ = f["at"], f["seg"]
            print("%-10s %-6s %s  pred-done %6.0f  factor %6.0f | entry->req %6.0f  req->landed %6.0f  "
                  "landed->pub %5.0f  pub->seen %5.0f  (seen at %6.0f) | later req->landed %5.0f"
                  % (out["label"], launch.split()[0], name, a["pred_done"], a["factor_landed"], s_["entry_to_request"],
                     s_["request_to_landed"], s_["landed_to_published"], s_["published_to_seen"], a["seen"],
                     f["later"]["request_to_landed"]), file=sys.stderr)
    out["kernel"] = eng.last_kernel_name()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
