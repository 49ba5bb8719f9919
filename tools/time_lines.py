"""Times the line detectors on a batch of synthetic frames (CUDA events around cs_detect_lines_batch's device part).

    python tools/time_lines.py [--frames 256] [--flavour lsd|edlines] [--seq] [--reps 5]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--flavour", default="lsd")
    ap.add_argument("--seq", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--real", action="store_true", help="use the object_slam fixture frames (cycled) instead of synthetic ones")
    args = ap.parse_args()
    import torch
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    if args.real:
        import cv2
        import glob
        fs = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "fixture_b", "raw_imgs", "*.jpg")))
        base = [cv2.imread(f, 1) for f in fs]
    batch = S.make_batch(20260922 + sum(map(ord, "c3")), args.frames, 640, 480, 3, poisson=True, distinct=min(args.frames, 32))
    imgs = batch[0]
    if args.real:
        imgs = np.stack([base[i % len(base)] for i in range(args.frames)])
    Ts, boxes = batch[1], batch[2]
    ctx = cs.Context(0, 640, 480, args.frames, 16, 8192)
    ctx.set_calibration(batch[4])
    det = cs.line_lbd_detect(context=ctx)
    det.use_LSD = args.flavour == "lsd"
    det.line_length_thres = 15
    flags = 128 if args.seq else 0
    ctx.set_profiling(1 | flags)
    ctx.upload_online(imgs, Ts, boxes, det.params(), cs.default_params())
    try:
        import subprocess
        print("GPU:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip(), flush=True)
    except (OSError, subprocess.SubprocessError):
        pass
    import ctypes as C
    prof = np.zeros(16, np.uint64)
    for r in range(args.reps):
        if args.flavour == "lsd":
            ctx.L.cs_debug_lsd_prof(ctx.h, None, 1)
        ctx.run()
        sm = ctx.stage_ms()
        msg = "%s %s frames %d: line stage %.3f ms (CUDA events), whole step %.3f ms" % (args.flavour, "seq" if args.seq else "par", args.frames, sm["lsd"], sm["total"])
        if args.flavour == "lsd":
            ctx.L.cs_debug_lsd_prof(ctx.h, prof.ctypes.data_as(C.POINTER(C.c_uint64)), 0)
            pf = prof.astype(np.float64) / args.frames
            msg += (" | Mcycles/frame: scan %.2f grow %.2f rect %.2f refine %.2f kernel %.2f, seeds grown/frame %.0f, region px/frame %.0f,"
                    " used-map re-checks/frame %.0f, region lists past the shared-memory part (LSD_SEQ_SCAP entries) %d (%.3f %% of seeds grown)") % (
                        pf[3] / 1e6, pf[0] / 1e6, pf[1] / 1e6, pf[2] / 1e6, pf[6] / 1e6, pf[5], pf[7], pf[4], int(prof[8]),
                        100.0 * float(prof[8]) / max(float(prof[4]), 1.0))
            hist = [int(prof[15]) >> s & ((1 << 21) - 1) for s in (0, 21, 42)]
            msg += ("\n    outside the growth pass, Mcycles/frame: hand-off (used-word re-read + seed mask) %.2f, density + candidate store %.2f,"
                    " reduce_region_radius %.2f (with its region2rect), unattributed %.2f"
                    " | per frame: seeds reaching region2rect %.1f, refines %.1f, reduce iterations %.1f,"
                    " region2rect sizes <=32 / <=64 / >64: %.1f / %.1f / %.1f") % (
                        pf[9] / 1e6, pf[10] / 1e6, pf[11] / 1e6,
                        (pf[6] - pf[3] - pf[0] - pf[1] - pf[2] - pf[10] - pf[11]) / 1e6,
                        pf[12], pf[13], pf[14], hist[0] / args.frames, hist[1] / args.frames, hist[2] / args.frames)
        print(msg, flush=True)


if __name__ == "__main__":
    main()
