"""Times BinaryDescriptor::compute on key lines of any octave (line_lbd_detect.compute_descriptors_octaves_batch) and prints one JSON line.

    python tools/time_lbd_compute_octaves.py [--frames 256] [--calls 10] [--warmup 2] [--ref-frames 4]

Workload: --frames synthetic VGA frames (cube_slam_b200.synthetic.make_batch) with the key lines LSDDetector::detect(img, 2, 3) returns for
each (3 octaves), described in one synchronous call; the median of --calls wall-clock times after --warmup calls.  The compiled reference
(oracle/_ref/liblinelbd_compute_octaves_ref.so: the reference's own BinaryDescriptor::compute, one host core) describes the first --ref-frames frames'
key lines where it is present, and its per-frame time is reported next to the product's.  The card's name, power limit and SM clock are read
in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_lsd_octaves import card, median_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-frames", type=int, default=4)
    args = ap.parse_args()
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs = np.ascontiguousarray(S.make_batch(0, args.frames, 640, 480, 3)[0])
    F, H, W = imgs.shape[:3]
    ctx = cs.Context(0, W, H, F, 1, 1)
    det = cs.line_lbd_detect(1, 1.0, context=ctx)
    kls = det.lsd.detect(list(imgs), 2, 3)
    n = [int(sum(np.sum(k["octave"] == o) for k in kls)) for o in range(3)]
    ms = median_ms(lambda: det.compute_descriptors_octaves_batch(imgs, kls), args.calls, args.warmup)
    ms_f = median_ms(lambda: det.compute_descriptors_octaves_batch(imgs, kls, want_float=True), args.calls, args.warmup)
    res = {"card": card(), "frames": F, "size": [W, H], "octaves": 3, "calls": args.calls, "warmup": args.warmup, "key_lines_per_octave": n,
           "median_ms": ms, "ms_per_frame": ms / F, "median_ms_with_float": ms_f}
    ctx.close()
    try:
        from oracle import pyoracle_compute_octaves as O
        if O.ref_available():
            r = min(args.ref_frames, F)
            t0 = time.perf_counter()
            for f in range(r):
                O.ref_lbd_compute_octaves(imgs[f], kls[f])
            res["reference_ms_per_frame_one_core"] = (time.perf_counter() - t0) * 1e3 / r
            res["reference_frames"] = r
        else:
            res["reference"] = "oracle/_ref/liblinelbd_compute_octaves_ref.so not built"
    except Exception as e:  # noqa: BLE001
        res["reference"] = "failed: %s" % e
    print(json.dumps(res))


if __name__ == "__main__":
    main()
