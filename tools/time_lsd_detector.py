"""Times the C++ LSDDetector drop-in (shim/lsd_detector_b200.cpp) and prints one JSON line.

    python tools/time_lsd_detector.py [--frames 256] [--octaves 1] [--calls 5] [--warmup 1] [--ref-frames 32]

Workload: --frames synthetic VGA BGR frames (cube_slam_b200.synthetic.make_batch), scale 2, --octaves octaves, no mask, through the test
harness oracle/_ref/libshim_lsd.so (the reference's line_lbd library with the drop-in in place of LSDDetector.cpp; built by build() where the
reference checkout exists):
  - vector:  one call of LSDDetector::detect(vector<Mat>, ...) over all frames (one batch on the GPU);
  - single:  the same frames as --frames calls of detect(Mat, vector<KeyLine>&, ...), one after the other on one host thread;
  - the reference's own LSDDetector (oracle/_ref/libref_lsd_detector.so, one host core) over the first --ref-frames frames, reported per frame.
Each GPU figure is the median of --calls wall-clock times after --warmup calls, and includes the Mat packing, the host-device copies and the
KeyLine fill.  The card's name, power limit and SM clock are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def median_ms(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--octaves", type=int, default=1)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-frames", type=int, default=32)
    args = ap.parse_args()
    import test_gpu_lsd_detector_shim as G
    from cube_slam_b200 import synthetic as S
    from time_lsd_octaves import card
    for p in (G.SHIM, G.REF):
        if not os.path.exists(p):
            sys.exit("%s is missing: build() compiles it where the reference checkout exists" % p)
    imgs = list(np.ascontiguousarray(S.make_batch(0, args.frames, 640, 480, 3)[0]))
    F, K = len(imgs), args.octaves
    shim, ref = G.Driver(G.SHIM), G.Driver(G.REF)
    cap = 4096 * K * F

    n_lines = []

    def vector():
        lists = shim.detect(G.VECTOR, imgs, 2, K, [None] * F, pre=[np.zeros(0, G.REC_DTYPE)] * F, cap=cap)[0]
        n_lines[:] = [len(l) for l in lists]

    def single():
        for img in imgs:
            shim.detect(G.FLAT, img, 2, K, cap=4096 * K)

    res = {"card": card(), "frames": F, "size": [640, 480], "octaves": K, "calls": args.calls, "warmup": args.warmup}
    res["vector_ms"] = median_ms(vector, args.calls, args.warmup)
    res["single_calls_ms"] = median_ms(single, args.calls, args.warmup)
    res["key_lines_per_frame"] = float(np.mean(n_lines))
    R = min(args.ref_frames, F)
    t0 = time.perf_counter()
    want = ref.detect(G.VECTOR, imgs[:R], 2, K, [None] * R, pre=[np.zeros(0, G.REC_DTYPE)] * R, cap=cap)[0]
    ref_ms = (time.perf_counter() - t0) * 1e3
    assert [len(l) for l in want] == n_lines[:R]
    res["reference_ms_per_frame"] = ref_ms / R
    res["reference_frames"] = R
    res["vector_ms_per_frame"] = res["vector_ms"] / F
    res["single_ms_per_frame"] = res["single_calls_ms"] / F
    print(json.dumps(res))


if __name__ == "__main__":
    main()
