"""Times the octave calls of a multi-octave LSD line_lbd_detect and prints one JSON line.

    python tools/time_lsd_octaves.py [--frames 256] [--calls 10] [--warmup 2] [--cap 2048] [--ref-frames 4]

Workload: --frames synthetic VGA frames (cube_slam_b200.synthetic.make_batch), use_LSD, line_length_thres 15, octave ratio 2, numoctaves
1 / 2 / 3.  For each count: detect_raw_lines_octaves_batch and detect_descrip_lines_octaves_batch, synchronous calls, the median of --calls
wall-clock times after --warmup calls.  The compiled reference (oracle/_ref/liblinelbd_octaves_ref.so: the reference's own class, one host core)
runs detect_descrip_lines_octaves on the first --ref-frames frames where it is present, and its per-frame time is reported next to the
product's per-frame time.  The card's name, power limit and SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [s.strip() for s in o.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "error": str(e)}


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
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cap", type=int, default=2048)
    ap.add_argument("--ref-frames", type=int, default=4)
    args = ap.parse_args()
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs = np.ascontiguousarray(S.make_batch(0, args.frames, 640, 480, 3)[0])
    F, H, W = imgs.shape[:3]
    res = {"card": card(), "frames": F, "size": [W, H], "calls": args.calls, "warmup": args.warmup, "octave_ratio": 2.0, "octaves": {}}
    ctx = cs.Context(0, W, H, F, 1, 1)
    for K in (1, 2, 3):
        det = cs.line_lbd_detect(K, 2.0, context=ctx)
        det.use_LSD = True
        det.line_length_thres = 15.0
        raw_ms = median_ms(lambda: det.detect_raw_lines_octaves_batch(imgs, args.cap), args.calls, args.warmup)
        out = det.detect_descrip_lines_octaves_batch(imgs, args.cap)
        desc_ms = median_ms(lambda: det.detect_descrip_lines_octaves_batch(imgs, args.cap), args.calls, args.warmup)
        res["octaves"][str(K)] = {"raw_median_ms": raw_ms, "descrip_median_ms": desc_ms, "descrip_ms_per_frame": desc_ms / F,
                                  "key_lines_per_octave": [int(sum(len(kls[k]) for kls, _ in out)) for k in range(K)]}
    ctx.close()
    try:
        from oracle import pyoracle_octaves as O
        if O.ref_available():
            n = min(args.ref_frames, F)
            for K in (1, 2, 3):
                t0 = time.perf_counter()
                for f in range(n):
                    O.ref_lsd_octaves(imgs[f], K, 2.0, 15.0, mode=2)
                res["octaves"][str(K)]["reference_ms_per_frame_one_core"] = (time.perf_counter() - t0) * 1e3 / n
            res["reference_frames"] = n
        else:
            res["reference"] = "oracle/_ref/liblinelbd_octaves_ref.so not built"
    except Exception as e:  # noqa: BLE001
        res["reference"] = "failed: %s" % e
    print(json.dumps(res))


if __name__ == "__main__":
    main()
