"""Times the line descriptor's detect-and-describe call on frames already in GPU memory against the host-frame call, and prints one JSON line.

    python tools/time_lbd_device_frames.py [--frames 256] [--calls 10] [--warmup 2] [--cap 2048]

Workload: --frames synthetic VGA frames (cube_slam_b200.synthetic.make_batch), both flavours (LSD, EDLines).  Three ways to call
line_lbd_detect, alternated per repetition in one process: detect_descrip_lines_batch on a pinned numpy batch (the host form), and
detect_descrip_lines_device on a packed BGR CUDA tensor and on a planar RGB view (permute of an NCHW tensor, through k_ingest_frames).
Every call is synchronous; after --warmup calls of each, the median of --calls wall-clock times per way.  The outputs of the three ways are
compared in the same run (key-line bytes and descriptor bytes).  The card's name and power limit are read in the same run."""
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
        o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        name, power = [s.strip() for s in o.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "error": str(e)}


def same(a, b):
    return len(a) == len(b) and all(ka.tobytes() == kb.tobytes() and da.tobytes() == db.tobytes() for (ka, da), (kb, db) in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cap", type=int, default=2048)
    args = ap.parse_args()
    import torch
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs = np.ascontiguousarray(S.make_batch(0, args.frames, 640, 480, 3)[0])
    F, H, W = imgs.shape[:3]
    pinned = torch.from_numpy(imgs).pin_memory().numpy()
    t = torch.from_numpy(imgs).cuda()
    planar_rgb = t.flip(-1).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    res = {"card": card(), "frames": F, "size": [W, H], "calls": args.calls, "warmup": args.warmup, "cap": args.cap, "flavours": {}}
    ctx = cs.Context(0, W, H, F, 1, 1)
    for flavour, use_lsd in (("lsd", True), ("edlines", False)):
        det = cs.line_lbd_detect(context=ctx)
        det.use_LSD = use_lsd
        det.line_length_thres = 15.0
        ways = [("host_pinned_numpy", lambda: det.detect_descrip_lines_batch(pinned, args.cap)),
                ("device_packed_bgr", lambda: det.detect_descrip_lines_device(t, "bgr", args.cap)),
                ("device_planar_rgb", lambda: det.detect_descrip_lines_device(planar_rgb, "rgb", args.cap))]
        out = {}
        for name, fn in ways:
            for _ in range(args.warmup):
                out[name] = fn()
        ms = {name: [] for name, _ in ways}
        for _ in range(args.calls):
            for name, fn in ways:
                t0 = time.perf_counter()
                out[name] = fn()
                ms[name].append((time.perf_counter() - t0) * 1e3)
        ref = out["host_pinned_numpy"]
        res["flavours"][flavour] = {"median_ms": {k: float(np.median(v)) for k, v in ms.items()}, "min_ms": {k: float(np.min(v)) for k, v in ms.items()},
                                    "key_lines": int(sum(len(k) for k, _ in ref)),
                                    "outputs_identical": bool(all(same(out[k], ref) for k in out))}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
