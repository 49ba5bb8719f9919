"""Times the online cuboid batch (LSD lines + detect_cuboid) over a VGA + KITTI-shaped mix, four ways, and prints one JSON line.

    python tools/time_cuboids_mixed.py [--calls 10] [--warmup 2] [--vga 128] [--kitti 128]

Workload: --vga synthetic 640 x 480 indoor frames (3 boxes each, their own K) and --kitti synthetic 1242 x 375 frames (8 boxes each, a KITTI
K), online LSD (line_length_thres 15), default cuboid parameters.  Each way is timed as the median of --calls after --warmup, host clock:
upload (host frames to the device and the tables; it waits for the context stream) and run + fetch (the fetch waits for the device) apart:
  mixed       one cs_batch_upload_online_mixed batch of both sets (each frame with its own K) on one context, the frames packed into one
              host buffer once, before the timing
  mixed_list  the same through Context.upload_online_mixed on the list of frames: the Python form, which packs the list on every call
  sequential  two one-size batches (cs_batch_upload_online), one per set, on one context, one after the other
  in_flight   the two one-size batches on two contexts: both uploaded, both run_async, then both fetched
The records of all four are compared byte for byte.  Then one profiled synchronous run each (cs_set_profiling bit 0, the chain on one
stream) of the mixed batch and of the two one-size batches gives the per-stage times (cs_stage_ms).  The card's name, power limit and SM clock are read in the same run."""
import argparse
import ctypes as C
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--vga", type=int, default=128)
    ap.add_argument("--kitti", type=int, default=128)
    a = ap.parse_args()
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib, synthetic as S
    from cube_slam_b200.detect_3d_cuboid import default_params

    sets = [S.make_batch(31, a.vga, 640, 480, 3, distinct=16), S.make_batch(32, a.kitti, 1242, 375, 8, kind="kitti", distinct=16)]
    F = a.vga + a.kitti
    prm = default_params()

    def ctx():
        c = cs.Context(0, 1280, 960, F, 16, 4096)
        lp = _lib.LineParams()
        c.L.cs_default_line_params(C.byref(lp))
        lp.use_LSD, lp.line_length_thres = 1, 15.0
        return c, lp

    cm, lp = ctx()
    c1, _ = ctx()
    c2, _ = ctx()
    imgs = [im for s in sets for im in s[0]]
    Ts = np.concatenate([s[1] for s in sets])
    boxes = [b for s in sets for b in s[2]]
    Ks = np.concatenate([np.broadcast_to(s[4], (len(s[0]), 3, 3)) for s in sets])
    out = {}
    buf, views, _, Ts_m, boxes_m, box_off_m, _, _, Ks_m = cm._pack_mixed(imgs, Ts, boxes, [np.zeros((0, 4))] * F, Ks)   # packed once
    d = lambda a: _lib.ptr(a, C.c_double)

    def upload_mixed():
        cm.check(cm.L.cs_batch_upload_online_mixed(cm.h, buf.ctypes.data, views, F, d(Ks_m), d(Ts_m), d(boxes_m), _lib.ptr(box_off_m, C.c_int32),
                                                   C.byref(lp), C.byref(prm)))
        cm._n_obj, cm._topk = int(box_off_m[-1]), int(prm.max_cuboid_num)

    def run_mixed():
        cm.run_async()
        out["mixed"] = cm.fetch()

    def upload_list():
        cm.upload_online_mixed(imgs, Ts, boxes, lp, prm, K=Ks)

    def run_list():
        cm.run_async()
        out["mixed_list"] = cm.fetch()

    def one(c, s):
        c.set_calibration(s[4])
        c.upload_online(s[0], s[1], s[2], lp, prm)

    seq = []

    def upload_seq():
        one(c1, sets[0])

    def run_seq():   # the first set's run, then the second set's upload and run
        c1.run_async()
        seq[:] = [c1.fetch()]
        one(c1, sets[1])
        c1.run_async()
        seq.append(c1.fetch())
        out["sequential"] = list(seq)

    def upload_both():
        for c, s in zip((c1, c2), sets):
            one(c, s)

    def run_both():
        for c in (c1, c2):
            c.run_async()
        out["in_flight"] = [c1.fetch(), c2.fetch()]

    res = {"workload": "%d VGA (3 boxes) + %d KITTI-shaped (8 boxes), online LSD" % (a.vga, a.kitti), "card": card()}
    for name, up, run in (("mixed", upload_mixed, run_mixed), ("mixed_list", upload_list, run_list), ("sequential", upload_seq, run_seq),
                          ("in_flight", upload_both, run_both)):
        t_up, t_run = [], []
        for i in range(a.warmup + a.calls):
            t0 = time.perf_counter()
            up()
            t1 = time.perf_counter()
            run()
            t2 = time.perf_counter()
            if i >= a.warmup:
                t_up.append((t1 - t0) * 1e3)
                t_run.append((t2 - t1) * 1e3)
        res[name] = {"total_ms": round(float(np.median(np.add(t_up, t_run))), 2), "upload_ms": round(float(np.median(t_up)), 2),
                     "run_fetch_ms": round(float(np.median(t_run)), 2)}
    cat = lambda pair: (np.concatenate([p[0] for p in pair]).tobytes(), np.concatenate([p[1] for p in pair]).tobytes())
    m = (out["mixed"][0].tobytes(), out["mixed"][1].tobytes())
    res["identical"] = m == (out["mixed_list"][0].tobytes(), out["mixed_list"][1].tobytes()) == cat(out["sequential"]) == cat(out["in_flight"])
    res["n_objects"] = int(len(out["mixed"][1]))
    stages = {}
    for name, c, up in (("mixed", cm, upload_mixed), ("vga", c1, lambda: one(c1, sets[0])), ("kitti", c1, lambda: one(c1, sets[1]))):
        c.set_profiling(True)
        up()
        c.run()
        stages[name] = {k: round(v, 2) for k, v in c.stage_ms().items()}
        c.set_profiling(False)
    res["stages_ms"] = stages
    print(json.dumps(res))
    for c in (cm, c1, c2):
        c.close()
    return 0 if res["identical"] else 1


if __name__ == "__main__":
    sys.exit(main())
