"""Times frames already in GPU memory (cs_device_frames) on one GPU and prints one JSON line.

    python tools/time_device_frames.py [--steps 120] [--repeats 3] [--launches 50]

(a) The layout step over 256 VGA frames, per layout: CUDA-event time of --launches cs_batch_upload_online_device calls on the context stream
    (the call a user pays: the step plus the batch's small host-to-device tables), and the kernel time of k_ingest_frames (or of the
    device-to-device copy for packed BGR) from torch.profiler in a phase of its own.  Bytes moved = the view's bytes read + the packed bytes
    written, over kernel time, against MEASURED_PEAKS.json's HBM figure when the file exists, else the H100 SXM data sheet's 3.35 TB/s.
(b) bench.py's c3 online path (LSD lines, 12 contexts as a rolling pipeline of upload + cs_batch_run_async + cs_batch_fetch), three ways,
    alternated in one process and repeated --repeats times: frames from one device tensor through cs_batch_upload_online_device; bench.py's
    e2e form with pinned host frames (cs_batch_upload_online); and the round trip of a torch user without this API, tensor -> pinned host
    memory -> cs_batch_upload_online.  ms per step for each, and whether the records of all three are equal.
The card's name and power limit are read in the same run."""
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
        o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in o.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "error": str(e)}


def layouts(torch, imgs):
    """(name, device view, order): the layouts of the GPU tests, at full size"""
    F, H, W, _ = imgs.shape
    t = torch.from_numpy(imgs).cuda()
    out = [("nhwc_bgr (copy)", t, "bgr"), ("nhwc_rgb", t.flip(-1).contiguous(), "rgb"),
           ("nchw_bgr", t.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1), "bgr")]
    big = torch.zeros((F, H + 16, W + 32, 3), dtype=torch.uint8, device="cuda")
    big[:, 8:8 + H, 16:16 + W] = t
    out.append(("crop", big[:, 8:8 + H, 16:16 + W], "bgr"))
    bgra = torch.zeros((F, H, W, 4), dtype=torch.uint8, device="cuda")
    bgra[..., :3] = t
    out.append(("bgra", bgra[..., :3], "bgr"))
    g = t[..., 1].contiguous()
    out.append(("gray (copy)", g, "bgr"))
    big_g = torch.zeros((F, H + 16, W + 32), dtype=torch.uint8, device="cuda")
    big_g[:, 8:8 + H, 16:16 + W] = g
    out.append(("gray_crop", big_g[:, 8:8 + H, 16:16 + W], "bgr"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=120)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--inflight", type=int, default=12)
    args = ap.parse_args()
    import torch
    import cube_slam_b200 as cs
    import bench
    res = {"card": card()}
    peak_gbs, peak_src = bench.measured_peaks()
    wl = bench.make_workload("c3", 0)
    imgs = np.ascontiguousarray(wl["imgs"])
    F, H, W = imgs.shape[:3]
    params = cs.default_params(**wl["over"])
    from cube_slam_b200 import _lib
    lp = _lib.LineParams()
    _lib.load().cs_default_line_params(C.byref(lp))
    lp.use_LSD = 1                                  # bench.py's c3 headline: online LSD
    lp.line_length_thres = bench.LINE_LENGTH_THRES
    ctxs = []
    for _ in range(args.inflight):
        cx = cs.Context(0, W, H, F, 16, 8192)
        cx.set_calibration(wl["K"])
        ctxs.append(cx)

    # ---- (a) the layout step
    ctx = ctxs[0]
    st = torch.cuda.ExternalStream(ctx.stream())
    views = layouts(torch, imgs)
    step = {}
    for name, v, order in views:
        ctx.upload_online_device(v, wl["Ts"], wl["boxes"], lp, params, order=order)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.launches):
            ctx.upload_online_device(v, wl["Ts"], wl["boxes"], lp, params, order=order)
        e1.record(st)
        torch.cuda.synchronize()
        ch = v.shape[3] if v.dim() == 4 else 1
        step[name] = {"upload_call_ms": e0.elapsed_time(e1) / args.launches, "bytes_moved": 2 * F * H * W * ch}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, v, order in views:
            for _ in range(10):
                ctx.upload_online_device(v, wl["Ts"], wl["boxes"], lp, params, order=order)
            torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and ("k_ingest_frames" in e.name or "Memcpy DtoD" in e.name)),
                  key=lambda e: e.time_range.start)
    # one layout step per call, in issue order: ten per layout
    per = len(kern) // len(views)
    res["profiled_layout_events"] = len(kern)
    for i, (name, v, order) in enumerate(views):
        ks = kern[i * per:(i + 1) * per]
        if not ks:
            continue
        us = float(np.median([e.time_range.elapsed_us() for e in ks]))
        gbs = step[name]["bytes_moved"] / (us * 1e3)
        step[name].update({"kernel": ks[0].name, "kernel_us": us, "hbm_gbs": gbs, "share_of_peak": gbs / peak_gbs})
    res["layout_step"] = {"frames": F, "size": [W, H], "launches": args.launches, "peak_gbs": peak_gbs, "peak_source": peak_src, "layouts": step}
    del views
    torch.cuda.synchronize()

    # ---- (b) the c3 online path, three ways
    frames_dev = torch.from_numpy(imgs).cuda()
    pinned = torch.from_numpy(imgs).pin_memory()
    roundtrip = torch.empty_like(pinned).pin_memory()
    K_ = len(ctxs)

    def issue_device(cx):
        cx.upload_online_device(frames_dev, wl["Ts"], wl["boxes"], lp, params)
        cx.run_async()

    def issue_pinned(cx):
        cx.upload_online(pinned.numpy(), wl["Ts"], wl["boxes"], lp, params)
        cx.run_async()

    def issue_roundtrip(cx):
        roundtrip.copy_(frames_dev)                 # tensor.cpu() into pinned memory: returns when the bytes are on the host
        cx.upload_online(roundtrip.numpy(), wl["Ts"], wl["boxes"], lp, params)
        cx.run_async()

    def run(issue, n_steps):
        issued = fetched = 0
        last = None
        while fetched < n_steps:
            while issued < n_steps and issued - fetched < K_:
                issue(ctxs[issued % K_])
                issued += 1
            r, c = ctxs[fetched % K_].fetch()
            last = (r.copy(), c.copy())
            fetched += 1
        return last

    modes = [("device_tensor", issue_device), ("pinned_host", issue_pinned), ("tensor_to_pinned_roundtrip", issue_roundtrip)]
    for _, fn in modes:
        run(fn, K_)
    torch.cuda.synchronize()
    times = {m: [] for m, _ in modes}
    recs = {}
    for _ in range(args.repeats):
        for m, fn in modes:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            recs[m] = run(fn, args.steps)
            torch.cuda.synchronize()
            times[m].append((time.perf_counter() - t0) * 1e3 / args.steps)
    same = all(recs[m][0].tobytes() == recs["pinned_host"][0].tobytes() and (recs[m][1] == recs["pinned_host"][1]).all() for m in recs)
    res["c3_online"] = {"frames": F, "contexts": K_, "steps": args.steps, "repeats": args.repeats, "ms_per_step": times,
                        "records_equal": bool(same)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
