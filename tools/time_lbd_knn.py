"""Times k-nearest-neighbour (k = 2) and radius (r = 25) matching of line descriptors on one GPU and prints one JSON object.

    python tools/time_lbd_knn.py [--frames 257] [--reps 10]

Workloads: every frame of a batch of synthetic VGA frames (the bench workload's generator) against the next one -- 256 pairs of
LSD descriptor sets of the size the c3 workload produces -- and one 4096 x 4096 pair of random codes (queries a few bit flips from a train
code).  Each call is one synchronous call of the C ABI
(cs_knn_match_line_descrip_batch, cs_radius_match_line_descrip_batch) with host buffers allocated beforehand: "call_ms" is CUDA events
recorded on the context's stream before and after it -- uploads, kernels, copies back and the host's conversion to cs_dmatch records --
and "wall_ms" the host's clock around it; the median of --reps calls after one warm-up.  "mirror_ms" is the Python mirror's batch call
(adds building one numpy array per query).  Beside them, the reference's own BinaryDescriptorMatcher::knnMatch / radiusMatch on one CPU core
(oracle/_ref/liblinelbd_knn_ref.so, when it was built), median of 3."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=257)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    det = cs.line_lbd_detect()
    det.use_LSD = True
    det.line_length_thres = 15
    imgs = np.ascontiguousarray(S.make_batch(20260922, args.frames, 640, 480, 3, poisson=True)[0])
    descs = [d for _, d in det.detect_descrip_lines_batch(imgs)]
    bdm = det.bdm
    import ctypes as C
    from cube_slam_b200 import _lib
    L, h = det._ctx.L, det._ctx.h
    stream = torch.cuda.ExternalStream(det._ctx.L.cs_stream(det._ctx.h), device="cuda:0")

    def timed(fn):
        fn()
        gpu, wall = [], []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            t0 = time.perf_counter()
            out = fn()
            wall.append((time.perf_counter() - t0) * 1e3)
            b.record(stream)
            b.synchronize()
            gpu.append(a.elapsed_time(b))
        return statistics.median(gpu), statistics.median(wall), out

    rng = np.random.default_rng(7)
    t4 = rng.integers(0, 256, (4096, 32), dtype=np.uint8)
    q4 = t4[rng.permutation(4096)].copy()
    flips = rng.integers(0, 256, (4096, 12))
    for i in range(4096):
        np.bitwise_xor.at(q4[i], flips[i] // 8, (1 << (flips[i] % 8)).astype(np.uint8))
    work = {"consecutive_pairs": (descs[:-1], descs[1:]), "pair_4096x4096": ([q4], [t4])}
    out = {"gpu": torch.cuda.get_device_name(0), "frames": len(imgs), "size": "640x480", "line_length_thres": 15, "reps": args.reps}
    from oracle import pyoracle_knn as K
    ref = K.ref_available()
    for name, (qs, ts) in work.items():
        rec = {"pairs": len(qs), "queries": int(sum(len(q) for q in qs)), "code_pairs": int(sum(len(q) * len(t) for q, t in zip(qs, ts)))}
        qo = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int32)
        to = np.concatenate([[0], np.cumsum([len(t) for t in ts])]).astype(np.int32)
        q, t = np.ascontiguousarray(np.concatenate(qs)), np.ascontiguousarray(np.concatenate(ts))
        nq = int(qo[-1])
        kout, kn = np.zeros(2 * nq, _lib.DMATCH_DTYPE), np.zeros(nq, np.int32)
        rout, roff = np.zeros(16 * nq, _lib.DMATCH_DTYPE), np.zeros(nq + 1, np.int64)
        P = lambda a, ty: _lib.ptr(a, ty)
        calls = {
            "knn2": (lambda: det._ctx.check(L.cs_knn_match_line_descrip_batch(h, P(q, C.c_uint8), P(qo, C.c_int32), P(t, C.c_uint8), P(to, C.c_int32),
                                                                            len(qs), 2, None, kout.ctypes.data, P(kn, C.c_int32))),
                     lambda: int(kn.sum()), lambda: bdm.knnMatch_batch(qs, ts, 2)),
            "radius25": (lambda: det._ctx.check(L.cs_radius_match_line_descrip_batch(h, P(q, C.c_uint8), P(qo, C.c_int32), P(t, C.c_uint8), P(to, C.c_int32),
                                                                                   len(qs), C.c_float(25.0), None, rout.ctypes.data, C.c_int64(len(rout)),
                                                                                   P(roff, C.c_int64))),
                         lambda: int(roff[-1]), lambda: bdm.radiusMatch_batch(qs, ts, 25.0)),
        }
        for kind, (fn, count, mirror) in calls.items():
            g, w, _ = timed(fn)
            _, mw, _ = timed(mirror)
            rec[kind] = {"call_ms": round(g, 4), "wall_ms": round(w, 4), "mirror_ms": round(mw, 3), "matches": count(),
                         "code_pairs_per_s": rec["code_pairs"] / (g * 1e-3)}
            if ref:
                arg = 2 if kind == "knn2" else 25.0
                cpu = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    for qq, tt in zip(qs, ts):
                        K.ref_matcher_call("knn" if kind == "knn2" else "radius", qq, tt, arg)
                    cpu.append((time.perf_counter() - t0) * 1e3)
                rec[kind]["reference_cpu_one_core_ms"] = round(statistics.median(cpu), 3)
        out[name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
