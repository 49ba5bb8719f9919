"""Times matching line descriptors against a device-resident collection (cs_lbd_collection_*) on one GPU and prints one JSON object.

    python tools/time_lbd_collection.py [--reps 10] [--queries 300] [--sizes 16384,131072,1048576]

Collections: the descriptors of fixture_b's 58 frames, both detector flavours (one image per frame and flavour), replicated with a few
random bit flips per code until the collection holds about the given number of codes.  Queries: --queries codes of fixture_b frames, a
few bit flips away.  Each collection call (match, knn with k = 1, 2, 10, radius 25) is one synchronous call of the C ABI with host buffers
allocated beforehand: "call_ms" is CUDA events recorded on the context's stream before and after it -- the query upload, the kernels, the
copies back and the host's conversion to cs_dmatch records -- the median of --reps calls after one warm-up.  "pairwise_call_ms" is what a caller
does without the collection: one cs_knn_match_line_descrip_batch call pairing the query set with every image (host clock), plus the host
merge of the per-image lists into the k best overall.  "reference_cpu_one_core_ms": the reference's own collection knnMatch after add()
(oracle/_ref/liblinelbd_collection_ref.so, when it was built), one call, where the collection is small enough.  The card's name and power
limit are read from nvidia-smi in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def flipped(rng, codes, n_bits):
    out = codes.copy()
    bits = rng.integers(0, 256, (len(codes), n_bits))
    rows = np.repeat(np.arange(len(codes)), n_bits)
    np.bitwise_xor.at(out, (rows, (bits // 8).reshape(-1)), (1 << (bits % 8)).reshape(-1).astype(np.uint8))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--queries", type=int, default=300)
    ap.add_argument("--sizes", default="16384,131072,1048576")
    args = ap.parse_args()
    import torch
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    from conftest import GOLD
    import cv2
    meta = json.load(open(os.path.join(GOLD, "fixture_b", "meta.json")))
    frames = np.stack([cv2.imread(os.path.join(GOLD, "fixture_b", "raw_imgs", "%04d_rgb_raw.jpg" % i), 1) for i in range(meta["n_frames"])])
    det = cs.line_lbd_detect()
    det.line_length_thres = 15
    base = []
    for use_lsd in (True, False):
        det.use_LSD = use_lsd
        base += [d for _, d in det.detect_descrip_lines_batch(frames)]
    n_base = sum(len(d) for d in base)
    rng = np.random.default_rng(20261016)
    allq = np.concatenate(base)
    queries = flipped(rng, allq[rng.choice(len(allq), args.queries, replace=False)], 6)
    L, h = det._ctx.L, det._ctx.h
    stream = torch.cuda.ExternalStream(L.cs_stream(h), device="cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi, "base_images": len(base), "base_codes": n_base,
           "queries": len(queries), "reps": args.reps}

    def timed(fn):
        fn()
        gpu = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            gpu.append(a.elapsed_time(b))
        return statistics.median(gpu)

    from oracle import pyoracle_collection as P
    ref = P.ref_available()
    q = np.ascontiguousarray(queries)
    nq = len(q)
    P_ = _lib.ptr
    for size in [int(s) for s in args.sizes.split(",")]:
        imgs = list(base)
        while sum(len(d) for d in imgs) < size:
            imgs += [flipped(rng, d, 4) for d in base]
        n = sum(len(d) for d in imgs)
        bdm = cs.line_lbd_detect(context=det._ctx).bdm
        bdm.add(imgs)
        ch = bdm._h
        rec = {"images": len(imgs), "codes": n}
        kout, kn = np.zeros(nq * 10, _lib.DMATCH_DTYPE), np.zeros(nq, np.int32)
        rout, roff = np.zeros(64 * nq, _lib.DMATCH_DTYPE), np.zeros(nq + 1, np.int64)
        mout, mn = np.zeros(nq, _lib.DMATCH_DTYPE), C.c_int32(0)
        calls = {"match": lambda: det._ctx.check(L.cs_lbd_collection_match(ch, P_(q, C.c_uint8), nq, None, 0, mout.ctypes.data, C.byref(mn)))}
        for k in (1, 2, 10):
            calls["knn%d" % k] = (lambda k=k: det._ctx.check(L.cs_lbd_collection_knn_match(ch, P_(q, C.c_uint8), nq, k, None, 0, kout.ctypes.data,
                                                                                           P_(kn, C.c_int32))))
        rcap = [len(rout)]

        def radius():
            buf = rout if rcap[0] <= len(rout) else np.zeros(rcap[0], _lib.DMATCH_DTYPE)
            rc = L.cs_lbd_collection_radius_match(ch, P_(q, C.c_uint8), nq, C.c_float(25.0), None, 0, buf.ctypes.data, C.c_int64(rcap[0]),
                                                  P_(roff, C.c_int64))
            if rc == -3:
                rcap[0] = int(roff[-1])
                return radius()
            det._ctx.check(rc)
        calls["radius25"] = radius
        radius()                                                            # size the buffer first: the timed calls do not retry
        rout = np.zeros(max(rcap[0], 1), _lib.DMATCH_DTYPE)
        for name, fn in calls.items():
            ms = timed(fn)
            rec[name] = {"call_ms": round(ms, 4), "queries_per_s": round(nq / (ms * 1e-3)), "code_pairs_per_s": nq * n / (ms * 1e-3)}
            rec[name]["entries"] = int(mn.value) if name == "match" else (int(roff[-1]) if name == "radius25" else int(kn.sum()))
        # what a caller does without the collection: one pairwise batch call of the C ABI over (queries, image) pairs, then a host merge
        # of the per-image k best into the k best overall (by distance; the collection's tie order is not reproduced by this merge)
        pairs = [im for im in imgs if len(im)]
        qo = (np.arange(len(pairs) + 1) * nq).astype(np.int32)
        to = np.concatenate([[0], np.cumsum([len(t) for t in pairs])]).astype(np.int32)
        qq, tt = np.ascontiguousarray(np.tile(q, (len(pairs), 1))), np.ascontiguousarray(np.concatenate(pairs))
        for k in (2, 10):
            pout, pn = np.zeros(len(qq) * k, _lib.DMATCH_DTYPE), np.zeros(len(qq), np.int32)
            t0 = time.perf_counter()
            det._ctx.check(L.cs_knn_match_line_descrip_batch(h, P_(qq, C.c_uint8), P_(qo, C.c_int32), P_(tt, C.c_uint8), P_(to, C.c_int32), len(pairs), k,
                                                             None, pout.ctypes.data, P_(pn, C.c_int32)))
            t1 = time.perf_counter()
            d = pout["distance"].reshape(len(pairs), nq, k).transpose(1, 0, 2).reshape(nq, -1).copy()
            d[(np.arange(k)[None, None, :] >= pn.reshape(len(pairs), nq, 1)).transpose(1, 0, 2).reshape(nq, -1)] = np.inf
            order = np.argsort(d, axis=1, kind="stable")[:, :k]
            ti = pout["train_idx"].reshape(len(pairs), nq, k).transpose(1, 0, 2).reshape(nq, -1)
            np.take_along_axis(ti, order, 1)
            t2 = time.perf_counter()
            rec["pairwise_knn%d" % k] = {"pairwise_call_ms": round((t1 - t0) * 1e3, 3), "host_merge_ms": round((t2 - t1) * 1e3, 3),
                                         "collection_speedup": round((t2 - t0) * 1e3 / rec["knn%d" % k]["call_ms"], 1)}
        if ref and n <= 20000:
            t0 = time.perf_counter()
            P.ref_collection_time("knn", imgs, q, 2)
            rec["knn2"]["reference_cpu_one_core_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
        out["collection_%d" % size] = rec
        del bdm
    print(json.dumps(out))


if __name__ == "__main__":
    main()
