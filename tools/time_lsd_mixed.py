"""Times LSD over frames of different sizes and the single-run octave pyramid, and prints one JSON line.

    python tools/time_lsd_mixed.py [--baseline-lib PATH] [--calls 10] [--warmup 2] [--rounds 2]

Two workloads, each timed as the median of --calls synchronous calls after --warmup calls, in a process of its own per library and round
(rounds alternate between the libraries, so the spread between rounds shows the run-to-run noise):
  vector    64 synthetic BGR frames in 4 sizes (640 x 480, 1241 x 376, 1226 x 370, 320 x 240; KITTI-like sizes among them), interleaved, at
            1 and 3 octaves: one cs_detect_raw_lines_octaves_batch_mixed call against one cs_detect_raw_lines_octaves_batch call per size
            (what LSDDetector's vector form makes).  The two answers are compared byte for byte.
  octaves   tools/time_lsd_octaves.py's workload at numoctaves 3: 256 synthetic VGA frames, cs_detect_raw_lines_octaves_batch and
            cs_detect_descrip_lines_octaves_batch (cap 2048).  With --baseline-lib (a build of the library from before LSD ran the octaves
            as one batch, e.g. the parent commit's cube_slam_b200/lib/libcubeslam_b200.so) the same calls are timed there too and the key
            lines, counts and descriptors of both libraries are compared byte for byte.
The card's name, power limit and SM clock are read in the same run.  Outputs go to a temporary directory; nothing is written in the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "cube_slam_b200", "lib", "libcubeslam_b200.so")
SIZES = [(640, 480), (1241, 376), (1226, 370), (320, 240)]
CAP = 2048


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


class Lib(object):
    """the octave calls of one build of the library, through ctypes (two builds never share a process)"""

    def __init__(self, path, max_w, max_h):
        from cube_slam_b200 import _lib
        self.T = _lib
        L = self.L = C.CDLL(path)
        vp, i, i32_p = C.c_void_p, C.c_int, C.POINTER(C.c_int32)
        L.cs_create.restype = vp
        L.cs_create.argtypes = [i] * 6
        L.cs_destroy.argtypes = [vp]
        L.cs_last_error.restype = C.c_char_p
        L.cs_last_error.argtypes = [vp]
        L.cs_default_line_params.argtypes = [C.POINTER(_lib.LineParams)]
        lp = C.POINTER(_lib.LineParams)
        L.cs_detect_raw_lines_octaves_batch.argtypes = [vp, vp, i, i, i, i, i, lp, vp, C.c_int32, i32_p]
        L.cs_detect_descrip_lines_octaves_batch.argtypes = [vp, vp, i, i, i, i, i, lp, vp, vp, C.c_int32, i32_p]
        if hasattr(L, "cs_detect_raw_lines_octaves_batch_mixed"):
            L.cs_detect_raw_lines_octaves_batch_mixed.argtypes = [vp, vp, C.POINTER(_lib.FrameView), i, lp, vp, C.c_int32, i32_p]
        self.h = L.cs_create(0, max_w, max_h, 1, 1, 1)
        if not self.h:
            raise RuntimeError("cs_create failed")

    def params(self, K):
        p = self.T.LineParams()
        self.L.cs_default_line_params(C.byref(p))
        p.use_LSD, p.numoctaves, p.octaveratio, p.line_length_thres = 1, K, 2.0 if K > 1 else 1.0, 15.0
        return p

    def check(self, rc):
        if rc != 0:
            raise RuntimeError("status %d: %s" % (rc, self.L.cs_last_error(self.h).decode()))

    def octaves(self, imgs, K, describe=False):
        """one-size call over F x H x W x 3 frames -> (key lines F x K x CAP, counts F x K, descriptors or None)"""
        F, H, W = imgs.shape[:3]
        kl = np.zeros((F, K, CAP), self.T.OCTAVE_KEYLINE_DTYPE)
        n = np.zeros((F, K), np.int32)
        p = self.params(K)
        if describe:
            d = np.zeros((F, K, CAP, 32), np.uint8)
            self.check(self.L.cs_detect_descrip_lines_octaves_batch(self.h, imgs.ctypes.data, F, W, H, W * 3, 3, C.byref(p), kl.ctypes.data,
                                                                     d.ctypes.data, CAP, n.ctypes.data_as(C.POINTER(C.c_int32))))
            return kl, n, d
        self.check(self.L.cs_detect_raw_lines_octaves_batch(self.h, imgs.ctypes.data, F, W, H, W * 3, 3, C.byref(p), kl.ctypes.data, CAP,
                                                             n.ctypes.data_as(C.POINTER(C.c_int32))))
        return kl, n, None

    def octaves_mixed(self, buf, views, F, K):
        kl = np.zeros((F, K, CAP), self.T.OCTAVE_KEYLINE_DTYPE)
        n = np.zeros((F, K), np.int32)
        p = self.params(K)
        self.check(self.L.cs_detect_raw_lines_octaves_batch_mixed(self.h, buf.ctypes.data, views, F, C.byref(p), kl.ctypes.data, CAP,
                                                                   n.ctypes.data_as(C.POINTER(C.c_int32))))
        return kl, n

    def close(self):
        self.L.cs_destroy(self.h)


def slots(kl, n):
    """the filled slots only: the bytes a caller reads"""
    return b"".join(kl[f, k, :n[f, k]].tobytes() for f in range(n.shape[0]) for k in range(n.shape[1])) + n.tobytes()


def worker_vector(lib, args):
    from cube_slam_b200 import _lib, synthetic as S
    per = 16
    frames = {s: np.ascontiguousarray(S.make_batch(40 + i, per, s[0], s[1], 3)[0]) for i, s in enumerate(SIZES)}
    order = [(i % len(SIZES), i // len(SIZES)) for i in range(per * len(SIZES))]      # sizes interleaved
    imgs = [frames[SIZES[s]][j] for s, j in order]
    buf, views = _lib.pack_frames(imgs)
    L = Lib(lib, max(w for w, _ in SIZES), max(h for _, h in SIZES))
    res = {"frames": len(imgs), "sizes": SIZES}
    for K in (1, 3):
        def per_size():
            return {s: L.octaves(frames[s], K) for s in SIZES}

        def one_call():
            return L.octaves_mixed(buf, views, len(imgs), K)
        t_sizes = median_ms(per_size, args.calls, args.warmup)
        t_mixed = median_ms(one_call, args.calls, args.warmup)
        got = per_size()
        kl, n = one_call()
        same = all(slots(kl[i:i + 1], n[i:i + 1]) == slots(got[SIZES[s]][0][j:j + 1], got[SIZES[s]][1][j:j + 1]) for i, (s, j) in enumerate(order))
        res[str(K)] = {"per_size_calls_ms": t_sizes, "one_mixed_call_ms": t_mixed, "outputs_identical": bool(same),
                       "key_lines": int(n.sum())}
    L.close()
    return res


def worker_octaves(lib, args, dump):
    from cube_slam_b200 import synthetic as S
    imgs = np.ascontiguousarray(S.make_batch(0, 256, 640, 480, 3)[0])
    L = Lib(lib, 640, 480)
    K = 3
    raw_ms = median_ms(lambda: L.octaves(imgs, K), args.calls, args.warmup)
    desc_ms = median_ms(lambda: L.octaves(imgs, K, True), args.calls, args.warmup)
    kl, n, _ = L.octaves(imgs, K)
    dkl, dn, d = L.octaves(imgs, K, True)
    L.close()
    with open(dump, "wb") as fh:
        fh.write(slots(kl, n))
        fh.write(slots(dkl, dn))
        fh.write(b"".join(d[f, k, :dn[f, k]].tobytes() for f in range(dn.shape[0]) for k in range(K)))
    return {"frames": int(imgs.shape[0]), "numoctaves": K, "raw_median_ms": raw_ms, "descrip_median_ms": desc_ms, "key_lines": int(n.sum())}


def run_worker(case, lib, args, dump):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", case, "--lib", lib, "--calls", str(args.calls), "--warmup", str(args.warmup),
           "--dump", dump]
    o = subprocess.run(cmd, capture_output=True, text=True)
    if o.returncode != 0:
        raise RuntimeError("%s worker on %s failed:\n%s" % (case, lib, o.stderr[-3000:]))
    return json.loads(o.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--worker", default=None)
    ap.add_argument("--lib", default=LIB)
    ap.add_argument("--dump", default=None)
    args = ap.parse_args()
    if args.worker:
        out = worker_vector(args.lib, args) if args.worker == "vector" else worker_octaves(args.lib, args, args.dump)
        print(json.dumps(out))
        return
    res = {"card": card(), "calls": args.calls, "warmup": args.warmup}
    with tempfile.TemporaryDirectory() as tmp:
        res["vector"] = [run_worker("vector", LIB, args, os.path.join(tmp, "v")) for _ in range(args.rounds)]
        libs = [("this", LIB)] + ([("baseline", os.path.abspath(args.baseline_lib))] if args.baseline_lib else [])
        octs = {name: [] for name, _ in libs}
        dumps = {}
        for r in range(args.rounds):
            for name, path in (libs if r % 2 == 0 else libs[::-1]):
                dumps[name] = os.path.join(tmp, "oct_%s_%d" % (name, r))
                octs[name].append(run_worker("octaves", path, args, dumps[name]))
        res["octaves"] = octs
        if args.baseline_lib:
            res["octaves_outputs_identical"] = open(dumps["this"], "rb").read() == open(dumps["baseline"], "rb").read()
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
