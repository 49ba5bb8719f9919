"""Worker of tests/test_gpu_pipeline.py: runs one scenario of the benchmarked configuration in a fresh process and writes what the library
returned to an .npz; the test computes the CPU oracle and compares.

    python tests/pipeline_worker.py SCENARIO OUT.npz        SCENARIO: full | inflight | rolling | threads | shapes

A process of its own, because (1) the once-per-device function attributes (cs_kernels.h: CS_ONCE_PER_DEVICE) must be unset when the
`threads` scenario's host threads reach the launchers together, and (2) CUDA_DEVICE_MAX_CONNECTIONS must be set before CUDA starts, as
bench.py sets it, so that the streams of batches in flight interleave as they do under the benchmark.

Every batch is a run of bench.py's generator call (make_workload below); its repeated frames (distinct=32) are what lets the test compare
frame f with oracle frame f % 32 and with its own first occurrence.  The .npz holds, per labelled run: `<label>.recs` (cuboid records, one row
per box), `<label>.counts` (records per box), `<label>.stats` (STATS fields of ctx.stats()), and for matcher runs `<label>.knn` / `.radius`
(DMATCH_DTYPE records of all lists) with `.knn_len` / `.radius_len` (list lengths).  `mem_free0` / `mem_free_min`: cudaMemGetInfo's free
bytes at start and the least seen after a run."""
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# bench.py's WORKLOADS (the test checks the copy): name -> (frames per GPU, width, height, boxes/frame, kind, poisson, param overrides)
WORKLOADS = {
    "c2": (1, 640, 480, 5, "indoor", False, {}),
    "c3": (256, 640, 480, 3, "indoor", True, {}),
    "c4": (128, 1242, 375, 8, "kitti", False, {}),
    "c5": (64, 1280, 960, 8, "indoor", False, dict(yaw_step_deg=0.5, top_sample_count_override=30)),
}
SEED_BASE = 20260922        # bench.py make_workload's seed_base
LINE_LENGTH_THRES = 15.0    # bench.py
DISTINCT = 32               # make_workload renders min(F, 32) distinct frames; the rest repeat them cyclically
STATS = ("n_frames", "n_objects", "n_candidates", "n_valid", "n_lines_in")
LINE_MODES = {"given": 0, "lsd": 1, "edlines": 2}   # oracle.pyoracle.detect_frames_batch's line_mode

# (a) full batches, one context each, bench's protocol
FULL_CASES = [("c3", "lsd"), ("c3", "edlines"), ("c3", "given"), ("c4", "lsd"), ("c5", "lsd")]
# (b) four contexts in flight: c3-shaped 64-frame batches of bench's generator at ranks 1..4 (so four different seeds)
INFLIGHT_RANKS = (1, 2, 3, 4)
INFLIGHT_STEPS = 2 * len(INFLIGHT_RANKS)
# (c) the rolling pipeline: five 64-frame batches (ranks 1..5), three contexts, nine steps; step s uploads batch s % 5 on context s % 3.
# Context ROLLING_DEVICE_CTX takes every other one of its uploads (its 2nd, 4th ...) from a CUDA tensor through upload_online_device.
ROLLING_RANKS = (1, 2, 3, 4, 5)
ROLLING_CTXS = 3
ROLLING_STEPS = 9
ROLLING_DEVICE_CTX = 1
# context ROLLING_SCRIBBLE_CTX overwrites its pinned staging buffer as soon as each upload returns (cs_batch_upload_online waits for its copy)
ROLLING_SCRIBBLE_CTX = 2
# (d) host threads started together: (label, workload, rank, frames, line mode, entry point)
THREAD_JOBS = [("t_lsd", "c3", 1, 64, "lsd", "detect_frames_host"), ("t_edl", "c4", 0, 32, "edlines", "detect_frames_host"),
               ("t_given", "c3", 2, 64, "given", "detect_batch_host")]
# two matcher threads, knnMatch k = 5 and radiusMatch on train sets whose sorted launches ask for 4 KB to 128 KB of shared memory
MATCH_JOBS = [("t_match0", 71, (300, 9000, 16384, 2000)), ("t_match1", 72, (16000, 700, 5000, 12000))]
MATCH_QUERIES, MATCH_K, MATCH_RADIUS = 48, 5, 60.0
# (e) one context at 1280 x 960 x 256, shapes changing between batches
SHAPES_CTX = (1280, 960, 256)
SHAPES_RUNS = [("s0_c3_lsd", "c3", "lsd"), ("s1_c4_lsd", "c4", "lsd"), ("s2_c2_lsd", "c2", "lsd"), ("s3_tiny_given", "tiny", "given"),
               ("s4_c3_edlines", "c3", "edlines")]


def make_workload(name, rank=0, frames=None):
    """bench.py's make_workload: the same generator call on the same seeds"""
    from cube_slam_b200 import synthetic as S
    if name == "tiny":
        return tiny_workload()
    F, w, h, nb, kind, poisson, over = WORKLOADS[name]
    if frames:
        F = frames
    imgs, Ts, boxes, lines, K = S.make_batch(SEED_BASE + 1000 * rank + sum(map(ord, name)), F, w, h, nb, kind=kind, poisson=poisson,
                                             distinct=min(F, DISTINCT))
    return dict(imgs=imgs, Ts=Ts, boxes=boxes, lines=lines, K=K, over=over, w=w, h=h, F=F, name=name)


def tiny_workload():
    """3 gray frames of 97 x 211 (an odd width: rows not a multiple of 4 bytes), boxes placed by hand (the generator places none at this
    size): one box per frame, two boxes covering the whole frame or reaching its right and bottom borders, one box without a valid proposal"""
    from cube_slam_b200 import synthetic as S
    imgs, Ts, _, lines, K = S.make_batch(97211, 3, 97, 211, 2)
    boxes = [np.array([[5, 120, 60, 70, 0.9]]), np.array([[0, 100, 97, 111, 0.9], [40, 130, 55, 80, 0.8]]),
             np.array([[20, 150, 50, 55, 0.9], [30, 110, 40, 90, 0.7]])]
    return dict(imgs=np.ascontiguousarray(imgs[..., 1]), Ts=Ts, boxes=boxes, lines=lines, K=K, over={}, w=97, h=211, F=3, name="tiny")


def digest(wl):
    """SHA-256 of a workload's inputs: frames, poses, calibration, boxes and lines"""
    import hashlib
    h = hashlib.sha256(wl["imgs"].tobytes() + wl["Ts"].tobytes() + wl["K"].tobytes())
    for b, l in zip(wl["boxes"], wl["lines"]):
        h.update(np.ascontiguousarray(b).tobytes() + np.ascontiguousarray(l).tobytes())
    return h.hexdigest()


def match_inputs(seed, n_train):
    """MATCH_QUERIES query codes near random train codes (a planted code with 0..139 bits flipped) and duplicated train codes"""
    rng = np.random.default_rng(seed * 100003 + n_train)
    t = rng.integers(0, 256, (n_train, 32), dtype=np.uint8)
    t[n_train - 1] = t[1]
    q = t[rng.integers(0, n_train, MATCH_QUERIES)].copy()
    for i in range(MATCH_QUERIES):
        flips = rng.integers(0, 256, int(rng.integers(0, 140)))
        np.bitwise_xor.at(q[i], flips // 8, (1 << (flips % 8)).astype(np.uint8))
    return q, t


class Recorder(object):
    def __init__(self, torch):
        self.torch = torch
        self.out = {}
        self.free0 = torch.cuda.mem_get_info(0)[0]
        self.free_min = self.free0
        self.lock = threading.Lock()

    def memory(self):
        free = self.torch.cuda.mem_get_info(0)[0]
        with self.lock:
            self.free_min = min(self.free_min, free)

    def batch(self, label, cx, recs, counts):
        st = cx.stats()
        self.memory()
        with self.lock:
            self.out[label + ".recs"] = np.ascontiguousarray(recs)
            self.out[label + ".counts"] = np.asarray(counts, np.int32)
            self.out[label + ".stats"] = np.array([st[k] for k in STATS], np.int64)

    def save(self, path):
        self.out["mem_free0"] = np.int64(self.free0)
        self.out["mem_free_min"] = np.int64(self.free_min)
        np.savez(path, **self.out)


def line_params(cs, cx, use_lsd):
    """bench.py's make_line_params"""
    det = cs.line_lbd_detect(context=cx)
    det.use_LSD = use_lsd
    det.line_length_thres = LINE_LENGTH_THRES
    return det.params()


def new_context(cs, wl, dims=None):
    w, h, F = dims or (wl["w"], wl["h"], wl["F"])
    cx = cs.Context(0, w, h, F, 16, 8192)     # bench.py's contexts
    cx.set_calibration(wl["K"])
    return cx


def upload(cs, cx, wl, mode):
    params = cs.default_params(**wl["over"])
    cx.set_calibration(wl["K"])
    if mode == "given":
        cx.upload(wl["imgs"], wl["Ts"], wl["boxes"], wl["lines"], params)
    else:
        cx.upload_online(wl["imgs"], wl["Ts"], wl["boxes"], line_params(cs, cx, mode == "lsd"), params)


def run_full(cs, rec):
    """(a) bench's protocol, one context per case: upload once, run_async three times without a fetch in between, then fetch"""
    for name, mode in FULL_CASES:
        wl = make_workload(name)
        cx = new_context(cs, wl)
        upload(cs, cx, wl, mode)
        for _ in range(3):
            cx.run_async()
        recs, counts = cx.fetch()
        rec.batch("%s_%s" % (name, mode), cx, recs, counts)
        cx.close()


def run_inflight(cs, rec):
    """(b) four contexts, four batches, run_async round-robin with no host sync, then a fetch of each"""
    wls = [make_workload("c3", r, 64) for r in INFLIGHT_RANKS]
    ctxs = [new_context(cs, wl) for wl in wls]
    for cx, wl in zip(ctxs, wls):
        upload(cs, cx, wl, "lsd")
    for i in range(INFLIGHT_STEPS):
        ctxs[i % len(ctxs)].run_async()
    for r, cx in zip(INFLIGHT_RANKS, ctxs):
        recs, counts = cx.fetch()
        rec.batch("inflight_r%d" % r, cx, recs, counts)
    for cx in ctxs:
        cx.close()


def run_rolling(cs, rec, torch):
    """(c) bench.py's e2e_run: step s is issued on context s % K (upload_online + run_async), then the oldest outstanding step is fetched.
    Frames come from a pinned staging buffer per context, refilled only after the step that read it has been fetched; on one context every
    other upload comes from a CUDA tensor instead, and another one zeroes its staging buffer as soon as the upload has returned, which the
    header allows (the upload waits for its copy)."""
    wls = [make_workload("c3", r, 64) for r in ROLLING_RANKS]
    ctxs = [new_context(cs, wls[0]) for _ in range(ROLLING_CTXS)]
    staging = [torch.empty(wls[0]["imgs"].shape, dtype=torch.uint8, pin_memory=True) for _ in ctxs]
    on_device = [torch.from_numpy(wl["imgs"]).cuda() for wl in wls]
    torch.cuda.synchronize()
    params = cs.default_params(**wls[0]["over"])
    lp = line_params(cs, ctxs[0], True)
    outstanding = [None] * ROLLING_CTXS     # the step each context is running, until it is fetched
    uploads = [0] * ROLLING_CTXS

    def issue(s):
        k = s % ROLLING_CTXS
        assert outstanding[k] is None, "staging buffer %d refilled before its step was fetched" % k
        wl, cx = wls[s % len(wls)], ctxs[k]
        if k == ROLLING_DEVICE_CTX and uploads[k] % 2 == 1:
            cx.upload_online_device(on_device[s % len(wls)], wl["Ts"], wl["boxes"], lp, params)
        else:
            staging[k].numpy()[...] = wl["imgs"]
            cx.upload_online(staging[k].numpy(), wl["Ts"], wl["boxes"], lp, params)
        if k == ROLLING_SCRIBBLE_CTX:
            staging[k].numpy()[...] = 0     # the upload has returned: the library holds its own copy
        cx.run_async()
        uploads[k] += 1
        outstanding[k] = s

    issued = fetched = 0
    while fetched < ROLLING_STEPS:
        while issued < ROLLING_STEPS and issued - fetched < ROLLING_CTXS:
            issue(issued)
            issued += 1
        k = fetched % ROLLING_CTXS
        recs, counts = ctxs[k].fetch()
        rec.batch("rolling_s%d" % fetched, ctxs[k], recs, counts)
        outstanding[k] = None
        fetched += 1
    for cx in ctxs:
        cx.close()


def run_threads(cs, rec):
    """(d) the first GPU work of the process: five host threads, each on its own context, released together by a barrier, each doing its
    work twice"""
    jobs = []
    for label, name, rank, F, mode, entry in THREAD_JOBS:
        wl = make_workload(name, rank, F)
        jobs.append((label, wl, mode, entry, new_context(cs, wl)))
    matchers = []
    for label, seed, sizes in MATCH_JOBS:
        det = cs.line_lbd_detect()
        matchers.append((label, [(n,) + match_inputs(seed, n) for n in sizes], det))
    gate = threading.Barrier(len(jobs) + len(matchers))
    errors = []

    def detect(label, wl, mode, entry, cx):
        params = cs.default_params(**wl["over"])
        lp = None if mode == "given" else line_params(cs, cx, mode == "lsd")
        gate.wait()
        for rep in range(2):
            if entry == "detect_frames_host":
                recs, counts = cx.detect_frames_host(wl["imgs"], wl["Ts"], wl["boxes"], lp, params)
            else:
                recs, counts = cx.detect_batch_host(wl["imgs"], wl["Ts"], wl["boxes"], wl["lines"], params)
            rec.batch("%s_rep%d" % (label, rep), cx, recs.copy(), counts.copy())

    def match(label, sets, det):
        gate.wait()
        for rep in range(2):
            for n, q, t in sets:
                for kind, lists in (("knn", det.bdm.knnMatch(q, t, MATCH_K)), ("radius", det.bdm.radiusMatch(q, t, MATCH_RADIUS))):
                    key = "%s_rep%d_n%d.%s" % (label, rep, n, kind)
                    with rec.lock:
                        rec.out[key] = np.concatenate(lists)
                        rec.out[key + "_len"] = np.array([len(x) for x in lists], np.int32)
        rec.memory()

    def guarded(fn, *args):
        try:
            fn(*args)
        except Exception as e:  # noqa: BLE001 -- reported in the exit code and on stderr
            errors.append("%s: %s: %s" % (args[0], type(e).__name__, e))
            gate.abort()

    threads = [threading.Thread(target=guarded, args=(detect,) + j) for j in jobs]
    threads += [threading.Thread(target=guarded, args=(match,) + m) for m in matchers]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for j in jobs:
        j[-1].close()
    for m in matchers:
        m[-1]._ctx.close()
    if errors:
        raise RuntimeError("; ".join(errors))


def run_shapes(cs, rec):
    """(e) one context sized for the largest batch, five batches of changing shape: grow-only arenas when a batch shrinks and when the frame
    width changes"""
    cx = None
    for label, name, mode in SHAPES_RUNS:
        wl = make_workload(name)
        if cx is None:
            cx = new_context(cs, wl, SHAPES_CTX)
        upload(cs, cx, wl, mode)
        cx.run_async()
        recs, counts = cx.fetch()
        rec.batch(label, cx, recs, counts)
    cx.close()


def main():
    scenario, out = sys.argv[1], sys.argv[2]
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # as bench.py, before CUDA starts
    import torch
    import cube_slam_b200 as cs
    torch.cuda.set_device(0)
    rec = Recorder(torch)
    if scenario == "full":
        run_full(cs, rec)
    elif scenario == "inflight":
        run_inflight(cs, rec)
    elif scenario == "rolling":
        run_rolling(cs, rec, torch)
    elif scenario == "threads":
        run_threads(cs, rec)
    elif scenario == "shapes":
        run_shapes(cs, rec)
    else:
        raise SystemExit("unknown scenario %r" % scenario)
    torch.cuda.synchronize()
    rec.save(out)
    print("pipeline_worker %s: peak device memory in use %.2f GB" % (scenario, (rec.free0 - rec.free_min) / 1e9), flush=True)


if __name__ == "__main__":
    main()
