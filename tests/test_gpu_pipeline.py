"""The configurations bench.py times, checked against the CPU oracle: full 256 / 128 / 64-frame batches under bench's protocol (upload once,
three run_async without a fetch), four batches in flight on four contexts, the rolling upload_online + run_async + fetch pipeline (pinned host
frames, and device frames on one context), host threads released together at process start on their own contexts (batch paths and the
knn / radius matcher), and one context taking batches of changing shape.  A kernel that goes wrong only at batch scale, state that leaks from
one batch into the next on a reused context, or a race between contexts or host threads shows here.

The GPU work runs in a fresh process (tests/pipeline_worker.py, one per scenario), so that the once-per-device function attributes are unset
when the host threads of the `threads` scenario reach the launchers together, and so that CUDA_DEVICE_MAX_CONNECTIONS is set before CUDA starts,
as under bench.py.  This process computes the oracle (oracle.pyoracle.detect_frames_batch over the batch's 32 distinct frames, OpenMP over the
host cores) while the worker runs, then compares: frame f of a batch with oracle frame f % 32 (records with _compare_cuboid's tolerances,
counts exactly), every repeated frame byte for byte with its first occurrence (what catches indexing mistakes in frames 32 to 255), and the
batch statistics (candidates, scored proposals, segments handed to the cuboid stage) with the oracle's sums.

Measured on one H100 80GB HBM3 at a 400 W power limit: the five GPU tests take 81 s in all, 15-20 s each, most of it process start-up and
input generation.  Peak device memory in use (cudaMemGetInfo's free bytes in the worker, at start and after each run) is 5.2 GB in `shapes`
and 1.5-3.3 GB in the others."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import pipeline_worker as PW
from test_gpu_cuboid_parity import _compare_cuboid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "pipeline_worker.py")


def test_workloads_table_is_bench_s():
    """the worker's copy of bench.py's table, seed base and line length, and its generator call, equal bench.py's own (bench.py is read in a
    subprocess: importing it here would set CUDA_DEVICE_MAX_CONNECTIONS for every later test)"""
    code = ("import inspect, json, sys\n"
            "sys.path[:0] = [%r, %r]\n"
            "import bench, pipeline_worker as PW\n"
            "print(json.dumps(dict(table={k: list(v[:7]) for k, v in bench.WORKLOADS.items()}, line_length=bench.LINE_LENGTH_THRES,\n"
            "                      seed_base=inspect.signature(bench.make_workload).parameters['seed_base'].default,\n"
            "                      c3_r1=PW.digest(bench.make_workload('c3', 1, frames=64)), c4_r0=PW.digest(bench.make_workload('c4', 0, frames=32)))))\n"
            ) % (ROOT, os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got["table"] == {k: list(v) for k, v in PW.WORKLOADS.items()}
    assert got["line_length"] == PW.LINE_LENGTH_THRES and got["seed_base"] == PW.SEED_BASE
    assert got["c3_r1"] == PW.digest(PW.make_workload("c3", 1, 64)) and got["c4_r0"] == PW.digest(PW.make_workload("c4", 0, 32))


@functools.lru_cache(maxsize=None)
def reference(name, rank, mode, n_distinct):
    """the batch's distinct frames and the oracle's answer on them (records, counts, box offsets, per-frame n_valid / n_cand / n_lines)"""
    from oracle import pyoracle as O
    wl = PW.make_workload(name, rank, n_distinct)
    ref = O.detect_frames_batch(wl["imgs"], wl["K"], wl["Ts"], wl["boxes"], wl["lines"] if mode == "given" else None, O.default_params(**wl["over"]),
                                line_mode=PW.LINE_MODES[mode], line_length_thres=PW.LINE_LENGTH_THRES, want_records=True)
    return wl, ref


def n_distinct(name, F):
    return 3 if name == "tiny" else min(F, PW.DISTINCT)


def run_worker(scenario, tmp_path, batches=()):
    """the scenario in a fresh process; the oracle of `batches` ((name, rank, mode, F) ...) is computed while it runs"""
    out = str(tmp_path / (scenario + ".npz"))
    env = dict(os.environ)
    env["CUDA_DEVICE_MAX_CONNECTIONS"] = "32"
    p = subprocess.Popen([sys.executable, WORKER, scenario, out], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, cwd=ROOT)
    try:
        for name, rank, mode, F in batches:
            reference(name, rank, mode, n_distinct(name, F))
    finally:
        so, se = p.communicate(timeout=900)
    assert p.returncode == 0, (so[-3000:], se[-3000:])
    print(so.strip())
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


def check_batch(got, label, name, rank, mode, F):
    """one fetched batch of F frames against the oracle of its distinct frames, and every repeated frame against its first occurrence"""
    wl, ref = reference(name, rank, mode, n_distinct(name, F))
    D = len(wl["imgs"])
    recs, counts, stats = got[label + ".recs"], got[label + ".counts"], dict(zip(PW.STATS, got[label + ".stats"].tolist()))
    nb = [len(wl["boxes"][f % D]) for f in range(F)]
    off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    assert len(counts) == off[-1] and stats["n_frames"] == F and stats["n_objects"] == off[-1], (label, len(counts), stats)
    every = [f % D for f in range(F)]
    assert stats["n_candidates"] == int(ref["n_cand"][every].sum()), (label, stats)
    assert stats["n_valid"] == int(ref["n_valid"][every].sum()), (label, stats)
    assert stats["n_lines_in"] == int(ref["n_lines"][every].sum()), (label, stats)
    assert int(counts.sum()) > 0, label
    for f in range(F):
        d = f % D
        for b in range(nb[f]):
            o, ro = off[f] + b, ref["box_off"][d] + b
            n = int(counts[o])
            assert n == int(ref["counts"][ro]), (label, "frame", f, "box", b, n, int(ref["counts"][ro]))
            if f >= D:
                o0 = off[d] + b
                a, a0 = recs[o, :n].copy(), recs[o0, :n].copy()
                a["pad_"] = 0
                a0["pad_"] = 0
                assert a.tobytes() == a0.tobytes(), (label, "frame", f, "box", b, "differs from frame", d)
                continue
            for k in range(n):
                try:
                    _compare_cuboid(recs[o, k], ref["records"][ro, k])
                except AssertionError as e:
                    raise AssertionError("%s: frame %d box %d record %d: %s" % (label, f, b, k, e)) from None


def check_lists(got, key, want):
    """the flattened DMATCH_DTYPE lists of the worker against the oracle's [(query, query_idx, train_idx, distance)]"""
    flat, lens = got[key], got[key + "_len"]
    assert len(lens) == len(want), (key, len(lens), len(want))
    o = 0
    for n, (i, qi, ti, di) in zip(lens.tolist(), want):
        g = flat[o:o + n]
        o += n
        assert n == len(ti), (key, i, n, len(ti))
        np.testing.assert_array_equal(g["query_idx"], qi, err_msg=key)
        np.testing.assert_array_equal(g["train_idx"], ti, err_msg=key)
        np.testing.assert_array_equal(g["distance"], di, err_msg=key)
        assert (g["img_idx"] == 0).all(), key
    assert o == len(flat), key


@pytest.mark.gpu
def test_full_batches_under_bench_protocol(oracle, tmp_path):
    """c3 with online LSD (the headline), online EDLines and lines given; c4 and c5 (dense 181 x 30 sweep) with online LSD: one context
    each, upload once, run_async three times, fetch"""
    cases = [(name, 0, mode, PW.WORKLOADS[name][0]) for name, mode in PW.FULL_CASES]
    got = run_worker("full", tmp_path, cases)
    for name, rank, mode, F in cases:
        check_batch(got, "%s_%s" % (name, mode), name, rank, mode, F)


@pytest.mark.gpu
def test_batches_in_flight_on_four_contexts(oracle, tmp_path):
    """four 64-frame batches of different seeds, run_async round-robin twice over with no host sync, then fetched: each equals its own
    oracle (no batch sees another context's frames, lines or records)"""
    cases = [("c3", r, "lsd", 64) for r in PW.INFLIGHT_RANKS]
    got = run_worker("inflight", tmp_path, cases)
    for name, r, mode, F in cases:
        check_batch(got, "inflight_r%d" % r, name, r, mode, F)


@pytest.mark.gpu
def test_rolling_upload_run_fetch_pipeline(oracle, tmp_path):
    """bench.py's e2e_run over three contexts and nine steps: every step a different batch from the previous one on its context, pinned host
    frames, device frames on every other upload of one context; each fetched step equals its batch's oracle"""
    cases = [("c3", r, "lsd", 64) for r in PW.ROLLING_RANKS]
    got = run_worker("rolling", tmp_path, cases)
    for s in range(PW.ROLLING_STEPS):
        r = PW.ROLLING_RANKS[s % len(PW.ROLLING_RANKS)]
        check_batch(got, "rolling_s%d" % s, "c3", r, "lsd", 64)


@pytest.mark.gpu
def test_host_threads_started_together_at_process_start(oracle, tmp_path):
    """five host threads, their own context each, released by one barrier as the process's first GPU work: cs_detect_frames_batch with LSD
    (64 VGA frames) and with EDLines (32 KITTI frames), cs_detect_cuboids_batch with lines given (64 VGA frames), and two matchers running
    knnMatch k = 5 and radiusMatch on train sets from 300 to 16384 codes; every thread twice, every answer the oracle's"""
    from oracle import pyoracle_knn as K
    cases = [(name, rank, mode, F) for _, name, rank, F, mode, _ in PW.THREAD_JOBS]
    got = run_worker("threads", tmp_path, cases)
    for label, name, rank, F, mode, _ in PW.THREAD_JOBS:
        for rep in range(2):
            check_batch(got, "%s_rep%d" % (label, rep), name, rank, mode, F)
    for label, seed, sizes in PW.MATCH_JOBS:
        for n in sizes:
            q, t = PW.match_inputs(seed, n)
            knn, rad = K.lbd_knn_lists(q, t, PW.MATCH_K), K.lbd_radius_lists(q, t, PW.MATCH_RADIUS)
            assert any(len(x[2]) for x in rad)
            for rep in range(2):
                check_lists(got, "%s_rep%d_n%d.knn" % (label, rep, n), knn)
                check_lists(got, "%s_rep%d_n%d.radius" % (label, rep, n), rad)


@pytest.mark.gpu
def test_one_context_changing_shapes(oracle, tmp_path):
    """one 1280 x 960 x 256 context: c3 with LSD, c4 (KITTI, 8 boxes), c2 (one frame), three 97 x 211 gray frames with lines given, c3 with
    EDLines -- the grow-only arenas when a batch shrinks and when the frame width changes"""
    cases = []
    for label, name, mode in PW.SHAPES_RUNS:
        F = 3 if name == "tiny" else PW.WORKLOADS[name][0]
        cases.append((label, name, 0, mode, F))
    got = run_worker("shapes", tmp_path, [c[1:] for c in cases])
    for label, name, rank, mode, F in cases:
        check_batch(got, label, name, rank, mode, F)
