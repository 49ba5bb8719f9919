"""The LSD seed loop's work after region growth, on the GPU: region2rect on regions of one, two and more 32-point chunks, refine, and
reduce_region_radius with its warp-parallel compaction (the reference's swap-with-last order, restated in closed form), on ordinary
frames and on lists of thousands of points.

Each batch goes through both instantiations of k_lsd_grow_seq.  The profiling one (cs_set_profiling bit 0) must show the regimes were
reached: refines, reduce iterations, and region2rect calls in each of its size classes (<= 32, <= 64, > 64 points).  Raw segments and the
filtered matrix equal the oracle's bit for bit in both."""
import ctypes as C

import numpy as np
import pytest

from test_oracle_ref_lsd_large_regions import frames

pytestmark = pytest.mark.gpu

SLOT_SEEDS_TO_RECT, SLOT_REFINES, SLOT_REDUCE_ITERS, SLOT_RECT_SIZES = 12, 13, 14, 15   # cs_debug_lsd_prof
CAP = 16384


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    yield d
    d._ctx.set_profiling(0)
    d._ctx.close()


def ordinary(seed, w, h):
    """a benchmark-like synthetic frame (bench.py's c3 generator)"""
    from cube_slam_b200 import synthetic as S
    return S.make_batch(seed, 1, w, h, 3, kind="indoor", poisson=True)[0][0]


def run(det, imgs, profiled):
    ctx = det._ctx
    ctx.set_profiling(1 if profiled else 0)
    try:
        ctx.check(ctx.L.cs_debug_lsd_prof(ctx.h, None, 1))
        lines = det.detect_filter_lines_batch(np.ascontiguousarray(imgs), cap=CAP)
        prof = np.zeros(16, np.uint64)
        ctx.check(ctx.L.cs_debug_lsd_prof(ctx.h, prof.ctypes.data_as(C.POINTER(C.c_uint64)), 0))
    finally:
        ctx.set_profiling(0)
    return lines, prof


def check_batch(det, oracle, named):
    """named: [(name, frame)] of one size and channel count -> the profiling run's counters"""
    imgs = np.stack([img for _, img in named])
    refs = [oracle.lsd_detect(img, 15.0, cap=CAP) for _, img in named]
    counters = None
    for profiled in (True, False):
        lines, prof = run(det, imgs, profiled)
        if profiled:
            counters = prof
        else:
            assert not prof[SLOT_SEEDS_TO_RECT:].any()   # the production kernel counts nothing
        for f, ((name, _), r) in enumerate(zip(named, refs)):
            dbg = det.debug_frame(f, CAP)
            assert len(dbg["raw_lines"]) == len(r["raw_lines"]), (name, profiled)
            np.testing.assert_array_equal(dbg["raw_lines"], r["raw_lines"], err_msg="%s profiled=%s" % (name, profiled))
            np.testing.assert_array_equal(lines[f], r["lines"], err_msg="%s profiled=%s" % (name, profiled))
    return counters


def rect_sizes(prof):
    v = int(prof[SLOT_RECT_SIZES])
    return [v >> s & ((1 << 21) - 1) for s in (0, 21, 42)]


@pytest.mark.parametrize("kind", ["bgr", "gray"])
def test_ordinary_vga_frames(det, oracle, kind):
    """c3-like frames: hundreds of region2rect calls per frame on either side of 32 and 64 points, dozens of refines and reduces"""
    named = []
    for s in range(6):
        img = ordinary(311 + s, 640, 480)
        named.append(("c3_%d" % s, img if kind == "bgr" else img[:, :, 1].copy()))
    prof = check_batch(det, oracle, named)
    assert int(prof[SLOT_REFINES]) > 0 and int(prof[SLOT_REDUCE_ITERS]) > 0, prof
    assert all(n > 0 for n in rect_sizes(prof)), rect_sizes(prof)
    assert int(prof[SLOT_SEEDS_TO_RECT]) > 0


@pytest.mark.parametrize("name", ["rings_vga", "saw30", "saw45", "bar_vga"])
def test_long_regions(det, oracle, name):
    """regions of thousands of points: the compaction moves points across many 32-point chunks, and past the shared-memory list"""
    prof = check_batch(det, oracle, [(name, frames()[name]), ("c3", ordinary(320, 640, 480)[:, :, 1].copy())])
    assert rect_sizes(prof)[2] > 0


def test_small_frames(det, oracle):
    """QVGA frames: short regions whose lists end inside the first or second 32-point chunk"""
    named = [("qvga_%d" % s, ordinary(330 + s, 320, 240)) for s in range(4)]
    prof = check_batch(det, oracle, named)
    assert rect_sizes(prof)[0] > 0 and rect_sizes(prof)[1] > 0
