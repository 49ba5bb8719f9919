"""The LSD seed loop on regions past the shared-memory part of its region list, on the GPU.

k_lsd_grow_seq keeps the first LSD_SEQ_SCAP = 2 048 entries of a seed's region list in shared memory and the rest in the frame's HBM arena
slice (LsdReg::get / put); refine's re-grow starts at the first pass's size, and reduce_region_radius swaps entries anywhere in the list.
The frames of tests/test_oracle_ref_lsd_large_regions.py reach that path (their regimes are asserted there, on the CPU, through the oracle's
statistics).  Here every one goes through cs_detect_lines_batch alone and in batches that mix it with ordinary frames, through both
instantiations of the seed loop: the profiling one (cs_set_profiling bit 0), whose counters of seeds, first-pass pixels and seeds whose list
outgrew shared memory must equal the oracle's counts exactly, and the production one.  Stage planes, raw segments and the filtered matrix
equal the oracle's bit for bit."""
import ctypes as C

import numpy as np
import pytest

from test_oracle_ref_lsd_large_regions import SPILL, frames

pytestmark = pytest.mark.gpu

SLOT_SEEDS, SLOT_FIRST_PIXELS, SLOT_SPILLED = 4, 7, 8   # cs_debug_lsd_prof
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


@pytest.fixture(scope="module")
def ref(oracle):
    """the oracle's stages, segments and statistics of every frame, computed once"""
    cache = {}

    def get(name, img):
        if name not in cache:
            r = oracle.lsd_detect(img, 15.0, cap=CAP, want_stages=True)
            r["stats"] = oracle.lsd_stats(img, cap=CAP)[1]
            cache[name] = r
        return cache[name]
    return get


def ordinary(seed, w, h):
    """a benchmark-like synthetic frame (bench.py's c3 generator)"""
    from cube_slam_b200 import synthetic as S
    return S.make_batch(seed, 1, w, h, 3, kind="indoor", poisson=True)[0][0]


def run(det, imgs, profiled):
    """one cs_detect_lines_batch; with profiled, through k_lsd_grow_seq<true> with the counters reset just before -> (lines, counters)"""
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


def check_batch(det, ref, named):
    """named: [(name, frame)] of one size and channel count -> per-frame oracle results; asserts both instantiations against them"""
    imgs = np.stack([img for _, img in named])
    refs = [ref(name, img) for name, img in named]
    for profiled in (True, False):
        lines, prof = run(det, imgs, profiled)
        if profiled:
            for slot, key in ((SLOT_SEEDS, "seeds"), (SLOT_FIRST_PIXELS, "first_sum"), (SLOT_SPILLED, "n_all_spill")):
                assert int(prof[slot]) == sum(r["stats"][key] for r in refs), ([n for n, _ in named], key, int(prof[slot]))
        else:
            assert not prof[[SLOT_SEEDS, SLOT_FIRST_PIXELS, SLOT_SPILLED]].any()   # the production kernel counts nothing
        for f, ((name, _), r) in enumerate(zip(named, refs)):
            dbg = det.debug_frame(f, CAP)
            st = r["stages"]
            np.testing.assert_array_equal(dbg["scaled"], st["scaled"], err_msg=name)
            np.testing.assert_array_equal(dbg["modgrad"][:-1, :-1], st["modgrad"][:-1, :-1], err_msg=name)
            np.testing.assert_array_equal(dbg["angles"], st["angles"], err_msg=name)
            np.testing.assert_array_equal(dbg["list"], st["list"][st["angles"].ravel()[st["list"]] != -1024.0], err_msg=name)
            assert len(dbg["raw_lines"]) == len(r["raw_lines"]), (name, profiled)
            np.testing.assert_array_equal(dbg["raw_lines"], r["raw_lines"], err_msg="%s profiled=%s" % (name, profiled))
            np.testing.assert_array_equal(lines[f], r["lines"], err_msg="%s profiled=%s" % (name, profiled))
    return refs


def test_the_shared_memory_part_is_still_2048_entries(det):
    """The frames were searched for region lists of 2 047 / 2 048 / 2 049 entries: a seed loop with another LSD_SEQ_SCAP must fail here, not
    quietly test a boundary it no longer has.  k_lsd_grow_seq's dynamic shared memory is LSD_SEQ_SCAP * 4 + 96 * 8 bytes."""
    from cube_slam_b200 import _lib
    out = np.zeros(14, np.int32)
    det._ctx.check(det._ctx.L.cs_debug_lsd_occupancy(det._ctx.h, _lib.ptr(out, C.c_int32)))
    assert out[3] == SPILL * 4 + 96 * 8, out


@pytest.mark.parametrize("name", sorted(frames()))
def test_each_frame_alone(det, ref, name):
    img = frames()[name]
    (r,) = check_batch(det, ref, [(name, img)])
    assert len(r["raw_lines"]) > 0


def test_mixed_vga_gray_batch(det, ref):
    """ordinary frames around the giant ones: the frame after a spilling frame starts from its own arena slice"""
    F = frames()
    named = [("c3_a", ordinary(91, 640, 480)[:, :, 1].copy())] + [(n, F[n]) for n in ("rings_vga", "saw0", "saw30", "saw45")]
    named += [("c3_b", ordinary(92, 640, 480)[:, :, 1].copy()), ("saw90", F["saw90"]), ("bar_vga", F["bar_vga"]),
              ("c3_c", ordinary(93, 640, 480)[:, :, 1].copy())]
    refs = check_batch(det, ref, named)
    assert sum(r["stats"]["n_all_spill"] for r in refs) > 100


def test_mixed_vga_bgr_batch(det, ref):
    F = frames()
    rings_as_bgr = np.ascontiguousarray(np.repeat(F["rings_vga"][:, :, None], 3, 2))   # equal channels: the same gray frame
    named = [("c3_bgr_a", ordinary(94, 640, 480)), ("rings_vga_as_bgr", rings_as_bgr), ("c3_bgr_b", ordinary(95, 640, 480)),
             ("rings_vga_bgr", F["rings_vga_bgr"]), ("saw30_bgr", F["saw30_bgr"]), ("c3_bgr_c", ordinary(96, 640, 480))]
    check_batch(det, ref, named)


def test_mixed_sxga_batch(det, ref):
    """1280 x 960: rings whose re-grows start hundreds of times in HBM, the sawtooth with a 17 731-entry region, then an ordinary frame"""
    F = frames()
    named = [("rings_sxga", F["rings_sxga"]), ("saw20_sxga", F["saw20_sxga"]), ("sxga_c", ordinary(97, 1280, 960)[:, :, 1].copy())]
    refs = check_batch(det, ref, named)
    assert refs[0]["stats"]["regrow_past"] > 500


def test_exact_boundary_sizes_in_one_batch(det, ref):
    """first passes of 2 049 and 2 047 entries and a list of 2 047, with an ordinary frame of the same size between them"""
    F = frames()
    named = [("first_2049", F["first_2049"]), ("qvga_c", ordinary(98, 320, 240)[:, :, 1].copy()), ("first_2047", F["first_2047"]),
             ("n_all_2047", F["n_all_2047"])]
    refs = check_batch(det, ref, named)
    assert all(r["stats"][k] >= 1 for r, k in zip(refs, ("first_2049", "seeds", "first_2047", "n_all_2047")))
    # the 2 048-entry bar twice in one batch (a 96 x 320 frame)
    refs = check_batch(det, ref, [("first_2048", F["first_2048"]), ("first_2048_again", F["first_2048"])])
    assert refs[0]["stats"]["first_2048"] == 1
