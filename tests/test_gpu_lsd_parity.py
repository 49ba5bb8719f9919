"""GPU parity of the LSD line detector (cs_detect_lines) against the CPU oracle's restatement of line_lbd's LSD path.

Streaming stages (blur, resize, gradient modulus / angle, pseudo-ordering) must be bit-exact; the detected segments are
float32 and must be identical (the only non-IEEE operations are double cos/sin/log of CUDA vs glibc, <= 2 ulp before the
float rounding)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True              # object_slam/src/main_obj.cpp:365
    d.line_length_thres = 15      # :366
    return d


def _check_frame(det, oracle, img, frame=0, cap=8192):
    ref = oracle.lsd_detect(img, 15.0, cap=cap, want_stages=True)
    dbg = det.debug_frame(frame, cap)
    np.testing.assert_array_equal(dbg["scaled"], ref["stages"]["scaled"])
    np.testing.assert_array_equal(dbg["modgrad"][:-1, :-1], ref["stages"]["modgrad"][:-1, :-1])
    np.testing.assert_array_equal(dbg["angles"], ref["stages"]["angles"])
    # the GPU list keeps only pixels with a defined angle (the seed loop skips the others): same order otherwise
    rl = ref["stages"]["list"]
    np.testing.assert_array_equal(dbg["list"], rl[ref["stages"]["angles"].ravel()[rl] != -1024.0])
    assert len(dbg["raw_lines"]) == len(ref["raw_lines"])
    np.testing.assert_array_equal(dbg["raw_lines"], ref["raw_lines"])
    return ref


def test_fixture_frames(det, oracle, fixture_a, fixture_b):
    imgs = [fixture_b["frames"][i][0] for i in (0, 17, 40)]
    lines = det.detect_filter_lines_batch(np.stack(imgs))
    for f, img in enumerate(imgs):
        ref = _check_frame(det, oracle, img, f)
        np.testing.assert_array_equal(lines[f], ref["lines"])
        assert len(lines[f]) > 5
    one = det.detect_filter_lines(fixture_a["img"])
    ref = _check_frame(det, oracle, fixture_a["img"], 0)
    np.testing.assert_array_equal(one, ref["lines"])


def test_synthetic_and_gray_input(det, oracle):
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, lines, K = S.make_batch(41, 4, 640, 480, 3)
    out = det.detect_filter_lines_batch(imgs)
    for f in range(4):
        ref = oracle.lsd_detect(imgs[f], 15.0)
        np.testing.assert_array_equal(out[f], ref["lines"])
    gray = np.ascontiguousarray(imgs[:, :, :, 1])
    out = det.detect_filter_lines_batch(gray)
    for f in range(4):
        np.testing.assert_array_equal(out[f], oracle.lsd_detect(gray[f], 15.0)["lines"])
    # a flat image has no gradient above the threshold: no lines, no crash
    flat = np.full((1, 240, 320, 3), 90, np.uint8)
    assert len(det.detect_filter_lines_batch(flat)[0]) == 0


def test_more_octaves_give_the_same_lines_and_bad_counts_fail_loudly(det, oracle, fixture_a):
    """filter_lines keeps octave 0 only (line_lbd_allclass.cpp:200-207) and octave 0 does not depend on the higher octaves: a detector built
    with 2 or 3 octaves returns the one-octave matrix (the compiled reference does: tests/test_oracle_ref_octaves.py)."""
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(context=det._ctx)
    d.use_LSD = True
    d.line_length_thres = 15
    want = oracle.lsd_detect(fixture_a["img"], 15.0)["lines"]
    for n in (2, 3):
        d.numoctaves_ = n
        np.testing.assert_array_equal(d.detect_filter_lines(fixture_a["img"]), want)
    d.numoctaves_ = 0
    with pytest.raises(cs.CubeSlamError, match="INVALID_ARG"):
        d.detect_filter_lines(np.zeros((64, 64), np.uint8))


def test_lines_feed_detect_cuboid(det, oracle, fixture_b):
    """The online path of object_slam: line_lbd lines -> detect_cuboid (main_obj.cpp:424-450), frame 0 (no sampling)."""
    import cube_slam_b200 as cs
    img, boxes = fixture_b["frames"][0]
    lines = det.detect_filter_lines(img)
    d3 = cs.detect_3d_cuboid()
    d3.set_calibration(fixture_b["K"])
    d3.nominal_skew_ratio = 2  # main_obj.cpp:360
    got = d3.detect_cuboid(img, fixture_b["T"], boxes, lines.astype(np.float64))
    ref_lines = oracle.lsd_detect(img, 15.0)["lines"].astype(np.float64)
    ref = oracle.detect_cuboid(img, fixture_b["K"], fixture_b["T"], boxes, ref_lines, oracle.default_params(nominal_skew_ratio=2))
    assert len(got) == len(boxes) == 1
    assert got[0][0].proposal_index == int(ref["cuboids"][0][0]["proposal_index"])
    assert abs(got[0][0].normalized_error - float(ref["cuboids"][0][0]["normalized_error"])) < 1e-9


def test_object_slam_sequence_parity(det, oracle, fixture_b):
    """north_star: best-proposal-index parity on the shipped object_slam/data sequence, online mode
    (object_slam/src/main_obj.cpp:392-450): LSD lines (length > 15) -> detect_cuboid with nominal_skew_ratio 2,
    roll/pitch sampling on every frame but the first, all frames at the first frame's pose."""
    import cube_slam_b200 as cs
    frames = fixture_b["frames"]
    K, T = fixture_b["K"], fixture_b["T"]
    imgs = np.stack([f[0] for f in frames])
    gpu_lines = det.detect_filter_lines_batch(imgs)
    ctx = cs.Context(0, 640, 480, len(frames), 8, 4096)
    ctx.set_calibration(K)
    n_checked = 0
    for sampling, ids in ((0, [0]), (1, list(range(1, len(frames))))):
        p = cs.default_params(whether_sample_cam_roll_pitch=sampling, nominal_skew_ratio=2.0)
        out, counts = ctx.detect_batch_host(imgs[ids], np.stack([T] * len(ids)), [frames[i][1] for i in ids],
                                            [gpu_lines[i].astype(np.float64) for i in ids], p)
        o = 0
        for i in ids:
            ref_lines = oracle.lsd_detect(frames[i][0], 15.0)["lines"]
            np.testing.assert_array_equal(gpu_lines[i], ref_lines)
            ref = oracle.detect_cuboid(frames[i][0], K, T, frames[i][1], ref_lines.astype(np.float64),
                                       oracle.default_params(whether_sample_cam_roll_pitch=sampling, nominal_skew_ratio=2.0))
            for b in range(len(frames[i][1])):
                assert counts[o] == len(ref["cuboids"][b]), (i, b)
                if counts[o]:
                    g, r = out[o, 0], ref["cuboids"][b][0]
                    assert int(g["proposal_index"]) == int(r["proposal_index"]), i
                    assert abs(float(g["normalized_error"]) - float(r["normalized_error"])) < 1e-4
                    np.testing.assert_allclose(g["pos"], r["pos"], rtol=1e-9, atol=1e-9)
                    np.testing.assert_array_equal(g["box_corners_2d"], r["box_corners_2d"])
                    n_checked += 1
                o += 1
    assert n_checked >= 45  # 51 of the 58 frames carry a box
    ctx.close()


def test_online_batch_equals_two_calls(det, oracle):
    """cs_detect_frames_batch (lines stay on the device) == cs_detect_lines_batch followed by cs_detect_cuboids_batch."""
    _online_equals_two_calls(det, oracle, 51, 5, 640, 480, 3, "indoor")


def test_online_batch_equals_two_calls_at_kitti_size(det, oracle):
    """The same at the KITTI size with 8 boxes a frame, as bench.py's c4 runs the online path."""
    _online_equals_two_calls(det, oracle, 52, 3, 1242, 375, 8, "kitti")


def _online_equals_two_calls(det, oracle, seed, F, w, h, n_boxes, kind):
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, _, K = S.make_batch(seed, F, w, h, n_boxes, kind=kind, poisson=(kind == "indoor"))
    ctx = cs.Context(0, w, h, F, 16, 2048)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    lp = det.params()
    out1, cnt1 = ctx.detect_frames_host(imgs, Ts, boxes, lp, p)
    out1, cnt1 = out1.copy(), cnt1.copy()
    lines = det.detect_filter_lines_batch(imgs)
    out2, cnt2 = ctx.detect_batch_host(imgs, Ts, boxes, [l.astype(np.float64) for l in lines], p)
    np.testing.assert_array_equal(cnt1, cnt2)
    assert out1.tobytes() == out2.tobytes()
    # and both equal the oracle's two-stage result
    from test_gpu_cuboid_parity import _compare_box
    o = 0
    n_knife = 0
    for f in range(F):
        rl = oracle.lsd_detect(imgs[f], float(lp.line_length_thres))["lines"].astype(np.float64)

        def redo(cut_flip=-1, f=f, rl=rl):
            return oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], rl, oracle.default_params(max_cuboid_num=2), cut_flip=cut_flip)
        ref = redo()
        for b in range(len(boxes[f])):
            n_knife += _compare_box(oracle, out1[o], cnt1[o], ref, b, redo)
            o += 1
    assert n_knife == 0
    ctx.close()


def test_sequence_against_the_shipped_matlab_cuboids(det, fixture_b):
    """The CUDA path end to end (cs_detect_lines -> cs_detect_cuboids_batch) against the cuboids the reference's authors ship for this
    sequence (object_slam/data/detect_cuboids_saved.txt, MATLAB, local ground frame) at the per-frame poses of pop_cam_poses_saved.txt.
    A soft check (another Canny / DT in MATLAB): same cuboid up to the sampling grid; tests/test_oracle_matlab_crosscheck.py is the CPU twin."""
    import os
    import cube_slam_b200 as cs
    from scipy.spatial.transform import Rotation
    from conftest import GOLD
    fb = os.path.join(GOLD, "fixture_b")
    pop = np.loadtxt(os.path.join(fb, "pop_cam_poses_saved.txt"))
    sav = np.loadtxt(os.path.join(fb, "detect_cuboids_saved.txt"))
    ids = [int(r[0]) for r in sav]
    frames = fixture_b["frames"]
    imgs = np.stack([frames[i][0] for i in ids])
    Ts = []
    for i in ids:
        T = np.eye(4)
        T[:3, :3] = Rotation.from_quat(pop[i][4:8]).as_matrix()
        T[:3, 3] = pop[i][1:4]
        Ts.append(T)
    lines = det.detect_filter_lines_batch(imgs)
    ctx = cs.Context(0, 640, 480, len(ids), 8, 4096)
    ctx.set_calibration(fixture_b["K"])
    out, counts = ctx.detect_batch_host(imgs, np.stack(Ts), [frames[i][1] for i in ids], [l.astype(np.float64) for l in lines],
                                        cs.default_params(nominal_skew_ratio=2.0))
    assert list(counts) == [1] * len(ids)
    rows = []
    for k, row in enumerate(sav):
        c = out[k, 0]
        d_pos = float(np.linalg.norm(np.array(c["pos"]) - row[1:4]))
        d_yaw = (float(c["rotY"]) - row[4] + np.pi / 4) % (np.pi / 2) - np.pi / 4
        swapped = abs(((float(c["rotY"]) - row[4] + np.pi / 2) % np.pi) - np.pi / 2) > np.pi / 4
        sc = np.array(c["scale"])[[1, 0, 2]] if swapped else np.array(c["scale"])
        rows.append((d_pos, abs(d_yaw), float((np.abs(sc - row[5:8]) / row[5:8]).max())))
    rows = np.array(rows)
    step = 6.0 / 180 * np.pi
    assert np.median(rows[:, 0]) < 0.05 and np.median(rows[:, 1]) < 0.02 and np.median(rows[:, 2]) < 0.15
    good = (rows[:, 0] < 0.15) & (rows[:, 1] < 2.1 * step) & (rows[:, 2] < 0.3)
    assert good.sum() >= 42, int(good.sum())     # 43 of 51, the oracle's own count (tests/test_oracle_matlab_crosscheck.py)
    ctx.close()


def test_seed_loop_on_a_giant_region(det, oracle):
    """A smooth ramp is one line-support region far larger than the shared-memory part of the region list (it spills to HBM):
    result unchanged."""
    ramp = np.tile((np.arange(640) * 0.35).astype(np.uint8)[None, :], (480, 1))
    ramp = np.ascontiguousarray(ramp)
    got = det.detect_filter_lines_batch(ramp[None])
    _, redo = det.seed_loop_stats(1)
    ref = oracle.lsd_detect(ramp, 15.0)
    np.testing.assert_array_equal(got[0], ref["lines"])
    np.testing.assert_array_equal(det.debug_frame(0)["raw_lines"], ref["raw_lines"])


def test_tma_staged_tiles_equal_byte_staged_tiles(det, oracle):
    """k_lsd_blur<true> / k_ed_front<true> (BGR tiles fetched by the copy engine, the default on 640 / 1280 wide BGR frames) against the
    byte-load instantiations (cs_set_profiling bit 8): identical segments for both detectors, and equal to the oracle."""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(71, 3, 640, 480, 3)[0]
    for use_lsd, ref_fn in ((True, oracle.lsd_detect), (False, oracle.edl_detect)):
        d = cs.line_lbd_detect(context=det._ctx)
        d.use_LSD = use_lsd
        d.line_length_thres = 15
        got = {}
        for flags in (0, 256):
            det._ctx.set_profiling(flags)
            got[flags] = d.detect_filter_lines_batch(imgs)
        det._ctx.set_profiling(0)
        for f in range(3):
            np.testing.assert_array_equal(got[0][f], got[256][f])
            np.testing.assert_array_equal(got[0][f], ref_fn(imgs[f], 15.0)["lines"])


# ---- shapes, strides and densities where the kernels' indexing can go wrong ----------------------------------------------------------

def test_kitti_and_sxga_bgr_batches(det, oracle):
    """KITTI 1242 x 375 BGR (rows of 3 726 bytes, not a multiple of 16: the byte-staged blur) and 1280 x 960 BGR (the TMA-staged blur), the
    frame shapes of bench.py's c4 and c5, stage by stage."""
    from cube_slam_b200 import synthetic as S
    for imgs in (S.make_batch(81, 3, 1242, 375, 3, kind="kitti")[0], S.make_batch(82, 2, 1280, 960, 3)[0]):
        lines = det.detect_filter_lines_batch(imgs)
        for f in range(len(imgs)):
            ref = _check_frame(det, oracle, imgs[f], f)
            np.testing.assert_array_equal(lines[f], ref["lines"])
            assert len(lines[f]) > 20


ODD_SHAPES = [(97, 211), (61, 64), (200, 333), (203, 241), (3, 3), (4, 5), (7, 9)]


def odd_size_batch(h, w, channels):
    """Three h x w frames: blocks of random levels (long straight edges, corners), a step edge with noise, pure noise."""
    from test_oracle_ref_lsd import tiny_frame
    rng = np.random.default_rng(h * 1000 + w + channels)
    c = (channels,) if channels == 3 else ()
    blocks = np.kron(rng.integers(0, 256, (h // 7 + 1, w // 9 + 1) + c), np.ones((7, 9) + (1,) * len(c), np.int64))[:h, :w]
    step = tiny_frame(h, w, h + w)
    if channels == 3:
        step = np.stack([step, step // 2 + 40, 255 - step], 2)
    noise = rng.integers(0, 256, (h, w) + c)
    return np.ascontiguousarray(np.stack([blocks, step, noise]).astype(np.uint8))


def test_odd_shapes_cover_unaligned_used_bitmaps():
    """The 0.8-scaled frame of some of these sizes is not a whole number of 32-pixel words, so frames 1 and 2 of a batch start mid-word in
    the seed loop's used bitmap, and its width is not a multiple of 32 (nor of the 128 pixels a seed-scan step reads)."""
    scaled = [(int(np.rint(0.8 * h)), int(np.rint(0.8 * w))) for h, w in ODD_SHAPES]
    assert any((H * W) % 32 for H, W in scaled) and all(W % 32 for H, W in scaled)


@pytest.mark.parametrize("channels", [1, 3], ids=["gray", "bgr"])
@pytest.mark.parametrize("shape", ODD_SHAPES, ids=["%dx%d" % s for s in ODD_SHAPES])
def test_odd_size_batches(det, oracle, shape, channels):
    imgs = odd_size_batch(shape[0], shape[1], channels)
    lines = det.detect_filter_lines_batch(imgs)
    for f in range(len(imgs)):
        ref = _check_frame(det, oracle, imgs[f], f)
        np.testing.assert_array_equal(lines[f], ref["lines"])


def test_frames_too_small_for_lsd(det):
    """lrint(0.8 * w) or lrint(0.8 * h) below 2: no gradient can be computed; the call fails instead of reading outside the frame."""
    import cube_slam_b200 as cs
    for shape in [(9, 1), (1, 9), (1, 1)]:
        with pytest.raises(cs.CubeSlamError, match="INVALID_ARG"):
            det.detect_filter_lines_batch(np.full((3,) + shape, 100, np.uint8))


def test_rectangles_disc_and_ragged_noise(det, oracle):
    """The frames tests/test_oracle_ref_lsd.py pins to the compiled reference: sharp rectangles (the reduce-radius and refine branches), a
    blurred disc (regions cut by the density test), noise at ragged sizes and a constant frame."""
    from test_oracle_ref_lsd import odd_and_degenerate_frames
    for name, img in odd_and_degenerate_frames().items():
        got = det.detect_filter_lines(img)
        ref = _check_frame(det, oracle, img, 0)
        np.testing.assert_array_equal(got, ref["lines"], err_msg=name)


def detect_strided(d, imgs, pad, cap=4096):
    """cs_detect_lines_batch on frames whose rows are `pad` bytes longer than width x channels (a cv::Mat ROI passed through the shim); the
    padding holds bytes that must not be read."""
    import ctypes as C
    from cube_slam_b200 import _lib
    F, H, W = imgs.shape[:3]
    ch = imgs.shape[3] if imgs.ndim == 4 else 1
    row = W * ch
    buf = np.full((F, H, row + pad), 0xA5, np.uint8)
    buf[:, :, :row] = imgs.reshape(F, H, row)
    out = np.zeros((F, cap, 4), np.float32)
    n = np.zeros(F, np.int32)
    p = d.params()
    rc = d._ctx.L.cs_detect_lines_batch(d._ctx.h, buf.ctypes.data, F, W, H, row + pad, ch, C.byref(p), _lib.ptr(out, C.c_float), cap,
                                        _lib.ptr(n, C.c_int32))
    assert rc == 0, d._ctx.L.cs_last_error(d._ctx.h).decode()
    return [out[f, :n[f]].copy() for f in range(F)]


def row_pads(row):
    """a pad that keeps rows 16-byte aligned and one that breaks the alignment"""
    aligned = (-row) % 16 or 16
    return aligned, next(p for p in (3, 5) if (row + p) % 16)


@pytest.mark.parametrize("use_lsd", [True, False], ids=["lsd", "edlines"])
def test_padded_rows_equal_packed_rows(det, oracle, use_lsd):
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    d = cs.line_lbd_detect(context=det._ctx)
    d.use_LSD = use_lsd
    d.line_length_thres = 15
    ref_fn = oracle.lsd_detect if use_lsd else oracle.edl_detect
    vga = S.make_batch(84, 3, 640, 480, 3)[0]
    for imgs in (S.make_batch(83, 3, 1242, 375, 3, kind="kitti")[0], vga, np.ascontiguousarray(vga[:, :, :, 1]), odd_size_batch(97, 211, 3)):
        packed = d.detect_filter_lines_batch(imgs)
        for f in range(len(imgs)):
            np.testing.assert_array_equal(packed[f], ref_fn(imgs[f], 15.0)["lines"])
        row = imgs.shape[2] * (imgs.shape[3] if imgs.ndim == 4 else 1)
        for pad in row_pads(row):
            got = detect_strided(d, imgs, pad)
            for f in range(len(imgs)):
                np.testing.assert_array_equal(got[f], packed[f], err_msg="row %d + pad %d, frame %d" % (row, pad, f))


def checkerboard_batch(name):
    """The checkerboard first, then a synthetic frame of the same size: the grown candidate buffer serves both."""
    from cube_slam_b200 import synthetic as S
    from test_oracle_ref_lsd import CHECKERBOARDS, checkerboard
    w, h = CHECKERBOARDS[name][:2]
    board = checkerboard(*CHECKERBOARDS[name])
    if w == 1280:   # BGR: the TMA-staged blur
        return np.stack([np.repeat(board[:, :, None], 3, 2), S.make_batch(85, 1, w, h, 3)[0][0]])
    return np.stack([board, S.make_batch(85, 1, w, h, 3)[0][0][:, :, 1]])


@pytest.mark.parametrize("name", ["vga_10px", "sxga_12px_noisy"])
def test_checkerboards_beyond_the_candidate_buffer(oracle, name):
    """More candidate rectangles in a frame than the seed loop's initial hand-off buffer holds (2 048): the synchronous entry point grows the
    buffer and runs again.  Every raw segment is the oracle's, and the filtered matrix is the reference's (empty: no segment of a
    checkerboard is longer than 15 pixels).  A fresh context, so that the first run overflows."""
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    cap = 16384
    imgs = checkerboard_batch(name)
    lines = d.detect_filter_lines_batch(imgs, cap=cap)
    for f in range(len(imgs)):
        ref = _check_frame(d, oracle, imgs[f], f, cap)
        np.testing.assert_array_equal(lines[f], ref["lines"])
    assert len(d.debug_frame(0, cap)["raw_lines"]) > 2048 and lines[0].shape == (0, 4) and len(lines[1]) > 20
    if oracle.ref_detect_filter_lines_available():
        np.testing.assert_array_equal(lines[0], oracle.ref_detect_filter_lines(imgs[0], True, 15.0, cap=cap))
    # again on the grown buffer, frames swapped
    again = d.detect_filter_lines_batch(imgs[::-1].copy(), cap=cap)
    np.testing.assert_array_equal(again[0], lines[1])
    np.testing.assert_array_equal(again[1], lines[0])
    d._ctx.close()


def test_descriptor_path_on_a_checkerboard(oracle):
    """cs_detect_descrip_lines with use_LSD on the 640 x 480 checkerboard (more than 2 048 candidate rectangles), no length filter: every
    octave-0 key line and its descriptor."""
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    img = checkerboard_batch("vga_10px")[0]
    lines, desc = d.detect_descrip_lines(img, cap=8192, as_mat=True)
    want = oracle.lbd_detect_keylines(img, True, -1.0)
    assert len(lines) == len(want) > 2048
    np.testing.assert_array_equal(lines, np.stack([want["sx"], want["sy"], want["ex"], want["ey"]], 1))
    np.testing.assert_array_equal(desc, oracle.lbd_compute(img, want))
    d._ctx.close()


def test_online_path_names_the_candidate_limit(det, oracle):
    """cs_detect_frames_batch does not add a host sync to re-run the detector: a batch with a frame of more candidate rectangles than the
    buffer holds fails with an error that names that limit (not max_lines_per_frame).  A synchronous detector call on the same context
    grows the buffer; the batch then runs and equals the two-call path."""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, _, K = S.make_batch(86, 2, 640, 480, 2)
    imgs[0] = np.repeat(checkerboard_batch("vga_10px")[0][:, :, None], 3, 2)
    ctx = cs.Context(0, 640, 480, 2, 16, 2048)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    lp = det.params()
    assert lp.use_LSD == 1
    with pytest.raises(cs.CubeSlamError, match="CAPACITY.*LSD candidate regions, more than the 2048 per frame"):
        ctx.detect_frames_host(imgs, Ts, boxes, lp, p)
    with pytest.raises(cs.CubeSlamError, match="CAPACITY.*LSD candidate regions"):   # still too small: nothing grew it
        ctx.detect_frames_host(imgs, Ts, boxes, lp, p)
    grow = cs.line_lbd_detect(context=ctx)
    grow.use_LSD = True
    grow.line_length_thres = 15
    np.testing.assert_array_equal(grow.detect_filter_lines_batch(imgs)[0], oracle.lsd_detect(imgs[0], 15.0)["lines"])
    out1, cnt1 = ctx.detect_frames_host(imgs, Ts, boxes, lp, p)
    out1, cnt1 = out1.copy(), cnt1.copy()
    lines = det.detect_filter_lines_batch(imgs)
    np.testing.assert_array_equal(lines[0], oracle.lsd_detect(imgs[0], 15.0)["lines"])
    out2, cnt2 = ctx.detect_batch_host(imgs, Ts, boxes, [l.astype(np.float64) for l in lines], p)
    np.testing.assert_array_equal(cnt1, cnt2)
    assert out1.tobytes() == out2.tobytes()
    ctx.close()
