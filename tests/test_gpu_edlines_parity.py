"""GPU parity of the EDLines line detector (cs_detect_lines, use_LSD = 0: the class default of line_lbd_detect,
line_lbd_allclass.cpp:121) against the CPU oracle's restatement of BinaryDescriptor / EDLineDetector.

Integer stages (blur, Sobel maps, gradient / direction maps, anchors in scan order, edge map after smart routing) must be
bit-exact; the fitted segments are float32 and must be identical."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()      # use_LSD = False, line_length_thres = 50: the constructor defaults
    assert d.use_LSD is False
    return d


def _check_frame(det, oracle, img, frame, thres):
    ref = oracle.edl_detect(img, thres, want_stages=True)
    h, w = img.shape[:2]
    dbg = det.debug_frame_edlines(w, h, frame)
    for k in ("blur", "dx", "dy", "g", "dir"):
        np.testing.assert_array_equal(dbg[k], ref["stages"][k], err_msg=k)
    np.testing.assert_array_equal(dbg["anchors"], ref["stages"]["anchors"])
    np.testing.assert_array_equal(dbg["edge"], ref["stages"]["edge"])
    assert len(dbg["raw_lines"]) == len(ref["raw_lines"])
    np.testing.assert_array_equal(dbg["raw_lines"], ref["raw_lines"])
    return ref


def test_fixture_frames(det, oracle, fixture_a, fixture_b):
    imgs = [fixture_b["frames"][i][0] for i in (0, 17, 40)]
    lines = det.detect_filter_lines_batch(np.stack(imgs))
    for f, img in enumerate(imgs):
        ref = _check_frame(det, oracle, img, f, 50.0)
        np.testing.assert_array_equal(lines[f], ref["lines"])
    one = det.detect_filter_lines(fixture_a["img"])
    ref = _check_frame(det, oracle, fixture_a["img"], 0, 50.0)
    np.testing.assert_array_equal(one, ref["lines"])
    assert len(one) > 5


def test_short_threshold_synthetic_gray_and_flat(det, oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    d = cs.line_lbd_detect(context=det._ctx)
    d.line_length_thres = 15
    imgs, Ts, boxes, lines, K = S.make_batch(43, 4, 640, 480, 3)
    out = d.detect_filter_lines_batch(imgs)
    total = 0
    for f in range(4):
        ref = _check_frame(d, oracle, imgs[f], f, 15.0)
        np.testing.assert_array_equal(out[f], ref["lines"])
        total += len(out[f])
    assert total > 10
    gray = np.ascontiguousarray(imgs[:, :, :, 1])
    out = d.detect_filter_lines_batch(gray)
    for f in range(4):
        np.testing.assert_array_equal(out[f], oracle.edl_detect(gray[f], 15.0)["lines"])
    flat = np.full((1, 240, 320, 3), 90, np.uint8)
    assert len(d.detect_filter_lines_batch(flat)[0]) == 0
    # odd sizes exercise the borders of the scan grid and of the routing walk
    rng = np.random.RandomState(5)
    odd = np.kron(rng.randint(0, 255, (9, 13)).astype(np.uint8), np.ones((23, 19), np.uint8))[:203, :241]
    got = d.detect_filter_lines(odd)
    ref = _check_frame(d, oracle, odd, 0, 15.0)
    np.testing.assert_array_equal(got, ref["lines"])
    assert len(got) > 5


def test_sequence_frames(det, oracle, fixture_b):
    """Every frame of the shipped object_slam sequence (object_slam/data/raw_imgs), one batch."""
    imgs = np.stack([fr[0] for fr in fixture_b["frames"]])
    out = det.detect_filter_lines_batch(imgs)
    for f in range(len(imgs)):
        ref = oracle.edl_detect(imgs[f], 50.0)
        np.testing.assert_array_equal(out[f], ref["lines"], err_msg="frame %d" % f)


def test_online_mode_with_edlines(det, oracle):
    """cs_detect_frames_batch with the EDLines flavour == cs_detect_lines_batch followed by cs_detect_cuboids_batch == oracle."""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    F = 4
    imgs, Ts, boxes, _, K = S.make_batch(53, F, 640, 480, 3, poisson=True)
    ctx = cs.Context(0, 640, 480, F, 16, 2048)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    d = cs.line_lbd_detect(context=det._ctx)
    d.line_length_thres = 15
    lp = d.params()
    assert lp.use_LSD == 0
    out1, cnt1 = ctx.detect_frames_host(imgs, Ts, boxes, lp, p)
    out1, cnt1 = out1.copy(), cnt1.copy()
    lines = d.detect_filter_lines_batch(imgs)
    out2, cnt2 = ctx.detect_batch_host(imgs, Ts, boxes, [l.astype(np.float64) for l in lines], p)
    np.testing.assert_array_equal(cnt1, cnt2)
    assert out1.tobytes() == out2.tobytes()
    o = 0
    for f in range(F):
        rl = oracle.edl_detect(imgs[f], 15.0)["lines"].astype(np.float64)
        ref = oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], rl, oracle.default_params(max_cuboid_num=2))
        for b in range(len(boxes[f])):
            assert cnt1[o] == len(ref["cuboids"][b])
            for k in range(cnt1[o]):
                assert int(out1[o, k]["proposal_index"]) == int(ref["cuboids"][b][k]["proposal_index"])
                assert abs(float(out1[o, k]["normalized_error"]) - float(ref["cuboids"][b][k]["normalized_error"])) < 1e-9
            o += 1
    ctx.close()


# ---- shapes, strides and the three routing regimes ----------------------------------------------------------------------------------

SM_NODES = 32766   # walk-graph nodes k_ed_route keeps in shared memory (cs_edlines.cu ed_sm_nodes)


def routing_regime(oracle, img):
    """Which of the three routing paths a frame takes, from the oracle's gradient map: the walk graph has one node per pixel with g > 0;
    up to SM_NODES it is walked in shared memory, up to w * h / 2 in HBM, beyond that k_ed_route_fit routes on the pixel maps."""
    g = oracle.edl_detect(img, 15.0, want_stages=True)["stages"]["g"]
    n = int((g > 0).sum())
    return "shared" if n <= SM_NODES else "hbm" if n <= g.size // 2 else "pixel_map"


@pytest.fixture(scope="module")
def det15(det):
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(context=det._ctx)
    d.line_length_thres = 15
    return d


def test_all_three_routing_regimes_in_one_batch(det15, oracle):
    """A batch whose frames take the three routing paths side by side (per-frame redo flags and graph offsets), then each regime alone,
    stage by stage; the regimes are asserted from the oracle's g map.  The 10-pixel checkerboard (pixel-map routing) has no segment."""
    from test_oracle_ref_edlines import dense_frames
    from test_oracle_ref_lsd import CHECKERBOARDS, checkerboard
    frames = dense_frames()
    board = np.repeat(checkerboard(*CHECKERBOARDS["vga_10px"])[:, :, None], 3, 2)
    batch = np.stack([frames["checkerboard_window"], frames["room"], frames["room_noise_band"], board])
    assert [routing_regime(oracle, img) for img in batch] == ["pixel_map", "shared", "hbm", "pixel_map"]
    for imgs in (batch, batch[1:2], batch[2:3], batch[0:1]):
        out = det15.detect_filter_lines_batch(imgs)
        for f in range(len(imgs)):
            ref = _check_frame(det15, oracle, imgs[f], f, 15.0)
            np.testing.assert_array_equal(out[f], ref["lines"])
    assert min(len(oracle.edl_detect(img, 15.0)["lines"]) for img in batch[:3]) >= 30


def test_kitti_and_sxga_bgr_batches(det15, oracle):
    """KITTI 1242 x 375 BGR (rows not a multiple of 16 bytes: byte-staged front end) and 1280 x 960 BGR (TMA-staged)."""
    from cube_slam_b200 import synthetic as S
    for imgs in (S.make_batch(91, 3, 1242, 375, 3, kind="kitti")[0], S.make_batch(92, 2, 1280, 960, 3)[0]):
        out = det15.detect_filter_lines_batch(imgs)
        for f in range(len(imgs)):
            ref = _check_frame(det15, oracle, imgs[f], f, 15.0)
            np.testing.assert_array_equal(out[f], ref["lines"])
            assert len(out[f]) > 20


@pytest.mark.parametrize("channels", [1, 3], ids=["gray", "bgr"])
@pytest.mark.parametrize("shape", [(97, 211), (61, 64), (200, 333), (203, 241), (3, 3), (4, 5), (7, 9)],
                         ids=lambda s: "%dx%d" % s)
def test_odd_size_batches(det15, oracle, shape, channels):
    """Batches of three frames at ragged sizes (test_gpu_lsd_parity.py's shape matrix); ed_run rejects frames under 8 x 8."""
    import cube_slam_b200 as cs
    from test_gpu_lsd_parity import odd_size_batch
    imgs = odd_size_batch(shape[0], shape[1], channels)
    if min(shape) < 8:
        with pytest.raises(cs.CubeSlamError, match="INVALID_ARG"):
            det15.detect_filter_lines_batch(imgs)
        return
    out = det15.detect_filter_lines_batch(imgs)
    for f in range(len(imgs)):
        ref = _check_frame(det15, oracle, imgs[f], f, 15.0)
        np.testing.assert_array_equal(out[f], ref["lines"])
