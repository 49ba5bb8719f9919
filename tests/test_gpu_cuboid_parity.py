"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same inputs.

Bars (BASELINE.json north_star): bit-exact for integer / byte / index work (gray, Canny, chamfer DT,
merged line set, valid-proposal set, kept ids, best-proposal index), 1e-4 on normalised scores
(we assert far tighter: the only non-IEEE operations are CUDA's atan2/sin/cos, <= 2 ulp)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-4   # north_star tolerance on normalised scores
TIGHT = 1e-9       # what we actually expect


@pytest.fixture(scope="module")
def cs():
    import cube_slam_b200 as cs
    return cs


def _oracle_params(O, **kw):
    return O.default_params(**kw)


def _compare_cuboid(g, o, tight=TIGHT):
    assert int(g["proposal_index"]) == int(o["proposal_index"])
    assert int(g["height_sample_id"]) == int(o["height_sample_id"])
    # NaN on both sides where every proposal of a box has the same errors (the reference's normalisation divides 0 by 0): equal.
    # The same infinity on both sides where weight_vp_angle = -1 divides by 1 + w = 0: equal
    gn, on = float(g["normalized_error"]), float(o["normalized_error"])
    assert abs(gn - on) < SCORE_TOL or (np.isnan(gn) and np.isnan(on)) or (np.isinf(gn) and gn == on)
    np.testing.assert_allclose(g["normalized_error"], o["normalized_error"], rtol=0, atol=tight)
    np.testing.assert_allclose(g["combined_score"], o["combined_score"], rtol=1e-9, atol=tight)
    np.testing.assert_allclose(g["edge_distance_error"], o["edge_distance_error"], rtol=1e-12, atol=1e-12)
    assert float(g["edge_angle_error"]) == float(o["edge_angle_error"])  # same arithmetic on both sides: bit for bit
    np.testing.assert_array_equal(g["box_corners_2d"], o["box_corners_2d"])
    np.testing.assert_array_equal(g["box_config_type"], o["box_config_type"])
    np.testing.assert_allclose(g["pos"], o["pos"], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(g["scale"], o["scale"], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(g["rotY"], o["rotY"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(g["box_corners_3d_world"], o["box_corners_3d_world"], rtol=1e-9, atol=1e-9)
    np.testing.assert_array_equal(g["rect_detect_2d"], o["rect_detect_2d"])
    np.testing.assert_allclose(g["skew_ratio"], o["skew_ratio"], rtol=1e-9)
    assert float(g["down_expand_height"]) == float(o["down_expand_height"])
    np.testing.assert_allclose(g["camera_roll_delta"], o["camera_roll_delta"], atol=1e-15)
    np.testing.assert_allclose(g["camera_pitch_delta"], o["camera_pitch_delta"], atol=1e-15)


def _compare_box(oracle, got, n_got, ref, b, redo=None):
    """One box's cuboids against the oracle, strictly: the atan2 of the angle-error chain is defined arithmetically on both sides
    (cs_pmath.h / oracle/pmath.h), so even fuse_normalize_scores_v2's cut through pairs of mathematically equal angle errors
    (object_3d_util.cpp:504-520) falls the same way."""
    assert n_got == len(ref["cuboids"][b])
    for k in range(n_got):
        _compare_cuboid(got[k], ref["cuboids"][b][k])
    return 0


def _run_frame(cs, ctx, img, K, T, boxes, lines, **kw):
    ctx.set_calibration(K)
    p = cs.default_params(**kw)
    ctx.upload(img[None], T[None], [boxes], [lines], p)
    ctx.run()
    return ctx.fetch()


MODES = {
    "default": {},
    "sample_roll_pitch": dict(whether_sample_cam_roll_pitch=1),
    "sample_height_top5": dict(whether_sample_bbox_height=1, max_cuboid_num=5),
    "config1_only": dict(consider_config_2=0),
    "config2_only": dict(consider_config_1=0),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_fixture_a_modes(cs, oracle, fixture_a, mode):
    fa = fixture_a
    kw = MODES[mode]
    ctx = cs.Context(0, 1280, 960, 1, 8, 4096)
    out, counts = _run_frame(cs, ctx, fa["img"], fa["K"], fa["T"], fa["boxes"], fa["lines"], **kw)
    ref = oracle.detect_cuboid(fa["img"], fa["K"], fa["T"], fa["boxes"], fa["lines"], _oracle_params(oracle, **kw), trace_object=0)
    st = ctx.stats()
    assert st["n_candidates"] == ref["n_candidates"] == fa["expected"][mode]["n_candidates"]
    assert st["n_valid"] == ref["n_valid"] == fa["expected"][mode]["n_valid"]
    assert counts[0] == len(ref["cuboids"][0])
    for k in range(counts[0]):
        _compare_cuboid(out[0, k], ref["cuboids"][0][k])
    # the committed golden pins the same best index
    assert int(out[0, 0]["proposal_index"]) == fa["expected"][mode]["cuboids"][0]["proposal_index"]
    ctx.close()


@pytest.mark.parametrize("split_kernels", [0, 32])
def test_fixture_a_stages(cs, oracle, fixture_a, split_kernels):
    """Stage by stage: gray/Canny/DT bit-exact, merged lines bit-exact, valid set + per-proposal errors.
    Default: hysteresis kernel + cone-form distance transform (two sweeps + row scans).  32 selects the two-pass raster-scan
    distance transform kernel."""
    fa = fixture_a
    ctx = cs.Context(0, 1280, 960, 1, 8, 4096)
    ctx.L.cs_set_profiling(ctx.h, split_kernels)
    _run_frame(cs, ctx, fa["img"], fa["K"], fa["T"], fa["boxes"], fa["lines"])
    ref = oracle.detect_cuboid(fa["img"], fa["K"], fa["T"], fa["boxes"], fa["lines"], trace_object=0)["trace"]
    roi = ctx.debug_roi(0)
    assert roi["roi"] == tuple(ref["roi"])
    np.testing.assert_array_equal(roi["canny"], ref["canny"])
    np.testing.assert_array_equal(roi["dist"], ref["dist"])
    assert roi["n_lines_roi"] == ref["n_lines_roi"] and roi["n_lines_merged"] == ref["n_lines_merged"]
    np.testing.assert_array_equal(roi["merged_lines"], ref["merged_lines"])
    cand = ctx.debug_candidates(0)
    assert cand["n"] == ref["n_candidates"]
    np.testing.assert_array_equal(np.nonzero(cand["valid"])[0], ref["cand_index"])
    np.testing.assert_allclose(cand["dist_err"][ref["cand_index"]], ref["rows"][:, 4], rtol=1e-13, atol=0)
    np.testing.assert_array_equal(cand["angle_err"][ref["cand_index"]], ref["rows"][:, 5])
    ctx.close()


@pytest.mark.parametrize("seed,w,h,kind,nb", [(11, 640, 480, "indoor", 3), (12, 640, 480, "indoor", 5), (13, 1242, 375, "kitti", 8),
                                              (14, 1280, 960, "indoor", 4)])
def test_synthetic_batch_matches_oracle(cs, oracle, seed, w, h, kind, nb):
    from cube_slam_b200 import synthetic as S
    F = 6
    imgs, Ts, boxes, lines, K = S.make_batch(seed, F, w, h, nb, kind=kind, poisson=(kind == "indoor"))
    ctx = cs.Context(0, w, h, F, 16, 4096)
    ctx.set_calibration(K)
    if seed == 11:
        ctx.L.cs_set_profiling(ctx.h, 8)  # one case through the CTA-wide selection kernel (k_fuse_rank)
    if seed == 13:
        ctx.L.cs_set_profiling(ctx.h, 32)  # one case through the raster-scan distance transform kernel
    p = cs.default_params(max_cuboid_num=3)
    out, counts = ctx.detect_batch_host(imgs, Ts, boxes, lines, p)
    st = ctx.stats()
    o = 0
    tot_c = tot_v = 0
    job = 0
    n_knife = 0
    for f in range(F):
        def redo(cut_flip=-1, f=f):
            return oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f], _oracle_params(oracle, max_cuboid_num=3), cut_flip=cut_flip)
        ref = redo()
        tot_c += ref["n_candidates"]
        tot_v += ref["n_valid"]
        for b in range(len(boxes[f])):
            n_knife += _compare_box(oracle, out[o], counts[o], ref, b, redo)
            o += 1
        # one traced ROI per frame: bit-exact image stages
        tr = oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f], trace_object=0)["trace"]
        roi = ctx.debug_roi(job)
        np.testing.assert_array_equal(roi["canny"], tr["canny"])
        np.testing.assert_array_equal(roi["dist"], tr["dist"])
        np.testing.assert_array_equal(roi["merged_lines"], tr["merged_lines"])
        job += len(boxes[f])
    assert st["n_candidates"] == tot_c and st["n_valid"] == tot_v
    ctx.close()


def test_canny_bits_match_oracle_on_every_roi(cs, oracle):
    """k_canny_nms on every ROI of two multi-frame batches (640 x 480 and 1280 x 960, several ROIs per frame, interior and border
    tiles): the edge bits equal the oracle's."""
    from cube_slam_b200 import synthetic as S
    for seed, w, h, nb in ((61, 640, 480, 4), (62, 1280, 960, 3)):
        imgs, Ts, boxes, lines, K = S.make_batch(seed, 3, w, h, nb, poisson=True)
        ctx = cs.Context(0, w, h, 3, 16, 4096)
        ctx.set_calibration(K)
        ctx.detect_batch_host(imgs, Ts, boxes, lines, cs.default_params(max_cuboid_num=2))
        rois = [ctx.debug_roi(j) for j in range(sum(len(b) for b in boxes))]
        ctx.close()
        job = 0
        for f in range(3):
            for b in range(len(boxes[f])):
                tr = oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f], trace_object=b)["trace"]
                np.testing.assert_array_equal(rois[job]["canny"], tr["canny"])
                job += 1


def test_dense_sweep_and_sampling(cs, oracle):
    """BASELINE config 5 shape (0.5 deg yaw step, 30 top-x samples) and roll/pitch sampling on synthetic frames."""
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, lines, K = S.make_batch(21, 2, 640, 480, 2)
    ctx = cs.Context(0, 640, 480, 2, 16, 4096)
    ctx.set_calibration(K)
    for kw in (dict(yaw_step_deg=0.5, top_sample_count_override=30), dict(whether_sample_cam_roll_pitch=1),
               dict(whether_sample_bbox_height=1, whether_sample_cam_roll_pitch=1, max_cuboid_num=4)):
        out, counts = ctx.detect_batch_host(imgs, Ts, boxes, lines, cs.default_params(**kw))
        o = 0
        for f in range(2):
            ref = oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f], _oracle_params(oracle, **kw))
            for b in range(len(boxes[f])):
                assert counts[o] == len(ref["cuboids"][b])
                if b == 0 or not kw.get("whether_sample_cam_roll_pitch"):
                    for k in range(counts[o]):
                        _compare_cuboid(out[o, k], ref["cuboids"][b][k])
                else:
                    # later boxes of a frame inherit the reference's mutated cam_pose (re-derived yaw, last ulp):
                    # indices must agree, continuous values to 1e-9
                    for k in range(counts[o]):
                        assert int(out[o, k]["proposal_index"]) == int(ref["cuboids"][b][k]["proposal_index"])
                        assert abs(out[o, k]["normalized_error"] - ref["cuboids"][b][k]["normalized_error"]) < 1e-9
                o += 1
    ctx.close()


@pytest.mark.parametrize("flags", [0, 32, 64])
def test_distance_transform_wide_sparse_and_empty_rois(cs, oracle, flags):
    """ROIs wider than 640 px (the row scans park their forward result in the row), an ROI with a single edge pixel
    (most pixels have no source in their vertical cone) and an edge-free ROI (DIST_MAX everywhere)."""
    rng = np.random.RandomState(3)
    K = np.array([[800.0, 0, 800], [0, 800, 250], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]])
    T[2, 3] = 1.4
    H, W = 500, 1600
    textured = np.kron(rng.randint(0, 255, (25, 80)).astype(np.uint8), np.ones((20, 20), np.uint8))
    flat = np.full((H, W), 120, np.uint8)
    dot = flat.copy()
    dot[240:243, 1370:1373] = 255          # a tiny blob: a handful of edge pixels far from most of the ROI
    ctx = cs.Context(0, W, H, 1, 8, 4096)
    ctx.L.cs_set_profiling(ctx.h, flags)
    for img, box in ((textured, [40, 30, 1500, 420, 0.9]), (dot, [30, 20, 1520, 450, 0.9]), (flat, [100, 60, 700, 300, 0.9])):
        img3 = np.ascontiguousarray(np.stack([img] * 3, -1))
        boxes = np.array([box], float)
        lines = np.array([[100.0, 100, 400, 110], [500, 300, 900, 310]])
        _run_frame(cs, ctx, img3, K, T, boxes, lines)
        tr = oracle.detect_cuboid(img3, K, T, boxes, lines, trace_object=0)["trace"]
        roi = ctx.debug_roi(0)
        assert roi["roi"] == tuple(tr["roi"]) and roi["roi"][2] > 640
        np.testing.assert_array_equal(roi["canny"], tr["canny"])
        np.testing.assert_array_equal(roi["dist"], tr["dist"])
    assert float(roi["dist"].min()) > 65000.0   # the flat frame: no edges, the transform saturates
    ctx.close()


def test_edge_cases(cs, oracle):
    """No lines at all, a box with no valid proposal, an empty frame list entry, gray input."""
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, lines, K = S.make_batch(31, 3, 640, 480, 2)
    ctx = cs.Context(0, 640, 480, 3, 16, 4096)
    ctx.set_calibration(K)
    boxes = [boxes[0], np.zeros((0, 5)), boxes[2]]
    lines = [np.zeros((0, 4)), lines[1], lines[2]]
    out, counts = ctx.detect_batch_host(imgs, Ts, boxes, lines, cs.default_params())
    o = 0
    for f in range(3):
        ref = oracle.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f])
        for b in range(len(boxes[f])):
            assert counts[o] == len(ref["cuboids"][b])
            for k in range(counts[o]):
                _compare_cuboid(out[o, k], ref["cuboids"][b][k])
            o += 1
    # single-channel input takes the `gray_img = rgb_img` branch (box_proposal_detail.cpp:65-66)
    gray = np.ascontiguousarray(imgs[:, :, :, 1])
    out_g, counts_g = ctx.detect_batch_host(gray, Ts, boxes, lines, cs.default_params())
    o = 0
    for f in range(3):
        ref = oracle.detect_cuboid(gray[f], K, Ts[f], boxes[f], lines[f])
        for b in range(len(boxes[f])):
            assert counts_g[o] == len(ref["cuboids"][b])
            for k in range(counts_g[o]):
                _compare_cuboid(out_g[o, k], ref["cuboids"][b][k])
            o += 1
    ctx.close()


def test_class_mirror_matches_reference_call_shape(cs, oracle, fixture_a):
    """detect_3d_cuboid mirror: same members / call as the reference demo (detect_3d_cuboid/src/main.cpp:56-66)."""
    fa = fixture_a
    det = cs.detect_3d_cuboid()
    det.whether_plot_detail_images = False
    det.whether_plot_final_images = False
    det.print_details = False
    det.set_calibration(fa["K"])
    det.whether_sample_bbox_height = False
    det.whether_sample_cam_roll_pitch = False
    all_object_cuboids = det.detect_cuboid(fa["img"], fa["T"], fa["boxes"], fa["lines"])
    assert len(all_object_cuboids) == 1 and len(all_object_cuboids[0]) == 1
    best = all_object_cuboids[0][0]
    assert best.proposal_index == fa["expected"]["default"]["cuboids"][0]["proposal_index"]
    np.testing.assert_allclose(det.cam_pose_raw.euler_angle, oracle.cam_pose(fa["K"], fa["T"])["euler"], atol=0)
    assert det.detect_cuboid(fa["img"], fa["T"], np.zeros((0, 5)), fa["lines"]) == []
