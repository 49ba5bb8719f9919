"""The oracle against the reference's own code with detect_cuboid's parameters off their defaults, on the CPU.

Where the reference takes a parameter as an argument, the oracle is pinned to the reference's function called with it (oracle/_ref/
libcuboid_ref.so, see oracle/ref/cuboid_ref.cpp), field for field and NaN == NaN:
  * the whole detect_3d_cuboid::detect_cuboid at the class members a caller can set: max_cut_skew, nominal_skew_ratio, max_cuboid_num
    (17 and 32, with height and roll / pitch sampling) and both configurations off.  The reference's partial_sort leaves ties undefined;
    the tie classifier of tests/test_oracle_ref_cuboid_edges.py decides those;
  * the free functions that take the others: merge_break_lines (distance, angle and length thresholds), VP_support_edge_infos (the two
    angle thresholds), box_edge_sum_dists (reweight_edge_distance), fuse_normalize_scores_v2 (weight_vp_angle, whether_normalize_two_errors)
    and linespace<double> (yaw range and step: 512 samples for the pair the product accepts, 513 for the one it refuses);
  * the Canny thresholds against cv2.Canny itself (L1 gradient, cv2.setUseOptimized(False)).

Inside detect_cuboid, shorted_edge_thre, the weights, the merge and length thresholds, the Canny thresholds and yaw_half_range_deg are
literals of the reference, and top_sample_count_override is an extension of this project: there they can only be checked against the
oracle (tests/test_gpu_cuboid_params.py does, on the device)."""
import numpy as np
import pytest

import test_oracle_ref_cuboid_edges as E
from test_gpu_cuboid_params import CS_MAX_YAW, YAW_RANGE, _step_for, linespace_count

MAX_CLASSIFIED = 12   # classified ties allowed over all detect_cuboid runs of this file

# two edge lists (pairs of corner ids) of the shape detect_cuboid gives box_edge_sum_dists: 9 and 7 edges, edges 4-6 reweighted
EDGES = (np.array([[0, 1], [1, 2], [2, 3], [3, 0], [1, 5], [2, 4], [3, 7], [4, 7], [4, 5]]),
         np.array([[0, 1], [1, 2], [2, 3], [3, 0], [1, 5], [2, 4], [4, 5]]))


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.ref_detect_cuboid_available():
        pytest.skip("oracle/_ref/libcuboid_ref.so not built (no reference checkout at build time)")
    oracle.lib().orc_set_portable_atan2(0)
    yield oracle
    oracle.lib().orc_set_portable_atan2(1)


@pytest.fixture(scope="module")
def tally():
    t = {"runs": 0, "classified": []}
    yield t
    print("\ncuboid parameter grid: %d oracle/reference runs, %d classified ties %s" % (t["runs"], len(t["classified"]), t["classified"]))
    assert len(t["classified"]) <= MAX_CLASSIFIED


RP = dict(whether_sample_cam_roll_pitch=1, whether_sample_bbox_height=1)
GRID = [("max_cut_skew_%g" % v, dict(max_cut_skew=v, max_cuboid_num=20)) for v in (0.5, 1.0, 1.5, 1e9)] + \
       [("nominal_skew_%g" % v, dict(nominal_skew_ratio=v, max_cuboid_num=20)) for v in (0.5, 3.0)] + \
       [("top%d_height_roll_pitch" % k, dict(max_cuboid_num=k, **RP)) for k in (17, 32)] + \
       [("configs_off", dict(consider_config_1=0, consider_config_2=0))]


@pytest.mark.parametrize("name,kw", GRID, ids=[g[0] for g in GRID])
def test_detect_cuboid_members(ref, tally, fixture_a, name, kw):
    frames = [("A", fixture_a["img"], fixture_a["K"], fixture_a["T"], fixture_a["boxes"], fixture_a["lines"])] + \
             [(t, img, K, T, boxes, lines) for t, img, K, T, boxes, lines in E.base_frames()[::2]]
    p = ref.default_params(**kw)
    moved = 0
    for tag, img, K, T, boxes, lines in frames:
        E._compare(ref, tally, "%s/%s" % (tag, name), img, K, T, boxes, lines, p)
        got = ref.detect_cuboid(img, K, T, boxes, lines, p)["cuboids"]
        base = ref.detect_cuboid(img, K, T, boxes, lines, ref.default_params(max_cuboid_num=max(int(p.max_cuboid_num), 1)))["cuboids"]
        moved += any(len(g) != len(b) or not np.array_equal(g["combined_score"], b["combined_score"], equal_nan=True) for g, b in zip(got, base))
        if name == "configs_off":
            assert all(len(g) == 0 for g in got)
        elif name.startswith("top"):
            assert any(len(g) == kw["max_cuboid_num"] for g in got), tag
    assert moved, "%s changes no record" % name


def _roi_line_sets():
    """The lines inside the ROI of each dense set of test_oracle_ref_cuboid_edges (random, dashes, odd lines), with its image and ROI."""
    out = []
    for tag, img, K, T, box, lines in E.dense_cases():
        h, w = img.shape[:2]
        l, t, r, b = E.roi_of(box, w, h)
        L = lines[[l <= min(x[0], x[2]) and max(x[0], x[2]) <= r and t <= min(x[1], x[3]) and max(x[1], x[3]) <= b for x in lines]]
        out.append((tag, img, (l, t, r, b), L - [l, t, l, t]))
    return out


def test_merge_break_lines(ref):
    n_cap = 0
    for tag, img, roi, L in _roi_line_sets():
        for dist in (0.0, 5.0, 20.0, 60.0, 1e6):
            for ang in (0.0, 1.0, 5.0, 20.0, 90.0, 180.0):
                for ln in (-1.0, 0.0, 30.0, 100.0, 1e6):
                    want = ref.ref_merge_break_lines(L, dist, ang, ln)
                    np.testing.assert_array_equal(ref.merge_break_lines(L, dist, ang, ln), want, err_msg="%s %g %g %g" % (tag, dist, ang, ln))
                    if ln == 1e6:
                        assert len(want) == 0
        n_cap += len(L) - len(ref.merge_break_lines(L, 1e6, 5.0, 0.0)) == 500
    assert n_cap >= 2   # the dashes reach the 500-merge cap with only the angle test limiting


def _vps_and_lines(rng, L):
    mids = np.stack([(L[:, 0] + L[:, 2]) / 2, (L[:, 1] + L[:, 3]) / 2], 1)
    ang = np.arctan2(L[:, 3] - L[:, 1], L[:, 2] - L[:, 0])
    ang = np.where(ang > np.pi / 2, ang - np.pi, np.where(ang < -np.pi / 2, ang + np.pi, ang))
    vps = np.array([[rng.uniform(-3000, 3000), rng.uniform(-3000, 3000)] for _ in range(3)])
    return vps, mids, ang


def test_vp_support_edge_infos(ref):
    rng = np.random.default_rng(11)
    n_nan = n_full = 0
    for tag, img, roi, L in _roi_line_sets():
        for _ in range(4):
            vps, mids, ang = _vps_and_lines(rng, L)
            for a, b in ((0.0, 0.0), (5.0, 5.0), (15.0, 10.0), (45.0, 30.0), (90.0, 90.0)):
                want = ref.ref_vp_support_edge_infos(vps, mids, ang, a, b)
                got = ref.vp_support_edge_infos(vps, mids, ang, a, b)
                np.testing.assert_array_equal(got, want, err_msg="%s %g %g" % (tag, a, b))
                n_nan += np.isnan(want).all()
                n_full += not np.isnan(want).any()
    assert n_nan > 0 and n_full > 0   # thresholds with no support and with support for all three points


def test_box_edge_sum_dists(ref):
    rng = np.random.default_rng(12)
    n_diff = 0
    for tag, img, (l, t, r, b), L in _roi_line_sets():
        gray = ref.bgr2gray(img)[t:b + 1, l:r + 1].copy()
        dist = ref.chamfer_dt(ref.canny(gray))
        h, w = dist.shape
        for _ in range(40):
            c = np.stack([rng.uniform(-5, w + 5, 8), rng.uniform(-5, h + 5, 8)])   # a few corners past the map: the reference's clamp
            for edges in EDGES:
                vals = []
                for rw in (0, 1):
                    want = ref.ref_box_edge_sum_dists(dist, c, edges, rw)
                    assert ref.box_edge_sum_dists(dist, c, edges, rw) == want, tag
                    vals.append(want)
                n_diff += vals[0] != vals[1]
    assert n_diff > 0


def test_fuse_normalize_scores_v2(ref):
    rng = np.random.default_rng(13)
    n_nan = 0
    for n in (1, 2, 4, 5, 6, 17, 40, 301):
        for trial in range(6):
            d = rng.uniform(0, 900, n)
            a = rng.uniform(0, 3, n)
            if trial == 1:
                a[:] = 1.25                                   # all angle errors equal: the angle term is left raw
            if trial == 2:
                a[np.argmin(d)] = a.min() - 0.5               # the same proposal is smallest in both errors: 0 / 0 at w = -1
            for w in (0.0, 0.3, 0.8, 5.0, -1.0):
                for norm in (0, 1):
                    kg, sg = ref.fuse_normalize_scores_v2(d, a, w, norm)
                    kw_, sw = ref.ref_fuse_normalize_scores_v2(d, a, w, norm)
                    np.testing.assert_array_equal(kg, kw_)
                    np.testing.assert_array_equal(sg, sw)   # NaN == NaN
                    n_nan += w == -1.0 and norm == 1 and np.isnan(sw).any()
    assert n_nan > 0


def test_linespace_yaw_counts(ref, fixture_a):
    yaw = ref.cam_pose(fixture_a["K"], fixture_a["T"])["yaw"] - np.pi / 2
    for half, step, n in ((YAW_RANGE, _step_for(CS_MAX_YAW - 1), CS_MAX_YAW), (YAW_RANGE, _step_for(CS_MAX_YAW), CS_MAX_YAW + 1),
                          (YAW_RANGE, 6.0, None), (0.0, 6.0, 1), (YAW_RANGE, _step_for(12), 13), (YAW_RANGE, _step_for(3), 4)):
        s, e, st = yaw - half / 180 * np.pi, yaw + half / 180 * np.pi, step / 180 * np.pi
        want = ref.ref_linespace(s, e, st)
        np.testing.assert_array_equal(ref.linespace(s, e, st), want)
        assert len(want) == linespace_count(s, e, st)
        if n is not None:
            assert len(want) == n


CANNY_PAIRS = ((0.0, 0.0), (0.0, 1.0), (80.0, 80.0), (200.0, 80.0), (79.5, 200.9), (2041.0, 3000.0))


def test_canny_thresholds_against_cv2(ref, fixture_a):
    cv2 = pytest.importorskip("cv2")
    cv2.setUseOptimized(False)
    cv2.setNumThreads(1)
    gray = ref.bgr2gray(fixture_a["img"])
    for lo, hi in CANNY_PAIRS:
        want = cv2.Canny(gray, lo, hi)
        got = ref.canny(gray, lo, hi)
        np.testing.assert_array_equal(got, want, err_msg="(%g, %g)" % (lo, hi))
        np.testing.assert_array_equal(ref.chamfer_dt(got), cv2.distanceTransform(255 - want, cv2.DIST_L2, 3))
    np.testing.assert_array_equal(ref.canny(gray, 200, 80), ref.canny(gray, 80, 200))
    np.testing.assert_array_equal(ref.canny(gray, 79.5, 200.9), ref.canny(gray, 79, 200))
    assert not ref.canny(gray, 2041, 3000).any()   # above 2 * 4 * 255, the largest L1 magnitude: no edge
    assert (ref.chamfer_dt(ref.canny(gray, 2041, 3000)) == ref.chamfer_dt(np.zeros((5, 5), np.uint8)).max()).all()
