"""GPU parity of the cuboid stage with every field of cs_cuboid_params off its default: the CUDA path (through the C ABI) against the CPU
oracle, one table entry per case, each on a small mixed batch -- fixture A, synthetic VGA, KITTI and 1280 x 960 frames with several boxes and
the lines given (one case detects its lines with the online LSD) -- through the default kernels and through the CTA-wide selection kernel
k_fuse_rank after the same warp sweep (cs_set_profiling bit 3).

Every record is compared with test_gpu_cuboid_parity's _compare_cuboid, the batch's candidate and valid counts with the oracle's, and for
one traced ROI per frame Canny, the distance map, the merged lines, the valid set and both error arrays bit for bit.  A field the kernels
ignored would still pass all of that wherever it changes nothing, so each case also shows from the oracle that it is not vacuous: its
result differs from the default one in the stage the field feeds (merged lines, Canny bits, valid set, distance errors, normalised errors,
combined score or rank, candidate count).  Where a case raises max_cuboid_num only to reach deeper ranks, the default it is measured
against returns as many cuboids (_baseline_kw), so that a list of another length cannot pass for a change.  The two Canny pairs that must mean the same as another show instead that they give exactly its
result: (200, 80) is swapped into the default (80, 200), (79.5, 200.9) is floored to (79, 200).

The limits: max_cuboid_num up to CS_MAX_TOPK = 32 (0 and 33 are refused with CS_ERR_CAPACITY and the next batch is right), 512 yaw samples
(CS_MAX_YAW; 513 are refused), more than 32 candidates per yaw in the warp sweep and more than 1 024 per box (the selection then runs in
k_fuse_rank).  weight_vp_angle = -1 makes 1 + w = 0: scores of -inf, +inf and NaN, where the ranking must put NaN after +inf."""
import re

import numpy as np
import pytest

import test_oracle_ref_cuboid_edges as E
from test_gpu_cuboid_parity import _compare_cuboid

pytestmark = pytest.mark.gpu

FW_CAP = 1024          # k_fuse_warp selects a batch whose boxes have at most this many candidates each
CS_MAX_TOPK = 32
CS_MAX_YAW = 512
LSD_THRES = 15.0       # line_length_thres object_slam uses with the LSD flavour
ROLL_PITCH_GROUPS = ("A", "vga")   # roll / pitch sampling (25 poses per box) runs on the two smaller groups
YAW_RANGE = 45.0


def _step_for(n_half):
    """A yaw step (deg) that puts 2 * YAW_RANGE / step half a step away from an integer: n_half + 0.5 steps, n_half + 1 samples."""
    return 2 * YAW_RANGE / (n_half + 0.5)


def linespace_count(start, end, step):
    """matrix_utils.cpp:350-363, the samples linespace<double> makes by accumulated double adds (and its stop after 1 001)."""
    n = 0
    while start <= end:
        n += 1
        start += step
        if n > 1000:
            break
    return n


def yaw_count(oracle, K, T, half_deg, step_deg):
    """The number of yaw samples detect_cuboid makes for a frame (box_proposal_detail.cpp:126-128), restated."""
    yaw_init = oracle.cam_pose(K, T)["yaw"] - 90.0 / 180.0 * np.pi
    return linespace_count(yaw_init - half_deg / 180.0 * np.pi, yaw_init + half_deg / 180.0 * np.pi, step_deg / 180.0 * np.pi)


CANNY_SAME = ((200.0, 80.0), (79.5, 200.9))
# what a "same" case must equal exactly: the default, or the pair the thresholds are floored to
SAME_AS = {"canny_79.5_200.9": dict(canny_low=79.0, canny_high=200.0)}
RP = dict(whether_sample_cam_roll_pitch=1, whether_sample_bbox_height=1)

# name -> (params, stage the non-default value must change in the oracle ("same": must not change at all), groups or None for all)
CASES = {}
for lo, hi in ((0.0, 0.0), (0.0, 1.0), (80.0, 80.0), (200.0, 80.0), (79.5, 200.9), (2041.0, 3000.0)):
    CASES["canny_%g_%g" % (lo, hi)] = (dict(canny_low=lo, canny_high=hi), "same" if (lo, hi) in CANNY_SAME else "canny", None)
for v in (0.0, 5.0, 60.0, 1e6):
    CASES["merge_dist_%g" % v] = (dict(pre_merge_dist_thre=v), "merged", None)
for v in (0.0, 1.0, 20.0, 90.0, 180.0):
    CASES["merge_angle_%g" % v] = (dict(pre_merge_angle_thre=v), "merged", None)
for v in (0.0, -1.0, 100.0, 1e6):
    CASES["edge_length_%g" % v] = (dict(edge_length_threshold=v), "merged", None)
for a, b in ((0.0, 0.0), (5.0, 5.0), (45.0, 30.0), (90.0, 90.0)):
    CASES["vp_thre_%g_%g" % (a, b)] = (dict(vp12_edge_angle_thre=a, vp3_edge_angle_thre=b), "angle_err", None)
for v in (-1.0, 0.0, 5.0, 60.0, 1e6):
    CASES["shorted_edge_%g" % v] = (dict(shorted_edge_thre=v), "valid", None)
CASES["no_reweight"] = (dict(reweight_edge_distance=0), "dist_err", None)
for w in (0.8, 0.0):
    CASES["no_normalize_w%g" % w] = (dict(whether_normalize_two_errors=0, weight_vp_angle=w), "norm", None)
for w in (0.0, 0.3, 5.0):
    CASES["weight_vp_%g" % w] = (dict(weight_vp_angle=w), "norm", None)
CASES["weight_vp_-1_top32"] = (dict(weight_vp_angle=-1.0, max_cuboid_num=32), "norm", None)
for w in (0.0, 0.5, 4.0):
    CASES["weight_skew_%g" % w] = (dict(weight_skew_error=w, max_cuboid_num=5), "score", None)
for v in (0.5, 3.0):
    CASES["nominal_skew_%g" % v] = (dict(nominal_skew_ratio=v, max_cuboid_num=5), "score", None)
for v in (0.5, 1.0, 1.5, 1e9):
    CASES["max_cut_skew_%g" % v] = (dict(max_cut_skew=v, max_cuboid_num=32), "score", None)   # deep enough to reach skews it cuts
CASES["configs_off"] = (dict(consider_config_1=0, consider_config_2=0), "valid", None)
for k in (6, 17, 31, 32):
    CASES["top%d" % k] = (dict(max_cuboid_num=k), "score", None)
    CASES["top%d_height_roll_pitch" % k] = (dict(max_cuboid_num=k, **RP), "ncand", ROLL_PITCH_GROUPS)
CASES["yaw_one"] = (dict(yaw_half_range_deg=0.0), "ncand", None)
CASES["yaw_13"] = (dict(yaw_step_deg=_step_for(12)), "ncand", None)
CASES["yaw_4"] = (dict(yaw_step_deg=_step_for(3)), "ncand", None)
CASES["yaw_512"] = (dict(yaw_step_deg=_step_for(CS_MAX_YAW - 1)), "ncand", ("A", "kitti"))
for t in (1, 2):
    CASES["top_x_%d" % t] = (dict(top_sample_count_override=t), "ncand", None)
CASES["top_x_64_warp"] = (dict(top_sample_count_override=64, yaw_step_deg=12.0), "ncand", None)        # 8 yaws: <= FW_CAP per box
CASES["top_x_64_fuse_rank"] = (dict(top_sample_count_override=64), "ncand", None)                      # 16 yaws: > FW_CAP per box
CASES["combo_rp_height_top32_cut"] = (dict(max_cuboid_num=32, max_cut_skew=1.2, **RP), "score", ROLL_PITCH_GROUPS)
CASES["combo_raw_errors_swapped_canny"] = (dict(whether_normalize_two_errors=0, reweight_edge_distance=0, canny_low=200.0, canny_high=80.0),
                                           "norm", None)
ONLINE_LSD_CASE = "merge_angle_20"


# ------------------------------------------------------------------------------------------- inputs
@pytest.fixture(scope="module")
def cs():
    import cube_slam_b200 as cs
    return cs


@pytest.fixture(scope="module")
def groups(fixture_a):
    """name -> (K, [(img, T, boxes, lines)]): one batch per frame size and calibration."""
    from cube_slam_b200 import synthetic as S
    out = {"A": (fixture_a["K"], [(fixture_a["img"], fixture_a["T"], fixture_a["boxes"], fixture_a["lines"])])}
    imgs, Ts, boxes, lines, K = S.make_batch(601, 2, 640, 480, 4)   # seed 601: boxes whose top 32 at weight_vp_angle = -1 reach a NaN score
    out["vga"] = (K, [(imgs[f], Ts[f], boxes[f], lines[f]) for f in range(2)])
    imgs, Ts, boxes, lines, K = S.make_batch(302, 1, 1242, 375, 4, kind="kitti")
    out["kitti"] = (K, [(imgs[0], Ts[0], boxes[0], lines[0])])
    img, K, T, boxes, lines = E.big_frame()
    out["big"] = (K, [(img, T, boxes, lines)])
    return out


def _dashes_group():
    """A VGA frame whose biggest box holds rows of collinear dashes (the 500-merge cap of merge_break_lines)."""
    tag, img, K, T, box, lines = next(c for c in E.dense_cases() if c[0].endswith("_dashes"))
    return K, [(img, T, np.array([box]), lines)]


def _online_group(oracle):
    """Two VGA frames whose lines come from the online LSD (the oracle's detect_filter_lines with use_LSD)."""
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, _, K = S.make_batch(611, 2, 640, 480, 3, poisson=True)
    return K, [(imgs[f], Ts[f], boxes[f], oracle.lsd_detect(imgs[f], LSD_THRES)["lines"].astype(np.float64)) for f in range(2)]


def _n_jobs_before(frames, f, kw):
    h = frames[0][0].shape[0]
    return sum(len(E.height_samples(bb, h)) if kw.get("whether_sample_bbox_height") else 1 for fr in frames[:f] for bb in fr[2])


class Oracle(object):
    """The oracle's records, counts and one traced ROI per frame (box 0, height sample 0) for one batch and one parameter set."""

    def __init__(self, oracle, K, frames, kw):
        self.K, self.frames, self.kw = K, frames, kw
        rp = bool(kw.get("whether_sample_cam_roll_pitch"))
        oracle.lib().orc_set_independent_boxes(int(rp))   # the device starts every box of a frame from the raw pose
        try:
            p = oracle.default_params(**kw)
            self.refs = [oracle.detect_cuboid(img, K, T, boxes, lines, p) for img, T, boxes, lines in frames]
            self.traces = [oracle.detect_cuboid(img, K, T, boxes, lines, p, trace_object=0, trace_caps=(4096, 1 << 21, 1 << 17))["trace"]
                           for img, T, boxes, lines in frames]
        finally:
            oracle.lib().orc_set_independent_boxes(0)
        self.jobs = [_n_jobs_before(frames, f, kw) for f in range(len(frames))]

    def stage(self, name):
        """What one stage of the pipeline made, as a list of arrays."""
        T, R = self.traces, self.refs
        if name == "canny":
            return [t["canny"] for t in T]
        if name == "merged":
            return [t["merged_lines"] for t in T]
        if name == "valid":
            return [t["cand_index"] for t in T] + [np.array([r["n_valid"] for r in R])]
        if name == "dist_err":
            return [t["rows"][:, 4] for t in T]
        if name == "angle_err":
            return [t["rows"][:, 5] for t in T]
        if name == "norm":
            return [c["normalized_error"] for r in R for c in r["cuboids"]] + [t["kept_scores"] for t in T]
        if name == "score":
            return [c[f] for r in R for c in r["cuboids"] for f in ("combined_score", "proposal_index", "height_sample_id")]
        if name == "ncand":
            return [np.array([r["n_candidates"] for r in R])]
        if name == "same":
            return self.stage("canny") + self.stage("merged") + self.stage("valid") + self.stage("dist_err") + self.stage("norm") + self.stage("score")
        raise KeyError(name)


def _same(a, b):
    return len(a) == len(b) and all(np.shape(x) == np.shape(y) and np.array_equal(np.asarray(x, np.float64), np.asarray(y, np.float64), equal_nan=True)
                                    for x, y in zip(a, b))


def _check(ctx, orc, out, counts):
    o = 0
    for f, ref in enumerate(orc.refs):
        for b in range(len(orc.frames[f][2])):
            assert counts[o] == len(ref["cuboids"][b]), (f, b, counts[o], len(ref["cuboids"][b]))
            for k in range(counts[o]):
                _compare_cuboid(out[o, k], ref["cuboids"][b][k])
            o += 1
    st = ctx.stats()
    assert st["n_candidates"] == sum(r["n_candidates"] for r in orc.refs)
    assert st["n_valid"] == sum(r["n_valid"] for r in orc.refs)
    for j, tr in zip(orc.jobs, orc.traces):
        roi = ctx.debug_roi(j)
        assert roi["roi"] == tuple(tr["roi"]), j
        np.testing.assert_array_equal(roi["canny"], tr["canny"], err_msg="job %d" % j)
        np.testing.assert_array_equal(roi["dist"], tr["dist"], err_msg="job %d" % j)
        assert (roi["n_lines_roi"], roi["n_lines_merged"]) == (tr["n_lines_roi"], tr["n_lines_merged"]), j
        np.testing.assert_array_equal(roi["merged_lines"], tr["merged_lines"], err_msg="job %d" % j)
        cand = ctx.debug_candidates(j)
        assert cand["n"] == tr["n_candidates"], j
        np.testing.assert_array_equal(np.nonzero(cand["valid"])[0], tr["cand_index"], err_msg="job %d" % j)
        np.testing.assert_array_equal(cand["dist_err"][tr["cand_index"]], tr["rows"][:, 4], err_msg="job %d" % j)
        np.testing.assert_array_equal(cand["angle_err"][tr["cand_index"]], tr["rows"][:, 5])


def _line_params(cs):
    import ctypes as C
    from cube_slam_b200 import _lib
    lp = _lib.LineParams()
    _lib.load().cs_default_line_params(C.byref(lp))
    lp.use_LSD = 1
    lp.line_length_thres = LSD_THRES
    return lp


def _run(cs, ctx, orc, flags, online=False):
    ctx.set_calibration(orc.K)
    ctx.L.cs_set_profiling(ctx.h, flags)
    imgs = np.stack([f[0] for f in orc.frames])
    Ts = np.stack([f[1] for f in orc.frames])
    p = cs.default_params(**orc.kw)
    if online:
        ctx.upload_online(imgs, Ts, [f[2] for f in orc.frames], _line_params(cs), p)
        ctx.run()
        out, counts = ctx.fetch()
    else:
        out, counts = ctx.detect_batch_host(imgs, Ts, [f[2] for f in orc.frames], [f[3] for f in orc.frames], p)
    _check(ctx, orc, out, counts)


@pytest.fixture(scope="module")
def ctx(cs):
    c = cs.Context(0, 1280, 960, 2, 8, 4096)
    yield c
    c.close()


_DEFAULTS = {}


def _baseline_kw(name, kw):
    """The parameters a case is measured against: the defaults, with the case's own max_cuboid_num where that only lets the case reach
    deeper ranks (a list of another length would differ whatever the field under test does).  The top-k cases are about max_cuboid_num
    itself and are measured against the defaults."""
    if re.match(r"top\d+", name) or "max_cuboid_num" not in kw:
        return {}
    return dict(max_cuboid_num=kw["max_cuboid_num"])


def _default(oracle, group, base_kw, K, frames):
    key = (group, tuple(sorted(base_kw.items())))
    if key not in _DEFAULTS:
        _DEFAULTS[key] = Oracle(oracle, K, frames, base_kw)
    return _DEFAULTS[key]


# ------------------------------------------------------------------------------------------- what a case has to reach
def _nan_after_inf(oracle, orc):
    """Boxes whose top 32 reaches the +inf scores while a NaN-scored cuboid of the same box (a kept proposal the lift does not drop) sits at
    an earlier kept position than one of the +inf records returned: ranked with the +inf ones by position, the NaN one would be returned
    in its place.  (No height sampling: one job per box, so a record's position is its place in the kept list.)"""
    n = 0
    every = oracle.default_params(**dict(orc.kw, max_cuboid_num=1 << 16))
    for f, (img, T, boxes, lines) in enumerate(orc.frames):
        allr = oracle.detect_cuboid(img, orc.K, T, boxes, lines, every)["cuboids"]
        for b in range(len(boxes)):
            kept = list(oracle.detect_cuboid(img, orc.K, T, boxes, lines, oracle.default_params(**orc.kw), trace_object=b)["trace"]["kept_ids"])
            inf_pos = [kept.index(int(r["proposal_index"])) for r in orc.refs[f]["cuboids"][b] if np.isposinf(r["combined_score"])]
            nan_pos = [kept.index(int(r["proposal_index"])) for r in allr[b] if np.isnan(r["combined_score"])]
            n += bool(inf_pos) and bool(nan_pos) and min(nan_pos) < max(inf_pos)
    return n


def _box_candidates(oracle, orc):
    """Candidates of each box on its own (one job per box: no height sampling)."""
    p = oracle.default_params(**orc.kw)
    return [oracle.detect_cuboid(img, orc.K, T, boxes[b:b + 1], lines, p)["n_candidates"] for img, T, boxes, lines in orc.frames
            for b in range(len(boxes))]


def _extra_checks(oracle, name, orcs):
    """Per-case evidence that the case reaches the regime it is there for."""
    kw = CASES[name][0]
    allo = list(orcs.values())
    if name == "merge_dist_1e+06":
        img, T, boxes, lines = orcs["dashes"].frames[0]
        h, w = img.shape[:2]
        l, t, r, b = E.roi_of(boxes[0], w, h)
        L = lines[[l <= min(x[0], x[2]) and max(x[0], x[2]) <= r and t <= min(x[1], x[3]) and max(x[1], x[3]) <= b for x in lines]]
        assert len(L) - len(oracle.merge_break_lines(L, dist_thre=1e6, len_thre=0)) == 500   # the merge loop stops at its cap
    if name == "edge_length_1e+06":
        assert all(t["n_lines_roi"] > 0 and t["n_lines_merged"] == 0 for o in allo for t in o.traces)
        # no line, no vanishing-point support: every angle error is the not-found penalty of all three VPs
        assert all(np.all(t["rows"][:, 5] == 3 * (30.0 / 180.0 * np.pi * 2)) for o in allo for t in o.traces)
    if name in ("shorted_edge_1e+06", "configs_off"):
        assert all(r["n_valid"] == 0 and all(len(c) == 0 for c in r["cuboids"]) for o in allo for r in o.refs)
    if name == "weight_vp_-1_top32":
        scores = np.concatenate([c["combined_score"] for o in allo for r in o.refs for c in r["cuboids"]])
        assert np.isneginf(scores).any() and np.isposinf(scores).any()
        assert _nan_after_inf(oracle, orcs["vga"]) >= 2
    if name.startswith("top") and not name.startswith("top_x"):
        k = kw["max_cuboid_num"]
        assert any(len(c) == k for o in allo for r in o.refs for c in r["cuboids"]), "no box fills its %d slots" % k
    if name == "yaw_one":
        assert all(yaw_count(oracle, o.K, fr[1], 0.0, 6.0) == 1 for o in allo for fr in o.frames)
    for tag, n in (("yaw_13", 13), ("yaw_4", 4), ("yaw_512", CS_MAX_YAW)):
        if name == tag:
            assert all(yaw_count(oracle, o.K, fr[1], YAW_RANGE, kw["yaw_step_deg"]) == n for o in allo for fr in o.frames)
    if name == "top_x_64_warp":
        per = [c for o in allo for c in _box_candidates(oracle, o)]
        assert max(per) <= FW_CAP and min(per) > 8 * 32, per    # 8 yaws, more than 32 candidates for each
    if name == "top_x_64_fuse_rank":
        assert max(c for o in allo for c in _box_candidates(oracle, o)) > FW_CAP


def _case_groups(oracle, groups, name):
    sel = CASES[name][2]
    out = {g: v for g, v in groups.items() if sel is None or g in sel}
    if name == "merge_dist_1e+06":
        out["dashes"] = _dashes_group()
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_param_case(cs, oracle, groups, ctx, name):
    kw, stage, _ = CASES[name]
    grp = _case_groups(oracle, groups, name)
    orcs = {g: Oracle(oracle, K, frames, kw) for g, (K, frames) in grp.items()}
    # not vacuous: the field changes what the oracle makes in the stage it feeds (or, for "same", changes nothing at all)
    if name in SAME_AS:
        base = {g: Oracle(oracle, K, frames, SAME_AS[name]) for g, (K, frames) in grp.items()}
    else:
        base = {g: _default(oracle, g, _baseline_kw(name, kw), *grp[g]) for g in grp}
    moved = [g for g, o in orcs.items() if not _same(o.stage(stage), base[g].stage(stage))]
    if stage == "same":
        assert moved == [], moved
    else:
        assert moved, "%s: the oracle's %s equals the default one in every group" % (name, stage)
    _extra_checks(oracle, name, orcs)
    online = _online_group(oracle) if name == ONLINE_LSD_CASE else None
    orc_online = Oracle(oracle, online[0], online[1], kw) if online else None
    for flags in (0, 8):
        for o in orcs.values():
            _run(cs, ctx, o, flags)
        if orc_online is not None:
            _run(cs, ctx, orc_online, flags, online=True)


def test_refused_parameters_leave_the_context_usable(cs, oracle, groups, ctx):
    """max_cuboid_num 0 and 33 and 513 yaw samples fail with CS_ERR_CAPACITY; the next batch on the same context is right."""
    K, frames = groups["vga"]
    good = Oracle(oracle, K, frames, dict(max_cuboid_num=3))
    step513 = _step_for(CS_MAX_YAW)
    assert all(yaw_count(oracle, K, fr[1], YAW_RANGE, step513) == CS_MAX_YAW + 1 for fr in frames)
    imgs = np.stack([f[0] for f in frames])
    Ts = np.stack([f[1] for f in frames])
    for flags in (0, 8):
        _run(cs, ctx, good, flags)
        for kw, text in ((dict(max_cuboid_num=0), "max_cuboid_num"), (dict(max_cuboid_num=CS_MAX_TOPK + 1), "max_cuboid_num"),
                         (dict(yaw_step_deg=step513), "too many yaw samples")):
            with pytest.raises(cs.CubeSlamError) as ei:
                ctx.detect_batch_host(imgs, Ts, [f[2] for f in frames], [f[3] for f in frames], cs.default_params(**kw))
            assert "CS_ERR_CAPACITY" in str(ei.value) and text in str(ei.value), str(ei.value)
            _run(cs, ctx, good, flags)
