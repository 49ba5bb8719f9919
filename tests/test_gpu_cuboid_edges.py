"""GPU parity of the cuboid stage at the image borders, on small boxes, on dense line sets up to its per-ROI capacities and on ROIs large
enough to leave shared memory: the inputs of tests/test_oracle_ref_cuboid_edges.py (there pinned oracle == the reference's own
detect_cuboid) through Context.detect_batch_host with the lines given, in mixed batches, against the CPU oracle.

Every stage is compared bit for bit where it is integer or byte work (ROI, Canny, distance map, lines inside the ROI, merged lines, valid
set, angle errors) and every record with a NaN-aware copy of test_gpu_cuboid_parity's comparison (normalized_error is 0 / 0 where a box
has few valid proposals).  Each test asserts from its own inputs that the path it is there for was taken."""
import numpy as np
import pytest

import test_oracle_ref_cuboid_edges as E

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-4   # north_star tolerance on normalised scores
TIGHT = 1e-9       # what we actually expect
HY_SMEM_PLANE_WORDS = (200 * 1024) // 4 // 2   # k_canny_hyst keeps a job's two bit planes in shared memory up to this many words each
DT_SMEM_PLANE_WORDS = (96 * 1024) // 4         # k_dt_bi stages a width class's bit planes in shared memory up to this many words
FU_SMEM_SORT = 4096                            # k_fuse_rank sorts a box's valid proposals in shared memory up to this many


@pytest.fixture(scope="module")
def cs():
    import cube_slam_b200 as cs
    return cs


def _same_or_nan(a, b):
    a, b = float(a), float(b)
    return (np.isnan(a) and np.isnan(b)) or a == b


def _compare_cuboid(g, o, tight=TIGHT):
    """test_gpu_cuboid_parity._compare_cuboid, with NaN == NaN on the scores."""
    assert int(g["proposal_index"]) == int(o["proposal_index"])
    assert int(g["height_sample_id"]) == int(o["height_sample_id"])
    gn, on = float(g["normalized_error"]), float(o["normalized_error"])
    assert np.isnan(gn) == np.isnan(on) and (np.isnan(gn) or abs(gn - on) < SCORE_TOL)
    np.testing.assert_allclose(g["normalized_error"], o["normalized_error"], rtol=0, atol=tight)
    np.testing.assert_allclose(g["combined_score"], o["combined_score"], rtol=1e-9, atol=tight)
    np.testing.assert_allclose(g["edge_distance_error"], o["edge_distance_error"], rtol=1e-12, atol=1e-12)
    assert _same_or_nan(g["edge_angle_error"], o["edge_angle_error"])  # same arithmetic on both sides: bit for bit
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


class Batch(object):
    """One batch (frames of one size and one K) with the oracle's records and, per ROI job, its stage trace, computed once and checked
    against any number of device runs."""

    def __init__(self, oracle, K, frames, kw, trace=True):
        self.K, self.frames, self.kw = K, frames, kw
        self.h, self.w = frames[0][0].shape[:2]
        self.refs, self.jobs = [], []
        for img, T, boxes, lines in frames:
            ref = oracle.detect_cuboid(img, K, T, boxes, lines, oracle.default_params(**kw))
            self.refs.append(ref)
            for b, box in enumerate(boxes):
                hss = E.height_samples(box, self.h) if kw.get("whether_sample_bbox_height") else [0]
                for hs, de in enumerate(hss):
                    tr = None
                    if trace:
                        tr = oracle.detect_cuboid(img, K, T, boxes, lines, oracle.default_params(**kw), trace_object=b, trace_height_sample=hs,
                                                  trace_caps=(4096, 1 << 21, 1 << 17))["trace"]
                    self.jobs.append(dict(box=box, down_expand=de, trace=tr, n_top=E.n_top_samples(box)))

    def run(self, cs, ctx, flags=0):
        ctx.set_calibration(self.K)
        ctx.L.cs_set_profiling(ctx.h, flags)
        imgs = np.stack([f[0] for f in self.frames])
        Ts = np.stack([f[1] for f in self.frames])
        out, counts = ctx.detect_batch_host(imgs, Ts, [f[2] for f in self.frames], [f[3] for f in self.frames], cs.default_params(**self.kw))
        self.check(ctx, out, counts)

    def check(self, ctx, out, counts):
        o = 0
        for f, ref in enumerate(self.refs):
            for b in range(len(self.frames[f][2])):
                assert counts[o] == len(ref["cuboids"][b]), (f, b)
                for k in range(counts[o]):
                    _compare_cuboid(out[o, k], ref["cuboids"][b][k])
                o += 1
        st = ctx.stats()
        assert st["n_candidates"] == sum(r["n_candidates"] for r in self.refs)
        assert st["n_valid"] == sum(r["n_valid"] for r in self.refs)
        for j, jb in enumerate(self.jobs):
            tr = jb["trace"]
            if tr is None:
                continue
            roi = ctx.debug_roi(j)
            assert roi["roi"] == tuple(tr["roi"]), j
            np.testing.assert_array_equal(roi["canny"], tr["canny"], err_msg="job %d" % j)
            np.testing.assert_array_equal(roi["dist"], tr["dist"], err_msg="job %d" % j)
            assert (roi["n_lines_roi"], roi["n_lines_merged"]) == (tr["n_lines_roi"], tr["n_lines_merged"]), j
            np.testing.assert_array_equal(roi["merged_lines"], tr["merged_lines"], err_msg="job %d" % j)
            cand = ctx.debug_candidates(j)
            assert cand["n"] == tr["n_candidates"], j
            np.testing.assert_array_equal(np.nonzero(cand["valid"])[0], tr["cand_index"], err_msg="job %d" % j)
            np.testing.assert_allclose(cand["dist_err"][tr["cand_index"]], tr["rows"][:, 4], rtol=1e-13, atol=0)
            np.testing.assert_array_equal(cand["angle_err"][tr["cand_index"]], tr["rows"][:, 5])


def _border_batches(oracle, kw):
    """Per frame size: every border, fractional, small and narrow box of E's two frames of that size, ten boxes to a frame, so that each
    launch mixes clamped and unclamped ROIs, several distance-transform width classes and jobs without a candidate."""
    rng = np.random.default_rng(7)
    by_size = {}
    for tag, img, K, T, obj, lines in E.base_frames():
        h, w = img.shape[:2]
        boxes = [bb for _, bb in E.border_boxes(obj, w, h) + E.small_boxes(w, h, rng)]
        perm = np.random.default_rng(len(boxes)).permutation(len(boxes))   # spread the narrow boxes over the frames
        boxes = [boxes[i] for i in perm]
        for i in range(0, len(boxes), 10):
            by_size.setdefault((w, h), [K, []])[1].append((img, T, np.array(boxes[i:i + 10]), lines))
    return {k: Batch(oracle, K, frames, kw) for k, (K, frames) in by_size.items()}


@pytest.mark.parametrize("mode,kw", (("default", dict(max_cuboid_num=2)), ("height", dict(whether_sample_bbox_height=1, max_cuboid_num=2))))
def test_border_and_small_boxes(cs, oracle, mode, kw):
    """Default kernels, the raster-scan DT (bit 5), the cone DT with global bit planes (bit 6) and TMA-staged Canny tiles (bit 9)."""
    batches = _border_batches(oracle, kw)
    clamp = dict(left=0, right=0, top=0, bottom=0)
    n_no_cand = n_dup = n_neg = 0
    classes = set()
    for (w, h), bt in batches.items():
        for jb in bt.jobs:
            ul, ut, ur, ub = E.roi_of(jb["box"], w, h, jb["down_expand"], clamp=False)
            rl, rt, rr, rb = E.roi_of(jb["box"], w, h, jb["down_expand"])
            assert (rl, rt, rr - rl, rb - rt) == tuple(jb["trace"]["roi"])
            clamp["left"] += ul < 0
            clamp["top"] += ut < 0
            clamp["right"] += ur > w - 1
            clamp["bottom"] += ub > h - 1
            n_no_cand += jb["n_top"] == 0
            classes.add(next(c for c, cw in enumerate((128, 256, 384, 512, 640, 1024, 2048)) if rr - rl <= cw))
            if kw.get("whether_sample_bbox_height"):
                hs = E.height_samples(jb["box"], h)
                n_dup += hs == [0, 0]
                n_neg += min(hs) < 0
        for flags in (0, 32, 64, 512):
            ctx = cs.Context(0, w, h, len(bt.frames), 10, 4096)
            bt.run(cs, ctx, flags)
            ctx.close()
    assert all(v > 0 for v in clamp.values()), clamp
    assert n_no_cand >= 2 * len(E.NARROW_SIZES) and len(classes) >= 4, (n_no_cand, classes)
    if kw.get("whether_sample_bbox_height"):
        assert n_dup > 0 and n_neg > 0, (n_dup, n_neg)


def _dense_batches(oracle, kw):
    """Per frame size: one frame per dense set (random / dashes / odd lines), each beside a small and a narrow box."""
    by_size = {}
    for tag, img, K, T, box, lines in E.dense_cases():
        h, w = img.shape[:2]
        boxes = np.array([box, [w - 41.0, h - 31.0, 40, 30, 0.5], [3.0, 5.0, 7, 50, 0.5]])
        by_size.setdefault((w, h), [K, [], []])
        by_size[(w, h)][1].append((img, T, boxes, lines))
        by_size[(w, h)][2].append(tag)
    return {k: (Batch(oracle, K, frames, kw), tags) for k, (K, frames, tags) in by_size.items()}


@pytest.mark.parametrize("mode,kw", (("top5", dict(max_cuboid_num=5)), ("height_top5", dict(whether_sample_bbox_height=1, max_cuboid_num=5))))
def test_dense_line_sets(cs, oracle, mode, kw):
    """The warp sweep / selection kernels and the CTA-wide ones (bit 3) on ROIs with about 700 lines inside and more than 200 merged, the 500-merge cap and odd lines."""
    reached_cap = reached_cta = 0
    for (w, h), (bt, tags) in _dense_batches(oracle, kw).items():
        for f, tag in enumerate(tags):
            img, T, boxes, lines = bt.frames[f]
            if tag.endswith("_dashes"):
                l, t, r, b = E.roi_of(boxes[0], w, h)
                L = lines[[l <= min(x[0], x[2]) and max(x[0], x[2]) <= r and t <= min(x[1], x[3]) and max(x[1], x[3]) <= b for x in lines]]
                reached_cap += len(L) - len(oracle.merge_break_lines(L, len_thre=0)) == 500
        reached_cta += any(jb["trace"]["n_lines_merged"] > 64 for jb in bt.jobs)
        for flags in (0, 8):
            ctx = cs.Context(0, w, h, len(bt.frames), 4, 8192)
            bt.run(cs, ctx, flags)
            ctx.close()
    assert reached_cap == 2 and reached_cta == 2, (reached_cap, reached_cta)


def test_large_roi_global_hysteresis_and_dt(cs, oracle):
    """A whole-frame box on a 1280 x 960 frame in one launch with small boxes: k_canny_hyst iterates the large ROI's planes in global
    memory and the others' in shared memory; the large ROI's DT width class stages from global memory, the small classes do not."""
    img, K, T, boxes, lines = E.big_frame()
    h, w = img.shape[:2]
    frames = [(img, T, np.array([[0.0, 0, w - 1, h - 1, 0.9], [5, 7, 60, 40, 0.5], [w - 80.0, h - 50, 70, 40, 0.5]]), lines),
              (img, T, np.array([[100.0, 400, 1100, 90, 0.9], boxes[0], [600, 0, 8, 30, 0.5]]), lines)]
    bt = Batch(oracle, K, frames, dict(max_cuboid_num=3))
    words = [(jb["trace"]["roi"][3] + 2) * ((jb["trace"]["roi"][2] + 31) // 32 + 2) for jb in bt.jobs]
    assert max(words) > HY_SMEM_PLANE_WORDS > min(words) and max(words) > DT_SMEM_PLANE_WORDS, words
    ctx = cs.Context(0, w, h, 2, 4, 4096)
    for flags in (0, 8):
        bt.run(cs, ctx, flags)
    ctx.close()


def test_global_memory_fuse_sort(cs, oracle):
    """Roll / pitch sampling with a 2 degree yaw step on a large object box: more than FU_SMEM_SORT valid proposals, so k_fuse_rank sorts
    in global memory; a whole-frame box (few valid proposals: its sorts stay in shared memory) rides along.  One box per frame: no pose
    is carried from box to box."""
    img, K, T, boxes, lines = E.big_frame()
    h, w = img.shape[:2]
    frames = [(img, T, boxes[:1], lines), (img, T, np.array([[0.0, 0, w - 1, h - 1, 0.9]]), lines)]
    bt = Batch(oracle, K, frames, dict(whether_sample_cam_roll_pitch=1, yaw_step_deg=2.0, max_cuboid_num=4), trace=False)
    assert bt.refs[0]["n_valid"] > FU_SMEM_SORT >= bt.refs[1]["n_valid"], (bt.refs[0]["n_valid"], bt.refs[1]["n_valid"])
    ctx = cs.Context(0, w, h, 2, 4, 4096)
    for flags in (0, 8):
        bt.run(cs, ctx, flags)
    ctx.close()


def test_per_roi_line_capacities(cs, oracle):
    """1024 lines inside one ROI and 256 merged lines return the oracle's records; one more of either fails with CS_ERR_CAPACITY
    naming the limit; the next batch on the same context is correct again (the error word is reset per run)."""
    cases = {tag: (img, K, T, box, lines) for tag, img, K, T, box, lines in E.capacity_cases()}
    img, K, T, box, lines = cases["cap1024_256"]
    h, w = img.shape[:2]
    good = Batch(oracle, K, [(img, T, box[None], lines), (img, T, np.array([[4.0, 4, 6, 20, 0.5]]), lines)], dict(max_cuboid_num=3))
    assert (good.jobs[0]["trace"]["n_lines_roi"], good.jobs[0]["trace"]["n_lines_merged"]) == (1024, 256)
    ctx = cs.Context(0, w, h, 2, 4, 4096)
    for flags in (0, 8):
        good.run(cs, ctx, flags)
        for tag, limit in (("cap1025_200", 1024), ("cap1000_257", 256)):
            img2, _, T2, box2, lines2 = cases[tag]
            tr = oracle.detect_cuboid(img2, K, T2, box2[None], lines2, trace_object=0)["trace"]
            assert (tr["n_lines_roi"], tr["n_lines_merged"]) == tuple(int(v) for v in tag[3:].split("_"))
            with pytest.raises(cs.CubeSlamError) as ei:
                ctx.detect_batch_host(np.stack([img2, img2]), np.stack([T2, T2]), [box2[None], box2[None]], [lines2, lines2],
                                      cs.default_params(max_cuboid_num=3))
            assert "CS_ERR_CAPACITY" in str(ei.value) and ("%d" % limit) in str(ei.value), str(ei.value)
            good.run(cs, ctx, flags)
    ctx.close()
