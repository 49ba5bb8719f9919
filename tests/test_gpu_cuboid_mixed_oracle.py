"""The cuboid batch over frames of different sizes and cameras (cs_detect_cuboids_batch_mixed, cs_detect_frames_batch_mixed, upload_mixed)
against the CPU oracle, stage by stage.

tests/test_gpu_cuboid_mixed_sizes.py compares the mixed call with the one-size call; both run the same per-frame tables (build_tables), the
same gray-plane addressing (CsJob::gray_off / gray_pitch) and the same Canny, distance-transform and sweep kernels, so a bug there cancels
out.  Here every expected value comes from oracle/pyoracle.py, run on each frame alone with that frame's own K and size, one box per call
(the product starts every box from the frame's raw pose): records, counts, the batch's candidate and valid totals and, per ROI job, the
ROI, Canny map, distance map, lines inside the ROI, merged lines and the valid candidates' errors.

The frame set puts the per-frame table where it can go wrong: frames at the context's maximum and one pixel below it, 3-channel rows that
are not a multiple of 16 bytes, gray frames whose planes start at odd offsets, a padded gray frame of odd width and a padded 3-channel
frame (both repacked by the upload), a crop view with its principal point moved, a 97 x 61 frame, KITTI-shaped frames, frames without
boxes, K with off-centre principal points and skew, boxes against each frame edge, small boxes, ROI widths either side of a
distance-transform width class and boxes where the height-sample clamp binds.  Each test asserts from its own inputs that these are there."""
import ctypes as C

import numpy as np
import pytest

import test_oracle_ref_cuboid_edges as E

pytestmark = pytest.mark.gpu

MAX_W, MAX_H = 1280, 960
TRACE_CAPS = (4096, 1 << 21, 1 << 17)
DT_CLASS_WIDTHS = (128, 256, 384, 512, 640, 1024, 2048)   # cs_dt_class_width
SETTINGS = {
    "default": dict(),
    "roll_pitch": dict(whether_sample_cam_roll_pitch=1),
    "bbox_height": dict(whether_sample_bbox_height=1, max_cuboid_num=5),
}
TRACED = ("default", "bbox_height")   # roll / pitch sampling: records only
TINY_LINES = [[5, 5, 60, 8], [10, 50, 90, 20], [80, 2, 82, 58], [3, 30, 40, 55], [20, 10, 75, 52]]   # few renders' segments fit 97 x 61


# ------------------------------------------------------------------------------------------- frames
def _render(seed, w, h, n_boxes, kind="indoor"):
    from cube_slam_b200 import synthetic as S
    img, T, boxes, lines, K = S.make_frame(np.random.default_rng(seed), w, h, n_boxes, kind)
    return dict(img=img, T=T, boxes=boxes, lines=lines, K=K)


def cam(K, fx=1.0, fy=1.0, dcx=0.0, dcy=0.0, skew=0.0):
    """K with its focal lengths scaled, its principal point moved and K[0, 1] set"""
    K = np.array(K, np.float64).reshape(3, 3).copy()
    K[0, 0] *= fx
    K[1, 1] *= fy
    K[0, 2] += dcx
    K[1, 2] += dcy
    K[0, 1] = skew
    return K


def lines_inside(lines, x0, y0, w, h, min_len=15.0):
    """the segments of a parent frame clipped to the crop (x0, y0, w, h) (Liang-Barsky), in the crop's coordinates; those left longer
    than min_len"""
    out = []
    for x1, y1, x2, y2 in np.asarray(lines, np.float64).reshape(-1, 4) - np.array([x0, y0, x0, y0], np.float64):
        dx, dy = x2 - x1, y2 - y1
        t0, t1 = 0.0, 1.0
        for p, q in ((-dx, x1), (dx, w - 1 - x1), (-dy, y1), (dy, h - 1 - y1)):
            if p == 0:
                t0, t1 = (t0, t1) if q >= 0 else (1.0, 0.0)
            elif p < 0:
                t0 = max(t0, q / p)
            else:
                t1 = min(t1, q / p)
        if t0 <= t1 and (t1 - t0) * np.hypot(dx, dy) > min_len:
            out.append([x1 + t0 * dx, y1 + t0 * dy, x1 + t1 * dx, y1 + t1 * dy])
    out = np.asarray(out, np.float64).reshape(-1, 4)
    out[:, [0, 2]] = np.clip(out[:, [0, 2]], 0, w - 1)
    out[:, [1, 3]] = np.clip(out[:, [1, 3]], 0, h - 1)
    return out


def boxes_inside(boxes, x0, y0, w, h):
    B = np.asarray(boxes, np.float64).reshape(-1, 5) - np.array([x0, y0, 0, 0, 0], np.float64)
    keep = (B[:, 0] >= 0) & (B[:, 1] >= 0) & (B[:, 0] + B[:, 2] <= w - 1) & (B[:, 1] + B[:, 3] <= h - 1)
    return B[keep]


def frame(name, img, T, K, boxes, lines, pad=0, rows=None, x0=0):
    """one frame: the image as the oracle sees it (contiguous) and the bytes the device call is given -- `rows` (h x stride) with the
    frame's first pixel at byte x0 of the first row; by default the image itself, `pad` filler bytes after each row"""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    if rows is None:
        rows = img.reshape(h, w * ch)
        if pad:
            rows = np.concatenate([rows, np.full((h, pad), 77, np.uint8)], axis=1)
    rows = np.ascontiguousarray(rows)
    assert (rows[:, x0:x0 + w * ch].reshape(img.shape) == img).all()
    return dict(name=name, img=img, T=np.asarray(T, np.float64).reshape(16), K=np.asarray(K, np.float64).reshape(3, 3),
                boxes=np.asarray(boxes, np.float64).reshape(-1, 5), lines=np.asarray(lines, np.float64).reshape(-1, 4), rows=rows, x0=x0)


def crop(name, R, x0, y0, w, h, boxes, gray=False, K=None, view=False, pad=0, lines=None):
    """a w x h crop of render R at (x0, y0), its principal point moved with it, with R's segments that lie inside it (or `lines`); view:
    handed to the device as a view into R's rows"""
    img = R["img"][y0:y0 + h, x0:x0 + w]
    K = cam(R["K"], dcx=-x0, dcy=-y0) if K is None else K
    rows, bx0 = None, 0
    if gray:
        img = img[..., 1]
    if view:
        assert not gray and not pad
        rows, bx0 = R["img"][y0:y0 + h].reshape(h, -1), 3 * x0
    lines = lines_inside(R["lines"], x0, y0, w, h) if lines is None else lines
    return frame(name, img, R["T"], K, boxes, lines, pad=pad, rows=rows, x0=bx0)


def whole(name, R, boxes=None, gray=False, K=None, pad=0):
    img = R["img"][..., 1] if gray else R["img"]
    return frame(name, img, R["T"], R["K"] if K is None else K, R["boxes"] if boxes is None else boxes, R["lines"], pad=pad)


def _cat(*b):
    return np.concatenate([np.asarray(x, np.float64).reshape(-1, 5) for x in b])


def _set_24(fixture_a, fixture_b):
    """23 frames of 13 sizes, 3-channel and gray, sizes interleaved in call order"""
    A = _render(101, 1280, 960, 3)
    B = _render(102, 1279, 959, 3)
    Cr = _render(103, 641, 479, 3)
    D = _render(104, 1242, 375, 4, "kitti")
    Ek = _render(105, 1242, 375, 3, "kitti")
    F = _render(106, 640, 480, 3)
    G = _render(107, 800, 600, 3)
    fa = fixture_a
    fb_img, fb_boxes = fixture_b["frames"][7]
    return [
        # the context's maximum: DT class boundary 256 / 257 (216 and 217 px wide boxes), the right edge, a bottom box whose height samples
        # are clamped by the frame's height (t + h = H - 16)
        whole("max_bgr", A, boxes=_cat(A["boxes"], [[400, 100, 216, 300, .9], [701, 500, 217, 300, .8], [1100, 300, 179, 200, .7],
                                                    [201, 700, 150, 244, .6]])),
        # 333 x 201 gray: the plane after it starts at an odd offset; boxes against the left and top edges, 108 / 109 px wide (ROI 128 / 129)
        crop("g333_a", Cr, 150, 140, 333, 201, [[0, 0, 60, 45, .9], [141, 31, 108, 150, .8], [31, 20, 109, 150, .7]], gray=True),
        whole("kitti_a", D, K=cam(D["K"], 1.03, 0.98, 7.5, -4.25)),
        # padded gray of odd width: stride = width + 13, a box against its right edge with an odd left edge
        crop("pad_gray", G, 201, 151, 415, 297, [[301, 41, 113, 200, .9], [17, 9, 150, 130, .6]], gray=True, pad=13),
        whole("max_m1", B, boxes=_cat(B["boxes"], [[1001, 757, 277, 201, .5]]), K=cam(B["K"], 0.97, 1.02, -11, 9, skew=0.8)),
        whole("no_boxes_a", F, boxes=np.zeros((0, 5))),
        # 641 x 479 BGR: rows of 1923 bytes (no TMA staging); a box against the top edge
        whole("bgr641", Cr, boxes=_cat(Cr["boxes"], [[51, 0, 130, 140, .9]]), K=cam(Cr["K"], 1.1, 1.1, 13, 6)),
        # 97 x 61: one box covering most of it (its ROI clamps on all four sides)
        crop("tiny_bgr", F, 383, 141, 97, 61, [[4, 3, 88, 55, .9]], lines=TINY_LINES),
        # 3-channel rows padded by 5 bytes: 1925-byte rows
        whole("pad_bgr", F, pad=5, K=cam(F["K"], 0.95, 0.96, -20, 15)),
        # a crop view: offset into the parent's rows, the parent's stride
        crop("crop_view", G, 37, 23, 561, 409, _cat(boxes_inside(G["boxes"], 37, 23, 561, 409), [[13, 17, 222, 180, .9]]), view=True),
        whole("kitti_gray", Ek, gray=True, K=cam(Ek["K"], 0.9, 0.92, -30, 11)),
        # a box against the right edge with a clamped height sample, one against the bottom edge
        crop("g333_b", Cr, 20, 10, 333, 201, [[232, 60, 100, 125, .7], [5.5, 150.2, 40, 50.8, .6]], gray=True, K=cam(Cr["K"], 1.2, 1.15, -40, -7)),
        frame("fixture_a", fa["img"], fa["T"], fa["K"], fa["boxes"], fa["lines"]),
        whole("no_boxes_kitti", D, boxes=np.zeros((0, 5))),
        crop("bgr477", A, 500, 400, 477, 355, [[3, 200, 140, 154, .9], [333, 7, 143, 121, .8]]),
        # small boxes (ROI expansion 10 px) against the edges of a small frame
        crop("small_bgr", G, 300, 200, 200, 150, [[0, 100, 30, 49, .9], [170, 0, 29, 25, .8], [61, 40, 50, 40, .7]],
             K=cam(G["K"], 1.0, 1.0, -300 + 17, -200 - 9, skew=-1.5)),
        frame("fixture_b", fb_img, fixture_b["T"], cam(fixture_b["K"], 1.04, 1.0, 3, -2), fb_boxes[:3], fa["lines"]),
        whole("max_gray", A, gray=True, boxes=_cat(A["boxes"][:2], [[0, 901, 300, 58, .5]]), K=cam(A["K"], 1.05, 1.01, 21, -13)),
        crop("g512", B, 101, 99, 512, 384, [[11, 21, 199, 250, .9], [400, 250, 111, 133, .8]], gray=True),
        whole("kitti_b", Ek, K=cam(Ek["K"], 1.0, 1.0, 0, 0, skew=2.0)),
        crop("no_boxes_g333", Cr, 300, 270, 333, 201, np.zeros((0, 5)), gray=True),
        crop("tiny_gray", F, 260, 130, 97, 61, [[0, 0, 96, 60, .9]], gray=True, lines=TINY_LINES),
        whole("gray641", Cr, gray=True, boxes=Cr["boxes"][:2], K=cam(Cr["K"], 0.93, 0.99, -17, 21)),
    ]


def _set_64():
    """64 frames of 16 sizes (each size four times, interleaved), crops of larger renders with random boxes, every third one gray"""
    sizes = ((1280, 960), (1279, 959), (1242, 375), (1001, 701), (800, 600), (730, 530), (641, 479), (640, 480), (561, 409), (512, 384),
             (477, 355), (415, 297), (333, 201), (200, 150), (161, 121), (97, 61))
    big = [_render(201, 1280, 960, 3), _render(202, 1280, 960, 4)]
    kitti = _render(203, 1242, 375, 4, "kitti")
    rng = np.random.default_rng(64)
    out = []
    for i in range(64):
        w, h = sizes[(i * 7) % 16]
        R = kitti if (w, h) == (1242, 375) else big[i % 2]
        x0, y0 = int(rng.integers(0, R["img"].shape[1] - w + 1)), int(rng.integers(0, R["img"].shape[0] - h + 1))
        boxes = list(boxes_inside(R["boxes"], x0, y0, w, h)[:2])
        for _ in range(0 if i % 5 == 4 else int(rng.integers(1, 3))):
            bw, bh = int(rng.integers(12, min(w - 1, 320))), int(rng.integers(12, min(h - 1, 320)))
            bx, by = int(rng.integers(0, w - bw)), int(rng.integers(0, h - bh))
            boxes.append([bx + rng.uniform(0, 0.9), by + rng.uniform(0, 0.9), bw, bh, 0.5])
        if i % 5 == 4:
            boxes = []
        K = cam(R["K"], rng.uniform(0.9, 1.1), rng.uniform(0.9, 1.1), -x0 + rng.uniform(-25, 25), -y0 + rng.uniform(-25, 25),
                skew=0.7 if i % 4 == 1 else 0.0)
        out.append(crop("f%02d_%dx%d" % (i, w, h), R, x0, y0, w, h, np.asarray(boxes, np.float64).reshape(-1, 5), gray=i % 3 == 1, K=K))
    return out


@pytest.fixture(scope="module")
def set24(fixture_a, fixture_b):
    return _set_24(fixture_a, fixture_b)


@pytest.fixture(scope="module")
def set64():
    return _set_64()


# ------------------------------------------------------------------------------------------- the oracle side (CPU only)
def n_jobs(box, img_h, kw):
    return len(E.height_samples(box, img_h)) if kw.get("whether_sample_bbox_height") else 1


def expect(oracle, frs, kw, lines_of=None, trace="all"):
    """The oracle's answer for a batch: per box (batch order) its records, the candidate / valid totals and, per ROI job in the order
    build_tables emits them (frame, box, height sample), its trace (None where not traced).  trace: "all", "first" (hs 0 of each frame's
    first box) or None.  lines_of(f): the lines frame f is detected with (default: its given lines)."""
    recs, jobs, n_cand, n_valid = [], [], 0, 0
    for f, fr in enumerate(frs):
        img, h = fr["img"], fr["img"].shape[0]
        lines = fr["lines"] if lines_of is None else lines_of(f)
        for b, box in enumerate(fr["boxes"]):
            nj = n_jobs(box, h, kw)
            for hs in range(nj):
                want = trace == "all" or (trace == "first" and b == 0 and hs == 0)
                if hs > 0 and not want:
                    jobs.append(None)
                    continue
                r = oracle.detect_cuboid(img, fr["K"], fr["T"].reshape(4, 4), box[None], lines, oracle.default_params(**kw),
                                         trace_object=0 if want else None, trace_height_sample=hs, trace_caps=TRACE_CAPS)
                if hs == 0:
                    recs.append(r["cuboids"][0])
                    n_cand += r["n_candidates"]
                    n_valid += r["n_valid"]
                jobs.append(r["trace"])
    return dict(recs=recs, jobs=jobs, n_cand=n_cand, n_valid=n_valid)


# ------------------------------------------------------------------------------------------- the device side
def new_ctx(max_frames=32):
    import cube_slam_b200 as cs
    return cs.Context(0, MAX_W, MAX_H, max_frames, 16, 4096)


def line_params(ctx, use_LSD):
    from cube_slam_b200 import _lib
    p = _lib.LineParams()
    ctx.L.cs_default_line_params(C.byref(p))
    p.use_LSD, p.line_length_thres = use_LSD, 15.0
    return p


def pack(frs):
    """the frames' bytes in one buffer with their cs_frame_views (strides, crop views and padding as each frame was given)"""
    from cube_slam_b200 import _lib
    views = (_lib.FrameView * len(frs))()
    parts, off = [], 0
    for i, f in enumerate(frs):
        h, w = f["img"].shape[:2]
        views[i].offset, views[i].width, views[i].height = off + f["x0"], w, h
        views[i].stride, views[i].channels = f["rows"].shape[1], 1 if f["img"].ndim == 2 else 3
        parts.append(f["rows"].reshape(-1))
        off += f["rows"].size
    return np.ascontiguousarray(np.concatenate(parts)), views


def tables(frs):
    Ts = np.ascontiguousarray(np.stack([f["T"] for f in frs]))
    Ks = np.ascontiguousarray(np.stack([f["K"].reshape(9) for f in frs]))
    box_off = np.concatenate([[0], np.cumsum([len(f["boxes"]) for f in frs])]).astype(np.int32)
    line_off = np.concatenate([[0], np.cumsum([len(f["lines"]) for f in frs])]).astype(np.int32)
    boxes = np.ascontiguousarray(np.concatenate([f["boxes"] for f in frs] + [np.zeros((1, 5))]))
    lines = np.ascontiguousarray(np.concatenate([f["lines"] for f in frs] + [np.zeros((1, 4))]))
    return Ts, Ks, box_off, line_off, boxes, lines


def mixed(ctx, frs, prm, mode="lines"):
    """cs_detect_cuboids_batch_mixed ("lines") or cs_detect_frames_batch_mixed ("lsd", "edlines") through the C ABI -> (records, counts)"""
    from cube_slam_b200 import _lib
    d = lambda a: _lib.ptr(a, C.c_double)
    buf, views = pack(frs)
    Ts, Ks, box_off, line_off, boxes, lines = tables(frs)
    n = int(box_off[-1])
    rec, cnt = np.zeros((max(n, 1), prm.max_cuboid_num), _lib.CUBOID_DTYPE), np.zeros(max(n, 1), np.int32)
    head = [ctx.h, buf.ctypes.data, views, len(frs), d(Ks), d(Ts), d(boxes), _lib.ptr(box_off, C.c_int32)]
    tail = [C.byref(prm), rec.ctypes.data, _lib.ptr(cnt, C.c_int32)]
    if mode == "lines":
        rc = ctx.L.cs_detect_cuboids_batch_mixed(*(head + [d(lines), _lib.ptr(line_off, C.c_int32)] + tail))
    else:
        rc = ctx.L.cs_detect_frames_batch_mixed(*(head + [C.byref(line_params(ctx, mode == "lsd"))] + tail))
    ctx.check(rc)
    return rec[:n], cnt[:n]


# ------------------------------------------------------------------------------------------- comparisons
def check_records(rec, cnt, want, label=""):
    from test_gpu_cuboid_edges import _compare_cuboid
    assert len(cnt) == len(want["recs"]), label
    for o, ref in enumerate(want["recs"]):
        assert cnt[o] == len(ref), (label, o)
        for k in range(cnt[o]):
            _compare_cuboid(rec[o, k], ref[k])


def check_stats(ctx, want, label=""):
    st = ctx.stats()
    assert st["n_roi_jobs"] == len(want["jobs"]), label
    assert st["n_candidates"] == want["n_cand"] and st["n_valid"] == want["n_valid"], (label, st, want["n_cand"], want["n_valid"])


def check_job(ctx, j, tr, label="", candidates=True):
    roi = ctx.debug_roi(j)
    assert roi["roi"] == tuple(tr["roi"]), (label, j)
    np.testing.assert_array_equal(roi["canny"], tr["canny"], err_msg="%s job %d canny" % (label, j))
    np.testing.assert_array_equal(roi["dist"], tr["dist"], err_msg="%s job %d dist" % (label, j))
    assert (roi["n_lines_roi"], roi["n_lines_merged"]) == (tr["n_lines_roi"], tr["n_lines_merged"]), (label, j)
    np.testing.assert_array_equal(roi["merged_lines"], tr["merged_lines"], err_msg="%s job %d merged lines" % (label, j))
    if candidates:
        cand = ctx.debug_candidates(j)
        assert cand["n"] == tr["n_candidates"], (label, j)
        np.testing.assert_array_equal(np.nonzero(cand["valid"])[0], tr["cand_index"], err_msg="%s job %d valid set" % (label, j))
        np.testing.assert_allclose(cand["dist_err"][tr["cand_index"]], tr["rows"][:, 4], rtol=1e-13, atol=0)
        np.testing.assert_array_equal(cand["angle_err"][tr["cand_index"]], tr["rows"][:, 5])


def check_traces(ctx, want, label="", candidates=True):
    n = 0
    for j, tr in enumerate(want["jobs"]):
        if tr is not None:
            check_job(ctx, j, tr, label, candidates)
            n += 1
    return n


# ------------------------------------------------------------------------------------------- what the inputs cover
def coverage(frs, kw):
    """from the inputs alone: what the batch's per-frame table meets"""
    cov = dict(sizes=set(), clamp=dict(left=0, right=0, top=0, bottom=0), small=0, classes=set(), widths=set(), odd_left=0, height_clamp=0,
               odd_gray_plane=0, unaligned_rows=0, repacked=0, skew=0, at_max=0, no_boxes=0, jobs=0)
    off = 0   # the mixed upload packs the frames back to back in call order; a gray frame is then read in place
    for f in frs:
        img = f["img"]
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else 3
        cov["sizes"].add((w, h))
        cov["odd_gray_plane"] += ch == 1 and off % 2 == 1
        cov["unaligned_rows"] += ch == 3 and (w * ch) % 16 != 0
        cov["repacked"] += f["rows"].shape[1] != w * ch
        cov["skew"] += f["K"][0, 1] != 0
        cov["at_max"] += (w, h) == (MAX_W, MAX_H)
        cov["no_boxes"] += len(f["boxes"]) == 0
        off += w * h * ch
        for box in f["boxes"]:
            cov["jobs"] += n_jobs(box, h, kw)
            ul, ut, ur, ub = E.roi_of(box, w, h, 0, clamp=False)
            l, t, r, b = E.roi_of(box, w, h, 0)
            cov["clamp"]["left"] += ul < 0
            cov["clamp"]["top"] += ut < 0
            cov["clamp"]["right"] += ur > w - 1
            cov["clamp"]["bottom"] += ub > h - 1
            cov["small"] += min(int(box[2]), int(box[3])) < 110
            cov["widths"].add(r - l)
            cov["classes"].add(next(c for c, cw in enumerate(DT_CLASS_WIDTHS) if r - l <= cw))
            cov["odd_left"] += l % 2 == 1
            bt, bh = int(box[1]), int(box[3])
            cov["height_clamp"] += h - bt - bh - 1 < max(min(20, bh - 90), 20)
    return cov


def _groups(frs):
    """EDLines' size groups in the mixed layout: (width, height, channels) in order of first appearance"""
    keys = [(f["img"].shape[1], f["img"].shape[0], f["img"].ndim) for f in frs]
    return list(dict.fromkeys(keys)), keys


# ------------------------------------------------------------------------------------------- tests
_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def test_frame_set_covers_the_table(set24):
    cov = coverage(set24, dict(whether_sample_bbox_height=1))
    assert len(set24) >= 20 and len(cov["sizes"]) >= 12, cov["sizes"]
    assert all(v > 0 for v in cov["clamp"].values()), cov["clamp"]
    assert {128, 129, 256, 257} <= cov["widths"] and len(cov["classes"]) >= 4, (cov["widths"], cov["classes"])
    for k in ("small", "odd_left", "height_clamp", "odd_gray_plane", "unaligned_rows", "skew", "at_max", "no_boxes"):
        assert cov[k] > 0, k
    assert cov["repacked"] >= 3   # the padded gray, the padded 3-channel frame and the crop view
    assert (MAX_W - 1, MAX_H - 1) in cov["sizes"] and (97, 61) in cov["sizes"] and (1242, 375) in cov["sizes"]
    ks = {tuple(np.round(f["K"].reshape(9), 9)) for f in set24}
    assert len(ks) >= 15


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_records_and_traces(set24, oracle, setting):
    """every box's records and counts, the batch's candidate / valid totals and (default, bbox_height) every ROI job's stage trace"""
    import cube_slam_b200 as cs
    kw = SETTINGS[setting]
    want = _cached(("set24", setting), lambda: expect(oracle, set24, kw, trace="all" if setting in TRACED else None))
    assert len(want["jobs"]) == coverage(set24, kw)["jobs"]
    ctx = new_ctx()
    try:
        rec, cnt = mixed(ctx, set24, cs.default_params(**kw))
        check_stats(ctx, want, setting)
        check_records(rec, cnt, want, setting)
        n = check_traces(ctx, want, setting)
        assert n == (len(want["jobs"]) if setting in TRACED else 0)
        assert cnt.sum() > 0
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", ("lsd", "edlines"))
def test_online_line_detectors(set24, oracle, mode):
    """cs_detect_frames_batch_mixed: each frame's lines are what the oracle's detector finds on that frame alone (line_length_thres 15),
    fed to detect_cuboid; records, counts, totals and, per frame, the first box's ROI trace with its merged lines"""
    import cube_slam_b200 as cs
    detect = oracle.lsd_detect if mode == "lsd" else oracle.edl_detect
    lines = _cached(("lines", mode), lambda: [detect(f["img"], 15.0)["lines"].astype(np.float64) for f in set24])
    want = _cached(("online", mode), lambda: expect(oracle, set24, {}, lines_of=lambda f: lines[f], trace="first"))
    if mode == "edlines":
        groups, keys = _groups(set24)
        order = [i for g in groups for i, k in enumerate(keys) if k == g]
        assert len(groups) >= 4 and order != sorted(order) and any(g[2] == 2 for g in groups), groups
        assert min(min(f["img"].shape[:2]) for f in set24) >= 8
    assert sum(len(l) for l in lines) > 0
    ctx = new_ctx()
    try:
        rec, cnt = mixed(ctx, set24, cs.default_params(), mode)
        check_stats(ctx, want, mode)
        check_records(rec, cnt, want, mode)
        n = check_traces(ctx, want, mode)
        assert n == sum(len(f["boxes"]) > 0 for f in set24)
    finally:
        ctx.close()


def test_full_batch_two_in_flight(set64, oracle):
    """64 frames of 16 sizes at max_frames = 64 on two contexts, the second in reverse order, both run_async before either fetch: every
    box's records against the oracle, and the first box's ROI trace of every frame"""
    import cube_slam_b200 as cs
    assert len(set64) == 64 and len({f["img"].shape[:2] for f in set64}) == 16
    prm = cs.default_params()
    batches = (set64, set64[::-1])
    wants = [_cached(("set64", k), lambda b=b: expect(oracle, b, {}, trace="first")) for k, b in enumerate(batches)]
    ctxs = [new_ctx(64), new_ctx(64)]
    try:
        for c, b in zip(ctxs, batches):
            c.upload_mixed([f["img"] for f in b], np.stack([f["T"] for f in b]), [f["boxes"] for f in b], [f["lines"] for f in b], prm,
                           K=np.stack([f["K"] for f in b]))
        for c in ctxs:
            c.run_async()
        for k, (c, w) in enumerate(zip(ctxs, wants)):
            rec, cnt = c.fetch()
            check_records(rec, cnt, w, "batch %d" % k)
            check_stats(c, w, "batch %d" % k)
        for k, (c, w) in enumerate(zip(ctxs, wants)):
            assert check_traces(c, w, "batch %d" % k, candidates=False) == sum(len(f["boxes"]) > 0 for f in set64)
    finally:
        for c in ctxs:
            c.close()


def _one_size_sets():
    """one-size batches whose gray planes are not the frames: padded gray of odd width (stride = width + 13) and 3-channel frames of
    odd w * h * 3 bytes (every other frame, and its gray plane, at an odd offset)"""
    G = _render(301, 800, 600, 3)
    gray = [crop("pg%d" % i, G, x, y, 415, 297, [[301, 41, 113, 200, .9], [31 + i, 9, 150, 130, .6]], gray=True, pad=13, K=G["K"])
            for i, (x, y) in enumerate(((201, 151), (0, 0), (385, 303)))]
    bgr = [crop("ob%d" % i, _render(302 + i, 641, 479, 3), 250, 200, 333, 201, [[1 + 2 * i, 11, 180, 185, .8], [151, 40, 181, 140, .7]])
           for i in range(3)]
    return dict(padded_gray=gray, odd_bgr=bgr)


@pytest.mark.parametrize("kind", ("padded_gray", "odd_bgr"))
def test_one_size_gray_plane(oracle, kind):
    """cs_detect_cuboids_batch (one size, cs_launch_gray into d_img + gray_base, k_canny_nms through gray_off / gray_pitch): records, and
    every ROI job's trace"""
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    frs = _one_size_sets()[kind]
    h, w = frs[0]["img"].shape[:2]
    ch = 1 if frs[0]["img"].ndim == 2 else 3
    stride = frs[0]["rows"].shape[1]
    assert stride > w if kind == "padded_gray" else (w * h * 3) % 2 == 1 and w % 2 == 1
    for kw in ({}, dict(whether_sample_bbox_height=1, max_cuboid_num=3)):
        want = expect(oracle, frs, kw)
        prm = cs.default_params(**kw)
        buf = np.ascontiguousarray(np.concatenate([f["rows"].reshape(-1) for f in frs]))
        Ts, _, box_off, line_off, boxes, lines = tables(frs)
        n = int(box_off[-1])
        rec, cnt = np.zeros((n, prm.max_cuboid_num), _lib.CUBOID_DTYPE), np.zeros(n, np.int32)
        ctx = new_ctx(4)
        try:
            ctx.set_calibration(frs[0]["K"])
            d = lambda a: _lib.ptr(a, C.c_double)
            ctx.check(ctx.L.cs_detect_cuboids_batch(ctx.h, buf.ctypes.data, len(frs), w, h, stride, ch, d(Ts), d(boxes), _lib.ptr(box_off, C.c_int32),
                                                    d(lines), _lib.ptr(line_off, C.c_int32), C.byref(prm), rec.ctypes.data, _lib.ptr(cnt, C.c_int32)))
            check_stats(ctx, want, kind)
            check_records(rec, cnt, want, kind)
            assert check_traces(ctx, want, kind) == len(want["jobs"])
        finally:
            ctx.close()
