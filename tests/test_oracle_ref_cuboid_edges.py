"""The cuboid stage at the image borders, on small boxes and on dense line sets up to its per-ROI capacities: the oracle against the
reference's own detect_3d_cuboid::detect_cuboid (oracle/_ref/libcuboid_ref.so, libm atan2), field for field.

The input set is built here, deterministically, and tests/test_gpu_cuboid_edges.py runs the same inputs on the device:
  * border boxes: each object of a synthetic VGA and KITTI frame moved flush against the left, right, top and bottom edges and 15 px past
    each (the ROI clamps of box_proposal_detail.cpp:155-161 fire; at the bottom, height sampling gives the duplicate sample {0, 0} and
    the negative sample {0, -15});
  * boxes with fractional and negative coordinates (truncated to int as the reference truncates them);
  * small boxes, 10-100 px a side (distance-map margin 10, ROIs smaller than one 32 x 32 Canny tile), and boxes narrower than 10 px
    (no top-x sample: zero candidates);
  * dense line sets added to real object boxes: 640 short random segments, dashes long enough to reach merge_break_lines' 500-merge cap,
    lines on the inclusive ROI border / right to left / vertical / zero-length / duplicated, and sets with exactly 1024 lines inside the
    ROI and exactly 256 merged lines (the product's per-ROI capacities), plus one more of each.

Where the two sides differ, the run counts as a classified divergence only if the test proves it is a tie the reference breaks by an
unspecified order: every rank the two disagree on has the same combined-score key (equal, or both NaN), or the reference's pick is
NaN-scored (the oracle ranks NaN last).  DESIGN.md section 2 calls these defined behaviours where the reference is undefined.
Boxes narrower than 10 px are not given to the reference: its linespace divides by a zero step there (SIGFPE)."""
import numpy as np
import pytest

FIELDS = ("pos", "rotY", "scale", "box_config_type", "box_corners_2d", "box_corners_3d_world", "rect_detect_2d", "edge_distance_error",
          "edge_angle_error", "normalized_error", "skew_ratio", "down_expand_height", "camera_roll_delta", "camera_pitch_delta")
PAST = 15          # px a border box reaches past the image edge
MAX_CLASSIFIED = 12  # classified divergences allowed over all runs of this file (a small minority of them)


# ------------------------------------------------------------------------------------------- inputs (shared with the GPU file)
def roi_of(box, img_w, img_h, down_expand=0, clamp=True):
    """The ROI box_proposal_detail.cpp:155-161 cuts for one box and height sample: (left, top, right, bottom), all inclusive; with
    clamp=False, before it is clipped to the image."""
    l, t = int(box[0]), int(box[1])
    w, h = int(box[2]), int(box[3])
    r = int(l + box[2])
    he = h + down_expand
    e = min(max(min(20, w - 100), 10), max(min(20, he - 100), 10))
    if not clamp:
        return l - e, t - e, r + e, t + he + e
    return max(0, l - e), max(0, t - e), min(img_w - 1, r + e), min(img_h - 1, t + he + e)


def height_samples(box, img_h):
    """box_proposal_detail.cpp:114-123 with whether_sample_bbox_height: the down-expand samples of one box."""
    t, h = int(box[1]), int(box[3])
    r = max(min(20, h - 90), 20)
    r = min(r, img_h - t - h - 1)
    return [0] + ([int(round(r / 2))] if r > 10 else []) + [r]


def n_top_samples(box):
    """Number of top-x samples (box_proposal_detail.cpp:144-146) -- 0 below 10 px wide."""
    l, w = int(box[0]), int(box[2])
    lo, hi = l + 5, int(l + box[2]) - 5
    step = int(round(min(20, w // 10)))
    if hi < lo:
        return 0
    assert step > 0
    return (hi - lo) // step + 1


def base_frames():
    """Two synthetic VGA (indoor camera) and two KITTI-shaped frames: (tag, img, K, T, object boxes, lines)."""
    from cube_slam_b200 import synthetic as S
    out = []
    for seed, w, h, kind, nb in ((301, 640, 480, "indoor", 3), (302, 1242, 375, "kitti", 4)):
        imgs, Ts, boxes, lines, K = S.make_batch(seed, 2, w, h, nb, kind=kind)
        for f in range(2):
            img = imgs[f].copy()
            img[h - 131:, w - 131:] = img[h - 131, w - 131]   # a flat corner: the small box there has an edge-free, saturated distance map
            out.append(("%s%d" % (kind, f), img, K, Ts[f], boxes[f], lines[f]))
    return out


def border_boxes(obj_boxes, img_w, img_h):
    """Each object flush against the left, right, top and bottom edges and PAST px beyond each; then fractional / negative ones."""
    out = []
    for b in obj_boxes:
        l, t, w, h, p = [float(v) for v in b]
        for dx in (0, PAST):
            out.append(("left%d" % dx, [-dx, t, w, h, p]))
            out.append(("right%d" % dx, [img_w - 1 - w + dx, t, w, h, p]))
            out.append(("top%d" % dx, [l, -dx, w, h, p]))
            out.append(("bottom%d" % dx, [l, img_h - 1 - h + dx, w, h, p]))
    l, t, w, h, p = [float(v) for v in obj_boxes[0]]
    out.append(("frac", [l + 0.7, t + 0.3, w - 0.6, h + 0.9, p]))
    out.append(("neg_frac_left", [-7.6, t + 0.5, w + 3.3, h - 0.2, p]))
    out.append(("neg_frac_top", [l - 0.4, -2.5, w + 0.45, h + 0.75, p]))
    out.append(("neg_frac_corner", [-0.9, -0.9, w + 0.99, h + 0.99, p]))
    return out


SMALL_SIZES = ((10, 10), (10, 100), (100, 10), (11, 37), (37, 64), (64, 23), (99, 99), (100, 100), (19, 19), (50, 12))
NARROW_SIZES = ((9, 60), (5, 5), (3, 40))


def small_boxes(img_w, img_h, rng):
    """Boxes of 10-100 px a side (some against the edges), and boxes narrower than 10 px (zero candidates)."""
    out = []
    for i, (w, h) in enumerate(SMALL_SIZES + NARROW_SIZES):
        if i % 4 == 0:
            x, y = 0.0, float(rng.integers(0, img_h - h))
        elif i % 4 == 1:
            x, y = float(img_w - 1 - w), float(img_h - 1 - h)
        else:
            x, y = float(rng.integers(0, img_w - w)), float(rng.integers(0, img_h - h))
        out.append(("small%dx%d" % (w, h), [x, y, float(w), float(h), 0.5]))
    return out


def _inside(box, img_w, img_h, margin=1.0):
    l, t, r, b = roi_of(box, img_w, img_h)
    return l + margin, t + margin, r - margin, b - margin


def random_segments(rng, box, img_w, img_h, n=640, lo=8.0, hi=40.0):
    """n short segments, both ends inside the box's ROI."""
    l, t, r, b = _inside(box, img_w, img_h)
    out = []
    while len(out) < n:
        x0, y0 = rng.uniform(l, r), rng.uniform(t, b)
        a, ln = rng.uniform(0, 2 * np.pi), rng.uniform(lo, hi)
        x1, y1 = x0 + ln * np.cos(a), y0 + ln * np.sin(a)
        if l <= x1 <= r and t <= y1 <= b:
            out.append([x0, y0, x1, y1])
    return np.array(out)


def dashes(box, img_w, img_h, angles_deg=(0, 30, 60, 90, 120, 150), spacing=21.0, dash=3.0, gap=2.0):
    """Families of collinear dashes (one family per direction, rows `spacing` apart) filling the box's ROI: merge_break_lines chains
    each row's dashes one merge at a time, so the set runs into the 500-merge cap."""
    l, t, r, b = _inside(box, img_w, img_h)
    cx, cy = (l + r) / 2, (t + b) / 2
    R = np.hypot(r - l, b - t) / 2
    out = []
    for a in np.deg2rad(angles_deg):
        u, n = np.array([np.cos(a), np.sin(a)]), np.array([-np.sin(a), np.cos(a)])
        for k in np.arange(-R, R, spacing):
            for s in np.arange(-R, R, dash + gap):
                p0 = np.array([cx, cy]) + n * k + u * s
                p1 = p0 + u * dash
                if l <= min(p0[0], p1[0]) and max(p0[0], p1[0]) <= r and t <= min(p0[1], p1[1]) and max(p0[1], p1[1]) <= b:
                    out.append([p0[0], p0[1], p1[0], p1[1]])
    return np.array(out)


def odd_lines(rng, box, img_w, img_h, frame_lines):
    """Lines exactly on the inclusive ROI border (and 0.5 px outside it), right to left, vertical, zero-length and duplicated."""
    l, t, r, b = [float(v) for v in roi_of(box, img_w, img_h)]
    out = [[l, t + 5, l, t + 45], [r, t + 5, r, t + 45], [l + 5, t, l + 55, t], [l + 5, b, l + 55, b],    # on the border: inside
           [l, t, r, b], [r, b, l, t], [l, b, r, t],                                                        # corner to corner
           [l - 0.5, t + 5, l + 30, t + 5], [l + 5, b + 0.5, l + 45, b - 3], [r + 0.5, t + 9, r - 40, t + 9]]  # just outside: dropped
    for _ in range(20):
        x0, y0 = rng.uniform(l + 1, r - 45), rng.uniform(t + 1, b - 10)
        out.append([x0 + 44, y0 + rng.uniform(0, 8), x0, y0])          # right to left
        out.append([x0 + 3, y0, x0 + 3, min(y0 + 40, b)])              # vertical, top down
        out.append([x0 + 7, min(y0 + 35, b), x0 + 7, y0])              # vertical, bottom up
        out.append([x0 + 11, y0 + 2, x0 + 11, y0 + 2])                 # zero length
    inside = [ln for ln in np.asarray(frame_lines).reshape(-1, 4)
              if l <= min(ln[0], ln[2]) and max(ln[0], ln[2]) <= r and t <= min(ln[1], ln[3]) and max(ln[1], ln[3]) <= b]
    out += [list(ln) for ln in inside[:15]] * 2                        # duplicated (twice more)
    out += out[10:30]
    return np.array(out, float)


def capacity_lines(box, img_w, img_h, n_inside, n_merged):
    """Exactly n_inside lines inside the box's ROI of which exactly n_merged survive merge_break_lines: n_merged 40 px horizontal
    segments that cannot merge (ends >= 20 px from any other start), the rest 3 px diagonal stubs stacked on a few spots (they merge
    among themselves or stay short, so the length filter drops them)."""
    l, t, r, b = _inside(box, img_w, img_h, 2.0)
    longs = []
    y = t
    while len(longs) < n_merged:
        x = l
        while x + 40 <= r and len(longs) < n_merged:
            longs.append([x, y, x + 40, y])
            x += 62
        y += 23
        assert y <= b, "box too small for %d separate segments" % n_merged
    spots = [(l + 51 + 62 * i, t + 11 + 46 * j) for j in range(4) for i in range(4)]
    stubs = [[sx, sy, sx + 2, sy + 2] for k in range(n_inside - n_merged) for sx, sy in [spots[k % len(spots)]]]
    return np.array(longs + stubs, float)


def n_inside_roi(lines, box, img_w, img_h, down_expand=0):
    l, t, r, b = roi_of(box, img_w, img_h, down_expand)
    L = np.asarray(lines).reshape(-1, 4)
    xs, ys = L[:, [0, 2]], L[:, [1, 3]]
    return int(((xs >= l) & (xs <= r) & (ys >= t) & (ys <= b)).all(1).sum())


def big_frame():
    """A 1280 x 960 synthetic frame (room for the capacity sets)."""
    from cube_slam_b200 import synthetic as S
    imgs, Ts, boxes, lines, K = S.make_batch(303, 1, 1280, 960, 2)
    return imgs[0], K, Ts[0], boxes[0], lines[0]


CAP_BOX = [150.0, 120.0, 1000.0, 620.0, 0.9]
CAP_SETS = ((1024, 256), (1025, 200), (1000, 257))   # (inside, merged): at both capacities, one past the line cap, one past the merged cap


def dense_cases():
    """(tag, img, K, T, box, lines) with the dense sets added to the frame's own lines; the box is a real object box of the frame."""
    rng = np.random.default_rng(404)
    out = []
    for tag, img, K, T, boxes, lines in base_frames()[::2]:
        h, w = img.shape[:2]
        box = max(boxes, key=lambda bb: bb[2] * bb[3])
        out.append((tag + "_random", img, K, T, box, np.concatenate([lines, random_segments(rng, box, w, h)])))
        out.append((tag + "_dashes", img, K, T, box, np.concatenate([lines, dashes(box, w, h)[:900]])))   # whole rows; the ROI stays within 1024 lines
        out.append((tag + "_odd", img, K, T, box, np.concatenate([lines, odd_lines(rng, box, w, h, lines)])))
    return out


def capacity_cases():
    img, K, T, _, _ = big_frame()
    h, w = img.shape[:2]
    return [("cap%d_%d" % (ni, nm), img, K, T, np.array(CAP_BOX), capacity_lines(CAP_BOX, w, h, ni, nm)) for ni, nm in CAP_SETS]


# ------------------------------------------------------------------------------------------- oracle vs reference
def combined_key(rec, p):
    """The score detect_cuboid sorts by (box_proposal_detail.cpp:517-536), from a record's own fields."""
    skew = p.weight_skew_error * max(float(rec["skew_ratio"]) - p.nominal_skew_ratio, 0.0)
    if float(rec["skew_ratio"]) > p.max_cut_skew:
        skew = 100
    return float(rec["normalized_error"]) + p.weight_skew_error * skew


def _same_key(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


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
    print("\ncuboid edge inputs: %d oracle/reference runs, %d classified divergences %s" % (t["runs"], len(t["classified"]), t["classified"]))
    assert len(t["classified"]) <= MAX_CLASSIFIED


def _compare(ref, tally, label, img, K, T, boxes, lines, p):
    """Oracle == reference on every box, or a proven tie (see the module docstring)."""
    k = max(int(p.max_cuboid_num), 1)
    got = ref.detect_cuboid(img, K, T, boxes, lines, p, topk_cap=k)["cuboids"]
    want = ref.ref_detect_cuboid(img, K, T, boxes, lines, p, cap_per_box=k)
    for b in range(len(want)):
        tally["runs"] += 1
        assert len(got[b]) == len(want[b]), (label, b)
        same = all(np.array_equal(np.asarray(got[b][j][f], np.float64), np.asarray(want[b][j][f], np.float64), equal_nan=True)
                   for j in range(len(want[b])) for f in FIELDS)
        if same:
            continue
        keys_g = [combined_key(r, p) for r in got[b]]
        keys_w = [combined_key(r, p) for r in want[b]]
        differ = [j for j in range(len(want[b])) if not all(np.array_equal(np.asarray(got[b][j][f], np.float64),
                                                                           np.asarray(want[b][j][f], np.float64), equal_nan=True) for f in FIELDS)]
        tie = all(_same_key(keys_g[j], keys_w[j]) for j in differ)
        nan_pick = len(want[b]) > 0 and np.isnan(float(want[b][0]["normalized_error"]))
        assert tie or nan_pick, "%s box %d: oracle and reference differ at ranks %s (keys %s vs %s)" % (label, b, differ, keys_g, keys_w)
        tally["classified"].append("%s/box%d" % (label, b))


MODES = (("default", {}), ("height", dict(whether_sample_bbox_height=1)), ("roll_pitch", dict(whether_sample_cam_roll_pitch=1)))


@pytest.mark.parametrize("mode,kw", MODES)
def test_border_fractional_and_small_boxes(ref, tally, mode, kw):
    rng = np.random.default_rng(7)
    n_dup = n_neg = 0
    for tag, img, K, T, obj, lines in base_frames():
        h, w = img.shape[:2]
        boxes = border_boxes(obj, w, h) + small_boxes(w, h, rng)
        wide = [(n, bb) for n, bb in boxes if int(bb[2]) >= 10]
        if kw.get("whether_sample_bbox_height"):
            for n, bb in wide:
                hs = height_samples(bb, h)
                n_dup += n.startswith("bottom0") and hs == [0, 0]
                n_neg += n.startswith("bottom%d" % PAST) and hs == [0, -PAST]
        # several boxes per call, as the reference is driven: with roll / pitch sampling later boxes start from the carried-over pose
        for i in range(0, len(wide), 8):
            chunk = wide[i:i + 8]
            _compare(ref, tally, "%s/%s/%s" % (tag, mode, chunk[0][0]), img, K, T, np.array([bb for _, bb in chunk]), lines,
                     ref.default_params(max_cuboid_num=1, **kw))
        # below 10 px wide the reference faults (linespace with a zero step); the oracle has no top-x sample, so no candidate
        narrow = np.array([bb for _, bb in boxes if int(bb[2]) < 10])
        assert len(narrow) == len(NARROW_SIZES) and all(n_top_samples(bb) == 0 for bb in narrow)
        res = ref.detect_cuboid(img, K, T, narrow, lines, ref.default_params(**kw))
        assert res["n_candidates"] == 0 and all(len(c) == 0 for c in res["cuboids"])
    if kw.get("whether_sample_bbox_height"):
        assert n_dup >= 4 and n_neg >= 4, (n_dup, n_neg)   # every frame has duplicate {0, 0} and negative {0, -15} samples


@pytest.mark.parametrize("mode,kw", (("top5", dict(max_cuboid_num=5)), ("height_top5", dict(whether_sample_bbox_height=1, max_cuboid_num=5))))
def test_dense_line_sets(ref, tally, mode, kw):
    for tag, img, K, T, box, lines in dense_cases():
        h, w = img.shape[:2]
        n_in = n_inside_roi(lines, box, w, h)
        assert (600 if "random" in tag or "dashes" in tag else 1) <= n_in <= 1024, (tag, n_in)
        for hs in range(len(height_samples(box, h))):   # within the product's per-ROI capacities for every height sample
            tr = ref.detect_cuboid(img, K, T, box[None], lines, ref.default_params(**kw), trace_object=0, trace_height_sample=hs)["trace"]
            assert tr["n_lines_roi"] <= 1024 and tr["n_lines_merged"] <= 256, (tag, hs, tr["n_lines_roi"], tr["n_lines_merged"])
        if tag.endswith("_dashes"):
            l, t, r, b = roi_of(box, w, h)
            L = lines[[l <= min(x[0], x[2]) and max(x[0], x[2]) <= r and t <= min(x[1], x[3]) and max(x[1], x[3]) <= b for x in lines]]
            assert len(L) - len(ref.merge_break_lines(L, len_thre=0)) == 500, tag   # the merge loop stops at its cap
        _compare(ref, tally, "%s/%s" % (tag, mode), img, K, T, box[None], lines, ref.default_params(**kw))


def test_capacity_line_sets(ref, tally):
    for tag, img, K, T, box, lines in capacity_cases():
        h, w = img.shape[:2]
        tr = ref.detect_cuboid(img, K, T, box[None], lines, trace_object=0, trace_caps=(4096, 1 << 21, 1 << 16))["trace"]
        ni, nm = [int(v) for v in tag[3:].split("_")]
        assert (tr["n_lines_roi"], tr["n_lines_merged"]) == (ni, nm), tag
        _compare(ref, tally, tag, img, K, T, box[None], lines, ref.default_params(max_cuboid_num=3))
