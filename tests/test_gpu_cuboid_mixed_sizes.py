"""detect_cuboid over frames of different sizes and cameras in one GPU batch (cs_batch_upload_mixed, cs_batch_upload_online_mixed,
cs_detect_cuboids_batch_mixed, cs_detect_frames_batch_mixed and the Context methods over them).

The expected records of every frame are what the one-size calls (cs_detect_cuboids_batch, cs_detect_frames_batch) return for that frame alone
with its own K set by cs_set_calibration, compared field by field with assert_array_equal; a subset is also compared with the oracle
(oracle/pyoracle.py::detect_cuboid, which takes K per call)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SETTINGS = {
    "default": (dict(), 0),
    "roll_pitch": (dict(whether_sample_cam_roll_pitch=1), 0),
    "bbox_height": (dict(whether_sample_bbox_height=1, max_cuboid_num=5), 0),
    "carried": (dict(whether_sample_cam_roll_pitch=1, max_cuboid_num=2), 1024),   # cs_set_profiling bit 10, several boxes per frame
}
MODES = ("lines", "lsd", "edlines")


def new_ctx(max_frames=16):
    import cube_slam_b200 as cs
    return cs.Context(0, 1280, 960, max_frames, 16, 4096)


def line_params(ctx, use_LSD):
    from cube_slam_b200 import _lib
    p = _lib.LineParams()
    ctx.L.cs_default_line_params(C.byref(p))
    p.use_LSD, p.line_length_thres = use_LSD, 15.0
    return p


def frame(img, T, boxes, lines, K, pad=0):
    return dict(img=np.ascontiguousarray(img, np.uint8), T=np.asarray(T, np.float64).reshape(16), boxes=np.asarray(boxes, np.float64).reshape(-1, 5),
                lines=np.asarray(lines, np.float64).reshape(-1, 4), K=np.asarray(K, np.float64).reshape(3, 3), pad=pad)


@pytest.fixture(scope="module")
def frames(fixture_a, fixture_b):
    """VGA indoor and KITTI-shaped BGR frames with their own K, a gray frame, a padded-stride view, a crop, a small frame with a box against
    its border, frames without boxes, and the fixture A and B images -- sizes interleaved, so that EDLines' size groups are not in call order"""
    from cube_slam_b200 import synthetic as S
    vi, vT, vb, vl, vK = S.make_batch(21, 3, 640, 480, 3)
    ki, kT, kb, kl, kK = S.make_batch(22, 2, 1242, 375, 5, kind="kitti")
    si, sT, sb, sl, sK = S.make_batch(23, 1, 320, 240, 1)
    small_box = np.array([[0, 140, 200, 99, 0.9]])          # left and bottom edges on the frame's border
    crop = vi[1][40:440, 60:620]                             # a 560 x 400 crop; K's principal point moves with it
    cK = vK.copy()
    cK[0, 2] -= 60
    cK[1, 2] -= 40
    cboxes = np.asarray(vb[1], float).reshape(-1, 5)
    inside = (cboxes[:, 0] >= 60) & (cboxes[:, 1] >= 40) & (cboxes[:, 0] + cboxes[:, 2] < 619) & (cboxes[:, 1] + cboxes[:, 3] < 439)
    cboxes = cboxes[inside] - np.array([60, 40, 0, 0, 0]) if inside.any() else np.array([[120.0, 90, 220, 180, 0.9]])
    clines = np.asarray(vl[1], float) - np.array([60, 40, 60, 40])
    a = fixture_a
    bimg, bboxes = fixture_b["frames"][7]
    return [frame(vi[0], vT[0], vb[0], vl[0], vK),
            frame(ki[0], kT[0], kb[0], kl[0], kK),
            frame(vi[1][..., 1], vT[1], vb[1], vl[1], vK),                      # gray
            frame(ki[1], kT[1], kb[1], kl[1], kK, pad=24),                      # padded rows
            frame(si[0], sT[0], small_box, sl[0], sK),
            frame(crop, vT[1], cboxes, clines, cK),
            frame(vi[2], vT[2], np.zeros((0, 5)), vl[2], vK),                   # no boxes
            frame(a["img"], a["T"], a["boxes"], a["lines"], a["K"]),
            frame(bimg, fixture_b["T"], bboxes[:3], a["lines"], fixture_b["K"]),
            frame(ki[0], kT[0], np.zeros((0, 5)), kl[0], kK)]                   # no boxes, KITTI


def pack(frs):
    """the frames in one buffer with their cs_frame_views (a frame with pad > 0 gets rows of width * channels + pad bytes)"""
    from cube_slam_b200 import _lib
    views = (_lib.FrameView * len(frs))()
    parts, off = [], 0
    for i, f in enumerate(frs):
        img = f["img"]
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else 3
        rows = img.reshape(h, w * ch)
        if f["pad"]:
            rows = np.concatenate([rows, np.full((h, f["pad"]), 77, np.uint8)], axis=1)
        views[i].offset, views[i].width, views[i].height, views[i].stride, views[i].channels = off, w, h, rows.shape[1], ch
        parts.append(rows.reshape(-1))
        off += rows.size
    return np.ascontiguousarray(np.concatenate(parts)), views


def tables(frs):
    Ts = np.ascontiguousarray(np.stack([f["T"] for f in frs]))
    Ks = np.ascontiguousarray(np.stack([f["K"].reshape(9) for f in frs]))
    box_off = np.concatenate([[0], np.cumsum([len(f["boxes"]) for f in frs])]).astype(np.int32)
    line_off = np.concatenate([[0], np.cumsum([len(f["lines"]) for f in frs])]).astype(np.int32)
    boxes = np.ascontiguousarray(np.concatenate([f["boxes"] for f in frs] + [np.zeros((1, 5))]))
    lines = np.ascontiguousarray(np.concatenate([f["lines"] for f in frs] + [np.zeros((1, 4))]))
    return Ts, Ks, box_off, line_off, boxes, lines


def mixed(ctx, frs, mode, prm, use_K=True):
    """the mixed call over frs -> (records, counts), through the C ABI"""
    from cube_slam_b200 import _lib
    d = lambda a: _lib.ptr(a, C.c_double)
    buf, views = pack(frs)
    Ts, Ks, box_off, line_off, boxes, lines = tables(frs)
    n = int(box_off[-1])
    rec, cnt = np.zeros((max(n, 1), prm.max_cuboid_num), _lib.CUBOID_DTYPE), np.zeros(max(n, 1), np.int32)
    head = [ctx.h, buf.ctypes.data, views, len(frs), d(Ks) if use_K else None, d(Ts), d(boxes), _lib.ptr(box_off, C.c_int32)]
    tail = [C.byref(prm), rec.ctypes.data, _lib.ptr(cnt, C.c_int32)]
    if mode == "lines":
        rc = ctx.L.cs_detect_cuboids_batch_mixed(*(head + [d(lines), _lib.ptr(line_off, C.c_int32)] + tail))
    else:
        rc = ctx.L.cs_detect_frames_batch_mixed(*(head + [C.byref(line_params(ctx, mode == "lsd"))] + tail))
    ctx.check(rc)
    return rec[:n], cnt[:n]


def alone(ctx, f, mode, prm):
    """the one-size call on frame f alone, its K set by cs_set_calibration"""
    ctx.set_calibration(f["K"])
    img = f["img"][None]
    if mode == "lines":
        return ctx.detect_batch_host(img, f["T"][None], [f["boxes"]], [f["lines"]], prm)
    return ctx.detect_frames_host(img, f["T"][None], [f["boxes"]], line_params(ctx, mode == "lsd"), prm)


def expected(ctx, frs, mode, prm):
    recs, cnts = zip(*[alone(ctx, f, mode, prm) for f in frs])
    return np.concatenate(recs), np.concatenate(cnts)


def assert_same(got, want):
    (gr, gc), (wr, wc) = got, want
    np.testing.assert_array_equal(gc, wc)
    assert gr.shape == wr.shape
    for name in gr.dtype.names:
        np.testing.assert_array_equal(gr[name], wr[name], err_msg=name)


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("mode", MODES)
def test_each_frame_is_its_one_size_answer(frames, mode, setting):
    import cube_slam_b200 as D
    kw, bits = SETTINGS[setting]
    prm = D.default_params(**kw)
    ctx = new_ctx()
    try:
        ctx.set_profiling(bits)
        got = mixed(ctx, frames, mode, prm)
        assert_same(got, expected(ctx, frames, mode, prm))
        assert got[1].sum() > 0
    finally:
        ctx.close()


def test_against_the_oracle(frames, oracle):
    import cube_slam_b200 as D
    from test_gpu_cuboid_edges import _compare_cuboid
    ctx = new_ctx()
    try:
        rec, cnt = mixed(ctx, frames, "lines", D.default_params())
    finally:
        ctx.close()
    o = 0
    for f in frames:
        img = f["img"]
        ref = oracle.detect_cuboid(img, f["K"], f["T"].reshape(4, 4), f["boxes"], f["lines"], oracle.default_params())
        for b in range(len(f["boxes"])):
            assert cnt[o] == len(ref["cuboids"][b])
            for k in range(cnt[o]):
                _compare_cuboid(rec[o, k], ref["cuboids"][b][k])
            o += 1


def test_per_frame_calibration(frames):
    """the same image twice with two calibrations: each slot is its own K's one-size answer, and the two differ"""
    import cube_slam_b200 as D
    f0 = frames[0]
    K2 = f0["K"].copy()
    K2[0, 0] *= 1.15
    K2[1, 1] *= 1.15
    pair = [f0, dict(f0, K=K2)]
    prm = D.default_params()
    ctx = new_ctx()
    try:
        for mode in MODES:
            got = mixed(ctx, pair, mode, prm)
            assert_same(got, expected(ctx, pair, mode, prm))
            n = len(f0["boxes"])
            assert got[0][:n].tobytes() != got[0][n:].tobytes(), mode
    finally:
        ctx.close()


def test_context_methods_and_two_batches_in_flight(frames):
    """upload_online_mixed on two contexts, both run_async before either fetch: the synchronous answers; and the Python methods' K forms"""
    import cube_slam_b200 as D
    prm = D.default_params()
    plain = [f for f in frames if not f["pad"]]
    halves = (plain[:5], plain[5:])
    want = []
    ref = new_ctx()
    try:
        for half in halves:
            want.append(expected(ref, half, "lsd", prm))
        ctxs = [new_ctx(), new_ctx()]
        lp = line_params(ctxs[0], 1)
        for c, half in zip(ctxs, halves):
            c.upload_online_mixed([f["img"] for f in half], np.stack([f["T"] for f in half]), [f["boxes"] for f in half], lp, prm,
                                  K=np.stack([f["K"] for f in half]))
        for c in ctxs:
            c.run_async()
        for c, w in zip(ctxs, want):
            assert_same(c.fetch(), w)
        # detect_*_mixed, and one K for every frame (None: the context's calibration)
        same_K = [dict(f, K=frames[0]["K"]) for f in plain[:4]]
        args = ([f["img"] for f in same_K], np.stack([f["T"] for f in same_K]), [f["boxes"] for f in same_K])
        w = expected(ref, same_K, "lines", prm)
        assert_same(ctxs[0].detect_batch_mixed(*args, [f["lines"] for f in same_K], prm, K=frames[0]["K"]), w)
        ctxs[1].set_calibration(frames[0]["K"])
        assert_same(ctxs[1].detect_batch_mixed(*args, [f["lines"] for f in same_K], prm), w)
        ctxs[1].upload_mixed(*args, [f["lines"] for f in same_K], prm)
        ctxs[1].run()
        assert_same(ctxs[1].fetch(), w)
        assert_same(ctxs[0].detect_frames_mixed(*args, line_params(ctxs[0], 0), prm, K=frames[0]["K"]), expected(ref, same_K, "edlines", prm))
        st = ctxs[0].stats()
        assert st["n_frames"] == 4 and st["n_lines_in"] > 0
        for c in ctxs:
            c.close()
    finally:
        ref.close()


def _refused(ctx, frs, mode, prm, status, text, use_K=True):
    from cube_slam_b200.detect_3d_cuboid import CubeSlamError
    with pytest.raises(CubeSlamError) as e:
        mixed(ctx, frs, mode, prm, use_K)
    assert status in str(e.value) and text in str(e.value), str(e.value)


def test_refusals_name_the_frame(frames):
    import cube_slam_b200 as D
    from cube_slam_b200 import _lib
    prm = D.default_params()
    few = frames[:3]
    ctx = new_ctx()
    try:
        _refused(ctx, few, "lines", prm, "CS_ERR_INVALID_ARG", "cs_set_calibration", use_K=False)
        big = few[:1] + [dict(few[1], img=np.zeros((100, 1300, 3), np.uint8), boxes=np.zeros((0, 5)))]
        _refused(ctx, big, "lines", prm, "CS_ERR_CAPACITY", "frame 1")
        for bad in (np.nan, np.inf):
            K = few[2]["K"].copy()
            K[0, 1] = bad
            _refused(ctx, few[:2] + [dict(few[2], K=K)], "lsd", prm, "CS_ERR_INVALID_ARG", "frame 2")
        _refused(ctx, [few[0], dict(few[1], K=np.zeros((3, 3)))], "lines", prm, "CS_ERR_INVALID_ARG", "frame 1: K has a zero determinant")
        tiny = few[:2] + [dict(few[2], img=np.zeros((6, 6), np.uint8), boxes=np.zeros((0, 5)))]
        _refused(ctx, tiny, "edlines", prm, "CS_ERR_INVALID_ARG", "frame 2: a 6 x 6 image is outside EDLines' sizes")
        tiny = few[:2] + [dict(few[2], img=np.zeros((1, 1), np.uint8), boxes=np.zeros((0, 5)))]
        _refused(ctx, tiny, "lsd", prm, "CS_ERR_INVALID_ARG", "frame 2: a 1 x 1 image is too small for LSD")
        # a view the frame checks refuse (cs_check_frame_views), through the C ABI
        buf, views = pack(few)
        views[1].channels = 2
        Ts, Ks, box_off, line_off, boxes, lines = tables(few)
        d = lambda a: _lib.ptr(a, C.c_double)
        out, cnt = np.zeros((16, 1), _lib.CUBOID_DTYPE), np.zeros(16, np.int32)
        rc = ctx.L.cs_detect_cuboids_batch_mixed(ctx.h, buf.ctypes.data, views, 3, d(Ks), d(Ts), d(boxes), _lib.ptr(box_off, C.c_int32), d(lines),
                                                 _lib.ptr(line_off, C.c_int32), C.byref(prm), out.ctypes.data, _lib.ptr(cnt, C.c_int32))
        assert rc == -1 and "frame 1: channels must be 1 or 3" in ctx.L.cs_last_error(ctx.h).decode()
        # the context is still good for a valid call
        for mode in MODES:
            assert_same(mixed(ctx, few, mode, prm), expected(ctx, few, mode, prm))
    finally:
        ctx.close()


def test_debug_reads_after_a_mixed_batch(frames):
    """cs_debug_roi / cs_debug_candidates read the mixed batch's jobs; cs_debug_lsd refuses after its online LSD run"""
    import cube_slam_b200 as D
    prm = D.default_params()
    ctx = new_ctx()
    try:
        mixed(ctx, frames[:3], "lsd", prm)
        roi = ctx.debug_roi(0)
        assert roi["roi"][2] > 0 and roi["canny"].any()
        assert ctx.debug_candidates(0)["n"] > 0
        assert ctx.L.cs_debug_lsd(ctx.h, 0, None, None, None, None, None, None, None, None, 0) == -6
    finally:
        ctx.close()


def test_lsd_candidate_overflow_fails_the_online_batch_at_fetch(frames):
    """a frame with more LSD candidate regions than the hand-off buffer holds fails the enqueue-only online batch at fetch with
    CS_ERR_CAPACITY, as the one-size online batch does; once a synchronous line call on the context has grown the buffer, every frame is its
    one-size answer"""
    import cube_slam_b200 as D
    from cube_slam_b200 import _lib
    from cube_slam_b200.detect_3d_cuboid import CubeSlamError
    rng = np.random.default_rng(3)
    board = np.ascontiguousarray(np.kron(rng.integers(0, 2, (240, 320)).astype(np.uint8) * 200 + 20, np.ones((4, 4), np.uint8)))  # 1280 x 960
    f0 = frames[0]
    frs = [f0, frame(board, f0["T"], [[100, 100, 300, 200, 0.9]], np.zeros((0, 4)), f0["K"]), frames[2]]
    prm = D.default_params()
    ctx, one = new_ctx(), new_ctx()
    try:
        for run, c in ((lambda: mixed(ctx, frs, "lsd", prm)), ctx), ((lambda: alone(one, frs[1], "lsd", prm)), one):
            with pytest.raises(CubeSlamError) as e:
                run()
            assert "CS_ERR_CAPACITY" in str(e.value) and "LSD candidate regions" in str(e.value), str(e.value)
            out, n = np.zeros((1, 4096, 4), np.float32), np.zeros(1, np.int32)
            c.check(c.L.cs_detect_lines_batch(c.h, board.ctypes.data, 1, 1280, 960, 1280, 1, C.byref(line_params(c, 1)), _lib.ptr(out, C.c_float), 4096,
                                              _lib.ptr(n, C.c_int32)))
        assert_same(mixed(ctx, frs, "lsd", prm), expected(one, frs, "lsd", prm))
    finally:
        ctx.close()
        one.close()
