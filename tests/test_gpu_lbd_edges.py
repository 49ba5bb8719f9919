"""The descriptor / matcher half of line_lbd_detect on the device (cs_lbd.cu, cs_lbd_kernels.cuh, cs_lbd_core.h, and the Sobel maps of
cs_edlines.cu: cs_edl_sobel_maps) at the shapes, strides, densities and routing regimes tests/test_z_gpu_lbd_parity.py does not reach:
1280 x 960 batches (TMA-staged front ends) and the same with byte staging, ragged and tiny frames, rows with padding through the C ABI,
cs_lbd_compute_batch over several frames with ragged key-line offsets, long and border lines, 13 463 key lines in one frame and the
capacity error one line short of it, the three EDLines routing regimes with key-line extras, one context across changing sizes, and the
matcher at scale and at its special cases.

Every comparison is exact against the CPU oracle, itself pinned to the compiled reference on the same inputs by
tests/test_oracle_ref_lbd_edges.py: key-line fields, class_id, 32-byte descriptors, 72-float descriptors (NaN in the same places), match
triples.  Each test asserts from its own inputs that the path it targets is taken."""
import ctypes as C

import numpy as np
import pytest

from test_oracle_ref_lbd_edges import (RAGGED_SHAPES, TIE_DISTANCES, TINY_GIVEN_SHAPES, TINY_LSD_SHAPES, given_rows, long_and_border_rows,
                                       matcher_cases, short_frame, short_frame_rows, sxga_frames, tiny_image)

pytestmark = pytest.mark.gpu

FIELDS = (("start_x", "sx"), ("start_y", "sy"), ("end_x", "ex"), ("end_y", "ey"), ("angle", "angle"), ("line_length", "line_length"),
          ("response", "response"), ("size", "size"), ("num_pixels", "num_pixels"))
BYTE_STAGING = 256      # cs_set_profiling bit 8: the front ends stage tiles with byte loads instead of TMA copies


@pytest.fixture(scope="module")
def ctx():
    import cube_slam_b200 as cs
    c = cs.Context(0, 2048, 2048, 1, 1, 1)
    yield c
    c.close()


def detector(ctx, use_lsd, thres=15.0):
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(context=ctx)
    d.use_LSD = use_lsd
    d.line_length_thres = thres
    return d


def product_keylines(kl):
    """oracle key lines -> cs_keyline records (the same 40-byte layout)"""
    from cube_slam_b200 import _lib
    return np.ascontiguousarray(kl).view(_lib.KEYLINE_DTYPE)


def same_keylines(got, want):
    assert len(got) == len(want)
    for a, b in FIELDS:
        np.testing.assert_array_equal(got[a], want[b], err_msg=a)
    np.testing.assert_array_equal(got["class_id"], np.arange(len(got)))


def same_results(a, b, what=""):
    """two [(key lines, descriptors)] lists of the library"""
    assert len(a) == len(b)
    for f, ((ka, da), (kb, db)) in enumerate(zip(a, b)):
        assert ka.tobytes() == kb.tobytes(), "%s frame %d: key lines differ" % (what, f)
        np.testing.assert_array_equal(da, db, err_msg="%s frame %d" % (what, f))


def check_frames(oracle, out, imgs, use_lsd, thres, cap=8192):
    n = 0
    for f, (kl, desc) in enumerate(out):
        want = oracle.lbd_detect_keylines(imgs[f], use_lsd, thres, cap)
        same_keylines(kl, want)
        np.testing.assert_array_equal(desc, oracle.lbd_compute(imgs[f], want))
        n += len(kl)
    return n


def frames_buffer(imgs, pad):
    """frames whose rows are `pad` bytes longer than width x channels; the padding holds 0xA5, which must not be read"""
    F, H, W = imgs.shape[:3]
    ch = imgs.shape[3] if imgs.ndim == 4 else 1
    row = W * ch
    buf = np.full((F, H, row + pad), 0xA5, np.uint8)
    buf[:, :, :row] = imgs.reshape(F, H, row)
    return buf, W, H, ch, row + pad


def descrip_strided(d, imgs, pad, cap=4096):
    """cs_detect_descrip_lines_batch with stride = row + pad"""
    from cube_slam_b200 import _lib
    buf, W, H, ch, stride = frames_buffer(imgs, pad)
    F = len(imgs)
    kl = np.zeros((F, cap), _lib.KEYLINE_DTYPE)
    desc = np.zeros((F, cap, 32), np.uint8)
    n = np.zeros(F, np.int32)
    p = d.params()
    d._ctx.check(d._ctx.L.cs_detect_descrip_lines_batch(d._ctx.h, buf.ctypes.data, F, W, H, stride, ch, C.byref(p), kl.ctypes.data,
                                                        _lib.ptr(desc, C.c_uint8), cap, _lib.ptr(n, C.c_int32)))
    return [(kl[f, :n[f]].copy(), desc[f, :n[f]].copy()) for f in range(F)]


def compute_batch(ctx, imgs, keylines, pad=0, want72=True):
    """cs_lbd_compute_batch: frame f's key lines are keylines[f] (cs_keyline records, any count including 0) -> [(n x 32, n x 72)] per frame"""
    from cube_slam_b200 import _lib
    buf, W, H, ch, stride = frames_buffer(imgs, pad)
    off = np.concatenate([[0], np.cumsum([len(k) for k in keylines])]).astype(np.int32)
    kl = np.ascontiguousarray(np.concatenate(keylines) if off[-1] else np.zeros(1, _lib.KEYLINE_DTYPE), _lib.KEYLINE_DTYPE)
    desc = np.zeros((max(int(off[-1]), 1), 32), np.uint8)
    f72 = np.zeros((max(int(off[-1]), 1), 72), np.float32)
    ctx.check(ctx.L.cs_lbd_compute_batch(ctx.h, buf.ctypes.data, len(imgs), W, H, stride, ch, kl.ctypes.data, _lib.ptr(off, C.c_int32),
                                         _lib.ptr(desc, C.c_uint8), _lib.ptr(f72, C.c_float) if want72 else None))
    return [(desc[off[f]:off[f + 1]].copy(), f72[off[f]:off[f + 1]].copy()) for f in range(len(imgs))]


def check_given(oracle, res, imgs, want_keylines):
    for f, (d, f72) in enumerate(res):
        wd, wf = oracle.lbd_compute(imgs[f], want_keylines[f], want_float=True)
        np.testing.assert_array_equal(d, wd, err_msg="frame %d" % f)
        np.testing.assert_array_equal(f72, wf, err_msg="frame %d" % f)      # NaN == NaN, in the same places


# ---- 1. shapes -------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("use_lsd", [True, False], ids=["lsd", "edlines"])
def test_sxga_batch_tma_and_byte_staging(ctx, oracle, use_lsd):
    """1280 x 960 BGR: rows of 3 840 bytes, a multiple of 16, so interior tiles of the Sobel-map (and LSD) front end are TMA copies; bit 8
    stages the same tiles with byte loads.  Both give the oracle's key lines and descriptors, detected and on given key lines."""
    imgs = sxga_frames()
    assert imgs.shape[1:] == (960, 1280, 3) and (3 * 1280) % 16 == 0
    d = detector(ctx, use_lsd)
    rows = np.concatenate([given_rows(960, 1280), long_and_border_rows()])
    kl = d.keylines_from_lines(rows, 1280, 960)
    want = [oracle.lbd_keylines_from_lsd(rows, 1280, 960)] * 2
    same_keylines(kl, want[0])
    got, given = {}, {}
    try:
        for flags in (0, BYTE_STAGING):
            ctx.set_profiling(flags)
            got[flags] = d.detect_descrip_lines_batch(imgs)
            given[flags] = compute_batch(ctx, imgs, [kl, kl])
    finally:
        ctx.set_profiling(0)
    assert check_frames(oracle, got[0], imgs, use_lsd, 15.0) > 40
    same_results(got[0], got[BYTE_STAGING], "byte staging")
    check_given(oracle, given[0], imgs, want)
    check_given(oracle, given[BYTE_STAGING], imgs, want)


@pytest.mark.parametrize("channels", [1, 3], ids=["gray", "bgr"])
@pytest.mark.parametrize("shape", RAGGED_SHAPES, ids=["%dx%d" % s for s in RAGGED_SHAPES])
def test_ragged_sizes(ctx, oracle, shape, channels):
    """Three-frame batches at sizes that cut the 64 x 32 front-end tiles, both flavours; then given key lines in every frame of the batch."""
    from test_gpu_lsd_parity import odd_size_batch
    h, w = shape
    imgs = odd_size_batch(h, w, channels)
    assert w % 64 or h % 32                   # partial tiles at the right or bottom edge
    for use_lsd in (True, False):
        check_frames(oracle, detector(ctx, use_lsd).detect_descrip_lines_batch(imgs), imgs, use_lsd, 15.0)
    rows = given_rows(h, w)
    d = detector(ctx, True)
    kl = d.keylines_from_lines(rows, w, h)
    want = oracle.lbd_keylines_from_lsd(rows, w, h)
    same_keylines(kl, want)
    check_given(oracle, compute_batch(ctx, imgs, [kl] * 3), imgs, [want] * 3)


# ---- 2. tiny frames ---------------------------------------------------------------------------------------------------------------------

def test_tiny_frames(ctx, oracle):
    """LSD flavour from 3 x 3: no key line and CS_OK (the reference describes nothing and makes no Sobel maps).  Given key lines in frames
    from 1 x 1: the oracle's descriptors, NaNs included.  The EDLines flavour keeps rejecting frames under 8 x 8, as its detection does."""
    import cube_slam_b200 as cs
    from test_gpu_lsd_parity import odd_size_batch
    lsd, edl = detector(ctx, True), detector(ctx, False)
    for h, w in TINY_LSD_SHAPES:
        assert min(h, w) < 8 and int(np.rint(0.8 * min(h, w))) >= 2
        for channels in (1, 3):
            imgs = odd_size_batch(h, w, channels)
            for thres in (15.0, -1.0):
                lsd.line_length_thres = thres
                out = lsd.detect_descrip_lines_batch(imgs)
                assert [len(k) for k, _ in out] == [0, 0, 0]
                assert all(len(oracle.lbd_detect_keylines(img, True, thres)) == 0 for img in imgs)
            with pytest.raises(cs.CubeSlamError, match="INVALID_ARG"):
                edl.detect_descrip_lines_batch(imgs)
    n_nan = 0
    for h, w in TINY_GIVEN_SHAPES:
        for channels in (1, 3):
            img = tiny_image(h, w, channels, h * 100 + w)
            rows = given_rows(h, w, 8)
            kl = lsd.keylines_from_lines(rows, w, h)
            want = oracle.lbd_keylines_from_lsd(rows, w, h)
            same_keylines(kl, want)
            d, f = lsd.compute_descriptors(img, kl, want_float=True)
            wd, wf = oracle.lbd_compute(img, want, want_float=True)
            np.testing.assert_array_equal(d, wd, err_msg="%dx%d" % (h, w))
            np.testing.assert_array_equal(f, wf, err_msg="%dx%d" % (h, w))
            n_nan += int(np.isnan(f).any(1).sum())
    assert n_nan > 0
    # several tiny frames in one compute batch
    imgs = np.stack([tiny_image(1, 9, 3, s) for s in range(3)])
    rows = given_rows(1, 9, 4)
    kl = lsd.keylines_from_lines(rows, 9, 1)
    check_given(oracle, compute_batch(ctx, imgs, [kl, kl[:0], kl]), imgs, [oracle.lbd_keylines_from_lsd(rows, 9, 1), kl[:0], oracle.lbd_keylines_from_lsd(rows, 9, 1)])


# ---- 3. padded rows -----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("use_lsd", [True, False], ids=["lsd", "edlines"])
def test_padded_rows_equal_packed_rows(ctx, oracle, use_lsd):
    """stride = row + pad through the C ABI (one pad keeps rows 16-byte aligned, one breaks it; a padded row turns TMA staging off), for
    detection with descriptors and for cs_lbd_compute_batch on the detected key lines: equal to the packed rows, which equal the oracle."""
    from cube_slam_b200 import synthetic as S
    from test_gpu_lsd_parity import odd_size_batch, row_pads
    d = detector(ctx, use_lsd)
    vga = S.make_batch(84, 3, 640, 480, 3)[0]
    for imgs in (S.make_batch(83, 3, 1242, 375, 3, kind="kitti")[0], vga, np.ascontiguousarray(vga[:, :, :, 1]), odd_size_batch(97, 211, 3)):
        packed = d.detect_descrip_lines_batch(imgs)
        assert check_frames(oracle, packed, imgs, use_lsd, 15.0) > 0
        kls = [k for k, _ in packed]
        given = compute_batch(ctx, imgs, kls)
        for f in range(len(imgs)):
            np.testing.assert_array_equal(given[f][0], packed[f][1])
        row = imgs.shape[2] * (imgs.shape[3] if imgs.ndim == 4 else 1)
        pads = row_pads(row)
        assert (row + pads[0]) % 16 == 0 and (row + pads[1]) % 16
        for pad in pads:
            same_results(descrip_strided(d, imgs, pad), packed, "row %d + pad %d" % (row, pad))
            for f, (dd, ff) in enumerate(compute_batch(ctx, imgs, kls, pad)):
                np.testing.assert_array_equal(dd, given[f][0])
                np.testing.assert_array_equal(ff, given[f][1])


# ---- 4. cs_lbd_compute_batch over several frames ------------------------------------------------------------------------------------

def test_compute_batch_ragged_offsets(ctx, oracle):
    """Seven VGA frames, frames 0, 3 and 6 without key lines; each frame's descriptors (bytes and floats) are its own one-frame oracle
    result.  Frames 1, 2 and 4 get the same given lines: their descriptors differ, so each line read its own frame's Sobel maps."""
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(96, 7, 640, 480, 3)[0]
    rows = given_rows(480, 640, 60)
    same = oracle.lbd_keylines_from_lsd(rows, 640, 480)
    want = [same[:0], same, same, same[:0], same, oracle.lbd_detect_keylines(imgs[5], True, 15.0), same[:0]]
    res = compute_batch(ctx, imgs, [product_keylines(k) for k in want])
    assert [len(r[0]) for r in res] == [len(k) for k in want] and len(want[5]) > 20
    check_given(oracle, res, imgs, want)
    assert (res[1][0] != res[2][0]).any() and (res[2][0] != res[4][0]).any()
    # without the float output
    res32 = compute_batch(ctx, imgs, [product_keylines(k) for k in want], want72=False)
    for f in range(7):
        np.testing.assert_array_equal(res32[f][0], res[f][0])


# ---- 5. long lines and borders ------------------------------------------------------------------------------------------------------

def test_long_and_border_lines(ctx, oracle):
    """Full-width / full-height / full-diagonal lines (numOfPixels 1 280, 960, 1 280: row walks eight times longer than any detected line
    so far), every border row and column, end points outside the frame, one-pixel lines; and a 1280 x 40 frame whose 63-row support regions
    leave it above and below.  BGR and gray."""
    d = detector(ctx, True)
    sxga = sxga_frames(1)[0]
    for img, rows in ((sxga, long_and_border_rows()), (short_frame(), short_frame_rows())):
        h, w = img.shape[:2]
        kl = d.keylines_from_lines(rows, w, h)
        want = oracle.lbd_keylines_from_lsd(rows, w, h)
        same_keylines(kl, want)
        assert kl["num_pixels"].max() == 1280
        if h == 960:
            assert {1280, 960, 1} <= set(kl["num_pixels"].tolist())
        for im in (img, np.ascontiguousarray(img[:, :, 1])):
            dd, ff = d.compute_descriptors(im, kl, want_float=True)
            wd, wf = oracle.lbd_compute(im, want, want_float=True)
            np.testing.assert_array_equal(dd, wd)
            np.testing.assert_array_equal(ff, wf)


# ---- 6. density and capacity --------------------------------------------------------------------------------------------------------

def test_thousands_of_keylines_and_the_capacity_error(oracle):
    """The noisy 1280 x 960 checkerboard with LSD and no length filter: 13 463 key lines, 13 463 describe CTAs in one launch.  Its 13 564
    raw segments are more candidate regions than the seed loop's first buffer (2 048) holds, so the fresh context grows it and runs the
    detector again.  One line short of the count: CS_ERR_CAPACITY naming max_lines_per_frame, and the next call is correct."""
    import cube_slam_b200 as cs
    from test_oracle_ref_lsd import CHECKERBOARDS, checkerboard
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    try:
        board = checkerboard(*CHECKERBOARDS["sxga_12px_noisy"])
        assert len(oracle.lsd_detect(board, -1.0, cap=16384)["raw_lines"]) > 2048
        want = oracle.lbd_detect_keylines(board, True, -1.0, cap=16384)
        assert len(want) == 13463
        wlines, wdesc = np.stack([want["sx"], want["sy"], want["ex"], want["ey"]], 1), oracle.lbd_compute(board, want)
        lines, desc = d.detect_descrip_lines(board, cap=16384, as_mat=True)
        np.testing.assert_array_equal(lines, wlines)
        np.testing.assert_array_equal(desc, wdesc)
        with pytest.raises(cs.CubeSlamError, match="CAPACITY.*13463 segments exceed max_lines_per_frame"):
            d.detect_descrip_lines(board, cap=len(want) - 1, as_mat=True)
        lines, desc = d.detect_descrip_lines(board, cap=len(want), as_mat=True)
        np.testing.assert_array_equal(lines, wlines)
        np.testing.assert_array_equal(desc, wdesc)
        vga = checkerboard(*CHECKERBOARDS["vga_10px"])
        want = oracle.lbd_detect_keylines(vga, True, -1.0, cap=16384)
        assert len(want) == 2760
        lines, desc = d.detect_descrip_lines(vga, cap=16384, as_mat=True)
        np.testing.assert_array_equal(lines, np.stack([want["sx"], want["sy"], want["ex"], want["ey"]], 1))
        np.testing.assert_array_equal(desc, oracle.lbd_compute(vga, want))
    finally:
        d._ctx.close()


# ---- 7. EDLines routing regimes ------------------------------------------------------------------------------------------------------

def test_edlines_descriptor_path_in_the_three_routing_regimes(ctx, oracle):
    """The key-line extras (direction -> angle, numOfPixels) come from k_ed_emit (walk-graph routing, in shared memory or HBM) or from
    k_ed_route_fit (pixel-map routing).  One batch with all three, then each frame alone; then detection-only calls (no extras) and
    descriptor calls alternating on a fresh context, whose extras buffers are allocated by the first descriptor call."""
    import cube_slam_b200 as cs
    from test_gpu_edlines_parity import routing_regime
    from test_oracle_ref_edlines import dense_frames
    fr = dense_frames()
    batch = np.stack([fr["checkerboard_window"], fr["room"], fr["room_noise_band"]])
    assert [routing_regime(oracle, img) for img in batch] == ["pixel_map", "shared", "hbm"]
    d = detector(ctx, False)
    for imgs in (batch, batch[0:1], batch[1:2], batch[2:3]):
        check_frames(oracle, d.detect_descrip_lines_batch(imgs), imgs, False, 15.0)
    fresh = cs.line_lbd_detect()
    fresh.line_length_thres = 15
    try:
        for _ in range(2):
            lines = fresh.detect_filter_lines_batch(batch)
            for f in range(3):
                np.testing.assert_array_equal(lines[f], oracle.edl_detect(batch[f], 15.0)["lines"])
            assert check_frames(oracle, fresh.detect_descrip_lines_batch(batch), batch, False, 15.0) >= 39 + 212 + 173
    finally:
        fresh._ctx.close()


# ---- 8. one context, changing sizes -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("use_lsd", [True, False], ids=["lsd", "edlines"])
def test_one_context_changing_sizes(oracle, use_lsd):
    """1280 x 960, then VGA, then tiny, then KITTI with padded rows, then a compute batch, on one context: grow-only buffers and Sobel maps
    left by a larger call must not leak into a smaller one."""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    from test_gpu_lsd_parity import odd_size_batch, row_pads
    d = cs.line_lbd_detect()
    d.use_LSD = use_lsd
    d.line_length_thres = 15
    try:
        sxga = sxga_frames(2, seed=97)
        check_frames(oracle, d.detect_descrip_lines_batch(sxga), sxga, use_lsd, 15.0)
        vga = S.make_batch(98, 2, 640, 480, 3)[0]
        check_frames(oracle, d.detect_descrip_lines_batch(vga), vga, use_lsd, 15.0)
        tiny = odd_size_batch(4, 5, 3)
        if use_lsd:
            assert [len(k) for k, _ in d.detect_descrip_lines_batch(tiny)] == [0, 0, 0]
        else:
            with pytest.raises(cs.CubeSlamError, match="INVALID_ARG"):
                d.detect_descrip_lines_batch(tiny)
        img5 = tiny_image(5, 5, 1, 55)
        rows = given_rows(5, 5, 8)
        dd, ff = d.compute_descriptors(img5, d.keylines_from_lines(rows, 5, 5), want_float=True)
        wd, wf = oracle.lbd_compute(img5, oracle.lbd_keylines_from_lsd(rows, 5, 5), want_float=True)
        np.testing.assert_array_equal(dd, wd)
        np.testing.assert_array_equal(ff, wf)
        kitti = S.make_batch(99, 2, 1242, 375, 3, kind="kitti")[0]
        check_frames(oracle, descrip_strided(d, kitti, row_pads(1242 * 3)[1]), kitti, use_lsd, 15.0)
        rows = given_rows(480, 640)
        kl = d.keylines_from_lines(rows, 640, 480)
        want = oracle.lbd_keylines_from_lsd(rows, 640, 480)
        check_given(oracle, compute_batch(d._ctx, vga, [kl, kl]), vga, [want, want])
    finally:
        d._ctx.close()


# ---- 9. the matcher --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["q2000_t5000", "ties", "pairs64_with_empty_sets", "far_and_never_met"])
def test_matcher_cases(ctx, oracle, name):
    d = detector(ctx, True)
    queries, trains, thresholds = matcher_cases()[name]
    got = {}
    for thres in thresholds:
        got[thres] = d.match_line_descrip_batch(queries, trains, thres)
        assert len(got[thres]) == len(queries)
        for p, (m, q, t) in enumerate(zip(got[thres], queries, trains)):
            wq, wt, wd = oracle.lbd_match(q, t, thres)
            np.testing.assert_array_equal(m["query_idx"], wq, err_msg="pair %d thres %g" % (p, thres))
            np.testing.assert_array_equal(m["train_idx"], wt, err_msg="pair %d thres %g" % (p, thres))
            np.testing.assert_array_equal(m["distance"], wd, err_msg="pair %d thres %g" % (p, thres))
            assert (m["img_idx"] == 0).all()
    if name == "q2000_t5000":
        assert len(queries[0]) == 2000 and len(trains[0]) == 5000 and len(got[25.0][0]) > 500
    elif name == "ties":
        m = got[300.0][0]
        np.testing.assert_array_equal(m["distance"], TIE_DISTANCES)
        in_32, in_33 = set(got[32.0][0]["query_idx"].tolist()), set(got[33.0][0]["query_idx"].tolist())
        assert in_32 == {1, 3, 5, 7} and in_33 == set(range(8))          # a distance equal to the threshold is rejected
        assert set(got[32.5][0]["query_idx"].tolist()) == in_33 and set(got[24.5][0]["query_idx"].tolist()) == in_32
        assert set(got[5.0][0]["query_idx"].tolist()) == {1, 5} and set(got[4.0][0]["query_idx"].tolist()) == set()
    elif name == "pairs64_with_empty_sets":
        for p in (0, 20, 31, 40, 63):
            assert all(len(got[t][p]) == 0 for t in thresholds)
        assert sum(len(m) for m in got[25.0]) > 100
    else:
        far = got[300.0][0]
        assert len(far) == len(queries[0]) and (far["distance"] > 128).all() and (far["train_idx"] == -1).all()
        assert all(len(got[t][k]) == 0 for t in thresholds for k in (1, 2, 3))     # never met (the `key == ~0` branch), and an empty train set


def test_sequence_pairs_in_one_call(ctx, oracle, fixture_b):
    """The LSD descriptors of the 58 frames of the shipped sequence, then every consecutive pair (57) matched in one launch."""
    d = detector(ctx, True)
    imgs = np.stack([fr[0] for fr in fixture_b["frames"]])
    out = d.detect_descrip_lines_batch(imgs)
    check_frames(oracle, out, imgs, True, 15.0)
    descs = [desc for _, desc in out]
    batch = d.match_line_descrip_batch(descs[:-1], descs[1:], 40.0)
    assert len(batch) == 57
    for p, m in enumerate(batch):
        wq, wt, wd = oracle.lbd_match(descs[p], descs[p + 1], 40.0)
        np.testing.assert_array_equal(m["query_idx"], wq)
        np.testing.assert_array_equal(m["train_idx"], wt)
        np.testing.assert_array_equal(m["distance"], wd)
    assert sum(len(m) for m in batch) > 100
