"""Every octave of a multi-octave LSD line_lbd_detect on the device (cs_lbd_octaves.cu: cs_detect_raw_lines_octaves_batch,
cs_detect_descrip_lines_octaves_batch and their device-frame forms, through line_lbd_detect.detect_raw_lines_octaves /
detect_descrip_lines_octaves).

The expected value is the oracle's restatement (pyoracle_octaves.lsd_octaves_raw / lsd_octaves_descrip), which tests/test_oracle_ref_lsd_octaves.py
pins to the reference's own class: every key-line field and every descriptor byte, compared with assert_array_equal.  Octave 0 must also be
what the one-octave calls return, and the device forms what the host forms return."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

THRES = 15.0


@pytest.fixture(scope="module")
def ctx():
    import cube_slam_b200 as cs
    c = cs.Context(0, 1280, 960, 1, 1, 1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def octo(oracle):
    """oracle/pyoracle_octaves.py: the multi-octave restatement (and the reference's own class where it can be built)"""
    from oracle import pyoracle_octaves
    return pyoracle_octaves


def detector(ctx, numoctaves=3, ratio=2.0, thres=THRES):
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(numoctaves, ratio, context=ctx)
    d.use_LSD = True
    d.line_length_thres = thres
    return d


def same_keylines(got, want, what):
    """product records (OCTAVE_KEYLINE_DTYPE) against the oracle's, field by field in declaration order"""
    assert len(got) == len(want), "%s: %d key lines, oracle %d" % (what, len(got), len(want))
    assert len(got.dtype.names) == len(want.dtype.names)
    for a, b in zip(got.dtype.names, want.dtype.names):
        np.testing.assert_array_equal(got[a], want[b], err_msg="%s field %s" % (what, a))


def check_descrip(out, imgs, numoctaves, ratio, octo, what):
    for f, (kls, descs) in enumerate(out):
        wk, wd = octo.lsd_octaves_descrip(imgs[f], numoctaves, ratio, THRES)
        assert len(kls) == len(descs) == numoctaves
        for k in range(numoctaves):
            same_keylines(kls[k], wk[k], "%s frame %d octave %d" % (what, f, k))
            np.testing.assert_array_equal(descs[k], wd[k], err_msg="%s frame %d octave %d descriptors" % (what, f, k))


def check_raw(out, imgs, numoctaves, ratio, octo, what):
    for f, kls in enumerate(out):
        want = octo.lsd_octaves_raw(imgs[f], numoctaves, ratio)
        assert len(kls) == numoctaves
        for k in range(numoctaves):
            same_keylines(kls[k], want[k], "%s frame %d octave %d" % (what, f, k))


def test_synthetic_vga_batch_of_256_three_octaves(ctx, octo):
    from cube_slam_b200 import synthetic
    imgs = synthetic.make_batch(11, 256, 640, 480)[0]
    d = detector(ctx, 3, 2.0)
    out = d.detect_descrip_lines_octaves_batch(imgs)
    assert sum(len(k) for kls, _ in out for k in kls[1:]) > 0      # the higher octaves did find lines
    check_descrip(out, imgs, 3, 2.0, octo, "vga")
    check_raw(d.detect_raw_lines_octaves_batch(imgs[:24]), imgs[:24], 3, 2.0, octo, "vga raw")


@pytest.mark.parametrize("numoctaves,ratio", [(2, 2.0), (3, 2.0), (3, 2.5)])
def test_fixture_b_batch(ctx, octo, fixture_b, numoctaves, ratio):
    imgs = np.stack([fr[0] for fr in fixture_b["frames"]])
    d = detector(ctx, numoctaves, ratio)
    check_descrip(d.detect_descrip_lines_octaves_batch(imgs), imgs, numoctaves, ratio, octo, "fixture B")
    check_raw(d.detect_raw_lines_octaves_batch(imgs[::7]), imgs[::7], numoctaves, ratio, octo, "fixture B raw")


@pytest.mark.parametrize("w,h", [(211, 97), (1242, 375), (161, 120)])
@pytest.mark.parametrize("gray", [False, True])
def test_odd_sizes(ctx, oracle, octo, w, h, gray):
    import cv2
    from cube_slam_b200 import synthetic
    imgs = np.stack([cv2.resize(x, (w, h), interpolation=cv2.INTER_AREA) for x in synthetic.make_batch(w + h, 3, 640, 480)[0]])
    if gray:
        imgs = np.ascontiguousarray(np.stack([oracle.bgr2gray(x) for x in imgs]))
    for ratio in (2.0, 2.5):
        d = detector(ctx, 3, ratio)
        check_descrip(d.detect_descrip_lines_octaves_batch(imgs), imgs, 3, ratio, octo, "%dx%d" % (w, h))
        check_raw(d.detect_raw_lines_octaves_batch(imgs), imgs, 3, ratio, octo, "%dx%d raw" % (w, h))


def test_octave_zero_is_the_one_octave_result(ctx, fixture_a, fixture_b):
    from cube_slam_b200 import synthetic
    imgs = [fixture_a["img"]] + [fixture_b["frames"][i][0] for i in (0, 5, 30)] + list(synthetic.make_batch(3, 4, 640, 480)[0])
    one = detector(ctx, 1, 1.0)
    for n in (1, 2, 3):
        d = detector(ctx, n, 2.0)
        for i, img in enumerate(imgs):
            kls, descs = d.detect_descrip_lines_octaves_batch(img[None])[0]
            [k1], [d1] = one.detect_descrip_lines_octaves(img)
            same_keylines(kls[0][list(k1.dtype.names)], k1, "frame %d, %d octaves" % (i, n))
            assert (kls[0]["octave"] == 0).all()
            np.testing.assert_array_equal(kls[0]["s_oct_x"], kls[0]["start_x"])
            np.testing.assert_array_equal(descs[0], d1)
            raw0 = d.detect_raw_lines_octaves(img)[0]
            rows = np.stack([raw0["start_x"], raw0["start_y"], raw0["end_x"], raw0["end_y"]], 1)
            np.testing.assert_array_equal(rows, one.detect_raw_lines(img))


def test_flat_raw_lines_are_every_octave_in_order(ctx, octo, fixture_b):
    img = fixture_b["frames"][5][0]
    d = detector(ctx, 3, 2.0)
    want = np.concatenate(octo.lsd_octaves_raw(img, 3, 2.0))
    rows = np.stack([want["sx"], want["sy"], want["ex"], want["ey"]], 1)
    np.testing.assert_array_equal(d.detect_raw_lines(img), rows)
    import cv2
    half = np.concatenate(octo.lsd_octaves_raw(cv2.resize(img, None, fx=0.5, fy=0.5), 3, 2.0))
    np.testing.assert_array_equal(d.detect_raw_lines(img, downsample_img=True),
                                  np.stack([half["sx"], half["sy"], half["ex"], half["ey"]], 1) * np.float32(2))


def test_device_forms_equal_host_forms(ctx):
    import torch
    from cube_slam_b200 import synthetic
    imgs = synthetic.make_batch(5, 6, 640, 480)[0]
    d = detector(ctx, 3, 2.0)
    want = d.detect_descrip_lines_octaves_batch(imgs)
    want_raw = d.detect_raw_lines_octaves_batch(imgs)
    gray = np.ascontiguousarray(np.stack([synthetic.cv2.cvtColor(x, synthetic.cv2.COLOR_BGR2GRAY) for x in imgs]))
    t = torch.from_numpy(imgs).cuda()
    planar_rgb = t.flip(-1).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)    # NCHW storage seen as NHWC, RGB order
    views = [(t, "bgr", want, want_raw), (planar_rgb, "rgb", want, want_raw),
             (torch.from_numpy(gray).cuda(), "bgr", d.detect_descrip_lines_octaves_batch(gray), d.detect_raw_lines_octaves_batch(gray))]
    for v, order, w, wr in views:
        got = d.detect_descrip_lines_octaves_device(v, order)
        got_raw = d.detect_raw_lines_octaves_device(v, order)
        for f in range(len(imgs)):
            for k in range(3):
                np.testing.assert_array_equal(got[f][0][k], w[f][0][k])
                np.testing.assert_array_equal(got[f][1][k], w[f][1][k])
                np.testing.assert_array_equal(got_raw[f][k], wr[f][k])
    torch.cuda.synchronize()


def test_refusals_return_their_status(ctx):
    from cube_slam_b200 import _lib
    L, h = ctx.L, ctx.h
    img = np.zeros((1, 64, 64), np.uint8)
    kl = np.zeros(64, _lib.OCTAVE_KEYLINE_DTYPE)
    desc = np.zeros((64, 32), np.uint8)
    n = np.zeros(8, np.int32)

    def call(use_lsd, numoctaves, ratio, cap=4, w=64, hh=64, describe=True):
        p = _lib.LineParams(int(use_lsd), numoctaves, ratio, THRES)
        a = np.zeros((1, hh, w), np.uint8)
        if describe:
            return L.cs_detect_descrip_lines_octaves_batch(h, a.ctypes.data, 1, w, hh, w, 1, C.byref(p), kl.ctypes.data, _lib.ptr(desc, C.c_uint8), cap,
                                                           _lib.ptr(n, C.c_int32))
        return L.cs_detect_raw_lines_octaves_batch(h, a.ctypes.data, 1, w, hh, w, 1, C.byref(p), kl.ctypes.data, cap, _lib.ptr(n, C.c_int32))

    for describe in (True, False):
        assert call(False, 2, 2.0, describe=describe) == -6                 # EDLines: CS_ERR_UNSUPPORTED
        assert call(True, 0, 2.0, describe=describe) == -1
        for ratio in (1.0, 3.0, 1.99):
            assert call(True, 2, ratio, describe=describe) == -1
            assert "pyrDown" in L.cs_last_error(h).decode()
        assert call(True, 1, 1.0, describe=describe) == 0                   # one octave never calls pyrDown
        assert call(True, 7, 2.0, describe=describe) == -1                   # octave 6 of 64 x 64 is 1 x 1
        assert "too small" in L.cs_last_error(h).decode()
    # capacity: a frame with more segments in octave 1 than the slots hold
    from cube_slam_b200 import synthetic
    frame = synthetic.make_batch(2, 1, 640, 480)[0]
    p = _lib.LineParams(1, 2, 2.0, THRES)
    big = np.zeros(2 * 8, _lib.OCTAVE_KEYLINE_DTYPE)
    bd = np.zeros((2 * 8, 32), np.uint8)
    rc = L.cs_detect_descrip_lines_octaves_batch(h, frame.ctypes.data, 1, 640, 480, 640 * 3, 3, C.byref(p), big.ctypes.data, _lib.ptr(bd, C.c_uint8), 8,
                                                 _lib.ptr(n, C.c_int32))
    assert rc == -3
    msg = L.cs_last_error(h).decode()
    assert "frame 0" in msg and "octave 0" in msg, msg
    d = detector(ctx, 2, 1.0)
    import cube_slam_b200 as cs
    with pytest.raises(cs.CubeSlamError):
        d.detect_descrip_lines_octaves(img[0])
    # the one-octave members keep working after a refusal
    assert len(detector(ctx, 2, 2.0).detect_descrip_lines_octaves(frame[0])[0]) == 2


def test_shim_matches_the_oracle(ctx, octo, fixture_b):
    """shim/line_lbd_b200.cpp's multi-octave members, built against the reference's own class header (oracle/_ref/libshim_line.so), return
    the restated oracle's key lines and descriptors -- the values tests/test_oracle_ref_lsd_octaves.py pins to the reference's own class --
    in every KeyLine field, with KeyLine::pt the mid point of the ends."""
    import os
    shim = os.path.join(os.path.dirname(octo.__file__), "_ref", "libshim_line.so")
    if not os.path.exists(shim):
        pytest.skip("oracle/_ref has no shim build")
    lib = C.CDLL(shim)
    if not hasattr(lib, "shim_lsd_octaves"):
        pytest.skip("the shim build predates the octave members")
    lib.shim_lsd_octaves.restype = C.c_int
    vp = C.c_void_p
    lib.shim_lsd_octaves.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, vp, vp, vp, C.c_int]
    for img in (fixture_b["frames"][0][0], fixture_b["frames"][30][0]):
        raw = octo.lsd_octaves_raw(img, 3, 2.0)
        wk, wd = octo.lsd_octaves_descrip(img, 3, 2.0, THRES)
        for mode in (0, 1, 2):
            cap = 8192
            kl = np.zeros((4, cap), octo.OCTAVE_KEYLINE_DTYPE)
            desc = np.zeros((4, cap, 32), np.uint8)
            cnt = np.zeros(4, np.int32)
            h, w = img.shape[:2]
            a = np.ascontiguousarray(img)
            k = lib.shim_lsd_octaves(a.ctypes.data, w, h, 3, 3, 2.0, THRES, mode, kl.ctypes.data, desc.ctypes.data, cnt.ctypes.data, cap)
            assert k == 3, k
            for o in range(3):
                np.testing.assert_array_equal(kl[o, :cnt[o]], wk[o] if mode == 2 else raw[o])
                if mode == 2:
                    np.testing.assert_array_equal(desc[o, :cnt[o]], wd[o])
