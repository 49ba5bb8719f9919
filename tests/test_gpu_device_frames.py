"""Frames already in GPU memory (cs_device_frames) through the batch cuboid path and the line detectors, on the device.

The expected value is always the host path on the equivalent numpy BGR (or gray) frames, which the other GPU suites pin to the oracle and
the reference: every record field is compared with assert_array_equal (NaN == NaN), and counts, lines and error statuses are compared as
well.  The views are torch CUDA tensors in every layout the descriptor stands for: packed NHWC BGR and gray (the device-to-device copy),
RGB, planar NCHW, crops, every other frame, BGRA / RGBA, and a base one byte into an allocation (k_ingest_frames).  Rejections are made on
the host by cs_check_device_frames; no case here lets the device read outside a live allocation."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINE_THRES = 15.0


@pytest.fixture(scope="module")
def torch():
    import torch as T
    assert T.cuda.is_available()
    return T


def _layouts(torch, imgs):
    """(name, device view, order) for a numpy BGR batch F x H x W x 3; each view holds exactly imgs' pixels"""
    F, H, W, _ = imgs.shape
    dev = torch.device("cuda", 0)
    t = torch.from_numpy(np.ascontiguousarray(imgs)).to(dev)
    out = [("nhwc_bgr", t, "bgr"),
           ("nhwc_rgb", t.flip(-1).contiguous(), "rgb"),
           ("nchw_bgr", t.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1), "bgr"),
           ("nchw_rgb", t.flip(-1).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1), "rgb")]
    big = torch.zeros((F, H + 6, W + 10, 3), dtype=torch.uint8, device=dev)
    big[:, 2:2 + H, 3:3 + W] = t
    out.append(("crop", big[:, 2:2 + H, 3:3 + W], "bgr"))
    every = torch.zeros((2 * F, H, W, 3), dtype=torch.uint8, device=dev)
    every[::2] = t
    out.append(("every_other_frame", every[::2], "bgr"))
    bgra = torch.full((F, H, W, 4), 255, dtype=torch.uint8, device=dev)
    bgra[..., :3] = t
    out.append(("bgra", bgra[..., :3], "bgr"))
    rgba = torch.full((F, H, W, 4), 7, dtype=torch.uint8, device=dev)
    rgba[..., :3] = t.flip(-1)
    out.append(("rgba", rgba[..., :3], "rgb"))
    flat = torch.zeros(F * H * W * 3 + 1, dtype=torch.uint8, device=dev)
    flat[1:] = t.reshape(-1)
    out.append(("offset_base", flat[1:].view(F, H, W, 3), "bgr"))
    flat_rgb = torch.zeros(F * H * W * 3 + 1, dtype=torch.uint8, device=dev)
    flat_rgb[1:] = t.flip(-1).reshape(-1)
    out.append(("offset_base_rgb", flat_rgb[1:].view(F, H, W, 3), "rgb"))
    return out


def _gray_layouts(torch, gray):
    F, H, W = gray.shape
    dev = torch.device("cuda", 0)
    g = torch.from_numpy(np.ascontiguousarray(gray)).to(dev)
    big = torch.zeros((F, H + 3, W + 5), dtype=torch.uint8, device=dev)
    big[:, 1:1 + H, 2:2 + W] = g
    every = torch.zeros((2 * F, H, W), dtype=torch.uint8, device=dev)
    every[::2] = g
    return [("gray", g, "bgr"), ("gray_crop", big[:, 1:1 + H, 2:2 + W], "bgr"), ("gray_every_other_frame", every[::2], "bgr")]


def _assert_records_equal(got, want, what):
    (r1, c1), (r2, c2) = got, want
    np.testing.assert_array_equal(c1, c2, err_msg=what)
    assert r1.dtype == r2.dtype and r1.shape == r2.shape, what
    for name in r1.dtype.names:
        np.testing.assert_array_equal(r1[name], r2[name], err_msg="%s: %s" % (what, name))


def _line_params(use_lsd):
    from cube_slam_b200 import _lib
    p = _lib.LineParams()
    _lib.load().cs_default_line_params(C.byref(p))
    p.use_LSD = int(use_lsd)
    p.line_length_thres = LINE_THRES
    return p


def _host_online(ctx, imgs, Ts, boxes, lp, p):
    ctx.upload_online(imgs, Ts, boxes, lp, p)
    ctx.run()
    r, c = ctx.fetch()
    return r.copy(), c.copy()


def _dev_online(ctx, view, order, Ts, boxes, lp, p, stream=None):
    ctx.upload_online_device(view, Ts, boxes, lp, p, order=order, stream=stream)
    ctx.run()
    r, c = ctx.fetch()
    return r.copy(), c.copy()


def _batch(seed, F, w, h, nb, kind="indoor"):
    from cube_slam_b200 import synthetic as S
    return S.make_batch(seed, F, w, h, nb, kind=kind, poisson=(kind == "indoor"))


@pytest.mark.parametrize("use_lsd", [1, 0])
def test_upload_online_device_every_layout(torch, use_lsd):
    import cube_slam_b200 as cs
    imgs, Ts, boxes, _, K = _batch(61, 3, 640, 480, 3)
    ctx = cs.Context(0, 640, 480, 3, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    lp = _line_params(use_lsd)
    want = _host_online(ctx, imgs, Ts, boxes, lp, p)
    assert want[1].sum() > 0
    for name, view, order in _layouts(torch, imgs):
        _assert_records_equal(_dev_online(ctx, view, order, Ts, boxes, lp, p), want, name)
    gray = np.ascontiguousarray(imgs[..., 1])
    want_g = _host_online(ctx, gray, Ts, boxes, lp, p)
    for name, view, order in _gray_layouts(torch, gray):
        _assert_records_equal(_dev_online(ctx, view, order, Ts, boxes, lp, p), want_g, name)
    ctx.close()


def test_upload_device_every_layout(torch):
    """the given-lines path (cs_batch_upload_device) against cs_batch_upload"""
    import cube_slam_b200 as cs
    imgs, Ts, boxes, lines, K = _batch(62, 3, 640, 480, 3)
    ctx = cs.Context(0, 640, 480, 3, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=3)
    ctx.upload(imgs, Ts, boxes, lines, p)
    ctx.run()
    want = tuple(a.copy() for a in ctx.fetch())
    assert want[1].sum() > 0
    for name, view, order in _layouts(torch, imgs):
        ctx.upload_device(view, Ts, boxes, lines, p, order=order)
        ctx.run()
        _assert_records_equal(tuple(a.copy() for a in ctx.fetch()), want, name)
    gray = np.ascontiguousarray(imgs[..., 2])
    ctx.upload(gray, Ts, boxes, lines, p)
    ctx.run()
    want_g = tuple(a.copy() for a in ctx.fetch())
    for name, view, order in _gray_layouts(torch, gray):
        ctx.upload_device(view, Ts, boxes, lines, p, order=order)
        ctx.run()
        _assert_records_equal(tuple(a.copy() for a in ctx.fetch()), want_g, name)
    ctx.close()


@pytest.mark.parametrize("w,h,nb,kind", [(1242, 375, 8, "kitti"), (1280, 960, 3, "indoor")])
def test_upload_online_device_at_kitti_and_sxga(torch, w, h, nb, kind):
    import cube_slam_b200 as cs
    imgs, Ts, boxes, _, K = _batch(63, 2, w, h, nb, kind)
    ctx = cs.Context(0, w, h, 2, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    lp = _line_params(1)
    want = _host_online(ctx, imgs, Ts, boxes, lp, p)
    assert want[1].sum() > 0
    for name, view, order in _layouts(torch, imgs):
        if name in ("nhwc_bgr", "nhwc_rgb", "nchw_rgb", "crop", "bgra", "offset_base_rgb"):
            _assert_records_equal(_dev_online(ctx, view, order, Ts, boxes, lp, p), want, name)
    ctx.close()


def _host_lines(det, imgs, cap=4096):
    try:
        return det.detect_filter_lines_batch(imgs, cap), None
    except Exception as e:   # noqa: BLE001 -- the error status is part of what is compared
        return None, str(e)


def _dev_lines(det, view, order, cap=4096):
    try:
        return det.detect_filter_lines_device(view, order, cap), None
    except Exception as e:   # noqa: BLE001
        return None, str(e)


@pytest.mark.parametrize("use_lsd", [True, False])
@pytest.mark.parametrize("w,h", [(640, 480), (1242, 375), (3, 3)])
def test_detect_filter_lines_device(torch, use_lsd, w, h):
    import cube_slam_b200 as cs
    if (w, h) == (3, 3):
        rng = np.random.default_rng(3)
        imgs = rng.integers(0, 256, (3, 3, 3, 3), dtype=np.uint8)
    else:
        imgs = _batch(64, 2, w, h, 3, "kitti" if w == 1242 else "indoor")[0]
    det = cs.line_lbd_detect(max_width=1280, max_height=960)
    det.use_LSD = use_lsd
    det.line_length_thres = LINE_THRES
    want, want_err = _host_lines(det, imgs)
    if (w, h) == (3, 3):
        if use_lsd:      # LSD on a 3 x 3 frame finds nothing and says CS_OK
            assert want_err is None and all(len(l) == 0 for l in want)
        else:            # the EDLines detector's own 8 x 8 minimum
            assert want is None and "CS_ERR_INVALID_ARG" in want_err
    else:
        assert want_err is None and sum(len(l) for l in want) > 0
    for name, view, order in _layouts(torch, imgs) + _gray_layouts(torch, np.ascontiguousarray(imgs[..., 0])):
        exp, exp_err = (want, want_err) if not name.startswith("gray") else _host_lines(det, np.ascontiguousarray(imgs[..., 0]))
        got, err = _dev_lines(det, view, order)
        assert err == exp_err, name
        if exp is not None:
            assert len(got) == len(exp)
            for f in range(len(exp)):
                np.testing.assert_array_equal(got[f], exp[f], err_msg="%s frame %d" % (name, f))


@pytest.mark.parametrize("use_lsd", [True, False])
def test_detecting_lines_between_upload_and_run_keeps_the_batch(torch, use_lsd):
    """Batch A uploaded from device frames, then lines detected from device frames B on the same context, then A run: A's records."""
    import cube_slam_b200 as cs
    imgs_a, Ts, boxes, _, K = _batch(65, 2, 640, 480, 3)
    imgs_b = _batch(66, 2, 640, 480, 3)[0]
    ctx = cs.Context(0, 640, 480, 2, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params()
    lp = _line_params(1)
    want = _host_online(ctx, imgs_a, Ts, boxes, lp, p)
    det = cs.line_lbd_detect(context=ctx)
    det.use_LSD = use_lsd
    det.line_length_thres = LINE_THRES
    want_b = det.detect_filter_lines_batch(imgs_b)
    a_view = _layouts(torch, imgs_a)[2][1]                     # planar: k_ingest_frames
    for name, b_view, order in _layouts(torch, imgs_b)[:2]:    # the copy and the kernel
        ctx.upload_online_device(a_view, Ts, boxes, lp, p)
        got_b = det.detect_filter_lines_device(b_view, order)
        for f in range(2):
            np.testing.assert_array_equal(got_b[f], want_b[f])
        ctx.run()
        _assert_records_equal(tuple(a.copy() for a in ctx.fetch()), want, name)
    ctx.close()


@pytest.mark.parametrize("layout", ["nhwc_bgr", "nhwc_rgb"])
def test_stream_order_without_host_sync(torch, layout):
    """Frames written on a side stream behind a sleep, uploaded with that stream and no synchronise: the library reads them after they are
    written; frames.zero_() queued on the same stream right after the upload returns runs after the library has read them."""
    import cube_slam_b200 as cs
    imgs, Ts, boxes, _, K = _batch(67, 3, 640, 480, 3)
    ctx = cs.Context(0, 640, 480, 3, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params(max_cuboid_num=2)
    lp = _line_params(1)
    want = _host_online(ctx, imgs, Ts, boxes, lp, p)
    src = imgs if layout == "nhwc_bgr" else np.ascontiguousarray(imgs[..., ::-1])
    host = torch.from_numpy(src).pin_memory()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    for explicit in (True, False):
        frames = torch.empty(host.shape, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(500_000_000)                      # ~0.25 s of GPU time before the frames are written
            frames.copy_(host, non_blocking=True)
            order = "bgr" if layout == "nhwc_bgr" else "rgb"
            if explicit:
                ctx.upload_online_device(frames, Ts, boxes, lp, p, order=order, stream=side)
            else:                                              # default: torch's current stream, here the side stream
                ctx.upload_online_device(frames, Ts, boxes, lp, p, order=order)
            frames.zero_()
        assert not side.query(), "the side stream finished before the checks could mean anything"
        ctx.run()
        _assert_records_equal(tuple(a.copy() for a in ctx.fetch()), want, "%s explicit=%s" % (layout, explicit))
        torch.cuda.synchronize()
        assert int(frames.max()) == 0                           # and the zero_ did run
    ctx.close()


def _segment_of(torch, ptr):
    """(base, size) of the cudaMalloc'ed segment of torch's caching allocator that holds ptr"""
    for s in torch.cuda.memory_snapshot():
        if s["address"] <= ptr < s["address"] + s["total_size"]:
            return s["address"], s["total_size"]
    raise AssertionError("no segment holds the tensor")


def test_check_device_frames_rejections(torch):
    from cube_slam_b200 import _lib
    L = _lib.load()
    F, H, W = 2, 48, 64
    t = torch.zeros((F, H, W, 3), dtype=torch.uint8, device="cuda")

    def check(d):
        rc = L.cs_check_device_frames(0, C.byref(d))
        return rc, L.cs_last_error(None).decode()

    good = _lib.device_frames(t)
    assert check(good)[0] == 0
    host = np.zeros((F, H, W, 3), np.uint8)                  # a host pointer
    d = _lib.device_frames(t)
    d.data = host.ctypes.data
    rc, msg = check(d)
    assert rc == -1 and "not device" in msg, msg
    # a packed view that ends exactly at the end of its allocation passes; one frame or one byte further does not
    base, size = _segment_of(torch, t.data_ptr())
    n = F * H * W * 3
    d = _lib.device_frames(t)
    d.data = base + size - n
    assert check(d)[0] == 0
    d.n_frames = F + 1
    d.data = base + size - n
    rc, msg = check(d)
    assert rc == -1 and "allocation" in msg, msg
    d = _lib.device_frames(t)
    d.data = base + size - n + 1
    rc, msg = check(d)
    assert rc == -1 and "allocation" in msg, msg
    for field, value, word in (("stride_col", -3, "negative"), ("channels", 2, "channels"), ("channel_order", 2, "order")):
        d = _lib.device_frames(t)
        setattr(d, field, value)
        rc, msg = check(d)
        assert rc == -1 and word in msg, (field, msg)


def test_entry_point_rejections_leave_the_context_usable(torch):
    import cube_slam_b200 as cs
    from cube_slam_b200.detect_3d_cuboid import CubeSlamError
    imgs, Ts, boxes, _, K = _batch(68, 2, 640, 480, 3)
    ctx = cs.Context(0, 640, 480, 2, 16, 4096)
    ctx.set_calibration(K)
    p = cs.default_params()
    lp = _line_params(1)
    want = _host_online(ctx, imgs, Ts, boxes, lp, p)
    t = torch.from_numpy(imgs).cuda()
    det = cs.line_lbd_detect(context=ctx)
    det.use_LSD = True
    det.line_length_thres = LINE_THRES
    want_lines = det.detect_filter_lines_batch(imgs)
    big = torch.zeros((3, 480, 640, 3), dtype=torch.uint8, device="cuda")
    wide = torch.zeros((2, 480, 648, 3), dtype=torch.uint8, device="cuda")
    cases = [("unknown order", lambda: ctx.upload_online_device(t, Ts, boxes, lp, p, order=5), "CS_ERR_INVALID_ARG"),
             ("zero frames", lambda: ctx.upload_online_device(t[:0], Ts[:0], [], lp, p), "CS_ERR_INVALID_ARG"),
             ("more frames than cs_create", lambda: ctx.upload_online_device(big, np.concatenate([Ts, Ts[:1]]), list(boxes) + [boxes[0]], lp, p),
              "CS_ERR_CAPACITY"),
             ("wider than cs_create", lambda: ctx.upload_online_device(wide, Ts, boxes, lp, p), "CS_ERR_CAPACITY"),
             ("given lines, unknown order", lambda: ctx.upload_device(t, Ts, boxes, [np.zeros((0, 4))] * 2, p, order=9), "CS_ERR_INVALID_ARG"),
             ("lines, unknown order", lambda: det.detect_filter_lines_device(t, order=3), "CS_ERR_INVALID_ARG"),
             ("lines, zero frames", lambda: det.detect_filter_lines_device(t[:0]), "CS_ERR_INVALID_ARG")]
    for name, call, status in cases:
        with pytest.raises(CubeSlamError) as ei:
            call()
        assert status in str(ei.value), (name, str(ei.value))
        if status == "CS_ERR_CAPACITY":
            assert "capacities" in str(ei.value)             # the host forms' wording
        _assert_records_equal(_dev_online(ctx, t, "bgr", Ts, boxes, lp, p), want, "after " + name)
        got = det.detect_filter_lines_device(t)
        for f in range(2):
            np.testing.assert_array_equal(got[f], want_lines[f])
    ctx.close()
