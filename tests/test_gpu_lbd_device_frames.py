"""The line descriptor's calls on frames already in GPU memory (cs_detect_descrip_lines_batch_device, cs_lbd_compute_batch_device through
line_lbd_detect.detect_descrip_lines_device / compute_descriptors_device), on the device.

The expected value is the host form on the equivalent numpy frames -- counts, every key-line field, descriptor bytes and the 72 floats,
compared with assert_array_equal -- and, on the fixture frames, the oracle as well.  The views are torch CUDA tensors in every layout of
tests/test_gpu_device_frames.py.  Rejections are made on the host before anything is enqueued; no case here lets the device read outside
a live allocation."""
import numpy as np
import pytest

from test_device_frames_host import FakeCudaArray
from test_gpu_device_frames import _assert_records_equal, _batch, _gray_layouts, _host_online, _layouts, _line_params, _segment_of
from test_gpu_lbd_edges import check_frames, compute_batch, same_results
from test_gpu_lsd_parity import checkerboard_batch

pytestmark = pytest.mark.gpu

THRES = 15.0


@pytest.fixture(scope="module")
def torch():
    import torch as T
    assert T.cuda.is_available()
    return T


@pytest.fixture(scope="module")
def ctx():
    import cube_slam_b200 as cs
    c = cs.Context(0, 1280, 960, 1, 1, 1)
    yield c
    c.close()


def detector(ctx, use_lsd, thres=THRES):
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(context=ctx)
    d.use_LSD = bool(use_lsd)
    d.line_length_thres = thres
    return d


def _mat(d, imgs, cap=4096):
    """the Mat overload of every frame through the host form: the batch call with no length filter"""
    keep = d.line_length_thres
    try:
        d.line_length_thres = -1.0
        out = d.detect_descrip_lines_batch(imgs, cap)
    finally:
        d.line_length_thres = keep
    return [(d._mat_rows(k), x) for k, x in out]


def _same_mat(got, want, what):
    assert len(got) == len(want)
    for f, ((la, da), (lb, db)) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(la, lb, err_msg="%s frame %d" % (what, f))
        np.testing.assert_array_equal(da, db, err_msg="%s frame %d" % (what, f))


def _frames(name, fixture_a, fixture_b):
    if name == "vga":
        return _batch(71, 3, 640, 480, 3)[0]
    if name == "kitti":
        return _batch(72, 2, 1242, 375, 8, "kitti")[0]
    if name == "fixture_a":
        return fixture_a["img"][None]
    fr = fixture_b["frames"]
    return np.stack([fr[0][0], fr[len(fr) // 2][0], fr[-1][0]])


@pytest.mark.parametrize("use_lsd", [1, 0], ids=["lsd", "edlines"])
@pytest.mark.parametrize("name", ["vga", "kitti", "fixture_a", "fixture_b"])
def test_every_layout_equals_the_host_form(torch, ctx, oracle, fixture_a, fixture_b, name, use_lsd):
    imgs = _frames(name, fixture_a, fixture_b)
    d = detector(ctx, use_lsd)
    want = d.detect_descrip_lines_batch(imgs)
    want_mat = _mat(d, imgs)
    assert sum(len(k) for k, _ in want) > 20
    gray = np.ascontiguousarray(imgs[..., 1])
    want_g = d.detect_descrip_lines_batch(gray)
    if name.startswith("fixture"):    # the host form is the oracle's here, and so is the device form
        assert check_frames(oracle, want, imgs, bool(use_lsd), THRES) > 20
        check_frames(oracle, want_g, gray, bool(use_lsd), THRES)
    for lname, view, order in _layouts(torch, imgs) + _gray_layouts(torch, gray):
        g = lname.startswith("gray")
        same_results(d.detect_descrip_lines_device(view, order), want_g if g else want, lname)
        if not g:
            _same_mat(d.detect_descrip_lines_device(view, order, as_mat=True), want_mat, lname + " as_mat")
    assert d.line_length_thres == THRES


def test_full_batch_of_256_vga_frames(torch, oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    imgs = np.ascontiguousarray(S.make_batch(73, 256, 640, 480, 3, distinct=32)[0])
    t = torch.from_numpy(imgs).cuda()
    planar_rgb = t.flip(-1).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    c = cs.Context(0, 640, 480, 256, 1, 1)
    for use_lsd in (1, 0):
        d = detector(c, use_lsd)
        want = d.detect_descrip_lines_batch(imgs, cap=2048)
        assert len(want) == 256 and sum(len(k) for k, _ in want) > 256 * 10
        same_results(d.detect_descrip_lines_device(t, cap=2048), want, "packed bgr")
        same_results(d.detect_descrip_lines_device(planar_rgb, "rgb", cap=2048), want, "planar rgb")
    c.close()


def test_given_keylines_equal_the_host_form(torch, ctx):
    imgs = _batch(74, 4, 640, 480, 3)[0]
    d = detector(ctx, 1)
    found = [k for k, _ in d.detect_descrip_lines_batch(imgs)]
    rows = np.array([[0, 0, 639, 479], [3, 400, 600, 20], [320, 5, 321, 470], [10.5, 10.25, 40.75, 12.5]], np.float32)
    given = d.keylines_from_lines(rows, 640, 480)
    per_frame = [found[0], given[:0], np.concatenate([found[2], given]), given]           # frame 1 has no key line
    want = compute_batch(ctx, imgs, per_frame)
    assert len(per_frame[0]) > 5
    gray = np.ascontiguousarray(imgs[..., 2])
    want_g = compute_batch(ctx, gray, per_frame)
    for lname, view, order in _layouts(torch, imgs) + _gray_layouts(torch, gray):
        exp = want_g if lname.startswith("gray") else want
        got = d.compute_descriptors_device(view, per_frame, want_float=True, order=order)
        codes = d.compute_descriptors_device(view, per_frame, order=order)
        for f in range(4):
            np.testing.assert_array_equal(got[f][0], exp[f][0], err_msg="%s frame %d" % (lname, f))
            np.testing.assert_array_equal(got[f][1], exp[f][1], err_msg="%s frame %d" % (lname, f))     # NaN == NaN, in the same places
            np.testing.assert_array_equal(codes[f], exp[f][0])
        assert got[1][0].shape == (0, 32) and got[1][1].shape == (0, 72)
    t = torch.from_numpy(imgs).cuda()
    empty = d.compute_descriptors_device(t, [given[:0]] * 4, want_float=True)            # an all-empty call: CS_OK, nothing described
    assert [(a.shape, b.shape) for a, b in empty] == [((0, 32), (0, 72))] * 4


def test_candidate_buffer_regrows_on_device_frames(torch):
    """A fresh context on the LSD checkerboard batch (more than 2 048 candidate rectangles in frame 0): the first run overflows the
    candidate buffer, which grows, and the run repeats on the frames still in the LSD frame buffer."""
    import cube_slam_b200 as cs
    imgs = checkerboard_batch("vga_10px")
    host = cs.line_lbd_detect()
    host.use_LSD, host.line_length_thres = True, THRES
    want = _mat(host, imgs, cap=8192)                                    # the host form, which regrows the same way
    host._ctx.close()
    dev = cs.line_lbd_detect()
    dev.use_LSD, dev.line_length_thres = True, THRES
    got = dev.detect_descrip_lines_device(torch.from_numpy(imgs).cuda(), cap=8192, as_mat=True)
    assert len(got[0][0]) > 2048 and len(got[1][0]) > 20
    _same_mat(got, want, "checkerboard")
    dev._ctx.close()


def test_frames_from_a_producer_stream(torch, ctx):
    """Frames written on a side stream behind a sleep and passed with that stream, no synchronise: the copy waits for them."""
    imgs = _batch(75, 3, 640, 480, 3)[0]
    d = detector(ctx, 1)
    want = d.detect_descrip_lines_batch(imgs)
    host = torch.from_numpy(np.ascontiguousarray(imgs[..., ::-1])).pin_memory()
    side = torch.cuda.Stream()
    for explicit in (True, False):
        frames = torch.zeros(host.shape, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(500_000_000)                      # ~0.25 s of GPU time before the frames are written
            frames.copy_(host, non_blocking=True)
            if explicit:
                got = d.detect_descrip_lines_device(frames, "rgb", stream=side)
            else:                                              # default: torch's current stream, here the side stream
                got = d.detect_descrip_lines_device(frames, "rgb")
        same_results(got, want, "explicit=%s" % explicit)
        frames2 = torch.zeros(host.shape, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        kls = [k for k, _ in want]
        with torch.cuda.stream(side):
            torch.cuda._sleep(500_000_000)
            frames2.copy_(host, non_blocking=True)
            codes = d.compute_descriptors_device(frames2, kls, order="rgb", stream=side if explicit else None)
        for f in range(3):
            np.testing.assert_array_equal(codes[f], want[f][1])
    torch.cuda.synchronize()


@pytest.mark.parametrize("use_lsd", [1, 0], ids=["lsd", "edlines"])
def test_descriptor_calls_leave_the_uploaded_batch_alone(torch, use_lsd):
    import cube_slam_b200 as cs
    imgs_a, Ts, boxes, _, K = _batch(76, 2, 640, 480, 3)
    imgs_b = _batch(77, 2, 640, 480, 3)[0]
    c = cs.Context(0, 640, 480, 2, 16, 4096)
    c.set_calibration(K)
    p = cs.default_params()
    lp = _line_params(1)
    want = _host_online(c, imgs_a, Ts, boxes, lp, p)
    assert want[1].sum() > 0
    d = detector(c, use_lsd)
    want_b = d.detect_descrip_lines_batch(imgs_b)
    a_view = _layouts(torch, imgs_a)[2][1]                      # planar: k_ingest_frames
    for lname, b_view, order in _layouts(torch, imgs_b)[:2]:    # the copy and the kernel
        c.upload_online_device(a_view, Ts, boxes, lp, p)
        same_results(d.detect_descrip_lines_device(b_view, order), want_b, lname)
        codes = d.compute_descriptors_device(b_view, [k for k, _ in want_b], order=order)
        for f in range(2):
            np.testing.assert_array_equal(codes[f], want_b[f][1])
        c.run()
        _assert_records_equal(tuple(a.copy() for a in c.fetch()), want, lname)
    c.close()


class _DeviceView(object):
    """__cuda_array_interface__ of packed bytes at an arbitrary device address"""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


def test_rejections_leave_the_context_usable(torch, ctx):
    from cube_slam_b200.detect_3d_cuboid import CubeSlamError
    imgs = _batch(78, 2, 640, 480, 3)[0]
    t = torch.from_numpy(imgs).cuda()
    d = detector(ctx, 1)
    want = d.detect_descrip_lines_batch(imgs)
    kls = [k for k, _ in want]
    counts = [len(k) for k in kls]
    assert min(counts) > 5
    base, size = _segment_of(torch, t.data_ptr())
    past = _DeviceView(base + size - imgs.nbytes + 1, imgs.shape)        # one byte beyond the allocation
    host_view = FakeCudaArray(imgs)                                       # a host pointer posing as a CUDA array

    def numoctaves_zero():
        d.numoctaves_ = 0
        try:
            d.detect_descrip_lines_device(t)
        finally:
            d.numoctaves_ = 1

    with pytest.raises(CubeSlamError) as host_cap:
        d.detect_descrip_lines_batch(imgs, cap=min(counts) - 1)
    cases = [("host pointer", lambda: d.detect_descrip_lines_device(host_view), "not device"),
             ("host pointer, given key lines", lambda: d.compute_descriptors_device(host_view, kls), "not device"),
             ("past the allocation", lambda: d.detect_descrip_lines_device(past), "allocation"),
             ("past the allocation, given key lines", lambda: d.compute_descriptors_device(past, kls), "allocation"),
             ("numoctaves 0", numoctaves_zero, "numoctaves"),
             ("capacity", lambda: d.detect_descrip_lines_device(t, cap=min(counts) - 1), "CS_ERR_CAPACITY")]
    for name, call, word in cases:
        with pytest.raises(CubeSlamError) as ei:
            call()
        assert word in str(ei.value), (name, str(ei.value))
        if name == "capacity":
            assert str(ei.value) == str(host_cap.value)                 # the host form's status and message
        same_results(d.detect_descrip_lines_device(t), want, "after " + name)
        codes = d.compute_descriptors_device(t, kls)
        for f in range(2):
            np.testing.assert_array_equal(codes[f], want[f][1], err_msg="after " + name)
