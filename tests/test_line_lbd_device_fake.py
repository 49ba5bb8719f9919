"""The Python mirror's descriptor calls on frames already in GPU memory (line_lbd_detect.detect_descrip_lines_device and
compute_descriptors_device), WITHOUT a GPU.  The two device entry points are replaced by a stand-in that reads the view through the
cs_device_frames it is given -- data pointer, strides, channel order -- from host memory behind a fake __cuda_array_interface__, and answers
from the CPU oracle through the same C signatures.  Checked here: the descriptor the mirror builds (strides, order, stream), the per-frame
slots it unpacks (empty frames included), and the arguments it refuses before calling the library.  What the kernels compute is tested on
the GPU (tests/test_gpu_lbd_device_frames.py)."""
import ctypes as C

import numpy as np
import pytest

from test_device_frames_host import FakeCudaArray
from test_line_lbd_mirror_fake import FakeContext, _view


def _frames_of(d):
    """the BGR (or gray) pixels a cs_device_frames stands for, read through its strides from host memory"""
    F, H, W, ch = d.n_frames, d.height, d.width, d.channels
    extent = (F - 1) * d.stride_frame + (H - 1) * d.stride_row + (W - 1) * d.stride_col + (2 * d.stride_channel if ch == 3 else 0) + 1
    raw = np.frombuffer((C.c_char * extent).from_address(d.data), np.uint8)
    if ch == 1:
        return np.lib.stride_tricks.as_strided(raw, (F, H, W), (d.stride_frame, d.stride_row, d.stride_col)).copy()
    v = np.lib.stride_tricks.as_strided(raw, (F, H, W, 3), (d.stride_frame, d.stride_row, d.stride_col, d.stride_channel))
    return np.ascontiguousarray(v[..., ::-1] if d.channel_order == 1 else v)


class FakeDeviceLib(object):
    """Delegates to the real libcubeslam_b200.so except for the two device-frame descriptor calls."""

    def __init__(self, real, oracle, _lib):
        self._real, self._o, self._lib = real, oracle, _lib
        self.calls = []

    def __getattr__(self, name):
        return getattr(self._real, name)

    @staticmethod
    def _descriptor(fr):
        d = fr._obj
        return dict(data=d.data, shape=(d.n_frames, d.height, d.width, d.channels), order=d.channel_order, stream=d.stream or 0,
                    strides=(d.stride_frame, d.stride_row, d.stride_col, d.stride_channel))

    def cs_detect_descrip_lines_batch_device(self, h, fr, params, kl, desc, cap, n):
        p, frames = params._obj, _frames_of(fr._obj)
        F = len(frames)
        k = _view(kl, self._lib.KEYLINE_DTYPE, F * cap).reshape(F, cap)
        d, nn = _view(desc, np.uint8, F * cap * 32).reshape(F, cap, 32), _view(n, np.int32, F)
        for f in range(F):
            want = self._o.lbd_detect_keylines(frames[f], bool(p.use_LSD), float(p.line_length_thres))
            k[f, :len(want)] = want.view(self._lib.KEYLINE_DTYPE)
            d[f, :len(want)] = self._o.lbd_compute(frames[f], want)
            nn[f] = len(want)
        self.calls.append(("detect_descrip_device", self._descriptor(fr), float(p.line_length_thres), cap))
        return 0

    def cs_lbd_compute_batch_device(self, h, fr, kl, off, desc, fdesc):
        frames = _frames_of(fr._obj)
        F = len(frames)
        o = _view(off, np.int32, F + 1).copy()
        self.calls.append(("compute_device", self._descriptor(fr), o, bool(fdesc)))
        if o[-1] == 0:
            return 0                                                       # no key line: outputs left as they are
        k = _view(kl, self._lib.KEYLINE_DTYPE, int(o[-1])).view(self._o.KEYLINE_DTYPE)
        dd, ff = _view(desc, np.uint8, int(o[-1]) * 32).reshape(-1, 32), _view(fdesc, np.float32, int(o[-1]) * 72).reshape(-1, 72) if fdesc else None
        for f in range(F):
            if o[f + 1] > o[f]:
                a, b = self._o.lbd_compute(frames[f], k[o[f]:o[f + 1]], want_float=True)
                dd[o[f]:o[f + 1]] = a
                if ff is not None:
                    ff[o[f]:o[f + 1]] = b
        return 0


@pytest.fixture()
def det(oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    d = cs.line_lbd_detect(context=FakeContext(FakeDeviceLib(_lib.load(), oracle, _lib)))
    d.line_length_thres = 15
    return d


@pytest.fixture(scope="module")
def imgs(fixture_b):
    """two fixture frames around a flat one, which has no line"""
    a, b = fixture_b["frames"][4][0], fixture_b["frames"][21][0]
    return np.stack([a, np.full_like(a, 90), b])


def _same_keylines(got, want):
    assert len(got) == len(want) and got.dtype.itemsize == 40
    for a, b in zip(got.dtype.names, want.dtype.names):
        np.testing.assert_array_equal(got[a], want[b], err_msg=a)


class _Stream(object):
    cuda_stream = 0x5150


def test_detect_descrip_lines_device_descriptor_and_slots(det, oracle, imgs):
    F, H, W, _ = imgs.shape
    planar = np.ascontiguousarray(imgs[..., ::-1].transpose(0, 3, 1, 2))          # NCHW RGB, as a decoder hands it over
    big = np.zeros((F, H + 4, W + 6, 3), np.uint8)
    big[:, 1:1 + H, 2:2 + W] = imgs
    gray = np.ascontiguousarray(imgs[..., 1])
    cases = [("nhwc_bgr", FakeCudaArray(imgs), "bgr", None, (H * W * 3, W * 3, 3, 1), 0, 0),
             ("nchw_rgb", FakeCudaArray(planar.transpose(0, 2, 3, 1)), "rgb", _Stream(), (3 * H * W, W, 1, H * W), 1, 0x5150),
             ("crop", FakeCudaArray(big[:, 1:1 + H, 2:2 + W], stream=0x77), "bgr", None, ((H + 4) * (W + 6) * 3, (W + 6) * 3, 3, 1), 0, 0x77),
             ("gray", FakeCudaArray(gray), "bgr", 0x99, (H * W, W, 1, 0), 0, 0x99)]
    for use_lsd in (True, False):
        det.use_LSD = use_lsd
        want = {c: [oracle.lbd_detect_keylines(x[f], use_lsd, 15.0) for f in range(F)] for c, x in (("bgr", imgs), ("gray", gray))}
        for name, view, order, stream, strides, code, handle in cases:
            out = det.detect_descrip_lines_device(view, order, cap=700, stream=stream)
            call = det._ctx.L.calls[-1]
            assert call[0] == "detect_descrip_device" and call[2] == 15.0 and call[3] == 700
            d = call[1]
            assert d["data"] == view.__cuda_array_interface__["data"][0], name
            assert d["strides"] == strides and d["order"] == code and d["stream"] == handle, (name, d)
            assert d["shape"] == (F, H, W, 1 if name == "gray" else 3)
            src = gray if name == "gray" else imgs
            assert len(out) == F
            for f, (kl, desc) in enumerate(out):
                w = want["gray" if name == "gray" else "bgr"][f]
                _same_keylines(kl, w)
                assert desc.shape == (len(w), 32) and desc.dtype == np.uint8
                np.testing.assert_array_equal(desc, oracle.lbd_compute(src[f], w))
            assert len(out[1][0]) == 0 and out[1][1].shape == (0, 32)            # the flat frame: an empty slot
            assert len(out[0][0]) > 10 and len(out[2][0]) > 10


def test_detect_descrip_lines_device_mat_overload(det, oracle, imgs):
    det.use_LSD = True
    out = det.detect_descrip_lines_device(FakeCudaArray(imgs[:2]), as_mat=True)
    assert det._ctx.L.calls[-1][2] == -1.0 and det.line_length_thres == 15
    for f, (lines, desc) in enumerate(out):
        want = oracle.lbd_detect_keylines(imgs[f], True, -1.0)
        assert lines.dtype == np.float32 and lines.shape == (len(want), 4)
        np.testing.assert_array_equal(lines, np.stack([want["sx"], want["sy"], want["ex"], want["ey"]], 1))
        np.testing.assert_array_equal(desc, oracle.lbd_compute(imgs[f], want))
    assert out[1][0].shape == (0, 4) and out[1][1].shape == (0, 32)


def test_compute_descriptors_device_csr_and_slots(det, oracle, imgs):
    F, H, W, _ = imgs.shape
    k0 = det.keylines_from_lines(np.array([[10, 20, 200, 40], [50, 300, 60, 100]], np.float32), W, H)
    k2 = det.keylines_from_lines(np.array([[5, 5, 400, 400], [600, 10, 30, 470], [100, 100, 140, 100]], np.float32), W, H)
    planar = np.ascontiguousarray(imgs.transpose(0, 3, 1, 2)).transpose(0, 2, 3, 1)
    for view, order in ((FakeCudaArray(imgs), "bgr"), (FakeCudaArray(planar), "bgr"), (FakeCudaArray(np.ascontiguousarray(imgs[..., ::-1])), "rgb")):
        out = det.compute_descriptors_device(view, [k0, k0[:0], k2], want_float=True, order=order, stream=0x42)
        call = det._ctx.L.calls[-1]
        assert call[0] == "compute_device" and call[1]["stream"] == 0x42 and call[3]
        np.testing.assert_array_equal(call[2], [0, 2, 2, 5])
        assert len(out) == 3 and out[1][0].shape == (0, 32) and out[1][1].shape == (0, 72)
        for f, k in ((0, k0), (2, k2)):
            wd, wf = oracle.lbd_compute(imgs[f], k.view(oracle.KEYLINE_DTYPE), want_float=True)
            np.testing.assert_array_equal(out[f][0], wd)
            np.testing.assert_array_equal(out[f][1], wf)
        codes = det.compute_descriptors_device(view, [k0, k0[:0], k2], order=order)
        assert not det._ctx.L.calls[-1][3]
        for f in range(3):
            np.testing.assert_array_equal(codes[f], out[f][0])
    empty = det.compute_descriptors_device(FakeCudaArray(imgs), [k0[:0]] * 3, want_float=True)     # an all-empty call
    np.testing.assert_array_equal(det._ctx.L.calls[-1][2], [0, 0, 0, 0])
    assert [(d.shape, f.shape) for d, f in empty] == [((0, 32), (0, 72))] * 3


def test_device_forms_refuse_bad_arguments_before_the_library(det, imgs):
    import cube_slam_b200 as cs
    k = det.keylines_from_lines(np.array([[10, 20, 200, 40]], np.float32), imgs.shape[2], imgs.shape[1])
    bad = [("host array", imgs, ValueError, "interface"),
           ("uint16", FakeCudaArray(imgs, typestr="<u2"), ValueError, "uint8"),
           ("rank 2", FakeCudaArray(imgs[0, :, :, 0]), ValueError, "shape"),
           ("rank 5", FakeCudaArray(imgs[..., None]), ValueError, "shape")]
    calls = len(det._ctx.L.calls)
    for name, x, exc, word in bad:
        with pytest.raises(exc, match=word):
            det.detect_descrip_lines_device(x)
        with pytest.raises(exc, match=word):
            det.compute_descriptors_device(x, [k] * 3)
    with pytest.raises(ValueError, match="order"):
        det.detect_descrip_lines_device(FakeCudaArray(imgs), order="bgra")
    with pytest.raises(cs.CubeSlamError, match="one key-line array per frame"):
        det.compute_descriptors_device(FakeCudaArray(imgs), [k, k])
    assert len(det._ctx.L.calls) == calls
