"""Frames already in GPU memory (cs_device_frames, cube_slam_b200/csrc/cs_ingest.cu) without a GPU.

The layout step -- k_ingest_frames and its launcher cs_launch_ingest, which picks a device-to-device copy for views that already are packed BGR
or gray -- is compiled from the source as it is under the CUDA-execution emulation of tests/host_core/cuda_emu_full.h (threads for CUDA
threads, host memory for device memory), and its output is compared byte for byte with numpy's ascontiguousarray of the equivalent BGR view.
The Python helper that turns __cuda_array_interface__ into the descriptor, and the argument checks of cs_check_device_frames that come
before any CUDA call, run here as well."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
SRC = os.path.join(ROOT, "cube_slam_b200", "csrc", "cs_ingest.cu")

PROLOGUE = r'''
#include "cuda_emu_full.h"
#include <cstdio>
#include "cube_slam_b200.h"
#define CS_SM_COUNT 132
'''
GLUE = r'''
extern "C" int emu_ingest(const cs_device_frames *fr, uint8_t *dst, int *launched)
{
    bool l = false;
    const int e = cs_launch_ingest(fr, dst, nullptr, &l);
    *launched = l ? 1 : 0;
    return e;
}
'''


class FakeCudaArray(object):
    """A host numpy array behind __cuda_array_interface__ (v3): what a torch CUDA tensor or a CuPy array hands over."""

    def __init__(self, a, stream=None, typestr="|u1", contiguous_as_none=True):
        self.a = a
        ai = a.__array_interface__
        self.__cuda_array_interface__ = {"shape": a.shape, "typestr": typestr, "data": (ai["data"][0], False), "version": 3,
                                         "strides": None if (contiguous_as_none and a.flags.c_contiguous) else a.strides}
        if stream is not None:
            self.__cuda_array_interface__["stream"] = stream


@pytest.fixture(scope="module")
def emu():
    bdir = os.path.join(HERE, "host_core", "_build")
    os.makedirs(bdir, exist_ok=True)
    gen, out = os.path.join(bdir, "cs_ingest_emu.cpp"), os.path.join(bdir, "libingestemu.so")
    hdr = os.path.join(HERE, "host_core", "cuda_emu_full.h")
    deps = [SRC, hdr, os.path.abspath(__file__), os.path.join(ROOT, "include", "cube_slam_b200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        text = open(SRC).read()
        body = text[text.index("#define ING_THREADS"):text.index("namespace {")]       # the kernel and its launcher, as they are
        body, n = re.subn(r"(\bk_ingest_frames<\d>)<<<([^,]+),\s*([^,]+),[^>]*>>>", r"EMU_LAUNCH(\1, \2, \3)", body)
        assert n == 2
        open(gen, "w").write(PROLOGUE + body + GLUE)
        subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-w", "-I", os.path.join(HERE, "host_core"),
                               "-I", os.path.join(HERE, "host_core", "fake_cuda_full"), "-I", os.path.join(ROOT, "include"), "-o", out, gen])
    return C.CDLL(out)


def _ingest(emu, view, order="bgr"):
    """the emulated copy of `view` (a numpy view of host bytes) -> (packed bytes, launched)"""
    from cube_slam_b200 import _lib
    d = _lib.device_frames(FakeCudaArray(view), order)
    total = d.n_frames * d.height * d.width * d.channels
    raw = np.full(total + 64 + 32, 0x5A, np.uint8)
    off = (-raw.ctypes.data) % 16                                       # the context's buffers are cudaMalloc'ed: 16-byte aligned
    launched = C.c_int(-1)
    assert emu.emu_ingest(C.byref(d), C.c_void_p(raw.ctypes.data + off), C.byref(launched)) == 0
    assert (raw[:off] == 0x5A).all() and (raw[off + total:] == 0x5A).all(), "wrote outside the packed frames"
    return raw[off:off + total].copy(), launched.value


def _rng_bytes(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


def _views(rng, F, H, W):
    """(name, view, order, BGR view it stands for, whether the layout kernel must run: True / False / None = either)"""
    nhwc = _rng_bytes(rng, (F, H, W, 3))
    nchw = _rng_bytes(rng, (F, 3, H, W))
    gray = _rng_bytes(rng, (F, H, W))
    big = _rng_bytes(rng, (F, H + 5, W + 7, 3))
    every = _rng_bytes(rng, (2 * F, H, W, 3))
    bgra = _rng_bytes(rng, (F, H, W, 4))
    raw = _rng_bytes(rng, F * H * W * 3 + 1)
    shifted = raw[1:].reshape(F, H, W, 3)                              # a base one byte past an allocation's start
    gbig = _rng_bytes(rng, (F, H + 2, W + 3))
    return [
        ("nhwc_bgr", nhwc, "bgr", nhwc, False),
        ("nhwc_rgb", nhwc, "rgb", nhwc[..., ::-1], True),
        ("nchw_bgr", nchw.transpose(0, 2, 3, 1), "bgr", nchw.transpose(0, 2, 3, 1), True),
        ("nchw_rgb", nchw.transpose(0, 2, 3, 1), "rgb", nchw.transpose(0, 2, 3, 1)[..., ::-1], True),
        ("gray", gray, "bgr", gray, False),
        ("gray_crop", gbig[:, 1:1 + H, 2:2 + W], "bgr", gbig[:, 1:1 + H, 2:2 + W], True),
        ("crop", big[:, 3:3 + H, 4:4 + W], "bgr", big[:, 3:3 + H, 4:4 + W], True),
        ("every_other_frame", every[::2], "rgb", every[::2][..., ::-1], True),
        ("every_other_frame_bgr", every[::2], "bgr", every[::2], None if F == 1 else True),
        ("bgra", bgra[..., :3], "bgr", bgra[..., :3], True),
        ("rgba", bgra[..., :3], "rgb", bgra[..., 2::-1], True),
        ("offset_base", shifted, "bgr", shifted, False),
        ("offset_base_rgb", shifted, "rgb", shifted[..., ::-1], True),
    ]


@pytest.mark.parametrize("F", [1, 3])
@pytest.mark.parametrize("W", [1242, 97, 61, 3])
def test_layout_kernel_equals_numpy(emu, F, W):
    H = 5
    rng = np.random.default_rng(W * 10 + F)
    seen = set()
    for name, view, order, want, kernel in _views(rng, F, H, W):
        got, launched = _ingest(emu, view, order)
        np.testing.assert_array_equal(got, np.ascontiguousarray(want).reshape(-1), err_msg=name)
        if kernel is not None:
            assert launched == int(kernel), name
        seen.add(launched)
    assert seen == {0, 1}                                               # both branches: the device-to-device copy and k_ingest_frames


def test_partial_last_chunk_and_one_pixel_rows(emu):
    """totals that are not a multiple of 16 bytes, rows of one pixel, one row per frame"""
    rng = np.random.default_rng(7)
    for F, H, W in ((1, 1, 1), (3, 1, 5), (2, 7, 1), (1, 3, 3)):
        a = _rng_bytes(rng, (F, H, W, 3))
        got, _ = _ingest(emu, a, "rgb")
        np.testing.assert_array_equal(got, np.ascontiguousarray(a[..., ::-1]).reshape(-1))
        p = _rng_bytes(rng, (F, 3, H, W)).transpose(0, 2, 3, 1)
        got, _ = _ingest(emu, p, "bgr")
        np.testing.assert_array_equal(got, np.ascontiguousarray(p).reshape(-1))


def test_descriptor_from_cuda_array_interface():
    from cube_slam_b200 import _lib
    a = np.zeros((4, 6, 10, 3), np.uint8)
    d = _lib.device_frames(FakeCudaArray(a))                             # strides None: C-contiguous
    assert (d.data, d.n_frames, d.height, d.width, d.channels) == (a.ctypes.data, 4, 6, 10, 3)
    assert (d.stride_frame, d.stride_row, d.stride_col, d.stride_channel) == (180, 30, 3, 1)
    assert d.channel_order == 0 and not d.stream
    v = np.zeros((2, 3, 8, 9), np.uint8).transpose(0, 2, 3, 1)[1:, 2:7, 1:]
    d = _lib.device_frames(FakeCudaArray(v), "rgb")
    assert (d.n_frames, d.height, d.width, d.channels) == (1, 5, 8, 3)
    assert (d.stride_frame, d.stride_row, d.stride_col, d.stride_channel) == (216, 9, 1, 72)
    assert d.data == v.__array_interface__["data"][0] and d.channel_order == 1
    g = np.zeros((3, 4, 5), np.uint8)[::2]
    d = _lib.device_frames(FakeCudaArray(g))
    assert (d.n_frames, d.channels, d.stride_frame, d.stride_row, d.stride_col, d.stride_channel) == (2, 1, 40, 5, 1, 0)
    d = _lib.device_frames(FakeCudaArray(np.zeros((1, 2, 2, 2), np.uint8)))   # 2 channels: passed on, the library refuses them
    assert d.channels == 2
    d = _lib.device_frames(FakeCudaArray(a), 7)                                # an integer order is passed on as well
    assert d.channel_order == 7


def test_descriptor_stream():
    from cube_slam_b200 import _lib

    class S(object):
        cuda_stream = 0x1234

    a = np.zeros((1, 2, 2, 3), np.uint8)
    assert _lib.device_frames(FakeCudaArray(a), stream=S()).stream == 0x1234       # a torch.cuda.Stream-like object
    assert _lib.device_frames(FakeCudaArray(a), stream=0x99).stream == 0x99         # a raw handle
    assert _lib.device_frames(FakeCudaArray(a, stream=0x77)).stream == 0x77         # the interface's stream
    assert _lib.device_frames(FakeCudaArray(a, stream=2)).stream == 2               # cudaStreamPerThread
    assert not _lib.device_frames(FakeCudaArray(a, stream=1)).stream                # the legacy default stream: NULL
    assert not _lib.device_frames(FakeCudaArray(a, stream=0x77), stream=0).stream   # an explicit 0 wins


def test_descriptor_rejects_wrong_dtype_rank_and_order():
    from cube_slam_b200 import _lib
    with pytest.raises(ValueError, match="uint8"):
        _lib.device_frames(FakeCudaArray(np.zeros((1, 2, 2, 3), np.uint8), typestr="<u2"))
    with pytest.raises(ValueError, match="uint8"):
        _lib.device_frames(FakeCudaArray(np.zeros((1, 2, 2, 3), np.float32).view(np.uint8)[..., :3], typestr="<f4"))
    for shape in ((4, 4), (1, 2, 2, 3, 1), (8,)):
        with pytest.raises(ValueError, match="shape"):
            _lib.device_frames(FakeCudaArray(np.zeros(shape, np.uint8)))
    with pytest.raises(ValueError, match="interface"):
        _lib.device_frames(np.zeros((1, 2, 2, 3), np.uint8))                 # host memory without the interface
    with pytest.raises(ValueError, match="order"):
        _lib.device_frames(FakeCudaArray(np.zeros((1, 2, 2, 3), np.uint8)), "bgra")


def test_new_symbols_are_exported_and_bound():
    from cube_slam_b200 import _lib
    L = _lib.load()
    for name in ("cs_check_device_frames", "cs_batch_upload_device", "cs_batch_upload_online_device", "cs_detect_lines_batch_device"):
        assert name in _lib.EXPORTS and hasattr(L, name)
        assert getattr(L, name).argtypes, name
    assert C.sizeof(_lib.DeviceFrames) == 8 + 4 * 4 + 4 * 8 + 8 + 8                # the header's layout: int32 order padded before the stream


def test_check_rejects_bad_descriptors_before_any_cuda_call():
    """The argument checks come before cudaPointerGetAttributes: on a host without a device these rejections are the same as on one."""
    from cube_slam_b200 import _lib
    L = _lib.load()
    a = np.zeros((2, 4, 5, 3), np.uint8)

    def check(**kw):
        d = _lib.device_frames(FakeCudaArray(a))
        for k, v in kw.items():
            setattr(d, k, v)
        rc = L.cs_check_device_frames(0, C.byref(d))
        return rc, L.cs_last_error(None).decode()

    assert check(stride_row=-15) == (-1, "negative stride")
    assert check(stride_channel=-1)[0] == -1
    rc, msg = check(channels=2)
    assert rc == -1 and "channels" in msg
    rc, msg = check(channel_order=5)
    assert rc == -1 and "order" in msg
    assert check(channels=1, channel_order=5)[1] != msg                        # the order is ignored for gray
    rc, msg = check(n_frames=0)
    assert rc == -1 and "empty" in msg
    rc, msg = check(data=None)
    assert rc == -1 and "null" in msg
    assert L.cs_check_device_frames(0, None) == -1
