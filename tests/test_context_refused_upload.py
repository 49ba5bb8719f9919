"""A refused upload leaves the prepared batch as it was.  cs_context.cu is compiled for the host (tests/host_core/context_refused_emu.cpp)
with launchers that record the frames, gray planes and ROI bytes they are asked to read and write, each checked against the batch's frame
buffer.  A 320 x 240 BGR batch is uploaded and run; then 1280 x 960 uploads -- one-size and mixed -- are refused for their box CSR, and a run
must still be the 320 x 240 batch's, inside its buffer.  An upload refused after the batch was given up runs nothing (CS_ERR_NOT_PREPARED)."""
import ctypes as C
import os
import subprocess

import numpy as np


def _build():
    here = os.path.dirname(os.path.abspath(__file__))
    csrc = os.path.join(here, "..", "cube_slam_b200", "csrc")
    src = os.path.join(here, "host_core", "context_refused_emu.cpp")
    out = os.path.join(here, "host_core", "_build", "libcontextrefused.so")
    deps = [src, os.path.join(here, "host_core", "cuda_emu.h"), os.path.join(here, "host_core", "fake_cuda", "cuda_runtime.h")]
    deps += [os.path.join(csrc, f) for f in ("cs_context.cu", "cs_carried.h", "cs_internal.h", "cs_kernels.h", "cs_host_pose.cpp", "cs_host_pose.h", "cs_nccl_impl.inc")]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-w", "-I", os.path.join(here, "host_core", "fake_cuda"),
                               "-x", "c++", "-o", out, src, os.path.join(csrc, "cs_host_pose.cpp"), "-ldl"])
    return out


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def test_a_refused_upload_leaves_the_prepared_batch_as_it_was():
    from cube_slam_b200 import _lib
    E = C.CDLL(_build())
    E.cs_create.restype = C.c_void_p
    E.cs_last_error.restype = C.c_char_p
    ctx = C.c_void_p(E.cs_create(0, 1280, 960, 4, 16, 4096))
    K = np.array([[400.0, 0, 160], [0, 400, 120], [0, 0, 1]])
    assert E.cs_set_calibration(ctx, _p(K, C.c_double)) == 0
    prm = _lib.CuboidParams()
    E.cs_default_cuboid_params(C.byref(prm))
    T = np.ascontiguousarray(np.tile(np.eye(4).reshape(16), (2, 1)))
    T[:, 11] = 1.0
    lines = np.array([[10.0, 10, 200, 20], [30, 200, 300, 150]] * 2)
    line_off = np.array([0, 2, 4], np.int32)
    rec = np.zeros(9, np.int64)

    def upload(w, h, box_off):
        imgs = np.zeros((2, h, w, 3), np.uint8)
        boxes = np.array([[50.0, 50, 100, 80, 0.9], [120, 60, 90, 100, 0.8]])
        return E.cs_batch_upload(ctx, imgs.ctypes.data_as(C.c_void_p), 2, w, h, w * 3, 3, _p(T, C.c_double), _p(boxes, C.c_double),
                                 _p(np.asarray(box_off, np.int32), C.c_int32), _p(lines, C.c_double), _p(line_off, C.c_int32), C.byref(prm))

    def run_and_check():
        assert E.cs_batch_run(ctx) == 0, E.cs_last_error(ctx)
        E.emu_record(_p(rec, C.c_int64))
        assert rec[1] == 0 and rec[3] == 0, rec                                  # nothing read or written outside the frame buffer
        assert tuple(rec[4:9]) == (2, 320, 240, 960, 3), rec                     # the prepared batch's frames

    assert upload(320, 240, [0, 1, 2]) == 0, E.cs_last_error(ctx)
    run_and_check()
    for box_off in ([1, 1, 2], [0, 2, 1]):                                       # first offset not 0; decreasing offsets
        assert upload(1280, 960, box_off) == -1
        run_and_check()
    views = (_lib.FrameView * 2)()
    for f, (w, h) in enumerate(((1280, 960), (640, 480))):
        views[f].offset, views[f].width, views[f].height, views[f].stride, views[f].channels = f * 1280 * 960 * 3, w, h, w * 3, 3
    boxes = np.array([[50.0, 50, 100, 80, 0.9], [120, 60, 90, 100, 0.8]])
    assert E.emu_store_mixed(ctx, views, 2, _p(T, C.c_double), _p(boxes, C.c_double), _p(np.array([1, 1, 2], np.int32), C.c_int32),
                             _p(lines, C.c_double), _p(line_off, C.c_int32), C.byref(prm)) == -1
    run_and_check()
    # refused after the batch was given up (an ROI outside the image fails the table build): nothing left to run
    assert E.cs_batch_upload(ctx, np.zeros((2, 240, 320, 3), np.uint8).ctypes.data_as(C.c_void_p), 2, 320, 240, 960, 3, _p(T, C.c_double),
                             _p(np.array([[400.0, 50, 100, 80, 0.9], [120, 60, 90, 100, 0.8]]), C.c_double), _p(np.array([0, 1, 2], np.int32), C.c_int32),
                             _p(lines, C.c_double), _p(line_off, C.c_int32), C.byref(prm)) == -1
    assert E.cs_batch_run(ctx) == -4
    E.cs_destroy(ctx)
