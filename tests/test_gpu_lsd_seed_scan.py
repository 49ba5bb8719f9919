"""The LSD seed loop's word-wise scan on the GPU (cube_slam_b200/csrc/cs_lsd.cu, k_lsd_grow_seq): seeds are taken from the row-padded
"angle defined" bit plane k_lsd_front writes and the used map in the same layout, so the scaled widths where a row does not fill its last
word (W % 32 != 0) are the ones to check, beside a wide frame and a frame dense enough to overflow the candidate buffer.  Every raw
segment must be the oracle's."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_lsd_parity import _check_frame, checkerboard_batch, odd_size_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    return d


def _defb(det, frame):
    """the defined-angle plane of the last run, unpacked to one bool per pixel of the scaled image"""
    from cube_slam_b200 import _lib
    L, h = det._ctx.L, det._ctx.h
    wh = np.zeros(2, np.int32)
    assert L.cs_debug_lsd(h, frame, _lib.ptr(wh, C.c_int32), None, None, None, None, None, None, None, 0) == 0
    W, H = int(wh[0]), int(wh[1])
    ww = C.c_int32(0)
    assert L.cs_debug_lsd_defb(h, frame, None, C.byref(ww)) == 0
    assert ww.value == (W + 31) // 32
    words = np.zeros(H * ww.value, np.uint32)
    assert L.cs_debug_lsd_defb(h, frame, words.ctypes.data_as(C.POINTER(C.c_uint32)), None) == 0
    bits = np.unpackbits(words.view(np.uint8).reshape(H, ww.value * 4), axis=1, bitorder="little")
    assert not bits[:, W:].any()          # the padding of each row's last word stays clear
    return bits[:, :W].astype(bool)


@pytest.mark.parametrize("w,h,kind", [(1242, 375, "kitti"), (641, 480, "indoor"), (1280, 960, "indoor")])
def test_widths_off_the_word_size(det, oracle, w, h, kind):
    """scaled widths 994, 513 (W % 32 != 0) and 1024"""
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(w + h, 2, w, h, 3, kind=kind)[0]
    lines = det.detect_filter_lines_batch(imgs)
    for f in range(len(imgs)):
        ref = _check_frame(det, oracle, imgs[f], f)
        np.testing.assert_array_equal(lines[f], ref["lines"])
    assert sum(len(x) for x in lines) > 10


@pytest.mark.parametrize("side", [39, 41])
def test_one_word_either_side(det, oracle, side):
    """scaled widths 31 and 33: a row of fewer pixels than a word, and one that spills a single pixel into a second word"""
    imgs = odd_size_batch(side, side, 3)
    det.detect_filter_lines_batch(imgs)
    for f in range(len(imgs)):
        _check_frame(det, oracle, imgs[f], f)


def test_checkerboard_beyond_the_candidate_buffer(oracle):
    """more candidate rectangles than the hand-off buffer holds: the re-run on the grown buffer returns the oracle's segments.  A fresh
    context, so that the first run overflows."""
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.use_LSD = True
    d.line_length_thres = 15
    imgs = checkerboard_batch("vga_10px")
    lines = d.detect_filter_lines_batch(imgs, cap=16384)
    for f in range(len(imgs)):
        ref = _check_frame(d, oracle, imgs[f], f, 16384)
        np.testing.assert_array_equal(lines[f], ref["lines"])
    assert len(d.debug_frame(0, 16384)["raw_lines"]) > 2048
    d._ctx.close()


@pytest.mark.parametrize("w,h", [(1242, 375), (640, 480), (39, 39)])
def test_defined_angle_plane_is_the_angle_map(det, w, h):
    """k_lsd_front's bit plane says "defined" exactly where the angle map holds an angle"""
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(7 * w + h, 2, w, h, 3)[0] if w > 100 else odd_size_batch(h, w, 3)
    det.detect_filter_lines_batch(imgs)
    for f in range(2):
        np.testing.assert_array_equal(_defb(det, f), det.debug_frame(f)["angles"] != -1024.0)
