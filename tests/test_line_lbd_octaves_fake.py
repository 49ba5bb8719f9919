"""The Python mirror's octave calls (line_lbd_detect.detect_raw_lines_octaves[_batch|_device], detect_raw_lines and
detect_descrip_lines_octaves[_batch|_device] of a multi-octave LSD detector), WITHOUT a GPU.  The four octave entry points are replaced by a
stand-in that answers from the CPU oracle (pyoracle_octaves.lsd_octaves_raw / lsd_octaves_descrip) through the same C signatures: slot (f, k) at
(f * numoctaves + k) * cap, n_lines holding n_frames * numoctaves counts.  Checked here: the 64-byte record, the per-frame and per-octave
split, which member calls which entry point, and the refusals the mirror makes before calling the library."""
import ctypes as C

import numpy as np
import pytest

from test_device_frames_host import FakeCudaArray
from test_line_lbd_device_fake import _frames_of
from test_line_lbd_mirror_fake import FakeContext, FakeLib, _view


class FakeOctaveLib(FakeLib):
    def __init__(self, real, oracle, _lib):
        super().__init__(real, oracle, _lib)
        from oracle import pyoracle_octaves
        self._octo = pyoracle_octaves

    def _fill(self, frames, params, kl, desc, cap, n, describe):
        p = params._obj
        K, F = p.numoctaves, len(frames)
        k = _view(kl, self._lib.OCTAVE_KEYLINE_DTYPE, F * K * cap).reshape(F, K, cap)
        nn = _view(n, np.int32, F * K).reshape(F, K)
        d = _view(desc, np.uint8, F * K * cap * 32).reshape(F, K, cap, 32) if describe else None
        for f in range(F):
            if describe:
                kls, descs = self._octo.lsd_octaves_descrip(frames[f], K, float(p.octaveratio), float(p.line_length_thres))
            else:
                kls, descs = self._octo.lsd_octaves_raw(frames[f], K, float(p.octaveratio)), None
            for o in range(K):
                assert len(kls[o]) <= cap
                k[f, o, :len(kls[o])] = kls[o].view(self._lib.OCTAVE_KEYLINE_DTYPE)
                k[f, o, len(kls[o]):] = np.frombuffer(b"\xee" * 64, self._lib.OCTAVE_KEYLINE_DTYPE)   # slots past the count
                if describe:
                    d[f, o, :len(kls[o])] = descs[o]
                nn[f, o] = len(kls[o])
        self.calls.append(("octaves", describe, K))
        return 0

    def cs_detect_raw_lines_octaves_batch(self, h, imgs, F, W, H, stride, ch, params, kl, cap, n):
        return self._fill(self._frames(imgs, F, W, H, stride, ch), params, kl, None, cap, n, False)

    def cs_detect_descrip_lines_octaves_batch(self, h, imgs, F, W, H, stride, ch, params, kl, desc, cap, n):
        return self._fill(self._frames(imgs, F, W, H, stride, ch), params, kl, desc, cap, n, True)

    def cs_detect_raw_lines_octaves_batch_device(self, h, fr, params, kl, cap, n):
        self.calls.append(("device",))
        return self._fill(_frames_of(fr._obj), params, kl, None, cap, n, False)

    def cs_detect_descrip_lines_octaves_batch_device(self, h, fr, params, kl, desc, cap, n):
        self.calls.append(("device",))
        return self._fill(_frames_of(fr._obj), params, kl, desc, cap, n, True)


@pytest.fixture(scope="module")
def octo(oracle):
    """oracle/pyoracle_octaves.py: the multi-octave restatement (and the reference's own class where it can be built)"""
    from oracle import pyoracle_octaves
    return pyoracle_octaves


@pytest.fixture()
def det(oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    d = cs.line_lbd_detect(3, 2.0, context=FakeContext(FakeOctaveLib(_lib.load(), oracle, _lib)))
    d.use_LSD = True
    d.line_length_thres = 15
    return d


def test_record_layout():
    from cube_slam_b200 import _lib
    from oracle import pyoracle_octaves
    dt = _lib.OCTAVE_KEYLINE_DTYPE
    assert dt.itemsize == 64 and pyoracle_octaves.OCTAVE_KEYLINE_DTYPE.itemsize == 64
    assert dt.names[:len(_lib.KEYLINE_DTYPE.names)] == _lib.KEYLINE_DTYPE.names
    assert [dt.fields[n][1] for n in _lib.KEYLINE_DTYPE.names] == [_lib.KEYLINE_DTYPE.fields[n][1] for n in _lib.KEYLINE_DTYPE.names]
    assert dt.names[len(_lib.KEYLINE_DTYPE.names):] == ("s_oct_x", "s_oct_y", "e_oct_x", "e_oct_y", "octave", "pad_")
    assert [dt.fields[n][1] for n in ("s_oct_x", "octave", "pad_")] == [40, 56, 60]


def test_batch_slots_and_octave_split(det, octo, fixture_b):
    imgs = np.stack([fixture_b["frames"][i][0] for i in (0, 9, 33)])
    out = det.detect_descrip_lines_octaves_batch(imgs, cap=512)
    raw = det.detect_raw_lines_octaves_batch(imgs, cap=512)
    assert len(out) == len(raw) == 3
    for f in range(3):
        wk, wd = octo.lsd_octaves_descrip(imgs[f], 3, 2.0, 15.0)
        wr = octo.lsd_octaves_raw(imgs[f], 3, 2.0)
        kls, descs = out[f]
        assert len(kls) == len(descs) == len(raw[f]) == 3
        for k in range(3):
            assert kls[k].dtype == raw[f][k].dtype and kls[k].dtype.itemsize == 64
            np.testing.assert_array_equal(kls[k].view(wk[k].dtype), wk[k])
            np.testing.assert_array_equal(descs[k], wd[k])
            np.testing.assert_array_equal(raw[f][k].view(wr[k].dtype), wr[k])
            assert (kls[k]["octave"] == k).all()


def test_single_frame_members(det, octo, fixture_a):
    img = fixture_a["img"]
    kls, descs = det.detect_descrip_lines_octaves(img)
    wk, wd = octo.lsd_octaves_descrip(img, 3, 2.0, 15.0)
    for k in range(3):
        np.testing.assert_array_equal(kls[k].view(wk[k].dtype), wk[k])
        np.testing.assert_array_equal(descs[k], wd[k])
    raw = np.concatenate(octo.lsd_octaves_raw(img, 3, 2.0))
    np.testing.assert_array_equal(det.detect_raw_lines(img), np.stack([raw["sx"], raw["sy"], raw["ex"], raw["ey"]], 1))
    assert [c[0] for c in det._ctx.L.calls] == ["octaves", "octaves"]
    assert len(det.detect_raw_lines_octaves(img)) == 3


def test_device_forms_read_the_view(det, octo, fixture_b):
    imgs = np.stack([fixture_b["frames"][i][0] for i in (0, 5)])
    host = det.detect_descrip_lines_octaves_batch(imgs, cap=512)
    rgb = FakeCudaArray(np.ascontiguousarray(imgs[..., ::-1]))
    got = det.detect_descrip_lines_octaves_device(rgb, order="rgb", cap=512)
    got_raw = det.detect_raw_lines_octaves_device(FakeCudaArray(imgs), cap=512)
    for f in range(2):
        for k in range(3):
            np.testing.assert_array_equal(got[f][0][k], host[f][0][k])
            np.testing.assert_array_equal(got[f][1][k], host[f][1][k])
            np.testing.assert_array_equal(got_raw[f][k].view(octo.OCTAVE_KEYLINE_DTYPE), octo.lsd_octaves_raw(imgs[f], 3, 2.0)[k])
    assert ("device",) in det._ctx.L.calls


def test_refusals_before_the_library(det, fixture_a):
    import cube_slam_b200 as cs
    img = fixture_a["img"]
    for ratio in (1.0, 3.0, 1.5):
        det.octaveratio_ = ratio
        with pytest.raises(cs.CubeSlamError):
            det.detect_descrip_lines_octaves(img)
        with pytest.raises(cs.CubeSlamError):
            det.detect_raw_lines(img)
    det.octaveratio_ = 2.0
    det.use_LSD = False
    for member in (det.detect_descrip_lines_octaves, det.detect_raw_lines, det.detect_raw_lines_octaves):
        with pytest.raises(cs.CubeSlamError):
            member(img)
    assert det._ctx.L.calls == []


def test_one_octave_keeps_its_entry_points(oracle, fixture_a):
    """numoctaves == 1: detect_raw_lines and detect_descrip_lines_octaves go through the one-octave entry points, whatever the ratio"""
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    img = fixture_a["img"]
    for ratio in (1.0, 2.0):
        d = cs.line_lbd_detect(1, ratio, context=FakeContext(FakeOctaveLib(_lib.load(), oracle, _lib)))
        d.use_LSD = True
        d.line_length_thres = 15
        d.detect_raw_lines(img)
        d.detect_descrip_lines_octaves(img)
        assert [c[0] for c in d._ctx.L.calls] == ["detect_lines", "detect_descrip"]
        assert len(d.detect_raw_lines_octaves(img)) == 1                  # the octave call itself also takes one octave
