"""BinaryDescriptor::compute on key lines of any octave on the device (cs_lbd_compute_octaves_batch[_device], through
line_lbd_detect.compute_descriptors_octaves[_batch|_device]).

The expected bytes are the oracle's restatement (pyoracle_compute_octaves.lbd_compute_octaves), which tests/test_oracle_ref_lbd_compute_octaves.py pins
to the reference's own BinaryDescriptor::compute; where oracle/_ref holds the compiled reference, the bytes and the 72-float descriptor are also
compared with it directly (assert_array_equal, as tests/test_z_gpu_lbd_parity.py compares the float descriptor).  The key lines come from
LSDDetector::detect(img, 2, K), as a caller of line_descriptor would take them, and from lists a detector never returns."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(1, 1.0, max_width=1280, max_height=960)
    d.use_LSD = True
    d.line_length_thres = 15.0
    yield d
    d._ctx.close()


@pytest.fixture(scope="module")
def octo(oracle):
    from oracle import pyoracle_compute_octaves
    return pyoracle_compute_octaves


@pytest.fixture(scope="module")
def has_ref(octo):
    return octo.ref_available()


def _synthetic(w, h, gray, seed):
    import cv2
    from cube_slam_b200 import synthetic
    img = synthetic.make_batch(seed, 1, 640, 480)[0][0]
    if (w, h) != (640, 480):
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
    return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)) if gray else img


def _gray(img):
    import cv2
    return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY))


def _check(det, octo, has_ref, img, kl, what):
    """the product's bytes and floats against the restatement and, where it is built, the reference's own compute"""
    got, gotf = det.compute_descriptors_octaves(img, kl, want_float=True)
    assert got.shape == (len(kl), 32) and gotf.shape == (len(kl), 72)
    np.testing.assert_array_equal(got, octo.lbd_compute_octaves(img, kl), err_msg=what)
    if has_ref:
        want, wantf = octo.ref_lbd_compute_octaves(img, kl, want_float=True)
        keys = list(zip(kl["class_id"].tolist(), kl["octave"].tolist()))
        rows = [i for i, k in enumerate(keys) if keys.index(k) == i]      # the reference never writes the later rows of a pair
        np.testing.assert_array_equal(got[rows], want[rows], err_msg=what + " (reference)")
        np.testing.assert_array_equal(gotf[rows], wantf[rows], err_msg=what + " (reference, float)")
    return got, gotf


@pytest.mark.parametrize("gray", [False, True])
def test_detector_lists_one_to_four_octaves(det, octo, has_ref, fixture_a, fixture_b, gray):
    frames = [("fixture A", fixture_a["img"])] + [("fixture B %d" % i, fixture_b["frames"][i][0]) for i in (0, 30)]
    frames += [("synthetic %d" % s, _synthetic(640, 480, False, s)) for s in (3, 4)]
    frames += [("641x479", _synthetic(641, 479, False, 5)), ("97x211", _synthetic(97, 211, False, 7))]
    deepest = []
    for name, img in frames:
        img = _gray(img) if gray else img
        full = det.lsd.detect(img, 2, 4)
        deepest.append(int(full["octave"].max()))
        for K in (1, 2, 3, 4):
            kl = full[full["octave"] < K]
            _check(det, octo, has_ref, img, kl, "%s, %d octaves" % (name, K))
    assert deepest.count(3) >= 5, deepest


def test_batch_of_vga_frames_is_each_frame_alone(det, octo):
    from cube_slam_b200 import synthetic
    imgs = synthetic.make_batch(11, 16, 640, 480)[0]
    kls = [det.lsd.detect(img, 2, 3) for img in imgs]
    out = det.compute_descriptors_octaves_batch(imgs, kls, want_float=True)
    for f, (d, fd) in enumerate(out):
        one, onef = det.compute_descriptors_octaves(imgs[f], kls[f], want_float=True)
        np.testing.assert_array_equal(d, one)
        np.testing.assert_array_equal(fd, onef)
        np.testing.assert_array_equal(d, octo.lbd_compute_octaves(imgs[f], kls[f]))


def test_lists_a_detector_never_returns(det, octo, has_ref, fixture_b):
    rng = np.random.default_rng(4)
    img = fixture_b["frames"][30][0]
    kl = det.lsd.detect(img, 2, 3)
    _check(det, octo, has_ref, img, kl[rng.permutation(len(kl))], "shuffled")
    deep = kl[kl["octave"] == 2]
    _check(det, octo, has_ref, img, deep, "deepest octave only")
    # repeated (class_id, octave) pairs: the first row of a pair gets the last one's descriptor, the others their own
    dup = np.concatenate([kl[:40], kl[5:15], kl[kl["octave"] == 1][:6], kl[:3]])
    dup["class_id"][40:50] = dup["class_id"][:10]
    got, gotf = _check(det, octo, has_ref, img, dup, "repeated pairs")
    pairs = octo.pair_rows(dup)
    assert len(pairs) == 10
    for i in range(len(dup)):
        own, ownf = det.compute_descriptors_octaves(img, dup[i:i + 1], want_float=True)
        j = pairs.get(i, i)
        src, srcf = det.compute_descriptors_octaves(img, dup[j:j + 1], want_float=True)
        np.testing.assert_array_equal(got[i], src[0])
        np.testing.assert_array_equal(gotf[i], srcf[0])
        if i not in pairs:
            np.testing.assert_array_equal(got[i], own[0])
    # in-octave ends on and beyond the octave's border
    h, w = img.shape[:2]
    edge = kl[:30].copy()
    for j, o in enumerate(edge):
        ow, oh = w >> int(o["octave"]), h >> int(o["octave"])
        edge[j]["s_oct_x"], edge[j]["e_oct_x"] = (ow - 1, ow + 3.5) if j % 3 == 0 else ((-2.5, 0) if j % 3 == 1 else (0, ow - 1))
        edge[j]["s_oct_y"], edge[j]["e_oct_y"] = (oh - 1, oh + 7) if j % 2 else (-4, oh - 1)
    _check(det, octo, has_ref, img, edge, "ends at the border")
    # a filtered subset skips class ids (the reference crashes there): each row is still its own descriptor
    sub = kl[kl["line_length"] > 30]
    got = det.compute_descriptors_octaves(img, sub)
    np.testing.assert_array_equal(got, octo.lbd_compute_octaves(img, sub))
    np.testing.assert_array_equal(got, np.concatenate([det.compute_descriptors_octaves(img, sub[i:i + 1]) for i in range(len(sub))]))
    # one batch: an empty frame, a 1-octave frame and a 4-octave frame
    from cube_slam_b200 import synthetic
    imgs = synthetic.make_batch(9, 3, 640, 480)[0]
    lists = [det.lsd.detect(imgs[0], 2, 1)[:0], det.lsd.detect(imgs[1], 2, 1), det.lsd.detect(imgs[2], 2, 4)]
    out = det.compute_descriptors_octaves_batch(imgs, lists, want_float=True)
    assert out[0][0].shape == (0, 32) and out[0][1].shape == (0, 72)
    for f in (1, 2):
        want, wantf = _check(det, octo, has_ref, imgs[f], lists[f], "mixed batch frame %d" % f)
        np.testing.assert_array_equal(out[f][0], want)
        np.testing.assert_array_equal(out[f][1], wantf)
    assert [len(x) for x in det.compute_descriptors_octaves_batch(imgs, [lists[0]] * 3)] == [0, 0, 0]


def test_octave_zero_is_cs_lbd_compute(det, fixture_a, fixture_b):
    from cube_slam_b200 import _lib
    for img in (fixture_a["img"], _gray(fixture_b["frames"][9][0]), _synthetic(641, 479, False, 12)):
        kl = det.lsd.detect(img, 2, 1)
        one = np.zeros(len(kl), _lib.KEYLINE_DTYPE)
        for f in _lib.KEYLINE_DTYPE.names:
            one[f] = kl[f]
        one["start_x"], one["start_y"], one["end_x"], one["end_y"] = kl["s_oct_x"], kl["s_oct_y"], kl["e_oct_x"], kl["e_oct_y"]
        d, fd = det.compute_descriptors(img, one, want_float=True)
        got, gotf = det.compute_descriptors_octaves(img, kl, want_float=True)
        np.testing.assert_array_equal(got, d)
        np.testing.assert_array_equal(gotf, fd)


def test_detect_descrip_lines_octaves_from_its_raw_key_lines(det, fixture_b):
    """cs_detect_raw_lines_octaves_batch's key lines, filtered as detect_descrip_lines_octaves filters them (line_lbd_allclass.cpp:312-317)
    and before its end swap, give the descriptors cs_detect_descrip_lines_octaves_batch returns"""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic
    imgs = np.concatenate([np.stack([fixture_b["frames"][i][0] for i in (0, 17, 40)]), synthetic.make_batch(21, 3, 640, 480)[0]])
    for ratio in (2.0, 2.5):
        d = cs.line_lbd_detect(3, ratio, context=det._ctx)
        d.use_LSD = True
        d.line_length_thres = 15.0
        raw = d.detect_raw_lines_octaves_batch(imgs)
        described = d.detect_descrip_lines_octaves_batch(imgs)
        kept = []
        for f in range(len(imgs)):
            kept.append(np.concatenate([o[o["line_length"] * np.float32(np.float32(ratio).astype(np.float64) ** k) > np.float32(15.0)]
                                        for k, o in enumerate(raw[f])]))
        out = d.compute_descriptors_octaves_batch(imgs, kept)
        for f in range(len(imgs)):
            np.testing.assert_array_equal(out[f], np.concatenate(described[f][1]), err_msg="frame %d, ratio %g" % (f, ratio))


def test_device_views_equal_the_host_form(det):
    import torch
    from cube_slam_b200 import synthetic
    big = synthetic.make_batch(6, 6, 640, 480)[0]
    crop = np.ascontiguousarray(big[:, 7:7 + 451, 3:3 + 601])
    t = torch.from_numpy(big).cuda()
    views = [(t[:, 7:7 + 451, 3:3 + 601], "bgr", crop), (t.flip(-1).contiguous(), "rgb", big), (t[::2], "bgr", big[::2]),
             (torch.from_numpy(np.ascontiguousarray(np.stack([_gray(x) for x in big]))).cuda(), "bgr", np.stack([_gray(x) for x in big]))]
    for v, order, host in views:
        kls = [det.lsd.detect(x, 2, 3) for x in host]
        want = det.compute_descriptors_octaves_batch(host, kls, want_float=True)
        got = det.compute_descriptors_octaves_device(v, kls, want_float=True, order=order)
        for f in range(len(host)):
            np.testing.assert_array_equal(got[f][0], want[f][0])
            np.testing.assert_array_equal(got[f][1], want[f][1])
    torch.cuda.synchronize()


def test_refusals_name_the_frame_and_row(det, fixture_a):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    L, h = det._ctx.L, det._ctx.h
    img = _synthetic(97, 211, True, 8)
    kl = det.lsd.detect(img, 2, 2)
    assert len(kl) > 6
    imgs = np.stack([img, img])
    off = np.array([0, 3, 6], np.int32)
    desc = np.full((6, 32), 7, np.uint8)

    def call(rows, offsets=off):
        rows = np.ascontiguousarray(rows, _lib.OCTAVE_KEYLINE_DTYPE)
        return L.cs_lbd_compute_octaves_batch(h, imgs.ctypes.data, 2, 97, 211, 97, 1, rows.ctypes.data, _lib.ptr(offsets, C.c_int32),
                                              _lib.ptr(desc, C.c_uint8), None)

    base = kl[:6].copy()
    for field, value, text in (("class_id", -1, "class_id -1"), ("octave", -2, "octave -2"), ("octave", 7, "pyrDown")):
        bad = base.copy()
        bad[field][4] = value
        assert call(bad) == -1
        msg = L.cs_last_error(h).decode()
        assert "frame 1, row 1" in msg and text in msg, msg
        assert (desc == 7).all()                                                  # nothing written
    ok = base.copy()
    ok["octave"][4] = 6                                                           # 97 x 211 -> ... -> 1 x 3: the deepest level pyrDown makes
    assert call(ok) == 0
    assert call(base, np.array([1, 3, 6], np.int32)) == -1 and "start at 0" in L.cs_last_error(h).decode()
    assert call(base, np.array([0, 4, 3], np.int32)) == -1 and "decrease" in L.cs_last_error(h).decode()
    with pytest.raises(cs.CubeSlamError, match="pyrDown"):
        bad = base.copy()
        bad["octave"][0] = 9
        det.compute_descriptors_octaves(img, bad)
    # the next call on the same context is correct
    full = det.lsd.detect(fixture_a["img"], 2, 3)
    from oracle import pyoracle_compute_octaves
    np.testing.assert_array_equal(det.compute_descriptors_octaves(fixture_a["img"], full),
                                  pyoracle_compute_octaves.lbd_compute_octaves(fixture_a["img"], full))
