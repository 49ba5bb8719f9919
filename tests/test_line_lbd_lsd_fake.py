"""The Python mirror of LSDDetector (line_lbd_detect.lsd: detect, detect_octaves, detect([images])) WITHOUT a GPU.  The library's
cs_detect_raw_lines_octaves_batch is replaced by the stand-in of tests/test_line_lbd_octaves_fake.py, which answers from the CPU oracle
(pyoracle_octaves.lsd_octaves_raw) through the same C signature, and here can also answer CS_ERR_CAPACITY below a given buffer size.
Checked: the per-octave and flat answers, the mask rule in numpy, one call per image size in the vector form, BGRA input, the capacity retry
and the refusals made before the library is called."""
import numpy as np
import pytest

from test_line_lbd_mirror_fake import FakeContext
from test_line_lbd_octaves_fake import FakeOctaveLib


class FakeCapacityLib(FakeOctaveLib):
    min_cap = 0

    def cs_detect_raw_lines_octaves_batch(self, h, imgs, F, W, H, stride, ch, params, kl, cap, n):
        self.calls.append(("raw", F, W, H, ch, cap))
        if cap < self.min_cap:
            return -3
        return self._fill(self._frames(imgs, F, W, H, stride, ch), params, kl, None, cap, n, False)


@pytest.fixture()
def lsd(oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    return cs.line_lbd_detect(context=FakeContext(FakeCapacityLib(_lib.load(), oracle, _lib))).lsd


@pytest.fixture(scope="module")
def octo(oracle):
    from oracle import pyoracle_octaves
    return pyoracle_octaves


def _masked(kl, mask):
    """LSDDetector.cpp:258-286 written out per line: erased when both truncated end points read 0"""
    keep = [i for i in range(len(kl)) if not (mask[int(kl["sy"][i]), int(kl["sx"][i])] == 0 and mask[int(kl["ey"][i]), int(kl["ex"][i])] == 0)]
    return kl[keep]


def test_octaves_flat_and_masks(lsd, octo, fixture_b):
    img, boxes = fixture_b["frames"][9]
    want = octo.lsd_octaves_raw(img, 3, 2.0)
    got = lsd.detect_octaves(img, 2, 3)
    assert len(got) == 3
    for k in range(3):
        np.testing.assert_array_equal(got[k].view(want[k].dtype), want[k])
    np.testing.assert_array_equal(lsd.detect(img, 2, 3).view(want[0].dtype), np.concatenate(want))
    rng = np.random.default_rng(3)
    mask = (rng.random(img.shape[:2]) < 0.3).astype(np.uint8)
    mask[:, :200] = 0
    for k, o in enumerate(lsd.detect_octaves(img, 2, 3, mask)):
        w = _masked(want[k], mask)
        assert 0 < len(w) < len(want[k])
        np.testing.assert_array_equal(o.view(w.dtype), w)                   # class_id keeps the gaps of the masked lines
    assert len(lsd.detect(img, 2, 1, np.zeros(img.shape[:2], np.uint8))) == 0
    assert len(lsd.detect(img, 5, 1)) == len(want[0])                       # one octave: scale unused
    assert lsd.detect_octaves(img, 2, 0) == [] and len(lsd.detect(img, 2, 0)) == 0


def test_vector_form_one_call_per_size(lsd, octo, fixture_b):
    import cv2
    a, b = fixture_b["frames"][0][0], fixture_b["frames"][5][0]
    small = cv2.resize(a, (320, 240), interpolation=cv2.INTER_AREA)
    gray = cv2.cvtColor(b, cv2.COLOR_BGR2GRAY)
    imgs = [a, small, gray, b, small[..., ::-1].copy(), np.dstack([b, np.full(b.shape[:2], 7, np.uint8)])]
    masks = [None, np.ones(small.shape[:2], np.uint8)]                     # fewer masks than images: the rest unmasked
    got = lsd.detect(imgs, 2, 2, masks)
    assert len(got) == len(imgs)
    for i, img in enumerate(imgs):
        want = np.concatenate(octo.lsd_octaves_raw(img[..., :3] if img.ndim == 3 else img, 2, 2.0))
        np.testing.assert_array_equal(got[i].view(want.dtype), want, err_msg=str(i))
    calls = [c for c in lsd._ctx.L.calls if c[0] == "raw"]
    # (480, 640, 3) x 3 (the BGRA frame packed to BGR), (240, 320, 3) x 2, (480, 640) gray x 1: three calls
    assert sorted((c[1], c[2], c[3], c[4]) for c in calls) == [(1, 640, 480, 1), (2, 320, 240, 3), (3, 640, 480, 3)]


def test_capacity_retry(lsd, octo, fixture_a):
    img = fixture_a["img"]
    lsd._ctx.L.min_cap = 9000
    got = lsd.detect(img, 2, 2)
    np.testing.assert_array_equal(got.view(octo.OCTAVE_KEYLINE_DTYPE), np.concatenate(octo.lsd_octaves_raw(img, 2, 2.0)))
    assert [c[5] for c in lsd._ctx.L.calls if c[0] == "raw"] == [2048, 4096, 8192, 16384]


def test_refusals_before_the_library(lsd, fixture_a):
    import cube_slam_b200 as cs
    img = fixture_a["img"]
    h, w = img.shape[:2]
    cases = [((img, 2, 1, np.ones((h, w + 1), np.uint8)), "Mask error"), ((img, 2, 1, np.ones((h, w), np.int16)), "Mask error"),
             ((img.astype(np.int16), 2, 1), "depth image"), ((img, 3, 2), "scale 2"), ((img, 2, -1), "negative"),
             (([img, img], 2, 1, [None, np.ones((3, 3), np.uint8)]), "Masks error"), (([img, img.astype(np.float32)], 2, 1), "depth image")]
    for args, text in cases:
        with pytest.raises(cs.CubeSlamError, match=text):
            lsd.detect(*args)
    assert lsd._ctx.L.calls == []
