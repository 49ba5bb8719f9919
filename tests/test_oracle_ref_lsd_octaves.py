"""Every octave of a multi-octave LSD line_lbd_detect: the oracle's restatement (pyoracle_octaves.lsd_octaves_raw / lsd_octaves_descrip: pyrDown,
lsd_oracle's LSD per octave, the KeyLine fill, the descriptor's blurred pyramid and Sobel maps, LBD per octave) against the REFERENCE'S OWN
class (oracle/ref/linelbd_octaves_ref.cpp, compiled on demand: ref_lsd_octaves) built with (numoctaves, octaveratio): every KeyLine field and every descriptor
byte, for both detect_raw_lines overloads and detect_descrip_lines_octaves.  Ratios whose integer part is not 2 make pyrDown throw in both."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import pyoracle_octaves
    if not pyoracle_octaves.ref_available():
        pytest.skip("oracle/_ref/liblinelbd_octaves_ref.so not built (no /root/reference on this machine)")
    return pyoracle_octaves


@pytest.fixture(scope="module")
def octo(oracle):
    """oracle/pyoracle_octaves.py: the multi-octave restatement (and the reference's own class where it can be built)"""
    from oracle import pyoracle_octaves
    return pyoracle_octaves


def _synthetic(w, h, gray):
    import cv2
    from cube_slam_b200 import synthetic
    img = synthetic.make_batch(w * 3 + h, 1, 640, 480)[0][0]
    if (w, h) != (640, 480):
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if gray else img


def _frames(fixture_a, fixture_b):
    out = [("fixture A", fixture_a["img"])] + [("fixture B %d" % i, fixture_b["frames"][i][0]) for i in (0, 5, 30)]
    for w, h in ((640, 480), (1242, 375), (211, 97)):
        for gray in (False, True):
            out.append(("%dx%d %s" % (w, h, "gray" if gray else "BGR"), _synthetic(w, h, gray)))
    return out


def _same(got, want, what):
    assert len(got) == len(want), what
    for k, (a, b) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(a, b, err_msg="%s octave %d" % (what, k))


@pytest.mark.parametrize("numoctaves,ratio", [(2, 2.0), (3, 2.0), (2, 2.5), (3, 2.5)])
def test_restated_octaves_equal_the_reference(ref, fixture_a, fixture_b, numoctaves, ratio):
    for what, img in _frames(fixture_a, fixture_b):
        raw = ref.lsd_octaves_raw(img, numoctaves, ratio)
        _same(raw, ref.ref_lsd_octaves(img, numoctaves, ratio, 15.0, mode=0), what + " vector<vector<KeyLine>>")
        _same(raw, ref.ref_lsd_octaves(img, numoctaves, ratio, 15.0, mode=1), what + " vector<KeyLine>")
        assert all(len(k) for k in raw), what                      # every octave found lines
        kls, descs = ref.lsd_octaves_descrip(img, numoctaves, ratio, 15.0)
        rk, rd = ref.ref_lsd_octaves(img, numoctaves, ratio, 15.0, mode=2)
        _same(kls, rk, what + " key lines")
        _same(descs, rd, what + " descriptors")


def test_ratio_decides_the_higher_octaves_kept(ref):
    img = _synthetic(640, 480, False)
    k2 = ref.lsd_octaves_descrip(img, 3, 2.0)[0]
    k25 = ref.lsd_octaves_descrip(img, 3, 2.5)[0]
    assert len(k2[0]) == len(k25[0])
    assert sum(map(len, k25[1:])) >= sum(map(len, k2[1:]))         # lineLength * 2.5^k keeps at least what 2^k keeps


@pytest.mark.parametrize("ratio", [1.0, 3.0])
def test_ratios_other_than_two_raise_in_both(ref, fixture_a, ratio):
    img = fixture_a["img"]
    with pytest.raises(RuntimeError):
        ref.ref_lsd_octaves(img, 2, ratio, 15.0, mode=2)
    with pytest.raises(ValueError):
        ref.lsd_octaves_descrip(img, 2, ratio)
    assert len(ref.ref_lsd_octaves(img, 1, ratio, 15.0, mode=0)) == 1   # one octave never calls pyrDown


def test_pyrdown_and_blurred_pyramid_equal_cv2(octo):
    import cv2
    rng = np.random.default_rng(1)
    for h, w in [(480, 640), (375, 1242), (97, 211), (120, 161), (7, 9)]:
        a = rng.integers(0, 256, (h, w), dtype=np.uint8)
        np.testing.assert_array_equal(octo.pyrdown(a, w // 2, h // 2), cv2.pyrDown(a, dstsize=(w // 2, h // 2)))
        blur = cv2.GaussianBlur(a, (5, 5), 1)
        want = [blur]
        for _ in range(2):
            want.append(cv2.pyrDown(want[-1], dstsize=(want[-1].shape[1] // 2, want[-1].shape[0] // 2)))
        if min(want[-1].shape) < 1:
            continue
        for k, (g, x) in enumerate(zip(octo.descriptor_pyramid(a, 3), want)):
            np.testing.assert_array_equal(g, x, err_msg="%dx%d level %d" % (w, h, k))
            dx, dy = octo.sobel_u8(g)
            np.testing.assert_array_equal(dx, cv2.Sobel(g, cv2.CV_16S, 1, 0, ksize=3))
            np.testing.assert_array_equal(dy, cv2.Sobel(g, cv2.CV_16S, 0, 1, ksize=3))
