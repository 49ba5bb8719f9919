"""BinaryDescriptor::compute on key lines of any octave: the oracle's restatement (pyoracle_compute_octaves.lbd_compute_octaves: the gray image, the
descriptor's blurred pyrDown pyramid of max(octave) + 1 levels, LBD per key line on its octave's Sobel maps, the (class_id, octave) row map)
against the REFERENCE'S OWN BinaryDescriptor::compute (oracle/ref/linelbd_compute_octaves_ref.cpp: ref_lbd_compute_octaves), byte for byte, on the key
lines LSDDetector returns for 1 to 4 octaves and on lists a detector never returns.  Runs on the CPU; skipped where the reference cannot be
built."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import pyoracle_compute_octaves
    if not pyoracle_compute_octaves.ref_available():
        pytest.skip("oracle/_ref/liblinelbd_compute_octaves_ref.so not built (no reference checkout on this machine)")
    return pyoracle_compute_octaves


@pytest.fixture(scope="module")
def octo(oracle):
    from oracle import pyoracle_octaves
    return pyoracle_octaves


def _synthetic(w, h, gray, seed):
    import cv2
    from cube_slam_b200 import synthetic
    img = synthetic.make_batch(seed, 1, 640, 480)[0][0]
    if (w, h) != (640, 480):
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if gray else img


def _frames(fixture_a, fixture_b):
    return [("fixture A", fixture_a["img"]), ("fixture B 9", fixture_b["frames"][9][0]), ("641x479 BGR", _synthetic(641, 479, False, 5)),
            ("641x479 gray", _synthetic(641, 479, True, 6)), ("97x211 BGR", _synthetic(97, 211, False, 7))]


def _keylines(octo, img, K):
    """LSDDetector::detect(img, keylines, 2, K): the flat list, octave after octave"""
    return np.concatenate(octo.lsd_octaves_raw(img, K))


def _alone(ref, img, row):
    """the reference's descriptor of one key line described on its own; class_id 0, since the reference reads the first line of every class_id
    up to the largest (binary_descriptor.cpp:1482-1490) and crashes on a list that skips one"""
    one = np.array([row], row.dtype)
    one["class_id"] = 0
    return ref.ref_lbd_compute_octaves(img, one)[0]


def test_detector_lists_one_to_four_octaves(ref, octo, fixture_a, fixture_b):
    for name, img in _frames(fixture_a, fixture_b):
        full = _keylines(octo, img, 4)
        for K in (1, 2, 3, 4):
            kl = full[full["octave"] < K]
            assert len(kl) and kl["octave"].max() == K - 1, (name, K)
            np.testing.assert_array_equal(ref.lbd_compute_octaves(img, kl), ref.ref_lbd_compute_octaves(img, kl), err_msg="%s, %d octaves" % (name, K))


def test_lists_a_detector_never_returns(ref, octo, fixture_b):
    rng = np.random.default_rng(4)
    img = fixture_b["frames"][30][0]
    kl = _keylines(octo, img, 3)
    for what, sub in (("shuffled", kl[rng.permutation(len(kl))]), ("deepest octave only", kl[kl["octave"] == 2])):
        np.testing.assert_array_equal(ref.lbd_compute_octaves(img, sub), ref.ref_lbd_compute_octaves(img, sub), err_msg=what)
    # repeated (class_id, octave) pairs: the first row gets the last one's descriptor; the others are the reference's own for that row alone
    dup = np.concatenate([kl[:40], kl[5:15], kl[kl["octave"] == 1][:6], kl[:3]])
    dup["class_id"][40:50] = dup["class_id"][:10]
    got, want = ref.lbd_compute_octaves(img, dup), ref.ref_lbd_compute_octaves(img, dup)
    pairs = ref.pair_rows(dup)
    assert len(pairs) == 10
    keys = list(zip(dup["class_id"].tolist(), dup["octave"].tolist()))
    shared = [i for i, k in enumerate(keys) if keys.count(k) > 1]
    alone = [i for i in range(len(dup)) if i not in shared]
    np.testing.assert_array_equal(got[alone], want[alone])
    for i in shared:
        if i in pairs:
            np.testing.assert_array_equal(got[i], want[i])
        np.testing.assert_array_equal(got[i], _alone(ref, img, dup[pairs.get(i, i)]))
    # in-octave ends on and beyond the octave's border
    h, w = img.shape[:2]
    edge = kl[:24].copy()
    for j, o in enumerate(edge):
        ow, oh = w >> int(o["octave"]), h >> int(o["octave"])
        edge[j]["s_oct_x"], edge[j]["e_oct_x"] = (ow - 1, ow + 3.5) if j % 3 == 0 else ((-2.5, 0) if j % 3 == 1 else (0, ow - 1))
        edge[j]["s_oct_y"], edge[j]["e_oct_y"] = (oh - 1, oh + 7) if j % 2 else (-4, oh - 1)
    np.testing.assert_array_equal(ref.lbd_compute_octaves(img, edge), ref.ref_lbd_compute_octaves(img, edge))
    assert ref.lbd_compute_octaves(img, kl[:0]).shape == (0, 32)
    assert ref.ref_lbd_compute_octaves(img, kl[:0]).shape == (0, 32)      # "keypoint list is empty": no error


def test_octave_beyond_the_pyramid_throws_in_both(ref, octo):
    img = _synthetic(97, 211, True, 8)
    kl = _keylines(octo, img, 2)[:4].copy()
    deepest = ref.deepest_octave(97, 211)
    assert deepest == 6                                                          # 97 x 211 -> ... -> 1 x 3
    kl["octave"][1] = deepest
    ref.ref_lbd_compute_octaves(img, kl)                                         # the last level pyrDown can make
    kl["octave"][1] = deepest + 1
    with pytest.raises(RuntimeError, match="pyrDown"):
        ref.ref_lbd_compute_octaves(img, kl)
    with pytest.raises(ValueError, match="pyrDown"):
        ref.lbd_compute_octaves(img, kl)
