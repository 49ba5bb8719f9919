"""The C++ drop-in for the reference's BinaryDescriptorMatcher, RUN: shim/binary_descriptor_matcher_b200.cpp compiled in place of
line_lbd/libs/binary_descriptor_matcher.cpp next to the reference's other line_lbd sources, driven by shim/test/matcher_shim_driver.cpp
(oracle/_ref/libshim_matcher.so, built by shim/test/Makefile where the reference checkout exists).  Every member a caller reaches -- match,
knnMatch and radiusMatch in both forms, add / train / clear -- on matchers made by hand and by line_lbd_detect's own constructor, compared
field for field (queryIdx, trainIdx, imgIdx, distance, in order, both values of compactResult) with the reference's own compiled matcher
(oracle/pyoracle_knn.py, oracle/pyoracle_collection.py) and with the C ABI's documented answer where the reference's is undefined."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import pyoracle_collection as P
from oracle import pyoracle_knn as K

from test_oracle_ref_lbd_collection import images_with_ties
from test_oracle_ref_lbd_knn import _planted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "oracle", "_ref", "libshim_matcher.so")
MATCH, KNN, RADIUS = 0, 1, 2


class Shim(object):
    """ctypes view of the driver: matcher handles and one call per member"""

    def __init__(self, path):
        L = self.L = C.CDLL(path)
        for f in ("shim_bdm_new", "shim_detector_new", "shim_detector_bdm"):
            getattr(L, f).restype = C.c_void_p
        for f in ("shim_bdm_free", "shim_bdm_recreate", "shim_detector_free", "shim_detector_bdm", "shim_bdm_train", "shim_bdm_clear"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.shim_bdm_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.shim_bdm_query.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64]
        L.shim_detector_match_line_descrip.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float] + [C.c_void_p] * 4
        L.shim_bdm_wrong_shape.argtypes = [C.c_void_p, C.c_int]
        L.shim_bdm_threads.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int64]

    def new(self):
        return self.L.shim_bdm_new()

    def add(self, m, images):
        ims = [np.ascontiguousarray(x, np.uint8).reshape(-1, 32) for x in images]
        off = np.concatenate([[0], np.cumsum([len(x) for x in ims])]).astype(np.int32)
        codes = np.ascontiguousarray(np.concatenate(ims + [np.zeros((1, 32), np.uint8)]))
        assert self.L.shim_bdm_add(m, codes.ctypes.data, off.ctypes.data, len(ims)) == 0

    def train(self, m):
        assert self.L.shim_bdm_train(m) == 0

    def clear(self, m):
        assert self.L.shim_bdm_clear(m) == 0

    def query(self, m, kind, q, train=None, k=0, r=0.0, masks=None, compact=False, mask=None, cap=None):
        """-> the lists the member appended, each (query_idx, train_idx, img_idx, distance) arrays (match: one list per DMatch), or the
        driver's negative code.  mask: the pairwise form's mask; masks: the collection form's; either as arrays whose 2-D shape is the Mat's
        (a 1-D array is an n x 1 mask)."""
        q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32)
        ms = [mask] if mask is not None else (masks or [])
        ms = [np.asarray(x, np.uint8).reshape(len(np.asarray(x)), -1) if np.asarray(x).ndim != 2 else np.asarray(x, np.uint8) for x in ms]
        shapes = np.array([x.shape for x in ms] + [(0, 0)], np.int32)
        mb = np.ascontiguousarray(np.concatenate([x.reshape(-1) for x in ms] + [np.zeros(1, np.uint8)]))
        t = None if train is None else np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
        nt = 0 if t is None else len(t)
        if cap is None:
            cap = max(len(q) * (max(nt, 1) if t is not None else max(int(k), 4096)), 1)
        lists = max(len(q), 1)
        ll = np.zeros(lists, np.int32)
        qi, ti, ii, d = (np.zeros(cap, x) for x in (np.int32, np.int32, np.int32, np.float32))
        qq = q if len(q) else np.zeros((1, 32), np.uint8)
        n = self.L.shim_bdm_query(m, kind, qq.ctypes.data, len(q), None if t is None else (t if nt else np.zeros((1, 32), np.uint8)).ctypes.data, nt, int(k),
                                  float(r), mb.ctypes.data, shapes.ctypes.data, len(ms), int(bool(compact)), ll.ctypes.data, qi.ctypes.data, ti.ctypes.data,
                                  ii.ctypes.data, d.ctypes.data, lists, cap)
        if n < 0:
            return n
        out, o = [], 0
        for l in range(n):
            out.append(tuple(x[o:o + ll[l]].copy() for x in (qi, ti, ii, d)))
            o += ll[l]
        return out


@pytest.fixture(scope="module")
def shim():
    if not os.path.exists(SHIM) or not K.ref_available() or not P.ref_available():
        pytest.skip("oracle/_ref/libshim_matcher.so or the reference's matchers not built (they need the reference's sources at build time)")
    import cube_slam_b200  # noqa: F401  (fails loudly if the product library is missing)
    return Shim(SHIM)


@pytest.fixture()
def bdm(shim):
    m = shim.new()
    yield m
    shim.L.shim_bdm_free(m)


def same(got, want, what=""):
    """got: the shim's lists; want: [(query, query_idx, train_idx, img_idx, distance)], or the pairwise [(query, query_idx, train_idx,
    distance)] whose img_idx is 0"""
    assert not isinstance(got, int), (what, got)
    assert len(got) == len(want), (what, len(got), len(want))
    for l, (g, w) in enumerate(zip(got, want)):
        w = w[1:] if len(w) == 5 else (w[1], w[2], np.zeros(len(w[1]), np.int32), w[3])
        for f, a, b in zip(("query_idx", "train_idx", "img_idx", "distance"), g, w):
            np.testing.assert_array_equal(a, np.asarray(b), err_msg="%s list %d %s" % (what, l, f))


def same_match(got, want, what=""):
    """got: the shim's match, one DMatch per list; want: (query_idx, train_idx, img_idx, distance) arrays"""
    assert not isinstance(got, int), (what, got)
    assert all(len(g[0]) == 1 for g in got)
    for j, f in enumerate(("query_idx", "train_idx", "img_idx", "distance")):
        np.testing.assert_array_equal(np.array([g[j][0] for g in got]).astype(np.asarray(want[j]).dtype).reshape(-1), want[j], err_msg="%s %s" % (what, f))


def as_match_lists(lists):
    """match's DMatches (one per list) in the lists' layout, from the nearest entry of each knn k = 1 list"""
    return [(x[0],) + tuple(np.asarray(y)[:1] for y in x[1:]) for x in lists if len(x[1])]


# ---------------------------------------------------------------------------------------------------------------- pairwise forms
def check_pairwise(shim, m, q, t, rng, ks=(0, 1, 2, 5, None), radii=(0.0, 25.0, 256.0), reference=True):
    """match, knnMatch (k None: more than the train set has) and radiusMatch of one pair, with and without a mask, both compactResult:
    the reference's own matcher where it is defined, the C ABI's documented answer (the oracle's restatement) everywhere"""
    for mask in (None, (rng.random(len(q)) < 0.6).astype(np.uint8)):
        want = as_match_lists(K.lbd_knn_lists(q, t, 1, mask, True))
        same(shim.query(m, MATCH, q, t, mask=mask), want, "match")
        if reference:
            same(shim.query(m, MATCH, q, t, mask=mask), as_match_lists(K.ref_knn_match(q, t, 1, mask, True)), "match vs reference")
        for compact in (False, True):
            for k in ks:
                k = len(t) + 3 if k is None else k
                got = shim.query(m, KNN, q, t, k=k, mask=mask, compact=compact)
                same(got, K.lbd_knn_lists(q, t, k, mask, compact), "knn %d %s" % (k, compact))
                if reference and k > 0:      # k = 0 is not run on the reference (a result buffer of 0 entries written to)
                    same(got, K.ref_knn_match(q, t, k, mask, compact), "knn %d %s vs reference" % (k, compact))
            for r in radii:
                got = shim.query(m, RADIUS, q, t, r=r, mask=mask, compact=compact)
                same(got, K.lbd_radius_lists(q, t, r, mask, compact), "radius %g %s" % (r, compact))
                if reference:
                    same(got, K.ref_radius_match(q, t, r, mask, compact), "radius %g %s vs reference" % (r, compact))


def golden_and_synthetic_descriptors(fixture_b):
    """LBD codes of frames of the golden sequence (tests/golden/fixture_b) and of a synthetic VGA batch, by detect_descrip_lines_batch with
    either detector"""
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    det = cs.line_lbd_detect()
    det.line_length_thres = 15
    golden = np.stack([fixture_b["frames"][i][0] for i in (0, 9, 17, 33)])
    out = []
    for imgs in (golden, S.make_batch(31, 3, 640, 480, 3)[0]):
        for use_lsd in (True, False):
            det.use_LSD = use_lsd
            out.append([d for _, d in det.detect_descrip_lines_batch(imgs)])
    return out


@pytest.mark.gpu
def test_pairwise_forms_on_golden_and_synthetic_descriptors(shim, bdm, oracle, fixture_b):
    rng = np.random.default_rng(3)
    sets = golden_and_synthetic_descriptors(fixture_b)
    assert len(sets) == 4 and all(len(s) >= 3 for s in sets)
    for descs in sets:
        q, t = descs[0], descs[1]
        assert len(q) > 5 and len(t) > 5
        check_pairwise(shim, bdm, q, t, rng)
    # one set against itself, and train codes planted at equal distances (ties the hash's order decides)
    check_pairwise(shim, bdm, sets[1][2], sets[1][2], rng, ks=(1, 2, 5), radii=(25.0,))
    q, t = _planted(np.random.default_rng(5), 60, 300)
    check_pairwise(shim, bdm, q, t, rng)


@pytest.mark.gpu
def test_pairwise_train_set_above_the_pairwise_cap(shim, bdm, oracle):
    """20 000 train codes: more than a pairwise C ABI call takes (16 384), so knnMatch / radiusMatch go through a temporary collection --
    the answer must still be the reference's"""
    rng = np.random.default_rng(20000)
    q, t = _planted(rng, 40, 20000)
    t[19990] = t[5]                                                   # an exact duplicate beyond the cap
    q[1] = t[19990]
    check_pairwise(shim, bdm, q, t, rng, ks=(1, 2, 7), radii=(25.0, 100.0))


@pytest.mark.gpu
def test_line_lbd_detect_bdm_from_the_reference_constructor(shim, oracle):
    """line_lbd_detect's own constructor (line_lbd_allclass.cpp:110-123) creates the shim's matcher as bdm; match_line_descrip (:341-356),
    the reference's code, reaches it too"""
    det = shim.L.shim_detector_new()
    try:
        m = shim.L.shim_detector_bdm(det)
        assert m
        rng = np.random.default_rng(11)
        q, t = _planted(rng, 50, 400)
        check_pairwise(shim, m, q, t, rng, ks=(1, 2, 5), radii=(25.0,))
        for thres in (25.0, 60.0):
            qi, ti, ii, d = (np.zeros(len(q), x) for x in (np.int32, np.int32, np.int32, np.float32))
            n = shim.L.shim_detector_match_line_descrip(det, q.ctypes.data, len(q), t.ctypes.data, len(t), thres, qi.ctypes.data, ti.ctypes.data, ii.ctypes.data,
                                                        d.ctypes.data)
            near = [x for x in as_match_lists(K.ref_knn_match(q, t, 1, None, True)) if x[3][0] < thres]
            assert n == len(near)
            np.testing.assert_array_equal(qi[:n], [x[1][0] for x in near])
            np.testing.assert_array_equal(ti[:n], [x[2][0] for x in near])
            np.testing.assert_array_equal(d[:n], [x[3][0] for x in near])
            assert (ii[:n] == 0).all()
        # the detector's matcher keeps a collection like any other
        imgs, q = images_with_ties(rng, [30, 0, 25], 20)
        shim.add(m, imgs)
        same(shim.query(m, KNN, q, k=3), P.ref_collection_knn(imgs, q, 3), "bdm collection knn")
    finally:
        shim.L.shim_detector_free(det)


# ---------------------------------------------------------------------------------------------------------------- collection forms
def check_collection(shim, m, imgs, q, rng, ks=(1, 2, 5), radii=(25.0, 60.0), masks=True):
    """the collection forms against the reference's own matcher after add(imgs) and against the documented answer"""
    opts = [None] + ([[(rng.random(len(q)) < 0.6).astype(np.uint8) for _ in imgs]] if masks else [])
    for ms in opts:
        got = shim.query(m, MATCH, q, masks=ms)
        same_match(got, P.collection_match_list(imgs, q, ms), "match")
        same_match(got, P.ref_collection_match(imgs, q, ms), "match vs reference")
        for compact in (False, True):
            for k in ks:
                got = shim.query(m, KNN, q, k=k, masks=ms, compact=compact)
                same(got, P.collection_knn_lists(imgs, q, k, ms, compact), "knn %d %s" % (k, compact))
                same(got, P.ref_collection_knn(imgs, q, k, ms, compact), "knn %d %s vs reference" % (k, compact))
            for r in radii:
                got = shim.query(m, RADIUS, q, r=r, masks=ms, compact=compact)
                same(got, P.collection_radius_lists(imgs, q, r, ms, compact), "radius %g %s" % (r, compact))
                same(got, P.ref_collection_radius(imgs, q, r, ms, compact), "radius %g %s vs reference" % (r, compact))


@pytest.mark.gpu
def test_collection_add_train_add_clear_and_reuse(shim, bdm, oracle):
    rng = np.random.default_rng(21)
    imgs, q = images_with_ties(rng, [9, 0, 14, 6, 0, 11], 40)
    first, second = imgs[:4], imgs[4:]
    shim.add(bdm, first[:2])
    shim.add(bdm, first[2:])                                          # two add()s before any train()
    check_collection(shim, bdm, first, q, rng)                        # the queries train() themselves
    shim.train(bdm)
    check_collection(shim, bdm, first, q, rng)
    shim.add(bdm, second)                                             # add after train: image 4 is empty and owns image 5's rows
    check_collection(shim, bdm, imgs, q, rng)
    shim.train(bdm)
    check_collection(shim, bdm, imgs, q, rng, masks=False)
    shim.clear(bdm)
    assert shim.query(bdm, MATCH, q) == []
    assert [len(x[0]) for x in shim.query(bdm, KNN, q, k=2)] == [0] * len(q) and shim.query(bdm, KNN, q, k=2, compact=True) == []
    assert shim.query(bdm, RADIUS, q, r=256.0, compact=True) == []
    fresh, q2 = images_with_ties(rng, [0, 17, 8], 30)
    shim.add(bdm, fresh)
    check_collection(shim, bdm, fresh, q2, rng)


@pytest.mark.gpu
def test_collection_of_golden_and_synthetic_keyframes(shim, bdm, oracle, fixture_b):
    rng = np.random.default_rng(22)
    for descs in golden_and_synthetic_descriptors(fixture_b):
        keys, held = descs[:-1] + [np.zeros((0, 32), np.uint8)], descs[-1]
        shim.clear(bdm)
        shim.add(bdm, keys)
        check_collection(shim, bdm, keys, held[:60], rng, ks=(1, 2, 5), radii=(25.0,))


@pytest.mark.gpu
def test_collection_larger_than_the_pairwise_cap(shim, bdm, oracle):
    rng = np.random.default_rng(23)
    imgs, q = images_with_ties(rng, [7000, 0, 9000, 5000], 30)
    shim.add(bdm, imgs)
    check_collection(shim, bdm, imgs, q, rng, ks=(1, 2, 6), radii=(25.0,))


@pytest.mark.gpu
def test_k_zero_and_empty_collection(shim, bdm, oracle):
    rng = np.random.default_rng(24)
    imgs, q = images_with_ties(rng, [12, 9], 10)
    assert shim.query(bdm, MATCH, q) == []                            # nothing added: no entries
    assert [len(x[0]) for x in shim.query(bdm, KNN, q, k=3)] == [0] * len(q)
    shim.add(bdm, imgs)
    assert [len(x[0]) for x in shim.query(bdm, KNN, q, k=0)] == [0] * len(q) and shim.query(bdm, KNN, q, k=0, compact=True) == []
    assert shim.query(bdm, KNN, q, k=-1) == -1                        # throws, as the reference's new[] of a negative size does


# ---------------------------------------------------------------------------------------------------------------- input errors
@pytest.mark.gpu
def test_input_errors_print_or_throw_where_the_reference_does(shim, bdm, oracle, capfd):
    rng = np.random.default_rng(25)
    imgs, q = images_with_ties(rng, [10, 12, 8], 16)
    t = imgs[0]
    shim.L.shim_cout_on()
    capfd.readouterr()
    assert shim.query(bdm, KNN, q[:0], t, k=2) == [] and "descriptors matrices cannot be void" in capfd.readouterr().out
    assert shim.query(bdm, KNN, q, t, k=2, mask=np.ones((len(q), 2))) == []
    assert "input mask should have %d rows and 1 column" % len(q) in capfd.readouterr().out
    # match / radiusMatch refuse only rows != n AND cols != 1; a 1-column mask of other length with too few bytes is refused here too
    assert shim.query(bdm, MATCH, q, t, mask=np.ones((3, 2))) == [] and "input mask should have" in capfd.readouterr().out
    assert shim.query(bdm, RADIUS, q, t, r=60.0, mask=np.ones(len(q) - 1)) == [] and "input mask should have" in capfd.readouterr().out
    shim.add(bdm, imgs)
    assert shim.query(bdm, KNN, q, k=2, masks=[np.ones(len(q))] * 2) == []
    assert "the number of images in dataset is 3 but knnMatch function received 2 masks" in capfd.readouterr().out
    # a per-image mask of the wrong shape: match leaves that image's matches out; knnMatch prints and stops at its first entry
    good = [(rng.random(len(q)) < 0.7).astype(np.uint8) for _ in imgs]
    bad = [good[0], np.ones((len(q), 2), np.uint8), good[2]]
    ones = [good[0], np.ones(len(q), np.uint8), good[2]]
    want = P.collection_match_list(imgs, q, ones)
    keep = want[2] != 1
    same_match(shim.query(bdm, MATCH, q, masks=bad), tuple(x[keep] for x in want), "match, bad mask")
    full = P.collection_knn_lists(imgs, q, 3, ones)
    stop = next(i for i, x in enumerate(full) if (x[3] == 1).any())
    got = shim.query(bdm, KNN, q, k=3, masks=bad)
    same(got, full[:stop], "knn, bad mask")
    assert "Error: mask 1 in knnMatch function should have %d and 1 column" % len(q) in capfd.readouterr().out


@pytest.mark.gpu
def test_descriptor_matrices_other_than_n_x_32_bytes_throw(shim, bdm, oracle):
    for which in range(3):                  # add(), a pairwise train matrix, a collection query: each throws std::invalid_argument
        assert shim.L.shim_bdm_wrong_shape(bdm, which) == 1, which


# ---------------------------------------------------------------------------------------------------------------- lifetime
@pytest.mark.gpu
def test_two_matchers_in_one_thread(shim, oracle):
    rng = np.random.default_rng(31)
    a_imgs, qa = images_with_ties(rng, [15, 0, 9], 20)
    b_imgs, qb = images_with_ties(rng, [0, 30], 20)
    a, b = shim.new(), shim.new()
    try:
        shim.add(a, a_imgs)
        shim.add(b, b_imgs)
        for _ in range(2):
            same(shim.query(a, KNN, qa, k=3), P.ref_collection_knn(a_imgs, qa, 3), "a")
            same(shim.query(b, KNN, qb, k=3), P.ref_collection_knn(b_imgs, qb, 3), "b")
        shim.clear(a)
        same(shim.query(b, RADIUS, qb, r=60.0), P.ref_collection_radius(b_imgs, qb, 60.0), "b after a.clear()")
    finally:
        shim.L.shim_bdm_free(a)
        shim.L.shim_bdm_free(b)


@pytest.mark.gpu
@pytest.mark.parametrize("clear_after", [1, 0])
def test_matchers_in_two_threads(shim, oracle, clear_after):
    rng = np.random.default_rng(32 + clear_after)
    imgs, q = images_with_ties(rng, [40, 0, 25, 30], 25)
    codes = np.ascontiguousarray(np.concatenate(imgs))
    off = np.concatenate([[0], np.cumsum([len(x) for x in imgs])]).astype(np.int32)
    k, cap_lists, cap = 4, len(q), len(q) * 4
    n = np.zeros(4, np.int32)
    ll = np.zeros(4 * cap_lists, np.int32)
    qi, ti, ii, d = (np.zeros(4 * cap, x) for x in (np.int32, np.int32, np.int32, np.float32))
    shim.L.shim_bdm_threads(2, codes.ctypes.data, off.ctypes.data, len(imgs), q.ctypes.data, len(q), k, clear_after, n.ctypes.data, ll.ctypes.data, qi.ctypes.data,
                            ti.ctypes.data, ii.ctypes.data, d.ctypes.data, cap_lists, cap)
    wants = (P.ref_collection_knn(imgs, q, k), K.ref_knn_match(q, codes, k))
    for s in range(4):
        assert n[s] == len(q), (s, n[s])
        lists, o = [], s * cap
        for l in range(n[s]):
            m = ll[s * cap_lists + l]
            lists.append(tuple(x[o:o + m] for x in (qi, ti, ii, d)))
            o += m
        same(lists, wants[s % 2], "thread %d form %d" % (s // 2, s % 2))


@pytest.mark.gpu
def test_matcher_constructed_again_at_a_freed_address(shim, oracle):
    rng = np.random.default_rng(33)
    old, q = images_with_ties(rng, [20, 0, 15], 20)
    new, q2 = images_with_ties(rng, [0, 12, 18], 20)
    m = shim.new()
    try:
        shim.add(m, old)
        same(shim.query(m, KNN, q, k=2), P.ref_collection_knn(old, q, 2), "before")
        shim.L.shim_bdm_recreate(m)                                   # destroyed (nothing freed) and constructed at the same address
        assert shim.query(m, MATCH, q) == [] and shim.query(m, KNN, q, k=2, compact=True) == []
        shim.add(m, new)
        check_collection(shim, m, new, q2, rng, ks=(1, 3), radii=(25.0,))
    finally:
        shim.L.shim_bdm_free(m)
