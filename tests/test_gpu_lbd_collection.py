"""Matching line descriptors against a device-resident collection of many images (cs_lbd_collection_*, kernels k_coll_scan / k_coll_merge2 /
k_coll_emit and CUB's segmented sort) through the Python mirror's collection forms (line_lbd_detect.bdm: add, match, knnMatch, radiusMatch
without a train matrix): field for field equal to the oracle's restatement (pinned to the reference by
tests/test_oracle_ref_lbd_collection.py) on random images with empty ones and ties, on fixture_b keyframes of both detector flavours queried
with member and held-out frames, and at 2^17 and 2^20 codes with duplicates planted in images that land in different train splits; the
collection forms against the pairwise ones; state (add after a query, clear, empty collections); errors and the radius retry."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import pyoracle_collection as P

from test_oracle_ref_lbd_collection import images_with_ties
from test_oracle_ref_lbd_knn import _flip, _planted

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import cube_slam_b200 as cs
    return cs.line_lbd_detect()._ctx


@pytest.fixture()
def det(ctx):
    """a detector of its own (and so a matcher and collection of its own) on the shared context"""
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect(context=ctx)
    d.line_length_thres = 15
    return d


def same(got, want, what=""):
    """got: the mirror's lists of DMATCH_DTYPE records; want: the oracle's [(query, query_idx, train_idx, img_idx, distance)]"""
    assert len(got) == len(want), (what, len(got), len(want))
    for g, w in zip(got, want):
        for f, v in zip(("query_idx", "train_idx", "img_idx", "distance"), w[1:]):
            np.testing.assert_array_equal(g[f], v, err_msg="%s %s" % (what, f))
        if len(g):
            assert (g["query_idx"] == w[0]).all()


def same_match(got, want, what=""):
    for f, v in zip(("query_idx", "train_idx", "img_idx", "distance"), want):
        np.testing.assert_array_equal(got[f], v, err_msg="%s %s" % (what, f))


def check(bdm, imgs, q, ks, radii, rng, masks=True):
    opts = [None] + ([[(rng.random(len(q)) < 0.6).astype(np.uint8) for _ in imgs]] if masks else [])
    for m in opts:
        same_match(bdm.match(q, m), P.collection_match_list(imgs, q, m), "match")
        for compact in (False, True):
            for k in ks:
                same(bdm.knnMatch(q, k, m, compact), P.collection_knn_lists(imgs, q, k, m, compact), "knn %d %s" % (k, compact))
            for r in radii:
                same(bdm.radiusMatch(q, r, m, compact), P.collection_radius_lists(imgs, q, r, m, compact), "radius %g %s" % (r, compact))


@pytest.mark.parametrize("sizes", [(9,), (0, 12), (7, 0, 5), (4, 6, 0), (0, 0, 3, 8, 0), (5, 1, 1, 0, 9, 2, 3, 0, 4, 6, 2, 1), (300, 0, 170, 90)])
def test_random_images_with_empty_ones_and_ties(det, oracle, sizes):
    rng = np.random.default_rng(sum(sizes) * 7 + len(sizes))
    imgs, q = images_with_ties(rng, list(sizes), 70)
    det.bdm.add(imgs)
    det.bdm.train()
    n = sum(sizes)
    check(det.bdm, imgs, q, [1, 2, 3, 7, n, n + 4], [0.0, 25.0, 128.0, math.inf], rng)


def test_codes_near_D_and_an_all_zero_mask(det, oracle):
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (12, 0, 15, 13)]
    base = np.concatenate(imgs)
    q = np.stack([_flip(base[i % 40], rng.choice(256, 110 + i % 30, replace=False)) for i in range(30)])
    det.bdm.add(imgs)
    check(det.bdm, imgs, q, [1, 2, 5, 40, 43], [127.0, 128.0, 129.0, 300.0], rng)
    q[:4] = imgs[2][:4]
    # image 1 is empty and starts at the same row as image 2, so it owns image 2's rows: its mask is the one consulted
    masks = [np.ones(len(q)), np.zeros(len(q)), np.ones(len(q)), np.ones(len(q))]
    got = det.bdm.match(q, masks)
    same_match(got, P.collection_match_list(imgs, q, masks))
    assert not np.isin(np.arange(4), got["query_idx"]).any()       # no fall-back to the next nearest code
    assert (det.bdm.match(q)["img_idx"][:4] == 1).all()


def test_fixture_b_keyframes_both_flavours(det, oracle, fixture_b):
    frames = np.stack([fixture_b["frames"][i][0] for i in range(0, 24, 2)])
    for use_lsd in (True, False):
        det.use_LSD = use_lsd
        descs = [d for _, d in det.detect_descrip_lines_batch(frames)]
        keys, held = descs[:-1], descs[-1]
        assert sum(len(d) for d in keys) > 100 and len(held) > 10
        det.bdm.clear()
        det.bdm.add(keys)
        rng = np.random.default_rng(int(use_lsd))
        for q in (held, keys[3]):
            check(det.bdm, keys, q, [1, 2, 3, 10], [0.0, 25.0, 60.0], rng)


def test_single_image_equals_pairwise(det, oracle):
    rng = np.random.default_rng(8)
    q, t = _planted(rng, 120, 400)
    det.bdm.add([t])

    def same_as_pairwise(a, b):
        """img_idx is 0 (the pairwise forms' value) wherever there is a train index; -1 with it beyond D = 128"""
        for f in ("query_idx", "train_idx", "distance"):
            np.testing.assert_array_equal(a[f], b[f])
        np.testing.assert_array_equal(a["img_idx"], np.where(a["train_idx"] < 0, -1, 0))

    same_as_pairwise(det.bdm.match(q), det.bdm.match(q, t))
    for k in (1, 2, 5, 400):
        got, want = det.bdm.knnMatch(q, k), det.bdm.knnMatch(q, t, k)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            same_as_pairwise(a, b)
    got, want = det.bdm.radiusMatch(q, 60.0, compactResult=True), det.bdm.radiusMatch(q, t, 60.0, compactResult=True)
    assert len(got) == len(want)
    for a, b in zip(got, want):
        same_as_pairwise(a, b)


def test_several_images_knn_equals_pairwise_over_the_concatenation(det, oracle):
    rng = np.random.default_rng(9)
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (5000, 0, 7000, 4384)]
    t = np.concatenate(imgs)
    q = np.concatenate([t[[3, 5100, 12100, 16383]], rng.integers(0, 256, (60, 32), dtype=np.uint8)])
    det.bdm.add(imgs)
    for k in (1, 2, 3, 9):
        got, want = det.bdm.knnMatch(q, k), det.bdm.knnMatch(q, t, k)
        for a, b in zip(got, want):
            for f in ("query_idx", "train_idx", "distance"):
                np.testing.assert_array_equal(a[f], b[f])


@pytest.mark.parametrize("log2n", [17, 20])
def test_large_collections_with_duplicates_across_splits(det, oracle, log2n):
    n = 1 << log2n
    rng = np.random.default_rng(log2n)
    sizes = [n // 4 - 1000, 0, n // 4 + 1000, n // 2]
    codes = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    q = np.concatenate([codes[rng.integers(0, n, 8)], np.stack([_flip(codes[7], [1, 2, 3])]), rng.integers(0, 256, (3, 32), dtype=np.uint8)])
    for r in (7, n // 3, n // 2 + 17, n - 2):                  # the same code in the first, third and fourth image, far apart
        codes[r] = codes[7]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    imgs = [codes[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    det.bdm.add(imgs)
    assert det.bdm.collection_size() == (4, n)
    rng_m = np.random.default_rng(1)
    masks = [(rng_m.random(len(q)) < 0.7).astype(np.uint8) for _ in imgs]
    for m in (None, masks):
        same_match(det.bdm.match(q, m), P.collection_match_list(imgs, q, m), "match")
        for k in (1, 2, 6):
            same(det.bdm.knnMatch(q, k, m), P.collection_knn_lists(imgs, q, k, m), "knn %d" % k)
        same(det.bdm.radiusMatch(q, 25.0, m, True), P.collection_radius_lists(imgs, q, 25.0, m, True), "radius")
    dup = det.bdm.knnMatch(q[8:9], 6)[0]
    assert set(dup["train_idx"][:4]) == {7, n // 3, n // 2 + 17, n - 2} and (dup["distance"][:4] == 3).all()


def test_split_at_its_largest_keeps_the_histogram_exact(det, oracle):
    """67 584 queries = 1056 query tiles, so the grid wants one split per tile column and the split size is clamped to 511 tiles (65 408
    codes), the bound of the 16-bit histogram bins of knn with k > 2.  70 000 codes: 65 600 copies of one code C (more than a 16-bit bin
    holds, had all of them landed in one split) and 4 400 codes one bit from it.  Four queries are C, the rest its complement (which meets
    nothing).  An overflowed bin would move the k-th distance to 1 and the gather past its segment."""
    rng = np.random.default_rng(65408)
    c = rng.integers(0, 256, 32, dtype=np.uint8)
    codes = np.tile(c, (70000, 1))
    near = rng.choice(70000, 4400, replace=False)
    bits = rng.integers(0, 256, 4400)
    codes[near, bits // 8] ^= (1 << (bits % 8)).astype(np.uint8)
    imgs = [codes[:30000], codes[:0], codes[30000:]]
    nq = 1056 * 64
    q = np.tile(~c, (nq, 1))
    at = np.array([0, 20000, 40000, nq - 1])
    q[at] = c
    det.bdm.add(imgs)
    for k in (3, 100):
        got = det.bdm.knnMatch(q, k)
        assert len(got) == nq and sum(len(x) for x in got) == 4 * k
        want = P.collection_knn_lists(imgs, q[at], k)
        for i, w in zip(at, want):
            g = got[i]
            assert (g["query_idx"] == i).all() and (g["distance"] == 0).all()
            for f, v in zip(("train_idx", "img_idx", "distance"), w[2:]):
                np.testing.assert_array_equal(g[f], v)


def test_state_add_after_query_clear_and_empty(det, oracle):
    import cube_slam_b200 as cs
    rng = np.random.default_rng(12)
    a, b = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (40, 0)], [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (0, 25, 30)]
    q = np.concatenate([a[0][:5], b[2][:5], rng.integers(0, 256, (10, 32), dtype=np.uint8)])
    bdm = det.bdm
    assert det.bdm is bdm                                      # one matcher per detector, as the reference creates it once
    assert bdm.collection_size() == (0, 0)
    assert len(bdm.match(q)) == 0 and all(len(x) == 0 for x in bdm.knnMatch(q, 3)) and bdm.radiusMatch(q, 25.0, compactResult=True) == []
    bdm.add([])
    assert bdm.collection_size() == (0, 0)
    bdm.add(a)
    same(bdm.knnMatch(q, 3), P.collection_knn_lists(a, q, 3))
    bdm.add(b)                                                 # after a query: the collection is everything added
    assert bdm.collection_size() == (5, 95)
    check(bdm, a + b, q, [1, 2, 4], [25.0], rng)
    assert bdm.knnMatch(q[:0], 2) == [] and len(bdm.match(q[:0])) == 0
    bdm.clear()
    assert bdm.collection_size() == (0, 0) and len(bdm.match(q)) == 0
    bdm.add(b)
    check(bdm, b, q, [1, 3], [25.0], rng)
    # a second detector on the same context has a collection of its own
    other = cs.line_lbd_detect(context=det._ctx)
    assert other.bdm is not bdm and other.bdm.collection_size() == (0, 0)


def test_errors_and_the_radius_retry(det, oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    rng = np.random.default_rng(4)
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (30, 50)]
    q = np.concatenate([imgs[0][:10], imgs[1][:10]])
    bdm = det.bdm
    bdm.add(imgs)
    with pytest.raises(cs.CubeSlamError, match="CS_ERR_INVALID_ARG.*masks"):
        bdm.knnMatch(q, 2, [np.ones(20)])
    with pytest.raises(cs.CubeSlamError, match="mask 1 has 19"):
        bdm.radiusMatch(q, 25.0, [np.ones(20), np.ones(19)])
    with pytest.raises(cs.CubeSlamError, match="CS_ERR_INVALID_ARG"):
        bdm.knnMatch(q, -1)
    want = P.collection_radius(imgs, q, 128.0)
    counts = [len(x[0]) for x in want]
    total = sum(counts)
    L, h = det._ctx.L, bdm._h
    off = np.full(len(q) + 1, -5, np.int64)
    out = np.zeros(total, _lib.DMATCH_DTYPE)
    qq = np.ascontiguousarray(q)
    rc = L.cs_lbd_collection_radius_match(h, _lib.ptr(qq, C.c_uint8), len(q), C.c_float(128.0), None, 0, out.ctypes.data, C.c_int64(total - 1),
                                          _lib.ptr(off, C.c_int64))
    assert rc == -3 and b"max_matches" in L.cs_last_error(det._ctx.h)
    np.testing.assert_array_equal(off, np.concatenate([[0], np.cumsum(counts)]))
    rc = L.cs_lbd_collection_radius_match(h, _lib.ptr(qq, C.c_uint8), len(q), C.c_float(128.0), None, 0, out.ctypes.data, C.c_int64(int(off[-1])),
                                          _lib.ptr(off, C.c_int64))
    assert rc == 0
    np.testing.assert_array_equal(out["train_idx"], np.concatenate([x[1] for x in want]))
    np.testing.assert_array_equal(out["img_idx"], np.concatenate([x[2] for x in want]))
    same(bdm._radius_collection(q, 128.0, max_matches=1), P.collection_radius_lists(imgs, q, 128.0), "retry")
