"""k-nearest-neighbour and radius matching of line descriptors on the GPU (cs_knn_match_line_descrip[_batch],
cs_radius_match_line_descrip[_batch]; kernels k_lbd_knn2 and k_lbd_match_sorted) through the Python mirror of BinaryDescriptorMatcher:
field for field equal to the oracle's knnMatch / radiusMatch (pinned to the reference by tests/test_oracle_ref_lbd_knn.py) on random codes
with planted ties, on descriptors of consecutive fixture_b frames, near D = 128, with masks and compactResult, in batches with uneven and
empty pairs; at the 16384-code bound and one above it; a radius buffer too small and the retry; k = 0 and k < 0."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import pyoracle_knn as K

from test_oracle_ref_lbd_knn import _flip, _planted

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    import cube_slam_b200 as cs
    d = cs.line_lbd_detect()
    d.line_length_thres = 15
    return d


def same(got, want, what=""):
    """got: the mirror's lists of DMATCH_DTYPE records; want: the oracle's [(query, query_idx, train_idx, distance)]"""
    assert len(got) == len(want), (what, len(got), len(want))
    for g, w in zip(got, want):
        assert g.dtype.itemsize == 16
        np.testing.assert_array_equal(g["query_idx"], w[1], err_msg=what)
        np.testing.assert_array_equal(g["train_idx"], w[2], err_msg=what)
        np.testing.assert_array_equal(g["distance"], w[3], err_msg=what)
        assert (g["img_idx"] == 0).all()
        if len(g):
            assert (g["query_idx"] == w[0]).all()


def check_batch(bdm, oracle, pairs, ks, radii=(0.0, 25.0, 128.0), seed=0):
    rng = np.random.default_rng(seed)
    qs, ts = [q for q, _ in pairs], [t for _, t in pairs]
    masks = [None if i % 3 == 0 else (rng.random(len(q)) < 0.6) for i, q in enumerate(qs)]
    for mk in (None, masks):
        for compact in (False, True):
            for k in ks:
                got = bdm.knnMatch_batch(qs, ts, k, mk, compact)
                for p in range(len(pairs)):
                    same(got[p], K.lbd_knn_lists(qs[p], ts[p], k, None if mk is None else mk[p], compact), "knn k=%d pair %d" % (k, p))
            for r in radii:
                got = bdm.radiusMatch_batch(qs, ts, r, mk, compact)
                for p in range(len(pairs)):
                    same(got[p], K.lbd_radius_lists(qs[p], ts[p], r, None if mk is None else mk[p], compact), "radius %g pair %d" % (r, p))


def test_random_codes_uneven_and_empty_pairs(det, oracle):
    rng = np.random.default_rng(31)
    shapes = [(7, 40), (0, 12), (5, 0), (1, 1), (19, 59), (3, 3), (12, 300), (0, 0), (4, 17)]
    pairs = [_planted(rng, nq, nt) if nq and nt else (rng.integers(0, 256, (nq, 32), dtype=np.uint8), rng.integers(0, 256, (nt, 32), dtype=np.uint8))
             for nq, nt in shapes]
    check_batch(det.bdm, oracle, pairs, [1, 2, 3, 5, 59, 303])
    # one pair at a time, through the single-pair entry points
    for q, t in pairs[:5]:
        for k in (1, 2, 5, len(t), len(t) + 3):
            same(det.bdm.knnMatch(q, t, k), K.lbd_knn_lists(q, t, k), "single knn")
        same(det.bdm.radiusMatch(q, t, 25.0, compactResult=True), K.lbd_radius_lists(q, t, 25.0, compact=True), "single radius")


def test_consecutive_fixture_b_frames_both_flavours(det, oracle, fixture_b):
    frames = np.stack([fixture_b["frames"][i][0] for i in range(6)])
    for use_lsd in (True, False):
        det.use_LSD = use_lsd
        descs = [d for _, d in det.detect_descrip_lines_batch(frames)]
        pairs = list(zip(descs[:-1], descs[1:]))
        assert sum(len(d) for d in descs) > 60
        check_batch(det.bdm, oracle, pairs, [1, 2, 5, max(len(b) for b in descs[1:]), max(len(b) for b in descs[1:]) + 3], seed=int(use_lsd))


def test_queries_near_D(det, oracle):
    rng = np.random.default_rng(5)
    t = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    q = np.stack([_flip(t[i % 40], rng.choice(256, 120 + i % 20, replace=False)) for i in range(30)])
    check_batch(det.bdm, oracle, [(q, t), (q[:7], t[:9])], [1, 2, 5, 40, 43], radii=(127.0, 128.0, 128.5, 129.0, 300.0, math.inf))
    far = np.concatenate(det.bdm.knnMatch(q, t, 40))
    assert (far["distance"] > 128).any() and (far["train_idx"][far["distance"] > 128] == -1).all()


def test_knn_1_is_match_line_descrip_without_threshold(det, oracle):
    rng = np.random.default_rng(8)
    q, t = _planted(rng, 200, 150)
    nearest = det.match_line_descrip(q, t, math.inf)
    one = det.bdm.knnMatch(q, t, 1, compactResult=True)
    flat = np.concatenate(one)
    np.testing.assert_array_equal(flat, nearest)
    np.testing.assert_array_equal(det.bdm.match(q, t), nearest)
    mask = rng.random(len(q)) < 0.5
    np.testing.assert_array_equal(det.bdm.match(q, t, mask), nearest[mask[nearest["query_idx"]]])


def test_train_sets_at_the_bound_and_above(det, oracle):
    import cube_slam_b200 as cs
    n = 16384
    rng = np.random.default_rng(77)
    t = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    q = np.stack([t[5], t[9000], _flip(t[123], range(0, 256, 3))])
    t[n - 1] = t[3]
    for k in (2, 5, n):
        same(det.bdm.knnMatch(q, t, k), K.lbd_knn_lists(q, t, k), "bound knn %d" % k)
    for r in (25.0, 100.0, 256.0):
        same(det.bdm.radiusMatch(q, t, r), K.lbd_radius_lists(q, t, r), "bound radius %g" % r)
    big = np.concatenate([t, t[:1]])
    for call in (lambda: det.bdm.knnMatch(q, big, 2), lambda: det.bdm.knnMatch(q, big, 5), lambda: det.bdm.radiusMatch(q, big, 25.0),
                 lambda: det.bdm.knnMatch_batch([q, q], [t[:10], big], 2)):
        with pytest.raises(cs.CubeSlamError, match="CS_ERR_CAPACITY.*16384"):
            call()


def test_radius_buffer_too_small_then_retry(det, oracle):
    from cube_slam_b200 import _lib
    rng = np.random.default_rng(12)
    pairs = [_planted(rng, 30, 80), (np.zeros((0, 32), np.uint8), rng.integers(0, 256, (5, 32), dtype=np.uint8)), _planted(rng, 25, 64)]
    q = np.ascontiguousarray(np.concatenate([p[0] for p in pairs]))
    t = np.ascontiguousarray(np.concatenate([p[1] for p in pairs]))
    qo = np.array([0, 30, 30, 55], np.int32)
    to = np.array([0, 80, 85, 149], np.int32)
    want = [K.lbd_radius_match(a, b, 100.0) for a, b in pairs]
    counts = [len(x[0]) for w in want for x in w]
    total = sum(counts)
    assert total > 10
    L, h = det._ctx.L, det._ctx.h
    off = np.full(56, -5, np.int64)
    out = np.zeros(total, _lib.DMATCH_DTYPE)
    rc = L.cs_radius_match_line_descrip_batch(h, _lib.ptr(q, C.c_uint8), _lib.ptr(qo, C.c_int32), _lib.ptr(t, C.c_uint8), _lib.ptr(to, C.c_int32), 3,
                                              C.c_float(100.0), None, out.ctypes.data, C.c_int64(total - 1), _lib.ptr(off, C.c_int64))
    assert rc == -3 and b"max_matches" in L.cs_last_error(h)
    np.testing.assert_array_equal(off, np.concatenate([[0], np.cumsum(counts)]))
    rc = L.cs_radius_match_line_descrip_batch(h, _lib.ptr(q, C.c_uint8), _lib.ptr(qo, C.c_int32), _lib.ptr(t, C.c_uint8), _lib.ptr(to, C.c_int32), 3,
                                              C.c_float(100.0), None, out.ctypes.data, C.c_int64(int(off[-1])), _lib.ptr(off, C.c_int64))
    assert rc == 0
    flat = np.concatenate([x[2] for w in want for x in w])
    np.testing.assert_array_equal(out["distance"], flat)
    np.testing.assert_array_equal(out["train_idx"], np.concatenate([x[1] for w in want for x in w]))
    # the mirror starts with a buffer of 1 and grows it once
    got = det.bdm.radiusMatch_batch([p[0] for p in pairs], [p[1] for p in pairs], 100.0, max_matches=1)
    for p in range(3):
        same(got[p], K.lbd_radius_lists(pairs[p][0], pairs[p][1], 100.0), "retry pair %d" % p)


def test_k_zero_negative_k_and_bad_masks(det, oracle):
    import cube_slam_b200 as cs
    rng = np.random.default_rng(4)
    q, t = _planted(rng, 9, 20)
    lists = det.bdm.knnMatch(q, t, 0)
    assert len(lists) == 9 and all(len(x) == 0 for x in lists)
    with pytest.raises(cs.CubeSlamError, match="CS_ERR_INVALID_ARG"):
        det.bdm.knnMatch(q, t, -1)
    for call in (lambda: det.bdm.knnMatch(q, t, 2, mask=np.ones(8)), lambda: det.bdm.radiusMatch(q, t, 25.0, mask=np.ones(10)),
                 lambda: det.bdm.match(q, t, mask=np.ones(3))):
        with pytest.raises(cs.CubeSlamError, match="mask"):
            call()
    assert det.bdm.knnMatch(q[:0], t, 2) == [] and det.bdm.radiusMatch(q, t[:0], 25.0) == []
