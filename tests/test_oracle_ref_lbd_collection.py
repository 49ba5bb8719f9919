"""Matching against a collection of images: the oracle's restatement (oracle/lbd_collection_oracle.cpp -- the pairwise restatement over the
concatenated images, the image map of add() and the mask post-filter) against the REFERENCE'S OWN BinaryDescriptorMatcher after add()
(line_lbd/libs/binary_descriptor_matcher.cpp:70-193, 344-428, 510-595, compiled into oracle/_ref/liblinelbd_collection_ref.so): match,
knnMatch and radiusMatch without a train matrix, with masks and compactResult.  The reference's answer is compared where it is defined
(the wrapper, oracle/ref/linelbd_collection_ref.cpp, cuts the rest); masked calls are made only where every entry the reference looks a
mask up for is defined.  The reference's collection radiusMatch is O(N^2) per query, so collections stay at a few hundred codes."""
import math

import numpy as np
import pytest

from oracle import pyoracle_collection as P

from test_oracle_ref_lbd_knn import _flip


@pytest.fixture(scope="module")
def ref(oracle):
    if not P.ref_available():
        pytest.skip("oracle/_ref/liblinelbd_collection_ref.so not built (no reference checkout on this machine)")
    return oracle


def same_lists(a, b, what=""):
    assert [x[0] for x in a] == [x[0] for x in b], (what, [x[0] for x in a], [x[0] for x in b])
    for x, y in zip(a, b):
        for u, v in zip(x[1:], y[1:]):
            np.testing.assert_array_equal(u, v, err_msg=what)


def same_match(a, b, what=""):
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v, err_msg=what)


def images_with_ties(rng, sizes, nq):
    """images of random codes; queries near codes of different images, and codes planted in several images at the same distance from
    query 0 and as exact duplicates across images"""
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in sizes]
    flat = [(i, j) for i, n in enumerate(sizes) for j in range(n)]
    q = []
    for _ in range(nq):
        i, j = flat[int(rng.integers(0, len(flat)))]
        q.append(_flip(imgs[i][j], rng.integers(0, 256, int(rng.integers(0, 60)))) if rng.random() < 0.8 else rng.integers(0, 256, 32, dtype=np.uint8))
    q = np.stack(q)
    nz = [i for i, n in enumerate(sizes) if n]
    for r, i in enumerate(nz[:6]):
        imgs[i][(r * 5) % sizes[i]] = _flip(q[0], [int(x) for x in rng.choice(256, 4, replace=False)])
    if len(nz) > 1:
        imgs[nz[-1]][-1] = imgs[nz[0]][0]
    return imgs, q


def defined_with_masks(imgs, q, k):
    """the reference looks masks up for every entry it builds: compare masked calls only where all of them are defined (each query meets
    k codes, all within D = 128)"""
    return all(len(x[0]) == k and (x[3] <= 128).all() for x in P.collection_knn(imgs, q, k))


def check(imgs, q, ks, radii, rng, masks=True):
    opts = [None]
    if masks:
        opts.append([(rng.random(len(q)) < 0.6).astype(np.uint8) for _ in imgs])
    for m in opts:
        if m is None or defined_with_masks(imgs, q, 1):
            same_match(P.collection_match_list(imgs, q, m), P.ref_collection_match(imgs, q, m), "match")
        for compact in (False, True):
            for k in ks:
                if m is None or defined_with_masks(imgs, q, k):
                    same_lists(P.collection_knn_lists(imgs, q, k, m, compact), P.ref_collection_knn(imgs, q, k, m, compact), "knn %d %s" % (k, compact))
            for r in radii:
                if m is None or r <= 128:
                    same_lists(P.collection_radius_lists(imgs, q, r, m, compact), P.ref_collection_radius(imgs, q, r, m, compact), "radius %g" % r)


@pytest.mark.parametrize("sizes", [(9,), (0, 12), (7, 0, 5), (4, 6, 0), (0, 0, 3, 8, 0), (5, 1, 1, 0, 9, 2, 3, 0, 4, 6, 2, 1)])
def test_images_with_empty_ones_and_ties(ref, sizes):
    """1-12 images, empty ones at the start, middle and end (the later image's rows report the empty image's index, and its mask); ties
    between images; k = 1, 2, 3 and beyond the collection; radius 0, 25, 128 and infinity"""
    rng = np.random.default_rng(sum(sizes) * 31 + len(sizes))
    imgs, q = images_with_ties(rng, list(sizes), 14)
    n = sum(sizes)
    check(imgs, q, [1, 2, 3, n, n + 4], [0.0, 25.0, 128.0, math.inf], rng)


def test_img_idx_of_rows_after_an_empty_image(ref):
    rng = np.random.default_rng(3)
    imgs = [np.zeros((0, 32), np.uint8), rng.integers(0, 256, (4, 32), dtype=np.uint8), np.zeros((0, 32), np.uint8), rng.integers(0, 256, (3, 32), dtype=np.uint8)]
    q = np.concatenate([imgs[1], imgs[3]])
    qi, ti, ii, d = P.ref_collection_match(imgs, q)
    np.testing.assert_array_equal(ti, np.arange(7))
    np.testing.assert_array_equal(ii, [0, 0, 0, 0, 2, 2, 2])      # the empty images own the rows that follow them
    same_match(P.collection_match_list(imgs, q), (qi, ti, ii, d))


def test_all_zero_mask_on_the_nearest_image(ref):
    """match does not fall back to the next nearest code when the nearest one's image masks the query"""
    rng = np.random.default_rng(11)
    imgs, q = images_with_ties(rng, [6, 8, 5], 10)
    q[:3] = imgs[1][:3]
    masks = [np.ones(len(q), np.uint8), np.zeros(len(q), np.uint8), np.ones(len(q), np.uint8)]
    got = P.collection_match_list(imgs, q, masks)
    same_match(got, P.ref_collection_match(imgs, q, masks))
    assert not np.isin([0, 1, 2], got[0]).any()
    for compact in (False, True):
        same_lists(P.collection_knn_lists(imgs, q, 2, masks, compact), P.ref_collection_knn(imgs, q, 2, masks, compact))
        same_lists(P.collection_radius_lists(imgs, q, 25.0, masks, compact), P.ref_collection_radius(imgs, q, 25.0, masks, compact))


def test_codes_near_D(ref):
    """distances around D = 128: train_idx and img_idx are -1 beyond it (no masks: the reference leaves trainIdx unwritten there)"""
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (12, 0, 15, 13)]
    base = np.concatenate(imgs)
    q = np.stack([_flip(base[i % 40], rng.choice(256, 120 + i % 20, replace=False)) for i in range(20)])
    check(imgs, q, [1, 2, 5, 40, 43], [127.0, 128.0, 129.0, 300.0], rng, masks=False)
    far = [x for x in P.collection_knn_lists(imgs, q, 40) if (x[4] > 128).any()]
    assert far and all((x[2][x[4] > 128] == -1).all() and (x[3][x[4] > 128] == -1).all() for x in far)


def test_fixture_b_frames_as_keyframes(ref, fixture_b):
    frames = [fixture_b["frames"][i][0] for i in (0, 2, 4, 6)]
    for use_lsd in (True, False):
        descs = [ref.lbd_compute(f, ref.lbd_detect_keylines(f, use_lsd, 15.0)) for f in frames]
        rng = np.random.default_rng(int(use_lsd))
        q = descs[-1][:40]
        check(descs[:-1], q, [1, 2, 3, 7], [0.0, 25.0], rng)
        check(descs, descs[1][:25], [1, 2, 5], [25.0], rng)


def test_restatement_edges():
    """what the library defines where the reference is not run: an empty collection, an empty query set, k = 0, k < 0"""
    rng = np.random.default_rng(2)
    q = rng.integers(0, 256, (5, 32), dtype=np.uint8)
    assert all(len(x[1]) == 0 for x in P.collection_knn_lists([np.zeros((0, 32), np.uint8)], q, 3))
    assert P.collection_knn_lists([], q, 2, compact=True) == [] and P.collection_radius_lists([], q, 25.0, compact=True) == []
    assert P.collection_knn_lists([q], q[:0], 2) == [] and len(P.collection_match_list([q], q[:0])[0]) == 0
    assert all(len(x[1]) == 0 for x in P.collection_knn_lists([q], q, 0))
    with pytest.raises(ValueError):
        P.collection_knn([q], q, -1)
    # masks drop entries beyond D = 128: they have no image
    far = np.stack([_flip(q[0], range(0, 256, 2))])
    assert P.collection_knn_lists([q], far, 5)[0][4].max() > 128
    kept = P.collection_knn_lists([q], far, 5, [np.ones(1)])[0]
    assert (kept[4] <= 128).all() and (kept[3] == 0).all()
