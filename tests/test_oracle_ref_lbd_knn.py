"""k-nearest-neighbour and radius matching of line descriptors: the oracle's restatement (oracle/lbd_knn_oracle.cpp: lbd_orc_knn_match,
lbd_orc_radius_match -- the met codes of a query in the multi-index hash's key order, first k / distance <= r) against the REFERENCE'S OWN
pairwise BinaryDescriptorMatcher::knnMatch / radiusMatch (line_lbd/libs/binary_descriptor_matcher.cpp:264-341, 431-507, compiled into
oracle/_ref/liblinelbd_knn_ref.so), with masks and compactResult.  The reference's answer is compared where it is defined: the first
min(k, met codes) entries of a knn list, the entries of a radius list that come from met codes, trainIdx where the distance is <= D = 128
(the wrapper, oracle/ref/linelbd_knn_ref.cpp, cuts the rest)."""
import numpy as np
import pytest

from oracle import pyoracle_knn as K


@pytest.fixture(scope="module")
def ref(oracle):
    if not K.ref_available():
        pytest.skip("oracle/_ref/liblinelbd_knn_ref.so not built (no reference checkout on this machine)")
    return oracle


def _flip(c, bits):
    c = c.copy()
    for b in bits:
        c[b // 8] ^= np.uint8(1 << (b % 8))
    return c


def _planted(rng, nq, nt):
    """train codes with planted ties (same distance to query 0, close in different bytes / patterns) and an exact duplicate; queries a
    few to many bit flips from a train code, or unrelated"""
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    q = np.stack([_flip(t[int(rng.integers(0, nt))], rng.integers(0, 256, int(rng.integers(0, 140)))) if rng.random() < 0.8
                  else rng.integers(0, 256, 32, dtype=np.uint8) for _ in range(nq)])
    k = int(rng.integers(2, 7))
    for j in range(min(6, nt)):
        t[(j * 7) % nt] = _flip(q[0], [int(x) for x in rng.choice(256, k, replace=False)])
    if nt > 1:
        t[nt - 1] = t[0]
    return q, t


def same_lists(a, b):
    assert [x[0] for x in a] == [x[0] for x in b], ([x[0] for x in a], [x[0] for x in b])
    for x, y in zip(a, b):
        for u, v in zip(x[1:], y[1:]):
            np.testing.assert_array_equal(u, v)


def check_pair(ref, q, t, ks=None, radii=(0.0, 25.0, 128.0), masks=True, rng=None):
    nt = len(t)
    ks = ks if ks is not None else sorted({1, 2, 5, nt, nt + 3})
    mask_opts = [None]
    if masks and len(q):
        rng = rng or np.random.default_rng(0)
        mask_opts.append((rng.random(len(q)) < 0.6).astype(np.uint8))
    for mask in mask_opts:
        for compact in (False, True):
            for k in ks:
                same_lists(K.lbd_knn_lists(q, t, k, mask, compact), K.ref_knn_match(q, t, k, mask, compact))
            for r in radii:
                same_lists(K.lbd_radius_lists(q, t, r, mask, compact), K.ref_radius_match(q, t, r, mask, compact))


def test_random_codes_with_planted_ties(ref):
    rng = np.random.default_rng(20261016)
    for trial in range(40):
        nq, nt = int(rng.integers(1, 20)), int(rng.integers(1, 60))
        q, t = _planted(rng, nq, nt)
        check_pair(ref, q, t, rng=rng)


def test_queries_near_D(ref):
    """distances around D = 128: a knn answer and a radius of 128 reach past it, where train_idx is -1"""
    rng = np.random.default_rng(5)
    t = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    q = np.stack([_flip(t[i % 40], rng.choice(256, 120 + i % 20, replace=False)) for i in range(30)])
    check_pair(ref, q, t, ks=[1, 2, 5, 40, 43], radii=(127.0, 128.0, 128.5, 129.0, 300.0))
    lists = K.lbd_knn_lists(q, t, 40)
    far = np.concatenate([x[3] for x in lists]) > 128
    assert far.any() and (np.concatenate([x[2] for x in lists])[far] == -1).all()


def test_consecutive_fixture_b_frames(ref, fixture_b):
    frames = [fixture_b["frames"][i][0] for i in (0, 1, 2)]
    for use_lsd in (True, False):
        descs = [ref.lbd_compute(f, ref.lbd_detect_keylines(f, use_lsd, 15.0)) for f in frames]
        for a, b in zip(descs[:-1], descs[1:]):
            assert len(a) > 10 and len(b) > 10
            check_pair(ref, a, b)


def test_empty_sides_and_k_zero(ref):
    rng = np.random.default_rng(9)
    q, t = _planted(rng, 6, 10)
    for a, b in ((q[:0], t), (q, t[:0]), (q[:0], t[:0])):
        assert K.lbd_knn_lists(a, b, 2) == [] and K.ref_knn_match(a, b, 2) == []
        assert K.lbd_radius_lists(a, b, 25.0) == [] and K.ref_radius_match(a, b, 25.0) == []
    # k = 0: the reference's query() writes every code it meets into a result buffer of 0 entries (not run); no entries here
    assert [x[0] for x in K.lbd_knn_lists(q, t, 0)] == list(range(6)) and all(len(x[1]) == 0 for x in K.lbd_knn_lists(q, t, 0))
    with pytest.raises(ValueError):
        K.lbd_knn_match(q, t, -1)
