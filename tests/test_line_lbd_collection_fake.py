"""The collection forms of the Python BinaryDescriptorMatcher mirror (cube_slam_b200/line_lbd.py) WITHOUT a GPU: which overload a call
selects (a descriptor matrix as the second argument: pairwise; a number, a list of masks or nothing: the collection), the image CSR of add(),
the n_images x n_query mask array and the mask-length check, the knn rows and the k asked for, the radius offsets and their one retry,
compactResult, and `line_lbd_detect.bdm` being one object -- against a stand-in for the cs_lbd_collection_* entry points that keeps the
images on the host and answers from the CPU oracle through the same C signatures.  What the kernels compute is tested on the GPU
(tests/test_gpu_lbd_collection.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle_collection as P

from test_line_lbd_matcher_fake import FakeMatcherLib
from test_line_lbd_mirror_fake import FakeContext, _view


class FakeCollectionLib(FakeMatcherLib):
    def __init__(self, *a):
        super().__init__(*a)
        self.colls = {}

    def cs_lbd_collection_create(self, h):
        key = 1000 + len(self.colls)
        self.colls[key] = []
        return key

    def cs_lbd_collection_destroy(self, c):
        self.colls.pop(c, None)

    def cs_lbd_collection_add(self, c, codes, offs, n):
        o = _view(offs, np.int32, n + 1)
        cc = _view(codes, np.uint8, max(int(o[-1]), 1) * 32).reshape(-1, 32)
        self.colls[c] += [cc[o[i]:o[i + 1]].copy() for i in range(n)]
        self.calls.append(("add", n, int(o[-1])))
        return 0

    def cs_lbd_collection_clear(self, c):
        self.colls[c] = []
        return 0

    def cs_lbd_collection_size(self, c, ni, nc):
        ni._obj.value, nc._obj.value = len(self.colls[c]), sum(len(x) for x in self.colls[c])
        return 0

    def _masks(self, m, n_masks, nq, c):
        if m is None:
            return None, n_masks == 0
        mm = _view(m, np.uint8, n_masks * max(nq, 1)).reshape(n_masks, -1)
        return list(mm), n_masks == len(self.colls[c])

    def cs_lbd_collection_knn_match(self, c, q, nq, k, m, n_masks, out, n):
        masks, ok = self._masks(m, n_masks, nq, c)
        self.calls.append(("knn", k, None if masks is None else np.array(masks)))
        if not ok or k < 0:
            return -1
        qq = _view(q, np.uint8, max(nq, 1) * 32).reshape(-1, 32)[:nq]
        o, nn = _view(out, self._lib.DMATCH_DTYPE, max(nq * k, 1)), _view(n, np.int32, max(nq, 1))
        for i, (a, b, d, e) in enumerate(P.collection_knn(self.colls[c], qq, k, masks) if k else [()] * nq):
            r = o[i * k:i * k + len(a)] if k else o[:0]
            if k:
                r["query_idx"], r["train_idx"], r["img_idx"], r["distance"] = a, b, d, e
            nn[i] = len(r)
        return 0

    def cs_lbd_collection_match(self, c, q, nq, m, n_masks, out, n):
        masks, ok = self._masks(m, n_masks, nq, c)
        self.calls.append(("match", None if masks is None else np.array(masks)))
        if not ok:
            return -1
        qq = _view(q, np.uint8, max(nq, 1) * 32).reshape(-1, 32)[:nq]
        a, b, d, e = P.collection_match_list(self.colls[c], qq, masks)
        o = _view(out, self._lib.DMATCH_DTYPE, max(nq, 1))
        o[:len(a)]["query_idx"], o[:len(a)]["train_idx"], o[:len(a)]["img_idx"], o[:len(a)]["distance"] = a, b, d, e
        n._obj.value = len(a)
        return 0

    def cs_lbd_collection_radius_match(self, c, q, nq, r, m, n_masks, out, cap, off):
        masks, ok = self._masks(m, n_masks, nq, c)
        self.calls.append(("radius", int(cap.value)))
        if not ok:
            return -1
        qq = _view(q, np.uint8, max(nq, 1) * 32).reshape(-1, 32)[:nq]
        rows = P.collection_radius(self.colls[c], qq, r.value, masks)
        offs = _view(off, np.int64, nq + 1)
        offs[:] = np.concatenate([[0], np.cumsum([len(x[0]) for x in rows])])
        if offs[-1] > cap.value:
            return -3
        o = _view(out, self._lib.DMATCH_DTYPE, max(int(offs[-1]), 1))
        for i, (a, b, d, e) in enumerate(rows):
            x = o[offs[i]:offs[i + 1]]
            x["query_idx"], x["train_idx"], x["img_idx"], x["distance"] = a, b, d, e
        return 0


@pytest.fixture()
def det(oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    return cs.line_lbd_detect(context=FakeContext(FakeCollectionLib(_lib.load(), oracle, _lib)))


def _data(seed):
    rng = np.random.default_rng(seed)
    imgs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (6, 0, 9, 4)]
    q = np.concatenate([imgs[0][:3], imgs[2][:3], rng.integers(0, 256, (4, 32), dtype=np.uint8)])
    masks = [(rng.random(len(q)) < 0.5).astype(np.uint8) for _ in imgs]
    return imgs, q, masks


def same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for f, v in zip(("query_idx", "train_idx", "img_idx", "distance"), w[1:]):
            np.testing.assert_array_equal(g[f], v)


def test_bdm_is_one_object(det):
    assert det.bdm is det.bdm


def test_dispatch_between_pairwise_and_collection(det):
    imgs, q, _ = _data(1)
    bdm = det.bdm
    bdm.add(imgs)
    L = det._ctx.L
    bdm.knnMatch(q, imgs[0], 2)
    assert L.calls[-1][0] == "knn" and len(L.calls[-1]) == 4          # the pairwise call (FakeMatcherLib records four fields)
    bdm.knnMatch(q, 2)
    assert L.calls[-1][:2] == ("knn", 2) and len(L.calls[-1]) == 3
    bdm.knnMatch(q, np.int64(3), compactResult=True)
    assert L.calls[-1][:2] == ("knn", 3)
    bdm.radiusMatch(q, imgs[2], 25.0)
    assert L.calls[-1][0] == "radius" and L.calls[-1][1] == 8 * len(q)
    bdm.radiusMatch(q, 25.0)
    bdm.radiusMatch(q, maxDistance=25.0)
    bdm.match(q)
    assert L.calls[-1][0] == "match"
    bdm.match(q, None)
    assert L.calls[-1][0] == "match"
    bdm.match(q, [np.ones(len(q))] * 4)
    assert L.calls[-1][0] == "match"
    n = len(L.calls)
    bdm.match(q, imgs[0])
    bdm.match(q, trainDescriptors=imgs[2])
    assert all(c[0] != "match" for c in L.calls[n:])                  # the pairwise match goes through cs_match_line_descrip


def test_add_csr_and_size(det):
    imgs, q, _ = _data(2)
    bdm = det.bdm
    assert bdm.collection_size() == (0, 0)
    bdm.add([])
    bdm.add(imgs[:2])
    bdm.add(imgs[2:])
    assert [c for c in det._ctx.L.calls if c[0] == "add"] == [("add", 2, 6), ("add", 2, 13)]
    assert bdm.collection_size() == (4, 19)
    bdm.clear()
    assert bdm.collection_size() == (0, 0)


@pytest.mark.parametrize("compact", [False, True])
def test_collection_lists_masks_and_k(det, compact):
    imgs, q, masks = _data(3)
    bdm = det.bdm
    bdm.add(imgs)
    for k in (1, 2, 5, 19, 40):
        same(bdm.knnMatch(q, k, masks, compact), P.collection_knn_lists(imgs, q, k, masks, compact))
        assert det._ctx.L.calls[-1][1] == min(k, 19)                   # never more slots than the collection has codes
        np.testing.assert_array_equal(det._ctx.L.calls[-1][2], np.stack(masks))
    same(bdm.knnMatch(q, 3, None, compact), P.collection_knn_lists(imgs, q, 3, None, compact))
    got = bdm.match(q, masks)
    for f, v in zip(("query_idx", "train_idx", "img_idx", "distance"), P.collection_match_list(imgs, q, masks)):
        np.testing.assert_array_equal(got[f], v)
    same(bdm.radiusMatch(q, 110.0, masks, compact), P.collection_radius_lists(imgs, q, 110.0, masks, compact))


def test_radius_retry(det):
    imgs, q, masks = _data(4)
    bdm = det.bdm
    bdm.add(imgs)
    got = bdm._radius_collection(q, 300.0, masks, False, max_matches=2)
    calls = [c for c in det._ctx.L.calls if c[0] == "radius"]
    assert calls[0][1] == 2 and calls[1][1] > 2 and len(calls) == 2
    same(got, P.collection_radius_lists(imgs, q, 300.0, masks))


def test_mask_validation_and_empty_queries(det):
    import cube_slam_b200 as cs
    imgs, q, masks = _data(5)
    bdm = det.bdm
    bdm.add(imgs)
    with pytest.raises(cs.CubeSlamError, match="mask 2 has 9 entries for 10"):
        bdm.knnMatch(q, 2, masks[:2] + [np.ones(9)] + masks[3:])
    with pytest.raises(AssertionError):                               # the fake context asserts rc == 0: a wrong count reaches the library
        bdm.knnMatch(q, 2, masks[:3])
    assert bdm.knnMatch(q[:0], 2) == [] and bdm.radiusMatch(q[:0], 25.0) == [] and len(bdm.match(q[:0])) == 0
    same(bdm.knnMatch(q, 2, []), P.collection_knn_lists(imgs, q, 2))  # [] is no masks, as in the reference
    assert det._ctx.L.calls[-1][2] is None


class FakeContextLib(FakeCollectionLib):
    """cs_create / cs_destroy stand-ins too, so that a real Context (its close() and its teardown order) runs without a device"""

    def cs_create(self, *a):
        self.calls.append(("cs_create",))
        return 77

    def cs_destroy(self, h):
        self.calls.append(("cs_destroy", h))

    def cs_lbd_collection_create(self, h):
        assert h == 77
        return super().cs_lbd_collection_create(h)

    def cs_lbd_collection_destroy(self, c):
        self.calls.append(("collection_destroy", c))
        super().cs_lbd_collection_destroy(c)


def test_context_close_releases_collections_first(oracle, monkeypatch):
    """the C ABI reads the context when a collection is destroyed: Context.close() destroys the collections made on it first, and a
    matcher collected after close() makes no call into the library; its collection forms then raise"""
    import gc
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    from cube_slam_b200.detect_3d_cuboid import Context
    fake = FakeContextLib(_lib.load(), oracle, _lib)
    monkeypatch.setattr(_lib, "load", lambda: fake)
    ctx = Context(0)
    det, idle = cs.line_lbd_detect(context=ctx), cs.line_lbd_detect(context=ctx)
    imgs, q, _ = _data(6)
    det.bdm.add(imgs)
    idle.bdm                                                            # a matcher without a collection: nothing to release
    handle = det.bdm._h
    ctx.close()
    names = [c[0] for c in fake.calls]
    assert names.index("collection_destroy") < names.index("cs_destroy")
    assert ("collection_destroy", handle) in fake.calls and names.count("collection_destroy") == 1
    with pytest.raises(cs.CubeSlamError, match="closed"):
        det.bdm.knnMatch(q, 2)
    with pytest.raises(cs.CubeSlamError, match="closed"):
        det.bdm.add(imgs)
    n = len(fake.calls)
    del det, idle
    gc.collect()
    assert fake.calls[n:] == []                                         # nothing reaches the destroyed context


def test_matcher_collected_before_close(oracle, monkeypatch):
    """a matcher collected while its context is open destroys its collection; close() then has nothing left to release"""
    import gc
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    from cube_slam_b200.detect_3d_cuboid import Context
    fake = FakeContextLib(_lib.load(), oracle, _lib)
    monkeypatch.setattr(_lib, "load", lambda: fake)
    ctx = Context(0)
    det = cs.line_lbd_detect(context=ctx)
    det.bdm.add(_data(7)[0])
    del det
    gc.collect()
    ctx.close()
    assert [c[0] for c in fake.calls if c[0] in ("collection_destroy", "cs_destroy")] == ["collection_destroy", "cs_destroy"]


def test_match_refuses_a_2d_array_that_is_not_a_train_matrix(det):
    import cube_slam_b200 as cs
    imgs, q, masks = _data(8)
    det.bdm.add(imgs)
    with pytest.raises(cs.CubeSlamError, match="list of per-image masks"):
        det.bdm.match(q, np.stack(masks))                               # masks as one array: refused, not taken for a train matrix
    same([det.bdm.match(q, list(np.stack(masks)))], [(0,) + P.collection_match_list(imgs, q, masks)])
