"""The Python mirror of BinaryDescriptorMatcher (cube_slam_b200/line_lbd.py: line_lbd_detect.bdm) WITHOUT a GPU: its marshalling -- pair
CSRs, the one mask array over a batch, the n_queries x k rows of the knn call and the k it asks for, the radius call's offsets and its one
retry after CS_ERR_CAPACITY, the compactResult views, the mask-length check -- exercised against a stand-in for the device entry points that
answers from the CPU oracle through the same C signatures.  What the kernels compute is tested elsewhere (tests/test_lbd_knn_host_emu.py,
tests/test_gpu_lbd_knn.py)."""
import numpy as np
import pytest

from oracle import pyoracle_knn as K

from test_line_lbd_mirror_fake import FakeContext, FakeLib, _view


class FakeMatcherLib(FakeLib):
    def _pairs(self, q, qo, t, to, n_pairs, mask):
        qo, to = _view(qo, np.int32, n_pairs + 1), _view(to, np.int32, n_pairs + 1)
        qq = _view(q, np.uint8, max(int(qo[-1]), 1) * 32).reshape(-1, 32)
        tt = _view(t, np.uint8, max(int(to[-1]), 1) * 32).reshape(-1, 32)
        m = None if mask is None else _view(mask, np.uint8, int(qo[-1]))
        return qo, to, qq, tt, m

    def cs_knn_match_line_descrip_batch(self, h, q, qo, t, to, n_pairs, k, mask, out, n):
        qo, to, qq, tt, m = self._pairs(q, qo, t, to, n_pairs, mask)
        nq = int(qo[-1])
        self.calls.append(("knn", k, n_pairs, None if m is None else m.copy()))
        if k < 0:
            return -1
        o, nn = _view(out, self._lib.DMATCH_DTYPE, max(nq * k, 1)), _view(n, np.int32, max(nq, 1))
        nn[:] = 0
        for p in range(n_pairs):
            if qo[p + 1] == qo[p] or to[p + 1] == to[p] or k == 0:
                continue
            res = K.lbd_knn_match(qq[qo[p]:qo[p + 1]], tt[to[p]:to[p + 1]], k, None if m is None else m[qo[p]:qo[p + 1]])
            for i, (a, b, c) in enumerate(res):
                g = qo[p] + i
                r = o[g * k:g * k + len(a)]
                r["query_idx"], r["train_idx"], r["img_idx"], r["distance"] = a, b, 0, c
                nn[g] = len(a)
        return 0

    def cs_radius_match_line_descrip_batch(self, h, q, qo, t, to, n_pairs, r, mask, out, cap, off):
        qo, to, qq, tt, m = self._pairs(q, qo, t, to, n_pairs, mask)
        nq = int(qo[-1])
        self.calls.append(("radius", int(cap.value), n_pairs))
        offs = _view(off, np.int64, nq + 1)
        rows = []
        for p in range(n_pairs):
            res = K.lbd_radius_match(qq[qo[p]:qo[p + 1]], tt[to[p]:to[p + 1]], r.value, None if m is None else m[qo[p]:qo[p + 1]])
            rows += res if to[p + 1] > to[p] else [(np.zeros(0),) * 3] * int(qo[p + 1] - qo[p])
        offs[:] = np.concatenate([[0], np.cumsum([len(x[0]) for x in rows])])
        if offs[-1] > cap.value:
            return -3
        o = _view(out, self._lib.DMATCH_DTYPE, max(int(offs[-1]), 1))
        for i, (a, b, c) in enumerate(rows):
            x = o[offs[i]:offs[i + 1]]
            x["query_idx"], x["train_idx"], x["img_idx"], x["distance"] = a, b, 0, c
        return 0


@pytest.fixture()
def bdm(oracle):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    d = cs.line_lbd_detect(context=FakeContext(FakeMatcherLib(_lib.load(), oracle, _lib)))
    return d.bdm


def _lists(recs):
    return [(r["query_idx"], r["train_idx"], r["distance"]) for r in recs]


def same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype.itemsize == 16 and (g["img_idx"] == 0).all()
        for a, b in zip((g["query_idx"], g["train_idx"], g["distance"]), w[1:]):
            np.testing.assert_array_equal(a, b)


def _data(seed):
    rng = np.random.default_rng(seed)
    qs = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (7, 0, 30, 4)]
    ts = [np.concatenate([q[::2], rng.integers(0, 256, (5, 32), dtype=np.uint8)]) for q in qs]
    ts[3] = ts[3][:0]
    masks = [rng.random(len(q)) < 0.5 for q in qs]
    masks[0] = None
    return qs, ts, masks


@pytest.mark.parametrize("compact", [False, True])
def test_knn_batch_marshalling(bdm, oracle, compact):
    qs, ts, masks = _data(1)
    for k in (1, 2, 3, 12, 40):
        got = bdm.knnMatch_batch(qs, ts, k, masks, compact)
        kind, k_asked, n_pairs, m = bdm._ctx.L.calls[-1]
        assert kind == "knn" and n_pairs == 4 and k_asked == min(k, max(len(t) for t in ts))    # never more slots than a train set has codes
        np.testing.assert_array_equal(m[:37], np.concatenate([np.ones(7), masks[2]]))
        for p in range(4):
            same(got[p], K.lbd_knn_lists(qs[p], ts[p], k, masks[p], compact))
    same(bdm.knnMatch(qs[2], ts[2], 2, masks[2], compact), K.lbd_knn_lists(qs[2], ts[2], 2, masks[2], compact))


@pytest.mark.parametrize("compact", [False, True])
def test_radius_batch_marshalling_and_retry(bdm, oracle, compact):
    qs, ts, masks = _data(2)
    got = bdm.radiusMatch_batch(qs, ts, 300.0, masks, compact, max_matches=3)
    calls = [c for c in bdm._ctx.L.calls if c[0] == "radius"]
    assert calls[0][1] == 3 and calls[1][1] > 3 and len(calls) == 2                     # one retry, with the size the call reported
    for p in range(4):
        same(got[p], K.lbd_radius_lists(qs[p], ts[p], 300.0, masks[p], compact))
    same(bdm.radiusMatch(qs[0], ts[0], 90.0, None, compact), K.lbd_radius_lists(qs[0], ts[0], 90.0, None, compact))


def test_mask_length_and_empty_sides(bdm):
    import cube_slam_b200 as cs
    qs, ts, _ = _data(3)
    for call in (lambda: bdm.knnMatch(qs[0], ts[0], 2, mask=np.ones(6)), lambda: bdm.radiusMatch(qs[0], ts[0], 25.0, mask=np.ones(8)),
                 lambda: bdm.knnMatch_batch(qs, ts, 2, [None, None, np.ones(29), None])):
        with pytest.raises(cs.CubeSlamError, match="mask"):
            call()
    assert bdm.knnMatch(qs[1], ts[1], 2) == [] and bdm.radiusMatch(qs[3], ts[3], 25.0) == []
    with pytest.raises(cs.CubeSlamError):
        bdm.knnMatch_batch(qs, ts[:3], 2)
