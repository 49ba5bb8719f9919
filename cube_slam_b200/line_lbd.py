"""Host-side mirror of `class line_lbd_detect` (line_lbd/include/line_lbd/line_lbd_allclass.h:22-70).

detect_filter_lines(img) -> n x 4 float32 [x1 y1 x2 y2]: what the reference writes into its `cv::Mat& linesmat_out`
(line_lbd/class/line_lbd_allclass.cpp:216-221).  The descriptor / matcher methods (get_line_descriptors, detect_descrip_lines,
detect_descrip_lines_octaves, match_line_descrip; :191-198,224-356) return numpy arrays: key lines as records of `_lib.KEYLINE_DTYPE`
(the KeyLine fields, octave 0), descriptors as n x 32 uint8 (the CV_8UC1 matrix), matches as records of `_lib.DMATCH_DTYPE` (cv::DMatch).
`line_lbd_detect.bdm` is the class's BinaryDescriptorMatcher (line_lbd_allclass.h:37): pairwise match, knnMatch and radiusMatch on the GPU,
and the collection forms (add / train / clear, then match / knnMatch / radiusMatch without a train matrix) against codes kept on the GPU.
`line_lbd_detect.lsd` is the class's LSDDetector (line_lbd_allclass.h:40): detect over the pyrDown pyramid with masks, per octave or flat,
and over a list of images with one library call per image size.
detect_filter_lines_device, detect_descrip_lines_device and compute_descriptors_device take frames that are already in GPU memory.
A detector built with more than one octave (LSD flavour, octaveratio 2) returns every octave from detect_raw_lines_octaves,
detect_raw_lines and detect_descrip_lines_octaves, key lines as records of `_lib.OCTAVE_KEYLINE_DTYPE`."""
import ctypes as C
import math
import numbers

import numpy as np

from . import _lib
from .detect_3d_cuboid import Context, CubeSlamError


def _codes(d):
    return np.ascontiguousarray(d, np.uint8).reshape(-1, 32)


def _is_number(x):
    return isinstance(x, numbers.Number) or (isinstance(x, np.ndarray) and x.ndim == 0)


class BinaryDescriptorMatcher(object):
    """Mirror of cv::line_descriptor::BinaryDescriptorMatcher on the device of `context`.  Descriptors are n x 32 uint8; a list of matches
    is a records array of `_lib.DMATCH_DTYPE`, a vector<vector<DMatch>> a Python list of them, one per query.

    Pairwise forms (binary_descriptor_matcher.cpp:196-341, 431-507): match(query, train, mask), knnMatch(query, train, k, mask, compactResult),
    radiusMatch(query, train, maxDistance, mask, compactResult).  mask: one value per query (0 = skip it), its length must be the number of
    queries.  Where the reference is undefined the library's definitions hold (include/cube_slam_b200.h): fewer than k entries when fewer
    codes are met, train_idx -1 beyond 128 bits, [] for an empty query or train set.  At most 16384 train codes per pair (CubeSlamError
    beyond).

    Collection forms (:70-193, 344-428, 510-595): add([descriptors of each image]), train(), clear(), then match(query, masks),
    knnMatch(query, k, masks, compactResult), radiusMatch(query, maxDistance, masks, compactResult) against every image added.  The codes
    stay on the GPU between queries.  train_idx is the global row over all images added, img_idx the image (an empty image followed by
    others at the same row owns that row, as in the reference); masks: None or one mask per image, each one value per query, applied to the
    entries after they are chosen.  Which form runs follows C++ overload resolution: a descriptor matrix as the second positional argument
    (or trainDescriptors=) selects the pairwise form; a number, a list of masks or nothing (match) the collection form."""

    def __init__(self, context):
        self._ctx = context
        self._h = None      # the cs_lbd_collection, created on the first add
        self._closed = False

    def _release(self):
        """Destroy the collection while its context is alive.  Context.close() calls this before it destroys the context (the C ABI
        requires that order); afterwards the collection forms raise CubeSlamError."""
        h, self._h, self._closed = self._h, None, True
        if h:
            self._ctx.L.cs_lbd_collection_destroy(h)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and not getattr(self, "_closed", True):
            try:
                self._ctx.L.cs_lbd_collection_destroy(h)
            except Exception:
                pass

    @staticmethod
    def _pairwise(args, kw, first_is_number):
        """True when the call names a train matrix: the pairwise overload"""
        if "trainDescriptors" in kw:
            return True
        if not args:
            return False
        x = args[0]
        if first_is_number:
            return not _is_number(x)
        return x is not None and not isinstance(x, (list, tuple))

    def match(self, queryDescriptors, *args, **kw):
        """match(query, train[, mask]) -- pairwise -- or match(query[, masks]) against the collection.  The collection's masks are a list
        (one mask per image); a 2-D array as second argument is a train matrix, so one that is not n x 32 is refused rather than guessed."""
        if self._pairwise(args, kw, False):
            t = kw.get("trainDescriptors", args[0] if args else None)
            if isinstance(t, np.ndarray) and t.ndim == 2 and t.shape[1] != 32:
                raise CubeSlamError("match(query, train): a train descriptor matrix is n x 32, got %s; pass the collection's masks as a "
                                    "list of per-image masks" % (t.shape,))
            return self._match_pair(queryDescriptors, *args, **kw)
        return self._match_collection(queryDescriptors, *args, **kw)

    def knnMatch(self, queryDescriptors, *args, **kw):
        """knnMatch(query, train, k[, mask, compactResult]) -- pairwise -- or knnMatch(query, k[, masks, compactResult]) against the
        collection."""
        if self._pairwise(args, kw, True):
            return self._knn_pair(queryDescriptors, *args, **kw)
        return self._knn_collection(queryDescriptors, *args, **kw)

    def radiusMatch(self, queryDescriptors, *args, **kw):
        """radiusMatch(query, train, maxDistance[, mask, compactResult]) -- pairwise -- or radiusMatch(query, maxDistance[, masks,
        compactResult]) against the collection."""
        if self._pairwise(args, kw, True):
            return self._radius_pair(queryDescriptors, *args, **kw)
        return self._radius_collection(queryDescriptors, *args, **kw)

    @staticmethod
    def _mask(mask, n):
        if mask is None:
            return None
        m = np.asarray(mask).reshape(-1)
        if len(m) != n:
            raise CubeSlamError("mask has %d entries for %d query descriptors" % (len(m), n))
        return np.ascontiguousarray(m != 0, np.uint8)

    def _pack(self, queries, trains, masks):
        qs, ts = [_codes(q) for q in queries], [_codes(t) for t in trains]
        if len(qs) != len(ts) or not qs:
            raise CubeSlamError("one train set per query set, at least one pair")
        masks = [None] * len(qs) if masks is None else list(masks)
        if len(masks) != len(qs):
            raise CubeSlamError("one mask (or None) per pair")
        ms = [self._mask(m, len(q)) for m, q in zip(masks, qs)]
        qo = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int32)
        to = np.concatenate([[0], np.cumsum([len(t) for t in ts])]).astype(np.int32)
        q = np.ascontiguousarray(np.concatenate(qs)) if qo[-1] else np.zeros((1, 32), np.uint8)
        t = np.ascontiguousarray(np.concatenate(ts)) if to[-1] else np.zeros((1, 32), np.uint8)
        m = None
        if any(x is not None for x in ms):
            m = np.ascontiguousarray(np.concatenate([x if x is not None else np.ones(len(qq), np.uint8) for x, qq in zip(ms, qs)] + [np.zeros(1, np.uint8)]))
        return qs, ts, ms, q, qo, t, to, m

    def _match_pair(self, queryDescriptors, trainDescriptors, mask=None):
        """match(query, train, matches, mask): the nearest code of every (unmasked) query -> DMATCH_DTYPE records, query order."""
        q, t = _codes(queryDescriptors), _codes(trainDescriptors)
        m = self._mask(mask, len(q))
        out = np.zeros(max(len(q), 1), _lib.DMATCH_DTYPE)
        n = C.c_int32(0)
        self._ctx.check(self._ctx.L.cs_match_line_descrip(self._ctx.h, _lib.ptr(q, C.c_uint8), len(q), _lib.ptr(t, C.c_uint8), len(t), C.c_float(math.inf),
                                                          out.ctypes.data, C.byref(n)))
        out = out[:n.value].copy()
        return out if m is None else out[m[out["query_idx"]] != 0]

    def _knn_pair(self, queryDescriptors, trainDescriptors, k, mask=None, compactResult=False):
        """knnMatch(query, train, matches, k, mask, compactResult): per query its first k codes; a masked query gives an empty list, or
        none with compactResult."""
        return self.knnMatch_batch([queryDescriptors], [trainDescriptors], k, None if mask is None else [mask], compactResult)[0]

    def _radius_pair(self, queryDescriptors, trainDescriptors, maxDistance, mask=None, compactResult=False):
        """radiusMatch(query, train, matches, maxDistance, mask, compactResult): per query every code at distance <= maxDistance; with
        compactResult empty lists are left out."""
        return self.radiusMatch_batch([queryDescriptors], [trainDescriptors], maxDistance, None if mask is None else [mask], compactResult)[0]

    def knnMatch_batch(self, queries, trains, k, masks=None, compactResult=False):
        """knnMatch over independent (query set, train set) pairs in one launch -> one vector<vector<DMatch>> per pair."""
        qs, ts, ms, q, qo, t, to, m = self._pack(queries, trains, masks)
        k = int(k)
        kk = min(k, max(len(x) for x in ts)) if k > 0 else k     # no query gets more entries than its train set has codes
        nq = int(qo[-1])
        out = np.zeros(max(nq * kk, 1), _lib.DMATCH_DTYPE)
        n = np.zeros(max(nq, 1), np.int32)
        self._ctx.check(self._ctx.L.cs_knn_match_line_descrip_batch(self._ctx.h, _lib.ptr(q, C.c_uint8), _lib.ptr(qo, C.c_int32), _lib.ptr(t, C.c_uint8),
                                                                    _lib.ptr(to, C.c_int32), len(qs), kk, None if m is None else _lib.ptr(m, C.c_uint8),
                                                                    out.ctypes.data, _lib.ptr(n, C.c_int32)))
        res = []
        for p in range(len(qs)):
            if not len(qs[p]) or not len(ts[p]):
                res.append([])
                continue
            res.append([out[i * kk:i * kk + n[i]].copy() for i in range(qo[p], qo[p + 1])
                        if not (compactResult and ms[p] is not None and not ms[p][i - qo[p]])])
        return res

    def radiusMatch_batch(self, queries, trains, maxDistance, masks=None, compactResult=False, max_matches=None):
        """radiusMatch over independent pairs in one call -> one vector<vector<DMatch>> per pair.  max_matches: the first buffer's size
        (default 8 per query); when the matches do not fit, the call is repeated once with the size the library reports."""
        qs, ts, ms, q, qo, t, to, m = self._pack(queries, trains, masks)
        nq = int(qo[-1])
        cap = int(max_matches) if max_matches is not None else 8 * nq
        off = np.zeros(nq + 1, np.int64)
        L, h = self._ctx.L, self._ctx.h
        for attempt in range(2):
            out = np.zeros(max(cap, 1), _lib.DMATCH_DTYPE)
            rc = L.cs_radius_match_line_descrip_batch(h, _lib.ptr(q, C.c_uint8), _lib.ptr(qo, C.c_int32), _lib.ptr(t, C.c_uint8), _lib.ptr(to, C.c_int32),
                                                      len(qs), C.c_float(maxDistance), None if m is None else _lib.ptr(m, C.c_uint8), out.ctypes.data,
                                                      C.c_int64(cap), _lib.ptr(off, C.c_int64))
            if rc == -3 and attempt == 0 and off[-1] > cap:        # CS_ERR_CAPACITY with the layout filled: resize and call again
                cap = int(off[-1])
                continue
            self._ctx.check(rc)
            break
        res = []
        for p in range(len(qs)):
            if not len(qs[p]) or not len(ts[p]):
                res.append([])
                continue
            lists = [out[off[i]:off[i + 1]].copy() for i in range(qo[p], qo[p + 1])]
            res.append([x for x in lists if len(x) or not compactResult])
        return res

    # ---------------------------------------------------------------- the collection ("from one image to a set")
    def _collection(self):
        if self._closed:
            raise CubeSlamError("the matcher's context is closed")
        if self._h is None:
            h = self._ctx.L.cs_lbd_collection_create(self._ctx.h)
            if not h:
                raise CubeSlamError("cs_lbd_collection_create failed")
            self._h = h
            depend = getattr(self._ctx, "_depend", None)
            if depend is not None:
                depend(self)                                         # close() of the context releases the collection first
        return self._h

    def add(self, descriptors):
        """add(vector<Mat>): append the codes of each image (n_i x 32 uint8, n_i may be 0) to the collection, uploaded to the GPU now."""
        ds = [_codes(d) for d in descriptors]
        if not ds:
            return
        off = np.concatenate([[0], np.cumsum([len(d) for d in ds])]).astype(np.int32)
        codes = np.ascontiguousarray(np.concatenate(ds)) if off[-1] else np.zeros((1, 32), np.uint8)
        self._ctx.check(self._ctx.L.cs_lbd_collection_add(self._collection(), _lib.ptr(codes, C.c_uint8), _lib.ptr(off, C.c_int32), len(ds)))

    def train(self):
        """train(): nothing to do -- the codes are searchable on the GPU as soon as add() returns (the query forms call train() in the
        reference too)."""

    def clear(self):
        """clear(): forget every image added, and return the collection's device memory."""
        if self._h is not None:
            self._ctx.check(self._ctx.L.cs_lbd_collection_clear(self._h))

    def collection_size(self):
        """(number of images, number of codes) added since creation or clear()"""
        if self._h is None:
            return 0, 0
        ni, nc = C.c_int32(0), C.c_int64(0)
        self._ctx.check(self._ctx.L.cs_lbd_collection_size(self._h, C.byref(ni), C.byref(nc)))
        return ni.value, nc.value

    @staticmethod
    def _masks(masks, nq):
        """one n_query byte row per image mask -> (array, count); None or [] -> no masks"""
        if masks is None or len(masks) == 0:
            return None, 0
        rows = []
        for i, m in enumerate(masks):
            m = np.asarray(m).reshape(-1)
            if len(m) != nq:
                raise CubeSlamError("mask %d has %d entries for %d query descriptors" % (i, len(m), nq))
            rows.append(m != 0)
        if not nq:
            return np.zeros(1, np.uint8), len(rows)
        return np.ascontiguousarray(np.stack(rows), np.uint8).reshape(-1), len(rows)

    def _query(self, queryDescriptors, masks):
        """(codes, n_query, mask pointer or None, number of masks); the mask array lives as long as the pointer's ctypes object"""
        q = _codes(queryDescriptors)
        m, n_masks = self._masks(masks, len(q))
        return q if len(q) else np.zeros((1, 32), np.uint8), len(q), None if m is None else _lib.ptr(m, C.c_uint8), n_masks

    def _match_collection(self, queryDescriptors, masks=None):
        """match(query, matches, masks): the nearest code of the collection for every query, unless the mask of its image skips the query
        (no fall-back to the next nearest) -> DMATCH_DTYPE records, query order."""
        q, nq, mp, n_masks = self._query(queryDescriptors, masks)
        out = np.zeros(max(nq, 1), _lib.DMATCH_DTYPE)
        n = C.c_int32(0)
        self._ctx.check(self._ctx.L.cs_lbd_collection_match(self._collection(), _lib.ptr(q, C.c_uint8), nq, mp, n_masks, out.ctypes.data, C.byref(n)))
        return out[:n.value].copy()

    def _knn_collection(self, queryDescriptors, k, masks=None, compactResult=False):
        """knnMatch(query, matches, k, masks, compactResult): the first k codes of the collection per query, then the masks; with
        compactResult lists left empty are dropped.  [] for an empty query set."""
        q, nq, mp, n_masks = self._query(queryDescriptors, masks)
        k = int(k)
        h = self._collection()
        kk = min(k, self.collection_size()[1]) if k > 0 else k     # no query gets more entries than the collection has codes
        out = np.zeros(max(nq * kk, 1), _lib.DMATCH_DTYPE)
        n = np.zeros(max(nq, 1), np.int32)
        self._ctx.check(self._ctx.L.cs_lbd_collection_knn_match(h, _lib.ptr(q, C.c_uint8), nq, kk, mp, n_masks, out.ctypes.data, _lib.ptr(n, C.c_int32)))
        lists = [out[i * kk:i * kk + n[i]].copy() for i in range(nq)]
        return [x for x in lists if len(x) or not compactResult]

    def _radius_collection(self, queryDescriptors, maxDistance, masks=None, compactResult=False, max_matches=None):
        """radiusMatch(query, matches, maxDistance, masks, compactResult): every code of the collection at distance <= maxDistance per
        query, then the masks; with compactResult lists left empty are dropped.  max_matches: the first buffer's size (default 8 per
        query); when the matches do not fit, the call is repeated once with the size the library reports."""
        q, nq, mp, n_masks = self._query(queryDescriptors, masks)
        h = self._collection()
        cap = int(max_matches) if max_matches is not None else 8 * nq
        off = np.zeros(nq + 1, np.int64)
        L = self._ctx.L
        for attempt in range(2):
            out = np.zeros(max(cap, 1), _lib.DMATCH_DTYPE)
            rc = L.cs_lbd_collection_radius_match(h, _lib.ptr(q, C.c_uint8), nq, C.c_float(maxDistance), mp, n_masks, out.ctypes.data, C.c_int64(cap),
                                                  _lib.ptr(off, C.c_int64))
            if rc == -3 and attempt == 0 and off[-1] > cap:        # CS_ERR_CAPACITY with the layout filled: resize and call again
                cap = int(off[-1])
                continue
            self._ctx.check(rc)
            break
        lists = [out[off[i]:off[i + 1]].copy() for i in range(nq)]
        return [x for x in lists if len(x) or not compactResult]


class LSDDetector(object):
    """Mirror of cv::line_descriptor::LSDDetector (descriptor.hpp:1004-1067, LSDDetector.cpp:104-287) on the device of `context`: LSD over the
    pyrDown pyramid, every KeyLine field, as records of `_lib.OCTAVE_KEYLINE_DTYPE` (KeyLine::pt is the mid point of start and end).

    detect(image, scale, numOctaves, mask=None) -> the flat list, octave after octave; detect_octaves(image, scale, numOctaves, mask=None) ->
    one array per octave; detect([images], scale, numOctaves, masks=None) -> one flat array per image, one library call per (height, width,
    channels) group.  Images are H x W gray, H x W x 3 BGR or H x W x 4 BGRA, uint8.  numOctaves == 1 ignores scale; numOctaves > 1 needs
    scale 2 (pyrDown's size rule); numOctaves == 0 detects nothing.  mask: an H x W uint8 array; a key line is dropped when the mask is 0 at
    both of its truncated end points (LSDDetector.cpp:258-286); class_id keeps counting the lines of an octave before the mask, as in the
    reference.  A masks list shorter than the images leaves the rest unmasked.  The arrays are new: the C++ overloads' append semantics and
    LSDOptions do not apply here.  Refusals raise CubeSlamError with the reference's message where it has one."""

    FIRST_CAP = 2048    # LSD segments per octave the first call has room for; doubled while the library answers CS_ERR_CAPACITY

    def __init__(self, context):
        self._ctx = context

    @staticmethod
    def _check(img, mask, scale, numOctaves, mask_message):
        img = np.asarray(img)
        if mask is not None:
            m = np.asarray(mask)
            if m.shape != img.shape[:2] or m.dtype != np.uint8:
                raise CubeSlamError(mask_message)
        if img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3, 4)):
            raise CubeSlamError("LSDDetector takes H x W gray, H x W x 3 BGR or H x W x 4 BGRA images, got shape %s" % (img.shape,))
        if img.dtype != np.uint8:
            raise CubeSlamError("Error, depth image!= 0")
        if numOctaves > 1 and int(scale) != 2:
            raise CubeSlamError("LSDDetector with more than one octave needs scale 2 (cv::pyrDown makes an octave of (cols / scale, rows / scale) "
                                "only when |2 * dst - src| <= 2), got %d" % int(scale))
        if numOctaves < 0:
            raise CubeSlamError("numOctaves must not be negative (the reference's vector::resize throws std::length_error)")

    @staticmethod
    def _gray_or_bgr(img):
        img = np.asarray(img)
        if img.ndim == 3 and img.shape[2] == 1:
            return img[..., 0]
        return img[..., :3] if img.ndim == 3 and img.shape[2] == 4 else img

    @staticmethod
    def _apply_mask(kl, mask):
        """LSDDetector.cpp:258-286: drop the lines whose two truncated end points both read 0 (a point outside the mask does not read 0)"""
        if mask is None or not len(kl):
            return kl
        m = np.asarray(mask)
        H, W = m.shape

        def zero_at(x, y):
            inside = (x > -1) & (y > -1) & (x < W) & (y < H)
            xi = np.where(inside, np.trunc(np.where(inside, x, 0)), 0).astype(np.int64)
            yi = np.where(inside, np.trunc(np.where(inside, y, 0)), 0).astype(np.int64)
            return inside & (m[yi, xi] == 0)
        drop = zero_at(kl["start_x"], kl["start_y"]) & zero_at(kl["end_x"], kl["end_y"])
        return kl[~drop]

    def _detect_group(self, frames, numOctaves):
        """frames of one size and channel count (F x H x W or F x H x W x 3) -> per frame, one OCTAVE_KEYLINE_DTYPE array per octave"""
        imgs = np.ascontiguousarray(frames, np.uint8)
        F, H, W = imgs.shape[:3]
        ch = 1 if imgs.ndim == 3 else imgs.shape[3]
        K = int(numOctaves)
        p = _lib.LineParams()
        L = self._ctx.L
        L.cs_default_line_params(C.byref(p))
        p.use_LSD, p.numoctaves, p.octaveratio = 1, K, 2.0 if K > 1 else 1.0
        n = np.zeros((F, K), np.int32)
        cap = self.FIRST_CAP
        while True:
            kl = np.zeros((F, K, cap), _lib.OCTAVE_KEYLINE_DTYPE)
            rc = L.cs_detect_raw_lines_octaves_batch(self._ctx.h, imgs.ctypes.data, F, W, H, W * ch, ch, C.byref(p), kl.ctypes.data, cap,
                                                     _lib.ptr(n, C.c_int32))
            if rc == -3 and cap < W * H:        # CS_ERR_CAPACITY: an octave holds more LSD segments than the buffer; twice the room
                cap *= 2
                continue
            self._ctx.check(rc)
            return [[kl[f, k, :n[f, k]].copy() for k in range(K)] for f in range(F)]

    def _octaves_of(self, images, numOctaves):
        """one call per (height, width, channels) group -> per image, its octaves"""
        out = [None] * len(images)
        if numOctaves < 1:
            return [[] for _ in images]
        groups = {}
        for i, img in enumerate(images):
            groups.setdefault(img.shape, []).append(i)
        for idx in groups.values():
            got = self._detect_group(np.stack([images[i] for i in idx]), numOctaves)
            for i, g in zip(idx, got):
                out[i] = g
        return out

    def _empty(self):
        return np.zeros(0, _lib.OCTAVE_KEYLINE_DTYPE)

    def detect(self, image, scale, numOctaves, mask=None, masks=None):
        """detect(image, scale, numOctaves, mask) -> the flat OCTAVE_KEYLINE_DTYPE array; detect([images], scale, numOctaves, masks) -> one
        per image (the fourth argument is then the list of masks)."""
        if isinstance(image, (list, tuple)):
            return self._detect_many(list(image), scale, numOctaves, masks if masks is not None else mask)
        octs = self.detect_octaves(image, scale, numOctaves, mask)
        return np.concatenate(octs) if octs else self._empty()

    def detect_octaves(self, image, scale, numOctaves, mask=None):
        """detect(image, vector<vector<KeyLine>>&, scale, numOctaves, opts, mask) -> one OCTAVE_KEYLINE_DTYPE array per octave"""
        numOctaves = int(numOctaves)
        self._check(image, mask, scale, numOctaves, "Mask error while detecting lines: please check its dimensions and that data type is CV_8UC1")
        octs = self._octaves_of([self._gray_or_bgr(image)], numOctaves)[0]
        return [self._apply_mask(o, mask) for o in octs]

    def _detect_many(self, images, scale, numOctaves, masks):
        numOctaves = int(numOctaves)
        masks = list(masks) if masks is not None else []
        ms = [masks[i] if i < len(masks) else None for i in range(len(images))]
        for img, m in zip(images, ms):
            self._check(img, m, scale, numOctaves, "Masks error while detecting lines: please check their dimensions and that data types are CV_8UC1")
        found = self._octaves_of([self._gray_or_bgr(x) for x in images], numOctaves)
        return [self._apply_mask(np.concatenate(o) if o else self._empty(), m) for o, m in zip(found, ms)]


class line_lbd_detect(object):
    def __init__(self, numoctaves=1, octaveratio=1.0, device=0, max_width=2048, max_height=2048, context=None):
        self.numoctaves_ = int(numoctaves)
        self.octaveratio_ = float(octaveratio)
        self.use_LSD = False            # line_lbd_allclass.cpp:121
        self.line_length_thres = 50.0   # :122
        self._ctx = context if context is not None else Context(device, max_width, max_height, 1, 1, 1)

    @property
    def bdm(self):
        """The class's BinaryDescriptorMatcher (line_lbd_allclass.h:37), on this detector's context: one object, created on first use as the
        reference creates it once in its constructor (:117), so that the images add() gives it stay for later queries."""
        if getattr(self, "_bdm", None) is None:
            self._bdm = BinaryDescriptorMatcher(self._ctx)
        return self._bdm

    @property
    def lsd(self):
        """The class's LSDDetector (line_lbd_allclass.h:40), on this detector's context: detect / detect_octaves over the pyrDown pyramid,
        with masks, and detect([images]) with one library call per image size."""
        if getattr(self, "_lsd", None) is None:
            self._lsd = LSDDetector(self._ctx)
        return self._lsd

    def params(self):
        p = _lib.LineParams()
        self._ctx.L.cs_default_line_params(C.byref(p))
        p.use_LSD = int(bool(self.use_LSD))
        p.numoctaves = self.numoctaves_
        p.octaveratio = self.octaveratio_
        p.line_length_thres = float(self.line_length_thres)
        return p

    def detect_filter_lines(self, gray_img, cap=8192):
        """One frame (H x W or H x W x 3 uint8) -> n x 4 float32."""
        return self.detect_filter_lines_batch(np.asarray(gray_img)[None], cap)[0]

    def detect_filter_lines_batch(self, imgs, cap=4096):
        imgs = np.ascontiguousarray(imgs, np.uint8)
        if imgs.ndim == 3:
            F, H, W = imgs.shape
            ch = 1
        else:
            F, H, W, ch = imgs.shape
        out = np.zeros((F, cap, 4), np.float32)
        n = np.zeros(F, np.int32)
        p = self.params()
        rc = self._ctx.L.cs_detect_lines_batch(self._ctx.h, imgs.ctypes.data, F, W, H, W * ch, ch, C.byref(p), _lib.ptr(out, C.c_float), cap,
                                               _lib.ptr(n, C.c_int32))
        if rc != 0:
            raise CubeSlamError("%s: %s" % (_lib.STATUS_NAMES.get(rc, rc), self._ctx.L.cs_last_error(self._ctx.h).decode()))
        return [out[f, :n[f]].copy() for f in range(F)]

    def detect_filter_lines_device(self, frames, order="bgr", cap=4096, stream=None):
        """detect_filter_lines_batch on frames already on the GPU: any object with __cuda_array_interface__ (a torch CUDA tensor, a CuPy array),
        uint8, (N, H, W, 3) or (N, H, W), any strides; order "bgr" or "rgb"; stream as Context.upload_device.  The frames go to the
        detector's own buffer, so a batch uploaded to the same context keeps its frames."""
        fr = _lib.device_frames(frames, order, stream)
        F = fr.n_frames
        out = np.zeros((F, cap, 4), np.float32)
        n = np.zeros(F, np.int32)
        p = self.params()
        self._ctx.check(self._ctx.L.cs_detect_lines_batch_device(self._ctx.h, C.byref(fr), C.byref(p), _lib.ptr(out, C.c_float), cap,
                                                                  _lib.ptr(n, C.c_int32)))
        return [out[f, :n[f]].copy() for f in range(F)]

    def detect_raw_lines(self, gray_img, downsample_img=False, cap=8192):
        """detect_raw_lines(gray_img, lines_mat, downsample_img) (line_lbd_allclass.cpp:174-189): every segment, no length filter -> n x 4
        float32; with downsample_img the image is halved first (cv::resize, as the reference does) and the lines scaled by 2.  One octave:
        the octave-0 segments.  More octaves (LSD flavour): the key lines of every octave, octave after octave, as keylines_to_mat writes
        them (start and end points in the input frame)."""
        octaves = self.numoctaves_ != 1
        if octaves and not self.use_LSD:
            raise CubeSlamError("detect_raw_lines with more than one octave is provided for the LSD flavour (use_LSD = True)")
        img = np.asarray(gray_img)
        if downsample_img:
            import cv2
            img = cv2.resize(img, None, fx=0.5, fy=0.5)
        if octaves:
            kl = np.concatenate(self.detect_raw_lines_octaves(img, cap))
            lines = np.stack([kl["start_x"], kl["start_y"], kl["end_x"], kl["end_y"]], 1).astype(np.float32).reshape(-1, 4)
            return lines * np.float32(2) if downsample_img else lines
        keep = self.line_length_thres
        try:
            self.line_length_thres = -1.0     # lineLength > -1: everything
            lines = self.detect_filter_lines(img, cap)
        finally:
            self.line_length_thres = keep
        return lines * np.float32(2) if downsample_img else lines

    # ---------------------------------------------------------------- every octave, LSD flavour (line_lbd_allclass.cpp:125-172,285-339)
    def _octave_params(self):
        """the detector's parameters for the octave calls; the refusals the reference makes (pyrDown's size rule) raise here"""
        if not self.use_LSD:
            raise CubeSlamError("the octave calls are provided for the LSD flavour (use_LSD = True)")
        if self.numoctaves_ > 1 and int(np.float32(self.octaveratio_)) != 2:
            raise CubeSlamError("numoctaves > 1 needs int(octaveratio) == 2 (got %g): cv::pyrDown makes an octave of (w / scale, h / scale) "
                                "only when |2 * dst - src| <= 2" % self.octaveratio_)
        return self.params()

    def _octave_lists(self, kl, desc, n, F):
        K = self.numoctaves_
        kls = [[kl[f, k, :n[f, k]].copy() for k in range(K)] for f in range(F)]
        if desc is None:
            return kls
        return [(kls[f], [desc[f, k, :n[f, k]].copy() for k in range(K)]) for f in range(F)]

    def _octaves_call(self, imgs, cap, describe):
        imgs, F, H, W, ch = self._frames(imgs)
        K = self.numoctaves_
        p = self._octave_params()
        kl = np.zeros((F, K, cap), _lib.OCTAVE_KEYLINE_DTYPE)
        desc = np.zeros((F, K, cap, 32), np.uint8) if describe else None
        n = np.zeros((F, K), np.int32)
        L = self._ctx.L
        if describe:
            self._ctx.check(L.cs_detect_descrip_lines_octaves_batch(self._ctx.h, imgs.ctypes.data, F, W, H, W * ch, ch, C.byref(p), kl.ctypes.data,
                                                                    _lib.ptr(desc, C.c_uint8), cap, _lib.ptr(n, C.c_int32)))
        else:
            self._ctx.check(L.cs_detect_raw_lines_octaves_batch(self._ctx.h, imgs.ctypes.data, F, W, H, W * ch, ch, C.byref(p), kl.ctypes.data, cap,
                                                                _lib.ptr(n, C.c_int32)))
        return self._octave_lists(kl, desc, n, F)

    def _octaves_device(self, frames, order, cap, stream, describe):
        fr = _lib.device_frames(frames, order, stream)
        F, K = fr.n_frames, self.numoctaves_
        p = self._octave_params()
        kl = np.zeros((F, K, cap), _lib.OCTAVE_KEYLINE_DTYPE)
        desc = np.zeros((F, K, cap, 32), np.uint8) if describe else None
        n = np.zeros((F, K), np.int32)
        L = self._ctx.L
        if describe:
            self._ctx.check(L.cs_detect_descrip_lines_octaves_batch_device(self._ctx.h, C.byref(fr), C.byref(p), kl.ctypes.data, _lib.ptr(desc, C.c_uint8),
                                                                           cap, _lib.ptr(n, C.c_int32)))
        else:
            self._ctx.check(L.cs_detect_raw_lines_octaves_batch_device(self._ctx.h, C.byref(fr), C.byref(p), kl.ctypes.data, cap, _lib.ptr(n, C.c_int32)))
        return self._octave_lists(kl, desc, n, F)

    def detect_raw_lines_octaves(self, gray_img, cap=8192):
        """detect_raw_lines(gray_img, vector<vector<KeyLine>>&) (line_lbd_allclass.cpp:149-172), LSD flavour: one array of
        _lib.OCTAVE_KEYLINE_DTYPE per octave -- every field of the reference's KeyLine (KeyLine::pt is the mid point of start and end).  The
        flat overload is the concatenation of the octaves.  Any numoctaves >= 1; more than one needs int(octaveratio) == 2."""
        return self.detect_raw_lines_octaves_batch(np.asarray(gray_img)[None], cap)[0]

    def detect_raw_lines_octaves_batch(self, imgs, cap=4096):
        """detect_raw_lines_octaves over frames of equal size -> per frame the list of octaves.  cap bounds the LSD segments of one octave."""
        return self._octaves_call(imgs, cap, False)

    def detect_raw_lines_octaves_device(self, frames, order="bgr", cap=4096, stream=None):
        """detect_raw_lines_octaves_batch on frames already on the GPU (frames, order, stream as detect_filter_lines_device)."""
        return self._octaves_device(frames, order, cap, stream, False)

    def debug_frame(self, frame=0, cap=8192):
        L = self._ctx.L
        wh = np.zeros(2, np.int32)
        self._ctx.check(L.cs_debug_lsd(self._ctx.h, frame, _lib.ptr(wh, C.c_int32), None, None, None, None, None, None, None, 0))
        W, H = int(wh[0]), int(wh[1])
        sc, mg, an = np.zeros((H, W)), np.zeros((H, W)), np.zeros((H, W))
        lst = np.zeros(W * H, np.int32)
        ll, nr = C.c_int32(), C.c_int32()
        raw = np.zeros((cap, 4), np.float32)
        self._ctx.check(L.cs_debug_lsd(self._ctx.h, frame, _lib.ptr(wh, C.c_int32), _lib.ptr(sc, C.c_double), _lib.ptr(mg, C.c_double),
                                       _lib.ptr(an, C.c_double), _lib.ptr(lst, C.c_int32), C.byref(ll), _lib.ptr(raw, C.c_float), C.byref(nr), cap))
        return dict(scaled=sc, modgrad=mg, angles=an, list=lst[:ll.value].copy(), raw_lines=raw[:nr.value].copy())

    def seed_loop_stats(self, n_frames):
        """Diagnostics of the last LSD run, kept for compatibility: (n_frames x 4 int32, all zero; redo flags, all 1 -- every frame
        goes through the one-warp-per-frame seed loop)."""
        st, redo = np.zeros((n_frames, 4), np.int32), np.zeros(n_frames, np.int32)
        self._ctx.check(self._ctx.L.cs_debug_lsd_stats(self._ctx.h, _lib.ptr(st, C.c_int32), _lib.ptr(redo, C.c_int32), n_frames))
        return st, redo

    def debug_frame_edlines(self, width, height, frame=0, cap=8192):
        """EDLineDetector's intermediate maps of one frame of the last use_LSD = False run (tests)."""
        L = self._ctx.L
        H, W = int(height), int(width)
        blur, dirm, edge = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
        dx, dy, g = np.zeros((H, W), np.int16), np.zeros((H, W), np.int16), np.zeros((H, W), np.int16)
        anchors = np.zeros(W * H // 5 + 1, np.int32)
        na, nr = C.c_int32(), C.c_int32()
        raw = np.zeros((cap, 4), np.float32)
        self._ctx.check(L.cs_debug_edlines(self._ctx.h, frame, _lib.ptr(blur, C.c_uint8), _lib.ptr(dx, C.c_int16), _lib.ptr(dy, C.c_int16),
                                           _lib.ptr(g, C.c_int16), _lib.ptr(dirm, C.c_uint8), _lib.ptr(anchors, C.c_int32), C.byref(na),
                                           _lib.ptr(edge, C.c_uint8), _lib.ptr(raw, C.c_float), C.byref(nr), cap))
        return dict(blur=blur, dx=dx, dy=dy, g=g, dir=dirm, anchors=anchors[:na.value].copy(), edge=edge, raw_lines=raw[:nr.value].copy())

    # ---------------------------------------------------------------- descriptors and matching (line_lbd_allclass.cpp:191-198,224-356)
    @staticmethod
    def _frames(imgs):
        imgs = np.ascontiguousarray(imgs, np.uint8)
        if imgs.ndim == 3:
            F, H, W = imgs.shape
            ch = 1
        else:
            F, H, W, ch = imgs.shape
        return imgs, F, H, W, ch

    def detect_descrip_lines_batch(self, imgs, cap=4096):
        """detect_descrip_lines(gray_img, keylines_out, line_descrips) (:253-272) over frames of equal size ->
        [(key lines, n x 32 uint8 descriptors)] per frame."""
        imgs, F, H, W, ch = self._frames(imgs)
        kl = np.zeros((F, cap), _lib.KEYLINE_DTYPE)
        desc = np.zeros((F, cap, 32), np.uint8)
        n = np.zeros(F, np.int32)
        p = self.params()
        self._ctx.check(self._ctx.L.cs_detect_descrip_lines_batch(self._ctx.h, imgs.ctypes.data, F, W, H, W * ch, ch, C.byref(p), kl.ctypes.data,
                                                                  _lib.ptr(desc, C.c_uint8), cap, _lib.ptr(n, C.c_int32)))
        return [(kl[f, :n[f]].copy(), desc[f, :n[f]].copy()) for f in range(F)]

    def detect_descrip_lines(self, gray_img, cap=8192, as_mat=False):
        """One frame -> (key lines, descriptors).  as_mat: the cv::Mat overload (:224-250) -- no length filter, lines as n x 4 float32."""
        if not as_mat:
            return self.detect_descrip_lines_batch(np.asarray(gray_img)[None], cap)[0]
        keep = self.line_length_thres
        try:
            self.line_length_thres = -1.0     # lineLength > -1: every octave-0 line, as the Mat overload keeps them
            kl, desc = self.detect_descrip_lines_batch(np.asarray(gray_img)[None], cap)[0]
        finally:
            self.line_length_thres = keep
        return self._mat_rows(kl), desc

    @staticmethod
    def _mat_rows(kl):
        """the Mat overload's lines: n x 4 float32 [start x, start y, end x, end y] of the key lines"""
        return np.stack([kl["start_x"], kl["start_y"], kl["end_x"], kl["end_y"]], 1).astype(np.float32).reshape(-1, 4)

    def detect_descrip_lines_device(self, frames, order="bgr", cap=4096, stream=None, as_mat=False):
        """detect_descrip_lines_batch on frames already on the GPU -> [(key lines, n x 32 uint8 descriptors)] per frame, the same values the
        host form returns for the same pixels.  frames, order and stream as detect_filter_lines_device: any object with
        __cuda_array_interface__, uint8, (N, H, W, 3) or (N, H, W), any strides.  as_mat: the cv::Mat overload of every frame, as
        detect_descrip_lines(..., as_mat=True) -- no length filter, lines as n x 4 float32."""
        fr = _lib.device_frames(frames, order, stream)
        F = fr.n_frames
        kl = np.zeros((F, cap), _lib.KEYLINE_DTYPE)
        desc = np.zeros((F, cap, 32), np.uint8)
        n = np.zeros(F, np.int32)
        p = self.params()
        if as_mat:
            p.line_length_thres = -1.0      # lineLength > -1: every octave-0 line, as the Mat overload keeps them
        self._ctx.check(self._ctx.L.cs_detect_descrip_lines_batch_device(self._ctx.h, C.byref(fr), C.byref(p), kl.ctypes.data,
                                                                         _lib.ptr(desc, C.c_uint8), cap, _lib.ptr(n, C.c_int32)))
        out = [(kl[f, :n[f]].copy(), desc[f, :n[f]].copy()) for f in range(F)]
        return [(self._mat_rows(k), d) for k, d in out] if as_mat else out

    def detect_descrip_lines_octaves(self, gray_img, cap=8192):
        """detect_descrip_lines_octaves (:285-339): the kept key lines with start x <= end x (ends swapped and the angle folded into
        [-pi/2, pi/2] where needed, :321-330) -> ([key lines], [descriptors]), one entry per octave.  One octave: records of
        _lib.KEYLINE_DTYPE.  More octaves (LSD flavour, int(octaveratio) == 2): records of _lib.OCTAVE_KEYLINE_DTYPE, every KeyLine field."""
        if self.numoctaves_ != 1:
            if not self.use_LSD:
                raise CubeSlamError("detect_descrip_lines_octaves with more than one octave is provided for the LSD flavour (use_LSD = True)")
            return self.detect_descrip_lines_octaves_batch(np.asarray(gray_img)[None], cap)[0]
        kl, desc = self.detect_descrip_lines(gray_img, cap)
        kl = kl.copy()
        PI = 3.14159265                     # line_lbd_allclass.cpp:19, a double: normalize_to_PI compares and folds in double (:272-281)
        sw = kl["start_x"] > kl["end_x"]
        sx, sy = kl["start_x"][sw].copy(), kl["start_y"][sw].copy()
        kl["start_x"][sw], kl["start_y"][sw] = kl["end_x"][sw], kl["end_y"][sw]
        kl["end_x"][sw], kl["end_y"][sw] = sx, sy
        a = kl["angle"][sw].astype(np.float64)
        kl["angle"][sw] = np.where(a > PI / 2, a - PI, np.where(a < -PI / 2, a + PI, a)).astype(np.float32)
        kl["class_id"] = np.arange(len(kl), dtype=np.int32)
        return [kl], [desc]

    def detect_descrip_lines_octaves_batch(self, imgs, cap=4096):
        """detect_descrip_lines_octaves of every octave (LSD flavour, any numoctaves >= 1) over frames of equal size -> per frame
        ([OCTAVE_KEYLINE_DTYPE records per octave], [n x 32 uint8 per octave])."""
        return self._octaves_call(imgs, cap, True)

    def detect_descrip_lines_octaves_device(self, frames, order="bgr", cap=4096, stream=None):
        """detect_descrip_lines_octaves_batch on frames already on the GPU (frames, order, stream as detect_filter_lines_device)."""
        return self._octaves_device(frames, order, cap, stream, True)

    def keylines_from_lines(self, lines, width, height):
        """KeyLine fields of n x 4 segment rows, as LSDDetector fills them (LSDDetector.cpp:226-250)."""
        lines = np.ascontiguousarray(lines, np.float32).reshape(-1, 4)
        kl = np.zeros(len(lines), _lib.KEYLINE_DTYPE)
        self._ctx.check(self._ctx.L.cs_keylines_from_lines(_lib.ptr(lines, C.c_float), len(lines), int(width), int(height), kl.ctypes.data))
        return kl

    def compute_descriptors(self, gray_img, keylines, want_float=False):
        """lbd->compute(gray_img, keylines, line_descrips): n x 32 uint8 (and the n x 72 float32 descriptor with want_float)."""
        imgs, F, H, W, ch = self._frames(np.asarray(gray_img)[None])
        kl = np.ascontiguousarray(keylines, _lib.KEYLINE_DTYPE)
        desc = np.zeros((len(kl), 32), np.uint8)
        fdesc = np.zeros((len(kl), 72), np.float32) if want_float else None
        self._ctx.check(self._ctx.L.cs_lbd_compute(self._ctx.h, imgs.ctypes.data, W, H, W * ch, ch, kl.ctypes.data, len(kl), _lib.ptr(desc, C.c_uint8),
                                                   _lib.ptr(fdesc, C.c_float) if want_float else None))
        return (desc, fdesc) if want_float else desc

    def compute_descriptors_device(self, frames, keylines_per_frame, want_float=False, order="bgr", stream=None):
        """lbd->compute on frames already on the GPU (frames, order, stream as detect_filter_lines_device), frame f with the key lines
        keylines_per_frame[f] (records of _lib.KEYLINE_DTYPE, any count including 0) -> per frame the n x 32 uint8 descriptors, or
        (n x 32 uint8, n x 72 float32) with want_float."""
        fr = _lib.device_frames(frames, order, stream)
        kls = [np.ascontiguousarray(k, _lib.KEYLINE_DTYPE).reshape(-1) for k in keylines_per_frame]
        if len(kls) != fr.n_frames:
            raise CubeSlamError("one key-line array per frame: %d for %d frames" % (len(kls), fr.n_frames))
        off = np.concatenate([[0], np.cumsum([len(k) for k in kls])]).astype(np.int32)
        n = int(off[-1])
        kl = np.ascontiguousarray(np.concatenate(kls)) if n else np.zeros(1, _lib.KEYLINE_DTYPE)
        desc = np.zeros((max(n, 1), 32), np.uint8)
        fdesc = np.zeros((max(n, 1), 72), np.float32) if want_float else None
        self._ctx.check(self._ctx.L.cs_lbd_compute_batch_device(self._ctx.h, C.byref(fr), kl.ctypes.data, _lib.ptr(off, C.c_int32),
                                                                _lib.ptr(desc, C.c_uint8), _lib.ptr(fdesc, C.c_float) if want_float else None))
        if want_float:
            return [(desc[off[f]:off[f + 1]].copy(), fdesc[off[f]:off[f + 1]].copy()) for f in range(fr.n_frames)]
        return [desc[off[f]:off[f + 1]].copy() for f in range(fr.n_frames)]

    def get_line_descriptors(self, gray_img, linesmat_src):
        """get_line_descriptors(gray_img, linesmat_src, line_descrips) (:191-198): descriptors of given n x 4 lines.  The reference builds
        the key lines with mat_to_keylines, which leaves class_id / octave unset (undefined there); the fields are filled here the way
        LSDDetector fills them for the same end points."""
        h, w = np.asarray(gray_img).shape[:2]
        return self.compute_descriptors(gray_img, self.keylines_from_lines(linesmat_src, w, h))

    def match_line_descrip(self, descrips_query, descrips_train, matching_dist_thres=25.0):
        """match_line_descrip (:341-356) -> records of DMATCH_DTYPE, query order."""
        q = np.ascontiguousarray(descrips_query, np.uint8).reshape(-1, 32)
        t = np.ascontiguousarray(descrips_train, np.uint8).reshape(-1, 32)
        out = np.zeros(max(len(q), 1), _lib.DMATCH_DTYPE)
        n = C.c_int32(0)
        self._ctx.check(self._ctx.L.cs_match_line_descrip(self._ctx.h, _lib.ptr(q, C.c_uint8), len(q), _lib.ptr(t, C.c_uint8), len(t),
                                                          C.c_float(matching_dist_thres), out.ctypes.data, C.byref(n)))
        return out[:n.value].copy()

    def match_line_descrip_batch(self, queries, trains, matching_dist_thres=25.0):
        """Several independent (query set, train set) pairs in one launch -> [records of DMATCH_DTYPE] per pair."""
        qs = [np.ascontiguousarray(q, np.uint8).reshape(-1, 32) for q in queries]
        ts = [np.ascontiguousarray(t, np.uint8).reshape(-1, 32) for t in trains]
        assert len(qs) == len(ts) and len(qs) > 0
        qo = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int32)
        to = np.concatenate([[0], np.cumsum([len(t) for t in ts])]).astype(np.int32)
        q = np.ascontiguousarray(np.concatenate(qs)) if qo[-1] else np.zeros((1, 32), np.uint8)
        t = np.ascontiguousarray(np.concatenate(ts)) if to[-1] else np.zeros((1, 32), np.uint8)
        out = np.zeros(max(int(qo[-1]), 1), _lib.DMATCH_DTYPE)
        n = np.zeros(len(qs), np.int32)
        self._ctx.check(self._ctx.L.cs_match_line_descrip_batch(self._ctx.h, _lib.ptr(q, C.c_uint8), _lib.ptr(qo, C.c_int32), _lib.ptr(t, C.c_uint8),
                                                                _lib.ptr(to, C.c_int32), len(qs), C.c_float(matching_dist_thres), out.ctypes.data,
                                                                _lib.ptr(n, C.c_int32)))
        return [out[qo[p]:qo[p] + n[p]].copy() for p in range(len(qs))]
