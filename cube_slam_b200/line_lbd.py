"""Host-side mirror of `class line_lbd_detect` (line_lbd/include/line_lbd/line_lbd_allclass.h:22-70).

detect_filter_lines(img) -> n x 4 float32 [x1 y1 x2 y2]: what the reference writes into its `cv::Mat& linesmat_out`
(line_lbd/class/line_lbd_allclass.cpp:216-221).  The descriptor / matcher methods (get_line_descriptors, detect_descrip_lines,
detect_descrip_lines_octaves, match_line_descrip; :191-198,224-356) return numpy arrays: key lines as records of `_lib.KEYLINE_DTYPE`
(the KeyLine fields, octave 0), descriptors as n x 32 uint8 (the CV_8UC1 matrix), matches as records of `_lib.DMATCH_DTYPE` (cv::DMatch).
`line_lbd_detect.bdm` is the class's BinaryDescriptorMatcher (line_lbd_allclass.h:37): pairwise match, knnMatch and radiusMatch on the GPU."""
import ctypes as C
import math

import numpy as np

from . import _lib
from .detect_3d_cuboid import Context, CubeSlamError


def _codes(d):
    return np.ascontiguousarray(d, np.uint8).reshape(-1, 32)


class BinaryDescriptorMatcher(object):
    """Mirror of cv::line_descriptor::BinaryDescriptorMatcher, the pairwise forms (binary_descriptor_matcher.cpp:196-341, 431-507), on the
    device of `context`.  Descriptors are n x 32 uint8; a list of matches is a records array of `_lib.DMATCH_DTYPE`, a vector<vector<DMatch>>
    a Python list of them, one per query.  mask: one value per query (0 = skip it), its length must be the number of queries.  Where the
    reference is undefined the library's definitions hold (include/cube_slam_b200.h): fewer than k entries when fewer codes are met,
    train_idx -1 beyond 128 bits, [] for an empty query or train set.  At most 16384 train codes per pair (CubeSlamError beyond)."""

    def __init__(self, context):
        self._ctx = context

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

    def match(self, queryDescriptors, trainDescriptors, mask=None):
        """match(query, train, matches, mask): the nearest code of every (unmasked) query -> DMATCH_DTYPE records, query order."""
        q, t = _codes(queryDescriptors), _codes(trainDescriptors)
        m = self._mask(mask, len(q))
        out = np.zeros(max(len(q), 1), _lib.DMATCH_DTYPE)
        n = C.c_int32(0)
        self._ctx.check(self._ctx.L.cs_match_line_descrip(self._ctx.h, _lib.ptr(q, C.c_uint8), len(q), _lib.ptr(t, C.c_uint8), len(t), C.c_float(math.inf),
                                                          out.ctypes.data, C.byref(n)))
        out = out[:n.value].copy()
        return out if m is None else out[m[out["query_idx"]] != 0]

    def knnMatch(self, queryDescriptors, trainDescriptors, k, mask=None, compactResult=False):
        """knnMatch(query, train, matches, k, mask, compactResult): per query its first k codes; a masked query gives an empty list, or
        none with compactResult."""
        return self.knnMatch_batch([queryDescriptors], [trainDescriptors], k, None if mask is None else [mask], compactResult)[0]

    def radiusMatch(self, queryDescriptors, trainDescriptors, maxDistance, mask=None, compactResult=False):
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


class line_lbd_detect(object):
    def __init__(self, numoctaves=1, octaveratio=1.0, device=0, max_width=2048, max_height=2048, context=None):
        self.numoctaves_ = int(numoctaves)
        self.octaveratio_ = float(octaveratio)
        self.use_LSD = False            # line_lbd_allclass.cpp:121
        self.line_length_thres = 50.0   # :122
        self._ctx = context if context is not None else Context(device, max_width, max_height, 1, 1, 1)

    @property
    def bdm(self):
        """The class's BinaryDescriptorMatcher (line_lbd_allclass.h:37, created at :117), on this detector's context."""
        return BinaryDescriptorMatcher(self._ctx)

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
        """detect_raw_lines(gray_img, lines_mat, downsample_img) (line_lbd_allclass.cpp:174-189): every octave-0 segment, no length filter ->
        n x 4 float32; with downsample_img the image is halved first (cv::resize, as the reference does) and the lines scaled by 2."""
        if self.numoctaves_ != 1:
            raise CubeSlamError("detect_raw_lines returns octave 0 only: build the detector with one octave")
        img = np.asarray(gray_img)
        if downsample_img:
            import cv2
            img = cv2.resize(img, None, fx=0.5, fy=0.5)
        keep = self.line_length_thres
        try:
            self.line_length_thres = -1.0     # lineLength > -1: everything
            lines = self.detect_filter_lines(img, cap)
        finally:
            self.line_length_thres = keep
        return lines * np.float32(2) if downsample_img else lines

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
        return np.stack([kl["start_x"], kl["start_y"], kl["end_x"], kl["end_y"]], 1).astype(np.float32).reshape(-1, 4), desc

    def detect_descrip_lines_octaves(self, gray_img, cap=8192):
        """detect_descrip_lines_octaves (:285-339) for the one octave the class is built with: the kept key lines with start x <= end x
        (ends swapped and the angle folded into [-pi/2, pi/2] where needed, :321-330) -> ([key lines], [descriptors]), one entry per octave."""
        if self.numoctaves_ != 1:
            raise CubeSlamError("detect_descrip_lines_octaves is provided for one octave (the library detects octave 0)")
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
