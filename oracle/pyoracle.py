"""ctypes binding of the CPU ORACLE (oracle/_build/liboracle.so).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may import
this module; the product package cube_slam_b200 never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")


def build(force=False):
    """Compile the oracle with the committed Makefile (g++ -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cpp", ".h"))]
    fresh = os.path.exists(_LIB_PATH) and all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in srcs)
    # oracle/_ref (the reference's own lsd.cpp) is built where the reference checkout exists; elsewhere the prebuilt file is used as it is
    ref_src = "/root/reference/line_lbd/libs/lsd.cpp"
    ref_libs = [os.path.join(_HERE, "_ref", n) for n in ("liblsd_ref.so", "libedl_ref.so", "liblinelbd_ref.so", "libcuboid_ref.so")]
    if os.path.exists(ref_src):
        deps = [ref_src, _LIB_PATH] + [os.path.join(_HERE, "ref", f) for f in os.listdir(os.path.join(_HERE, "ref")) if f.endswith((".cpp", ".hpp"))]
        fresh = fresh and all(os.path.exists(r) and all(os.path.getmtime(r) >= os.path.getmtime(d) for d in deps) for r in ref_libs)
    if not force and fresh:
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB_PATH


class Params(C.Structure):
    _fields_ = [
        ("consider_config_1", C.c_int), ("consider_config_2", C.c_int),
        ("whether_sample_cam_roll_pitch", C.c_int), ("whether_sample_bbox_height", C.c_int),
        ("max_cuboid_num", C.c_int),
        ("nominal_skew_ratio", C.c_double), ("max_cut_skew", C.c_double),
        ("vp12_edge_angle_thre", C.c_double), ("vp3_edge_angle_thre", C.c_double),
        ("shorted_edge_thre", C.c_double), ("reweight_edge_distance", C.c_int),
        ("whether_normalize_two_errors", C.c_int),
        ("weight_vp_angle", C.c_double), ("weight_skew_error", C.c_double),
        ("pre_merge_dist_thre", C.c_double), ("pre_merge_angle_thre", C.c_double),
        ("edge_length_threshold", C.c_double),
        ("canny_low", C.c_double), ("canny_high", C.c_double),
        ("yaw_half_range_deg", C.c_double), ("yaw_step_deg", C.c_double),
        ("top_sample_count_override", C.c_int),
    ]


class Cuboid(C.Structure):
    _fields_ = [
        ("pos", C.c_double * 3), ("scale", C.c_double * 3), ("rotY", C.c_double),
        ("box_config_type", C.c_double * 2),
        ("box_corners_2d", C.c_int32 * 16),
        ("box_corners_3d_world", C.c_double * 24),
        ("rect_detect_2d", C.c_double * 4),
        ("edge_distance_error", C.c_double), ("edge_angle_error", C.c_double),
        ("normalized_error", C.c_double), ("skew_ratio", C.c_double),
        ("down_expand_height", C.c_double),
        ("camera_roll_delta", C.c_double), ("camera_pitch_delta", C.c_double),
        ("combined_score", C.c_double),
        ("proposal_index", C.c_int32), ("height_sample_id", C.c_int32),
        ("valid", C.c_int32), ("pad_", C.c_int32),
    ]


CUBOID_DTYPE = np.dtype([
    ("pos", "f8", 3), ("scale", "f8", 3), ("rotY", "f8"), ("box_config_type", "f8", 2),
    ("box_corners_2d", "i4", (2, 8)), ("box_corners_3d_world", "f8", (3, 8)),
    ("rect_detect_2d", "f8", 4), ("edge_distance_error", "f8"), ("edge_angle_error", "f8"),
    ("normalized_error", "f8"), ("skew_ratio", "f8"), ("down_expand_height", "f8"),
    ("camera_roll_delta", "f8"), ("camera_pitch_delta", "f8"), ("combined_score", "f8"),
    ("proposal_index", "i4"), ("height_sample_id", "i4"), ("valid", "i4"), ("pad_", "i4"),
])
assert CUBOID_DTYPE.itemsize == C.sizeof(Cuboid)


class Trace(C.Structure):
    _fields_ = [
        ("want_object", C.c_int), ("want_height_sample", C.c_int),
        ("roi", C.c_int * 4), ("n_lines_roi", C.c_int), ("n_lines_merged", C.c_int),
        ("merged_lines", C.POINTER(C.c_double)), ("cap_lines", C.c_int),
        ("canny", C.POINTER(C.c_uint8)), ("dist", C.POINTER(C.c_float)), ("cap_px", C.c_int),
        ("n_candidates", C.c_int), ("n_valid", C.c_int),
        ("rows", C.POINTER(C.c_double)), ("corners", C.POINTER(C.c_double)),
        ("cand_index", C.POINTER(C.c_int32)), ("cap_valid", C.c_int),
        ("n_kept", C.c_int), ("kept_ids", C.POINTER(C.c_int32)), ("kept_scores", C.POINTER(C.c_double)),
    ]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_default_params.argtypes = [C.POINTER(Params)]
        _lib.orc_detect_cuboid.restype = C.c_int
        _lib.orc_merge_break_lines.restype = C.c_int
        for name in ("lsd_orc_detect", "edl_orc_detect"):
            if hasattr(_lib, name):
                getattr(_lib, name).restype = C.c_int
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def default_params(**kw):
    p = Params()
    lib().orc_default_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def bgr2gray(bgr, fixed15=True):
    bgr = np.ascontiguousarray(bgr, np.uint8)
    h, w = bgr.shape[:2]
    out = np.empty((h, w), np.uint8)
    lib().orc_bgr2gray(_p(bgr, C.c_uint8), w, h, w * 3, _p(out, C.c_uint8), w, int(fixed15))
    return out


def canny(gray, low=80.0, high=200.0):
    gray = np.ascontiguousarray(gray, np.uint8)
    h, w = gray.shape
    out = np.empty((h, w), np.uint8)
    lib().orc_canny(_p(gray, C.c_uint8), w, h, w, C.c_double(low), C.c_double(high), _p(out, C.c_uint8))
    return out


def chamfer_dt(edges):
    edges = np.ascontiguousarray(edges, np.uint8)
    h, w = edges.shape
    out = np.empty((h, w), np.float32)
    lib().orc_chamfer_dt(_p(edges, C.c_uint8), w, h, _p(out, C.c_float))
    return out


def merge_break_lines(lines, dist_thre=20.0, angle_thre_deg=5.0, len_thre=30.0):
    lines = np.ascontiguousarray(lines, np.float64).reshape(-1, 4)
    out = np.empty_like(lines)
    n = lib().orc_merge_break_lines(_p(lines, C.c_double), len(lines), C.c_double(dist_thre),
                                    C.c_double(angle_thre_deg), C.c_double(len_thre), _p(out, C.c_double))
    return out[:n].copy()


def _vp_support(L, name, vps, mids, angles, thre12_deg, thre3_deg):
    vps = np.ascontiguousarray(vps, np.float64).reshape(3, 2)
    mids = np.ascontiguousarray(mids, np.float64).reshape(-1, 2)
    angles = np.ascontiguousarray(angles, np.float64).reshape(-1)
    out = np.zeros((3, 2))
    getattr(L, name)(_p(vps, C.c_double), _p(mids, C.c_double), _p(angles, C.c_double), len(angles), C.c_double(thre12_deg),
                     C.c_double(thre3_deg), _p(out, C.c_double))
    return out


def _box_edge_sum_dists(L, name, dist, corners, edges, reweight):
    dist = np.ascontiguousarray(dist, np.float32)
    corners = np.ascontiguousarray(corners, np.float64).reshape(2, 8)
    edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
    f = getattr(L, name)
    f.restype = C.c_double
    return f(_p(dist, C.c_float), dist.shape[1], dist.shape[0], _p(corners, C.c_double), _p(edges, C.c_int32), len(edges), int(bool(reweight)))


def _fuse_normalize(L, name, dist_err, angle_err, weight_vp_angle, normalize):
    d = np.ascontiguousarray(dist_err, np.float64)
    a = np.ascontiguousarray(angle_err, np.float64)
    comb = np.zeros(max(len(d), 1))
    keep = np.zeros(max(len(d), 1), np.int32)
    f = getattr(L, name)
    f.restype = C.c_int
    m = f(_p(d, C.c_double), _p(a, C.c_double), len(d), C.c_double(weight_vp_angle), int(bool(normalize)), _p(comb, C.c_double), _p(keep, C.c_int32))
    return keep[:m].copy(), comb[:m].copy()


def _linespace(L, name, start, end, step, cap=1024):
    out = np.zeros(cap)
    f = getattr(L, name)
    f.restype = C.c_int
    n = f(C.c_double(start), C.c_double(end), C.c_double(step), _p(out, C.c_double), cap)
    return out[:min(n, cap)].copy()


def vp_support_edge_infos(vps, mids, angles, thre12_deg=15.0, thre3_deg=10.0):
    """VP_support_edge_infos (object_3d_util.cpp:380-425): 3 x 2 bounding edge angles per vanishing point, NaN where none supports it."""
    return _vp_support(lib(), "orc_vp_support_edge_infos", vps, mids, angles, thre12_deg, thre3_deg)


def box_edge_sum_dists(dist, corners, edges, reweight=True):
    """box_edge_sum_dists (object_3d_util.cpp:427-453) on a float32 distance map; corners 2 x 8, edges n x 2 corner ids."""
    return _box_edge_sum_dists(lib(), "orc_box_edge_sum_dists", dist, corners, edges, reweight)


def fuse_normalize_scores_v2(dist_err, angle_err, weight_vp_angle=0.8, normalize=True):
    """fuse_normalize_scores_v2 (object_3d_util.cpp:495-565) -> (kept indices, their combined scores)."""
    return _fuse_normalize(lib(), "orc_fuse_normalize_scores_v2", dist_err, angle_err, weight_vp_angle, normalize)


def linespace(start, end, step, cap=1024):
    """linespace<double> (matrix_utils.cpp:350-363): the samples (the loop stops after 1001)."""
    return _linespace(lib(), "orc_linespace_d", start, end, step, cap)


def cam_pose(K, T):
    K = np.ascontiguousarray(K, np.float64)
    T = np.ascontiguousarray(T, np.float64)
    out = np.empty(13)
    lib().orc_cam_pose(_p(K, C.c_double), _p(T, C.c_double), _p(out, C.c_double))
    return {"euler": out[:3].copy(), "KinvR": out[3:12].reshape(3, 3).copy(), "yaw": out[12]}


def detect_cuboid(img, K, T_wc, boxes, lines, params=None, topk_cap=None, trace_object=None,
                  trace_height_sample=0, trace_caps=(4096, 1 << 21, 1 << 16), cut_flip=-1):
    """detect_3d_cuboid::detect_cuboid for one frame (box_proposal_detail.cpp:56-557).

    Returns dict(cuboids=[structured array per bbox], n_candidates, n_valid, trace=dict|None)."""
    L = lib()
    if params is None:
        params = default_params()
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    K = np.ascontiguousarray(K, np.float64).reshape(3, 3)
    T_wc = np.ascontiguousarray(T_wc, np.float64).reshape(4, 4)
    boxes = np.ascontiguousarray(boxes, np.float64).reshape(-1, 5)
    lines = np.ascontiguousarray(lines, np.float64).reshape(-1, 4)
    N = len(boxes)
    if topk_cap is None:
        topk_cap = max(int(params.max_cuboid_num), 1)
    out = np.zeros((max(N, 1), topk_cap), CUBOID_DTYPE)
    counts = np.zeros(max(N, 1), np.int32)
    ncand = C.c_int64(0)
    nvalid = C.c_int64(0)
    tr = None
    bufs = None
    if trace_object is not None:
        cap_lines, cap_px, cap_valid = trace_caps
        bufs = dict(
            merged_lines=np.zeros((cap_lines, 4)), canny=np.zeros(cap_px, np.uint8), dist=np.zeros(cap_px, np.float32),
            rows=np.zeros((cap_valid, 9)), corners=np.zeros((cap_valid, 16)), cand_index=np.zeros(cap_valid, np.int32),
            kept_ids=np.zeros(cap_valid, np.int32), kept_scores=np.zeros(cap_valid))
        tr = Trace()
        tr.want_object = trace_object
        tr.want_height_sample = trace_height_sample
        tr.merged_lines = _p(bufs["merged_lines"], C.c_double)
        tr.cap_lines = cap_lines
        tr.canny = _p(bufs["canny"], C.c_uint8)
        tr.dist = _p(bufs["dist"], C.c_float)
        tr.cap_px = cap_px
        tr.rows = _p(bufs["rows"], C.c_double)
        tr.corners = _p(bufs["corners"], C.c_double)
        tr.cand_index = _p(bufs["cand_index"], C.c_int32)
        tr.cap_valid = cap_valid
        tr.kept_ids = _p(bufs["kept_ids"], C.c_int32)
        tr.kept_scores = _p(bufs["kept_scores"], C.c_double)
    L.orc_last_cut_margin.restype = C.c_double
    L.orc_last_cut_margin.argtypes = [C.c_int]
    L.orc_set_cut_flip(int(cut_flip))
    try:
        rc = L.orc_detect_cuboid(_p(img, C.c_uint8), w, h, img.strides[0], ch, _p(K, C.c_double), _p(T_wc, C.c_double),
                                 _p(boxes, C.c_double), N, _p(lines, C.c_double), len(lines), C.byref(params), topk_cap,
                                 out.ctypes.data_as(C.POINTER(Cuboid)), _p(counts, C.c_int),
                                 C.byref(ncand), C.byref(nvalid), C.byref(tr) if tr is not None else None)
        cut_margin = [float(L.orc_last_cut_margin(b)) for b in range(min(N, 64))]
    finally:
        L.orc_set_cut_flip(-1)
    if rc != 0:
        raise RuntimeError("orc_detect_cuboid failed: %d" % rc)
    # cut_margin[b]: how close fuse_normalize_scores_v2's `angle_error(cut) > angle_error(cut - 1)` came to a tie for box b (relative gap;
    # 1e300 when the comparison never ran).  cut_flip=b takes the other branch for box b where the gap is < 1e-13.
    res = {"cuboids": [out[i, :counts[i]].copy() for i in range(N)], "n_candidates": ncand.value,
           "n_valid": nvalid.value, "trace": None, "cut_margin": cut_margin}
    if tr is not None:
        rw, rh = tr.roi[2], tr.roi[3]
        npx = max(rw, 0) * max(rh, 0)
        res["trace"] = dict(
            roi=tuple(tr.roi), n_lines_roi=tr.n_lines_roi, n_lines_merged=tr.n_lines_merged,
            merged_lines=bufs["merged_lines"][:tr.n_lines_merged].copy(),
            canny=bufs["canny"][:npx].reshape(rh, rw).copy() if npx <= trace_caps[1] else None,
            dist=bufs["dist"][:npx].reshape(rh, rw).copy() if npx <= trace_caps[1] else None,
            n_candidates=tr.n_candidates, n_valid=tr.n_valid,
            rows=bufs["rows"][:tr.n_valid].copy(), corners=bufs["corners"][:tr.n_valid].copy(),
            cand_index=bufs["cand_index"][:tr.n_valid].copy(),
            n_kept=tr.n_kept, kept_ids=bufs["kept_ids"][:tr.n_kept].copy(), kept_scores=bufs["kept_scores"][:tr.n_kept].copy())
    return res


# ------------------------------------------------------------------------------------------- LSD
def lsd_fast_atan2(y, x):
    L = lib()
    L.lsd_orc_fast_atan2.restype = C.c_float
    L.lsd_orc_fast_atan2.argtypes = [C.c_float, C.c_float]
    return L.lsd_orc_fast_atan2(y, x)


def lsd_blur_resize(img64):
    """GaussianBlur(7x7, 0.75) then resize(x0.8, INTER_LINEAR) on a float64 image (lsd.cpp:450-459)."""
    src = np.ascontiguousarray(img64, np.float64)
    h, w = src.shape
    blur = np.empty_like(src)
    dw, dh = C.c_int(), C.c_int()
    scaled = np.empty((int(round(h * 0.8)) + 2) * (int(round(w * 0.8)) + 2), np.float64)
    lib().lsd_orc_blur_resize(_p(src, C.c_double), w, h, _p(blur, C.c_double), _p(scaled, C.c_double), C.byref(dw), C.byref(dh))
    return blur, scaled[:dw.value * dh.value].reshape(dh.value, dw.value).copy()


def lsd_detect(img, line_length_thres=15.0, cap=8192, want_stages=False, refine_mode=2):
    """line_lbd_detect::detect_filter_lines with use_LSD = true (line_lbd_allclass.cpp:216-221) -> n x 4 float32."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros((cap, 4), np.float32)
    raw = np.zeros((cap, 4), np.float32)
    n_raw = C.c_int(0)
    sw, sh = int(round(w * 0.8)), int(round(h * 0.8))
    st = None
    args = [None, None, None, None, None]
    if want_stages:
        st = dict(scaled=np.zeros((sh, sw)), modgrad=np.zeros((sh, sw)), angles=np.zeros((sh, sw)), list=np.zeros(sw * sh, np.int32))
        ll = C.c_int(0)
        args = [_p(st["scaled"], C.c_double), _p(st["modgrad"], C.c_double), _p(st["angles"], C.c_double), _p(st["list"], C.c_int32), C.byref(ll)]
    n = lib().lsd_orc_detect(_p(img, C.c_uint8), w, h, img.strides[0], ch, C.c_float(line_length_thres), _p(out, C.c_float), cap,
                             _p(raw, C.c_float), cap, C.byref(n_raw), *args, int(refine_mode))
    res = dict(lines=out[:min(n, cap)].copy(), raw_lines=raw[:min(n_raw.value, cap)].copy())
    if want_stages:
        st["list"] = st["list"][:ll.value].copy()
        res["stages"] = st
    return res


LSD_STAT_NAMES = ("seeds", "first_sum", "n_all_spill", "regrow_past", "reduce_past", "first_max", "n_all_max",
                  "first_2047", "first_2048", "first_2049", "n_all_2047", "n_all_2048", "n_all_2049", "nfa_max_n", "nfa_past_table")


def lsd_stats(img, cap=16384):
    """lsd_detect's raw segments and what the call did, in the GPU seed loop's terms (oracle/lsd_oracle.cpp, lsd_orc_detect_stats): seeds grown,
    the sum of first-pass region sizes, seeds whose region list (n_all = first pass + refine's re-grow) is longer than the 2 048 entries the
    seed loop keeps in shared memory, re-grows that start at or past entry 2 048, reduce-radius iterations on a list longer than 2 048, the
    largest first pass and n_all, how many first passes / n_all were exactly 2 047, 2 048, 2 049, the largest NFA n and the NFA calls that take
    log_gamma at an argument past the device's 16 384-entry table.  -> (raw n x 4 float32, dict)"""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros((cap, 4), np.float32)
    raw = np.zeros((cap, 4), np.float32)
    n_raw = C.c_int(0)
    st = np.zeros(len(LSD_STAT_NAMES), np.int64)
    L = lib()
    L.lsd_orc_detect_stats.restype = C.c_int
    L.lsd_orc_detect_stats(_p(img, C.c_uint8), w, h, img.strides[0], ch, C.c_float(15.0), _p(out, C.c_float), cap, _p(raw, C.c_float), cap,
                           C.byref(n_raw), 2, _p(st, C.c_int64))
    return raw[:min(n_raw.value, cap)].copy(), {k: int(v) for k, v in zip(LSD_STAT_NAMES, st)}


def lsd_nfa(n, k, p, logNT, lsd_first_term=True):
    """The reference's nfa(n, k, p) (lsd.cpp's (n + 1) first term, or descriptor.hpp's log_gamma(n + 1)) -> (value, i at which the tail loop
    stopped: n + 1 when it ran to the end, -1 for the early returns and the underflow branch)"""
    L = lib()
    L.orc_lsd_nfa.restype = C.c_double
    L.orc_lsd_nfa.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(C.c_int)]
    b = C.c_int(0)
    v = L.orc_lsd_nfa(int(n), int(k), float(p), float(logNT), int(bool(lsd_first_term)), C.byref(b))
    return v, b.value


def lsd_nfa_many(n, k, p, logNT, lsd_first_term=True):
    """lsd_nfa over arrays (one logNT and form for all) -> (values float64, break indices int32)"""
    n = np.ascontiguousarray(n, np.int32)
    k = np.ascontiguousarray(k, np.int32)
    p = np.ascontiguousarray(np.broadcast_to(p, n.shape), np.float64)
    out = np.zeros(len(n))
    brk = np.zeros(len(n), np.int32)
    lib().orc_lsd_nfa_many(_p(n, C.c_int32), _p(k, C.c_int32), _p(p, C.c_double), len(n), C.c_double(logNT), int(bool(lsd_first_term)),
                           _p(out, C.c_double), _p(brk, C.c_int32))
    return out, brk


_REF_LSD = None
_REF_LSD_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "liblsd_ref.so")


def ref_lsd_available():
    return os.path.exists(_REF_LSD_PATH)


def ref_lsd_detect(img, cap=8192):
    """The reference's OWN LSD (line_lbd/libs/lsd.cpp compiled from /root/reference into oracle/_ref/liblsd_ref.so, see oracle/ref/):
    createLineSegmentDetector(LSD_REFINE_ADV)->detect(gray) as LSDDetector::detectImpl calls it for octave 0 -> n x 4 float32, the raw
    segments before the key-line filter.  BGR input is converted with the oracle's cvtColor restatement (pinned to cv2)."""
    global _REF_LSD
    lib()  # liblsd_ref.so resolves the three OpenCV primitives from liboracle.so
    if _REF_LSD is None:
        _REF_LSD = C.CDLL(_REF_LSD_PATH)
        _REF_LSD.ref_lsd_detect.restype = C.c_int
    img = np.ascontiguousarray(img, np.uint8)
    gray = img if img.ndim == 2 else np.ascontiguousarray(bgr2gray(img))
    out = np.zeros((cap, 4), np.float32)
    n = _REF_LSD.ref_lsd_detect(_p(gray, C.c_uint8), gray.shape[1], gray.shape[0], _p(out, C.c_float), cap)
    if n < 0:
        raise RuntimeError("ref_lsd_detect failed")
    return out[:min(n, cap)].copy()


_REF_EDL = None
_REF_EDL_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libedl_ref.so")


def ref_edl_available():
    return os.path.exists(_REF_EDL_PATH)


def ref_edl_detect(img, cap=8192):
    """The reference's OWN EDLines detector (line_lbd/libs/binary_descriptor.cpp compiled from /root/reference into
    oracle/_ref/libedl_ref.so, see oracle/ref/edl_ref.cpp): BinaryDescriptor::detect with one octave, as line_lbd_detect::detect_raw_lines
    drives it for use_LSD = false -> n x 4 float32 key-line end points, before detect_filter_lines' length filter."""
    global _REF_EDL
    lib()
    if _REF_EDL is None:
        _REF_EDL = C.CDLL(_REF_EDL_PATH)
        _REF_EDL.ref_edl_detect.restype = C.c_int
    img = np.ascontiguousarray(img, np.uint8)
    gray = img if img.ndim == 2 else np.ascontiguousarray(bgr2gray(img))
    out = np.zeros((cap, 4), np.float32)
    n = _REF_EDL.ref_edl_detect(_p(gray, C.c_uint8), gray.shape[1], gray.shape[0], _p(out, C.c_float), cap)
    if n < 0:
        raise RuntimeError("ref_edl_detect failed")
    return out[:min(n, cap)].copy()


_REF_ALL = None
_REF_ALL_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "liblinelbd_ref.so")


def ref_detect_filter_lines_available():
    return os.path.exists(_REF_ALL_PATH)


def ref_detect_filter_lines(img, use_LSD=True, line_length_thres=50.0, cap=8192):
    """The reference's OWN line_lbd_detect::detect_filter_lines(image, lines_mat), whole (oracle/_ref/liblinelbd_ref.so: lsd.cpp,
    LSDDetector.cpp, binary_descriptor.cpp and line_lbd_allclass.cpp compiled from /root/reference, see oracle/ref/linelbd_ref.cpp), called
    as object_slam/src/main_obj.cpp:363-366,428 calls it -> the n x 4 CV_32F matrix as float32.  img: gray or BGR."""
    global _REF_ALL
    lib()
    if _REF_ALL is None:
        _REF_ALL = C.CDLL(_REF_ALL_PATH)
        _REF_ALL.ref_detect_filter_lines.restype = C.c_int
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros((cap, 4), np.float32)
    n = _REF_ALL.ref_detect_filter_lines(_p(img, C.c_uint8), w, h, ch, int(bool(use_LSD)), C.c_float(line_length_thres), _p(out, C.c_float), cap)
    if n < 0:
        raise RuntimeError("ref_detect_filter_lines failed (%d)" % n)
    return out[:min(n, cap)].copy()


_REF_CUB = None
_REF_CUB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libcuboid_ref.so")
REF_CUBOID_DTYPE = np.dtype([
    ("pos", "f8", 3), ("rotY", "f8"), ("scale", "f8", 3), ("box_config_type", "f8", 2), ("box_corners_2d", "f8", (2, 8)),
    ("box_corners_3d_world", "f8", (3, 8)), ("rect_detect_2d", "f8", 4), ("edge_distance_error", "f8"), ("edge_angle_error", "f8"),
    ("normalized_error", "f8"), ("skew_ratio", "f8"), ("down_expand_height", "f8"), ("camera_roll_delta", "f8"), ("camera_pitch_delta", "f8")])
assert REF_CUBOID_DTYPE.itemsize == 60 * 8


def ref_detect_cuboid_available():
    return os.path.exists(_REF_CUB_PATH)


def _ref_cub():
    global _REF_CUB
    lib()
    if _REF_CUB is None:
        _REF_CUB = C.CDLL(_REF_CUB_PATH)
        _REF_CUB.ref_detect_cuboid_skew.restype = C.c_int
        _REF_CUB.ref_merge_break_lines.restype = C.c_int
    return _REF_CUB


def ref_merge_break_lines(lines, dist_thre=20.0, angle_thre_deg=5.0, len_thre=30.0):
    """The reference's OWN merge_break_lines (object_3d_util.cpp:300)."""
    lines = np.ascontiguousarray(lines, np.float64).reshape(-1, 4)
    out = np.empty((max(len(lines), 1), 4))
    n = _ref_cub().ref_merge_break_lines(_p(lines, C.c_double), len(lines), C.c_double(dist_thre), C.c_double(angle_thre_deg),
                                         C.c_double(len_thre), _p(out, C.c_double))
    return out[:n].copy()


def ref_vp_support_edge_infos(vps, mids, angles, thre12_deg=15.0, thre3_deg=10.0):
    """The reference's OWN VP_support_edge_infos (object_3d_util.cpp:380)."""
    return _vp_support(_ref_cub(), "ref_vp_support_edge_infos", vps, mids, angles, thre12_deg, thre3_deg)


def ref_box_edge_sum_dists(dist, corners, edges, reweight=True):
    """The reference's OWN box_edge_sum_dists (object_3d_util.cpp:427)."""
    return _box_edge_sum_dists(_ref_cub(), "ref_box_edge_sum_dists", dist, corners, edges, reweight)


def ref_fuse_normalize_scores_v2(dist_err, angle_err, weight_vp_angle=0.8, normalize=True):
    """The reference's OWN fuse_normalize_scores_v2 (object_3d_util.cpp:495)."""
    return _fuse_normalize(_ref_cub(), "ref_fuse_normalize_scores_v2", dist_err, angle_err, weight_vp_angle, normalize)


def ref_linespace(start, end, step, cap=1024):
    """The reference's OWN linespace<double> (matrix_utils.cpp:350)."""
    return _linespace(_ref_cub(), "ref_linespace_d", start, end, step, cap)


def ref_detect_cuboid(img, K, T_wc, boxes, lines, params=None, cap_per_box=8):
    """The reference's OWN detect_3d_cuboid::detect_cuboid (detect_3d_cuboid/src/*.cpp compiled from /root/reference into
    oracle/_ref/libcuboid_ref.so against oracle/ref/minieigen.hpp / minicv.hpp, see oracle/ref/cuboid_ref.cpp), driven as
    object_slam/src/main_obj.cpp:354-361,449 drives it, with the members of params it has (the configs, both sampling flags,
    max_cuboid_num, nominal_skew_ratio, max_cut_skew).  Returns a list (one entry per box) of REF_CUBOID_DTYPE arrays, best first."""
    _ref_cub()
    if params is None:
        params = default_params()
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    K = np.ascontiguousarray(K, np.float64).reshape(3, 3)
    T_wc = np.ascontiguousarray(T_wc, np.float64).reshape(4, 4)
    boxes = np.ascontiguousarray(boxes, np.float64).reshape(-1, 5)
    lines = np.ascontiguousarray(lines, np.float64).reshape(-1, 4)
    N = len(boxes)
    flags = np.array([params.consider_config_1, params.consider_config_2, params.whether_sample_cam_roll_pitch, params.whether_sample_bbox_height], np.int32)
    out = np.zeros((max(N, 1), cap_per_box), REF_CUBOID_DTYPE)
    counts = np.zeros(max(N, 1), np.int32)
    rc = _REF_CUB.ref_detect_cuboid_skew(_p(img, C.c_uint8), w, h, ch, _p(K, C.c_double), _p(T_wc, C.c_double), _p(boxes, C.c_double), N,
                                         _p(lines, C.c_double), len(lines), _p(flags, C.c_int32), C.c_double(params.nominal_skew_ratio),
                                         C.c_double(params.max_cut_skew), int(params.max_cuboid_num), out.ctypes.data_as(C.POINTER(C.c_double)),
                                         cap_per_box, _p(counts, C.c_int32))
    if rc != 0:
        raise RuntimeError("ref_detect_cuboid failed (%d)" % rc)
    return [out[b, :min(counts[b], cap_per_box)].copy() for b in range(N)]


# ------------------------------------------------------------------------------------------- EDLines
def edl_detect(img, line_length_thres=50.0, cap=8192, want_stages=False):
    """line_lbd_detect::detect_filter_lines with use_LSD = false (EDLines, the class default) -> n x 4 float32."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros((cap, 4), np.float32)
    raw = np.zeros((cap, 4), np.float32)
    n_raw = C.c_int(0)
    st = None
    args = [None] * 8
    if want_stages:
        st = dict(blur=np.zeros((h, w), np.uint8), dx=np.zeros((h, w), np.int16), dy=np.zeros((h, w), np.int16), g=np.zeros((h, w), np.int16),
                  dir=np.zeros((h, w), np.uint8), anchors=np.zeros(w * h // 4 + 16, np.int32), edge=np.zeros((h, w), np.uint8))
        na = C.c_int(0)
        args = [_p(st["blur"], C.c_uint8), _p(st["dx"], C.c_int16), _p(st["dy"], C.c_int16), _p(st["g"], C.c_int16), _p(st["dir"], C.c_uint8),
                _p(st["anchors"], C.c_int32), C.byref(na), _p(st["edge"], C.c_uint8)]
    L = lib()
    L.edl_orc_detect.restype = C.c_int
    n = L.edl_orc_detect(_p(img, C.c_uint8), w, h, img.strides[0], ch, C.c_float(line_length_thres), _p(out, C.c_float), cap,
                         _p(raw, C.c_float), cap, C.byref(n_raw), *args)
    if n < 0:
        raise RuntimeError("edl_orc_detect failed (%d)" % n)
    res = dict(lines=out[:min(n, cap)].copy(), raw_lines=raw[:min(n_raw.value, cap)].copy())
    if want_stages:
        st["anchors"] = st["anchors"][:na.value].copy()
        res["stages"] = st
    return res


# ------------------------------------------------------------------------------------------- LBD descriptors + matcher (SURVEY 8 f4)
KEYLINE_DTYPE = np.dtype([("sx", np.float32), ("sy", np.float32), ("ex", np.float32), ("ey", np.float32), ("angle", np.float32),
                          ("line_length", np.float32), ("response", np.float32), ("size", np.float32), ("num_pixels", np.int32),
                          ("class_id", np.int32)])


def _img_args(img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    return img, w, h, ch


def lbd_detect_keylines(img, use_LSD=True, line_length_thres=15.0, cap=8192):
    """The key lines line_lbd_detect::detect_descrip_lines(gray, keylines_out, descrips) keeps (line_lbd_allclass.cpp:253-272)."""
    img, w, h, ch = _img_args(img)
    out = np.zeros(cap, KEYLINE_DTYPE)
    L = lib()
    L.lbd_orc_detect_keylines.restype = C.c_int
    n = L.lbd_orc_detect_keylines(_p(img, C.c_uint8), w, h, img.strides[0], ch, int(bool(use_LSD)), C.c_float(line_length_thres), out.ctypes.data_as(C.c_void_p), cap)
    if n < 0:
        raise RuntimeError("lbd_orc_detect_keylines failed (%d)" % n)
    return out[:n].copy()


def lbd_keylines_from_lsd(lines, w, h):
    """KeyLine fields of the LSD flavour from the n x 4 rows detect_filter_lines returns (LSDDetector.cpp:226-250)."""
    lines = np.ascontiguousarray(lines, np.float32).reshape(-1, 4)
    out = np.zeros(len(lines), KEYLINE_DTYPE)
    lib().lbd_orc_keylines_from_lsd(_p(lines, C.c_float), len(lines), int(w), int(h), out.ctypes.data_as(C.c_void_p))
    return out


def lbd_order_keylines(kl):
    """detect_descrip_lines_octaves' start / end swap and angle fold (line_lbd_allclass.cpp:321-330) on a copy."""
    kl = np.ascontiguousarray(kl, KEYLINE_DTYPE).copy()
    lib().lbd_orc_order_keylines(kl.ctypes.data_as(C.c_void_p), len(kl))
    return kl


def lbd_compute(img, keylines, want_float=False):
    """BinaryDescriptor::compute(image, keylines, descriptors) -> n x 32 uint8 (and n x 72 float32 with want_float)."""
    img, w, h, ch = _img_args(img)
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    n = len(kl)
    desc = np.zeros((n, 32), np.uint8)
    fdesc = np.zeros((n, 72), np.float32)
    L = lib()
    L.lbd_orc_compute.restype = C.c_int
    rc = L.lbd_orc_compute(_p(img, C.c_uint8), w, h, img.strides[0], ch, kl.ctypes.data_as(C.c_void_p), n, _p(desc, C.c_uint8), _p(fdesc, C.c_float))
    if rc < 0:
        raise RuntimeError("lbd_orc_compute failed (%d)" % rc)
    return (desc, fdesc) if want_float else desc


def lbd_match(query, train, thres=25.0):
    """line_lbd_detect::match_line_descrip -> (query_idx, train_idx, distance) of the good matches, query order."""
    q = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
    qi = np.zeros(max(len(q), 1), np.int32)
    ti = np.zeros(max(len(q), 1), np.int32)
    di = np.zeros(max(len(q), 1), np.float32)
    L = lib()
    L.lbd_orc_match.restype = C.c_int
    n = L.lbd_orc_match(_p(q, C.c_uint8), len(q), _p(t, C.c_uint8), len(t), C.c_float(thres), _p(qi, C.c_int32), _p(ti, C.c_int32), _p(di, C.c_float))
    return qi[:n].copy(), ti[:n].copy(), di[:n].copy()


def lbd_tables():
    """(F_g 63 doubles, F_l 21 doubles, rank of each one-byte xor pattern in Mihasher::query's enumeration)."""
    G = np.zeros(63, np.float64)
    Lw = np.zeros(21, np.float64)
    rank = np.zeros(256, np.int32)
    lib().lbd_orc_gauss_tables(_p(G, C.c_double), _p(Lw, C.c_double))
    lib().lbd_orc_pattern_rank(_p(rank, C.c_int32))
    return G, Lw, rank


def _ref_all():
    global _REF_ALL
    lib()
    if _REF_ALL is None:
        _REF_ALL = C.CDLL(_REF_ALL_PATH)
        _REF_ALL.ref_detect_filter_lines.restype = C.c_int
    for name in ("ref_detect_descrip_lines", "ref_detect_descrip_lines_octaves", "ref_lbd_compute", "ref_match_line_descrip"):
        getattr(_REF_ALL, name).restype = C.c_int
    return _REF_ALL


def ref_detect_descrip_lines(img, use_LSD=True, line_length_thres=15.0, cap=8192):
    """The reference's OWN detect_descrip_lines(gray, keylines_out, line_descrips) -> (key lines, n x 32 descriptors)."""
    img, w, h, ch = _img_args(img)
    kl = np.zeros(cap, KEYLINE_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    n = _ref_all().ref_detect_descrip_lines(_p(img, C.c_uint8), w, h, ch, int(bool(use_LSD)), C.c_float(line_length_thres), kl.ctypes.data_as(C.c_void_p),
                                            _p(desc, C.c_uint8), cap)
    if n < 0 or n > cap:
        raise RuntimeError("ref_detect_descrip_lines failed (%d)" % n)
    return kl[:n].copy(), desc[:n].copy()


def ref_detect_descrip_lines_octaves(img, use_LSD=True, line_length_thres=15.0, cap=8192):
    """The reference's OWN detect_descrip_lines_octaves, octave 0 -> (key lines with start x <= end x, n x 32 descriptors)."""
    img, w, h, ch = _img_args(img)
    kl = np.zeros(cap, KEYLINE_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    n = _ref_all().ref_detect_descrip_lines_octaves(_p(img, C.c_uint8), w, h, ch, int(bool(use_LSD)), C.c_float(line_length_thres),
                                                    kl.ctypes.data_as(C.c_void_p), _p(desc, C.c_uint8), cap)
    if n < 0 or n > cap:
        raise RuntimeError("ref_detect_descrip_lines_octaves failed (%d)" % n)
    return kl[:n].copy(), desc[:n].copy()


def ref_lbd_compute(img, keylines, want_float=False):
    """The reference's OWN BinaryDescriptor::compute on the given key lines."""
    img, w, h, ch = _img_args(img)
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    n = len(kl)
    desc = np.zeros((n, 32), np.uint8)
    fdesc = np.zeros((n, 72), np.float32)
    rc = _ref_all().ref_lbd_compute(_p(img, C.c_uint8), w, h, ch, kl.ctypes.data_as(C.c_void_p), n, _p(desc, C.c_uint8), _p(fdesc, C.c_float) if want_float else None)
    if rc < 0:
        raise RuntimeError("ref_lbd_compute failed (%d)" % rc)
    return (desc, fdesc) if want_float else desc


def ref_match_line_descrip(query, train, thres=25.0):
    """The reference's OWN match_line_descrip."""
    q = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
    qi = np.zeros(max(len(q), 1), np.int32)
    ti = np.zeros(max(len(q), 1), np.int32)
    di = np.zeros(max(len(q), 1), np.float32)
    n = _ref_all().ref_match_line_descrip(_p(q, C.c_uint8), len(q), _p(t, C.c_uint8), len(t), C.c_float(thres), _p(qi, C.c_int32), _p(ti, C.c_int32), _p(di, C.c_float))
    if n < 0:
        raise RuntimeError("ref_match_line_descrip failed (%d)" % n)
    return qi[:n].copy(), ti[:n].copy(), di[:n].copy()


# ------------------------------------------------------------------------------------------- batch driver (OpenMP, no Python in the loop)
def max_threads():
    return int(lib().orc_max_threads())


def detect_frames_batch(imgs, K, Ts, boxes_list, lines_list=None, params=None, line_mode=0, line_length_thres=15.0, n_threads=None,
                        want_records=False):
    """oracle/batch_oracle.cpp: the per-frame path (detect_filter_lines when line_mode > 0, then detect_cuboid) over a batch,
    frames over `n_threads` host threads with a static OpenMP schedule.  Returns dict(n_valid, n_cand, n_lines per frame
    [, records, counts])."""
    L = lib()
    if params is None:
        params = default_params()
    imgs = np.ascontiguousarray(imgs, np.uint8)
    F, h, w = imgs.shape[:3]
    ch = 1 if imgs.ndim == 3 else imgs.shape[3]
    K = np.ascontiguousarray(K, np.float64).reshape(3, 3)
    Ts = np.ascontiguousarray(Ts, np.float64).reshape(F, 16)
    box_off = np.zeros(F + 1, np.int32)
    box_off[1:] = np.cumsum([len(b) for b in boxes_list])
    boxes = np.ascontiguousarray(np.concatenate([np.asarray(b, np.float64).reshape(-1, 5) for b in boxes_list]) if box_off[-1] else np.zeros((0, 5)))
    if line_mode == 0:
        line_off = np.zeros(F + 1, np.int32)
        line_off[1:] = np.cumsum([len(l) for l in lines_list])
        lines = np.ascontiguousarray(np.concatenate([np.asarray(l, np.float64).reshape(-1, 4) for l in lines_list]) if line_off[-1] else np.zeros((0, 4)))
        lines_p, off_p = _p(lines, C.c_double), _p(line_off, C.c_int32)
    else:
        lines_p, off_p = None, None
    topk = max(int(params.max_cuboid_num), 1)
    nb = max(int(box_off[-1]), 1)
    out = np.zeros((nb, topk), CUBOID_DTYPE) if want_records else None
    counts = np.zeros(nb, np.int32) if want_records else None
    nv, nc, nl = np.zeros(F, np.int64), np.zeros(F, np.int64), np.zeros(F, np.int32)
    if n_threads is None:
        n_threads = max_threads()
    L.orc_detect_frames_batch.restype = C.c_int
    rc = L.orc_detect_frames_batch(_p(imgs, C.c_uint8), F, w, h, w * ch, ch, _p(K, C.c_double), _p(Ts, C.c_double), _p(boxes, C.c_double),
                                   _p(box_off, C.c_int32), lines_p, off_p, int(line_mode), C.c_float(line_length_thres), C.byref(params),
                                   int(n_threads), topk, out.ctypes.data_as(C.POINTER(Cuboid)) if want_records else None,
                                   _p(counts, C.c_int) if want_records else None, _p(nv, C.c_int64), _p(nc, C.c_int64), _p(nl, C.c_int32))
    if rc != 0:
        raise RuntimeError("orc_detect_frames_batch failed: %d" % rc)
    res = dict(n_valid=nv, n_cand=nc, n_lines=nl)
    if want_records:
        res["records"], res["counts"], res["box_off"] = out, counts, box_off
    return res


def ref_detect_filter_lines_octaves(img, use_LSD=True, line_length_thres=15.0, numoctaves=2, cap=8192):
    """The reference's OWN detect_filter_lines from a detector built with `numoctaves` octaves (ratio 2) -> (n x 4 float32, number of raw key
    lines over all octaves)."""
    img, w, h, ch = _img_args(img)
    L = _ref_all()
    L.ref_detect_filter_lines_octaves.restype = C.c_int
    out = np.zeros((cap, 4), np.float32)
    n_raw = C.c_int(0)
    n = L.ref_detect_filter_lines_octaves(_p(img, C.c_uint8), w, h, ch, int(bool(use_LSD)), C.c_float(line_length_thres), int(numoctaves), _p(out, C.c_float), cap,
                                          C.byref(n_raw))
    if n < 0 or n > cap:
        raise RuntimeError("ref_detect_filter_lines_octaves failed (%d)" % n)
    return out[:n].copy(), n_raw.value


def ref_minicv_pyrdown(gray, dw, dh):
    gray = np.ascontiguousarray(gray, np.uint8)
    out = np.zeros((dh, dw), np.uint8)
    _ref_all().ref_minicv_pyrdown(_p(gray, C.c_uint8), gray.shape[1], gray.shape[0], _p(out, C.c_uint8), dw, dh)
    return out


def ref_minicv_resize_half(gray):
    gray = np.ascontiguousarray(gray, np.uint8)
    h, w = gray.shape
    out = np.zeros((int(np.rint(h * 0.5)), int(np.rint(w * 0.5))), np.uint8)
    _ref_all().ref_minicv_resize_half(_p(gray, C.c_uint8), w, h, _p(out, C.c_uint8))
    return out
