"""ctypes binding of the CPU ORACLE for k-nearest-neighbour and radius matching of line descriptors.  TEST INFRASTRUCTURE ONLY.

lbd_knn_match / lbd_radius_match: the restatement in oracle/lbd_knn_oracle.cpp (part of oracle/_build/liboracle.so).
lbd_knn_lists / lbd_radius_lists: the vector<vector<DMatch>> the reference's knnMatch / radiusMatch build from it (mask, compactResult).
ref_knn_match / ref_radius_match: the reference's own matcher (oracle/ref/linelbd_knn_ref.cpp -> oracle/_ref/liblinelbd_knn_ref.so, built
here with oracle/Makefile's flags for liblinelbd_ref.so where the reference checkout exists; elsewhere a library built before is used).
Only tests/ and tools/ import this module; the product package cube_slam_b200 never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_KNN_PATH = os.path.join(_HERE, "_ref", "liblinelbd_knn_ref.so")
_REFERENCE = "/root/reference"
_REF_SRCS = [os.path.join(_REFERENCE, "line_lbd", "libs", f) for f in ("lsd.cpp", "LSDDetector.cpp", "binary_descriptor.cpp", "binary_descriptor_matcher.cpp")] + \
    [os.path.join(_REFERENCE, "line_lbd", "class", "line_lbd_allclass.cpp")]
_REF_KNN = None
_p = pyoracle._p


def _orc():
    L = pyoracle.lib()
    L.lbd_orc_knn_match.restype = C.c_int
    L.lbd_orc_radius_match.restype = C.c_int64
    return L


def build_ref():
    """Compile oracle/_ref/liblinelbd_knn_ref.so where the reference checkout exists and the library is missing or older than its sources."""
    pyoracle.build()
    if not os.path.exists(_REF_SRCS[0]):
        return _REF_KNN_PATH
    deps = _REF_SRCS + [pyoracle._LIB_PATH] + [os.path.join(_HERE, "ref", f) for f in os.listdir(os.path.join(_HERE, "ref")) if f.endswith((".cpp", ".hpp"))]
    if os.path.exists(_REF_KNN_PATH) and all(os.path.getmtime(_REF_KNN_PATH) >= os.path.getmtime(d) for d in deps):
        return _REF_KNN_PATH
    os.makedirs(os.path.dirname(_REF_KNN_PATH), exist_ok=True)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-w",
                           "-I", "ref/fakecv", "-I", os.path.join(_REFERENCE, "line_lbd", "include"), "-I", os.path.join(_REFERENCE, "line_lbd", "libs"),
                           "-o", _REF_KNN_PATH, "ref/linelbd_knn_ref.cpp", "-L", "_build", "-loracle", "-Wl,-rpath,$ORIGIN/../_build"], cwd=_HERE)
    return _REF_KNN_PATH


def ref_available():
    return os.path.exists(build_ref())


def _ref_knn():
    global _REF_KNN
    if _REF_KNN is None:
        _REF_KNN = C.CDLL(build_ref())
        _REF_KNN.ref_knn_match.restype = C.c_int
        _REF_KNN.ref_radius_match.restype = C.c_int
    return _REF_KNN


def _codes(query, train, mask):
    q = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
    m = None if mask is None else np.ascontiguousarray(np.asarray(mask).reshape(-1) != 0, np.uint8)
    assert m is None or len(m) == len(q)
    return q, t, m


def lbd_knn_match(query, train, k, mask=None):
    """BinaryDescriptorMatcher::knnMatch(query, train, matches, k, mask), restated: per query (query_idx, train_idx, distance) of the
    first k met codes in the hash's order (train_idx -1 beyond D = 128)."""
    q, t, m = _codes(query, train, mask)
    nq, kk = len(q), max(int(k), 1)
    n = np.zeros(max(nq, 1), np.int32)
    qi, ti, di = np.zeros(max(nq * kk, 1), np.int32), np.zeros(max(nq * kk, 1), np.int32), np.zeros(max(nq * kk, 1), np.float32)
    rc = _orc().lbd_orc_knn_match(_p(q, C.c_uint8), nq, _p(t, C.c_uint8), len(t), int(k), None if m is None else _p(m, C.c_uint8), _p(n, C.c_int32),
                                 _p(qi, C.c_int32), _p(ti, C.c_int32), _p(di, C.c_float))
    if rc < 0:
        raise ValueError("k must not be negative")
    return [(qi[i * kk:i * kk + n[i]].copy(), ti[i * kk:i * kk + n[i]].copy(), di[i * kk:i * kk + n[i]].copy()) for i in range(nq)]


def lbd_radius_match(query, train, max_distance, mask=None):
    """BinaryDescriptorMatcher::radiusMatch(query, train, matches, maxDistance, mask), restated: per query (query_idx, train_idx, distance)
    of every met code with distance <= max_distance, in the hash's order."""
    q, t, m = _codes(query, train, mask)
    nq = len(q)
    off = np.zeros(nq + 1, np.int64)
    L = _orc()
    args = (_p(q, C.c_uint8), nq, _p(t, C.c_uint8), len(t), C.c_float(max_distance), None if m is None else _p(m, C.c_uint8), _p(off, C.c_int64))
    total = L.lbd_orc_radius_match(*args, None, None, None, C.c_int64(0))
    qi, ti, di = np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.float32)
    L.lbd_orc_radius_match(*args, _p(qi, C.c_int32), _p(ti, C.c_int32), _p(di, C.c_float), C.c_int64(total))
    return [(qi[off[i]:off[i + 1]].copy(), ti[off[i]:off[i + 1]].copy(), di[off[i]:off[i + 1]].copy()) for i in range(nq)]


def lbd_knn_lists(query, train, k, mask=None, compact=False):
    """The vector<vector<DMatch>> of knnMatch(..., mask, compactResult) from lbd_knn_match -> [(query, query_idx, train_idx, distance)]:
    nothing for an empty side; a masked query is an empty list, or absent with compactResult."""
    q, t, m = _codes(query, train, mask)
    if len(q) == 0 or len(t) == 0:
        return []
    per = lbd_knn_match(q, t, k, m)
    return [(i,) + per[i] for i in range(len(q)) if not (compact and m is not None and not m[i])]


def lbd_radius_lists(query, train, max_distance, mask=None, compact=False):
    """The vector<vector<DMatch>> of radiusMatch(..., mask, compactResult) from lbd_radius_match: with compactResult every empty list is
    left out (masked or not)."""
    q, t, m = _codes(query, train, mask)
    if len(q) == 0 or len(t) == 0:
        return []
    per = lbd_radius_match(q, t, max_distance, m)
    return [(i,) + per[i] for i in range(len(q)) if not (compact and len(per[i][0]) == 0)]


def _ref_lists(fn, query, train, arg, mask, compact):
    q, t, m = _codes(query, train, mask)
    nq, nt = len(q), len(t)
    cap = max(nq * max(nt, 1), 1)
    lq, ll = np.zeros(max(nq, 1), np.int32), np.zeros(max(nq, 1), np.int32)
    qi, ti, di = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.float32)
    n = fn(_p(q, C.c_uint8), nq, _p(t, C.c_uint8), nt, arg, None if m is None else _p(m, C.c_uint8), int(bool(compact)), _p(lq, C.c_int32), _p(ll, C.c_int32),
           _p(qi, C.c_int32), _p(ti, C.c_int32), _p(di, C.c_float), cap)
    if n < 0:
        raise RuntimeError("reference matcher failed (%d)" % n)
    out, o = [], 0
    for l in range(n):
        out.append((int(lq[l]), qi[o:o + ll[l]].copy(), ti[o:o + ll[l]].copy(), di[o:o + ll[l]].copy()))
        o += ll[l]
    return out


def ref_matcher_call(kind, query, train, arg):
    """The reference's knnMatch (kind "knn", arg = k) or radiusMatch ("radius", arg = maxDistance) alone, nothing returned: for timing."""
    q, t, _ = _codes(query, train, None)
    fn = _ref_knn().ref_knn_match if kind == "knn" else _ref_knn().ref_radius_match
    z = np.zeros(1, np.int32)
    fn(_p(q, C.c_uint8), len(q), _p(t, C.c_uint8), len(t), int(arg) if kind == "knn" else C.c_float(arg), None, 0, _p(z, C.c_int32), _p(z, C.c_int32),
       _p(z, C.c_int32), _p(z, C.c_int32), _p(z.view(np.float32), C.c_float), -1)


def ref_knn_match(query, train, k, mask=None, compact=False):
    """The reference's OWN pairwise knnMatch, defined part only -> [(query, query_idx, train_idx, distance)] per list it returns."""
    return _ref_lists(_ref_knn().ref_knn_match, query, train, int(k), mask, compact)


def ref_radius_match(query, train, max_distance, mask=None, compact=False):
    """The reference's OWN pairwise radiusMatch, defined part only -> [(query, query_idx, train_idx, distance)] per list it returns."""
    return _ref_lists(_ref_knn().ref_radius_match, query, train, C.c_float(max_distance), mask, compact)


