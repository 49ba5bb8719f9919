"""ctypes binding of the CPU ORACLE for matching line descriptors against a collection of images.  TEST INFRASTRUCTURE ONLY.

collection_knn / collection_radius: the restatement in oracle/lbd_collection_oracle.cpp (part of oracle/_build/liboracle.so).
collection_match_list / collection_knn_lists / collection_radius_lists: what the reference's match / knnMatch / radiusMatch without a train
matrix return from it (masks, compactResult).
ref_collection_match / ref_collection_knn / ref_collection_radius: the reference's own matcher after add() (oracle/ref/linelbd_collection_ref.cpp
-> oracle/_ref/liblinelbd_collection_ref.so, built here like liblinelbd_knn_ref.so where the reference checkout exists).
Lists are [(query, query_idx, train_idx, img_idx, distance)]; `images` is a list of n_i x 32 uint8 code matrices.
Only tests/ and tools/ import this module; the product package cube_slam_b200 never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle, pyoracle_knn

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_PATH = os.path.join(_HERE, "_ref", "liblinelbd_collection_ref.so")
_REF = None
_p = pyoracle._p


def _orc():
    L = pyoracle.lib()
    L.lbd_orc_collection_knn.restype = C.c_int
    L.lbd_orc_collection_radius.restype = C.c_int64
    return L


def build_ref():
    """Compile oracle/_ref/liblinelbd_collection_ref.so where the reference checkout exists and the library is missing or older than its
    sources."""
    pyoracle.build()
    srcs = pyoracle_knn._REF_SRCS
    if not os.path.exists(srcs[0]):
        return _REF_PATH
    deps = srcs + [pyoracle._LIB_PATH] + [os.path.join(_HERE, "ref", f) for f in os.listdir(os.path.join(_HERE, "ref")) if f.endswith((".cpp", ".hpp"))]
    if os.path.exists(_REF_PATH) and all(os.path.getmtime(_REF_PATH) >= os.path.getmtime(d) for d in deps):
        return _REF_PATH
    os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
    ref = pyoracle_knn._REFERENCE
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-w",
                           "-I", "ref/fakecv", "-I", os.path.join(ref, "line_lbd", "include"), "-I", os.path.join(ref, "line_lbd", "libs"),
                           "-o", _REF_PATH, "ref/linelbd_collection_ref.cpp", "-L", "_build", "-loracle", "-Wl,-rpath,$ORIGIN/../_build"], cwd=_HERE)
    return _REF_PATH


def ref_available():
    return os.path.exists(build_ref())


def _ref():
    global _REF
    if _REF is None:
        _REF = C.CDLL(build_ref())
        _REF.ref_collection_query.restype = C.c_int
    return _REF


def _pack(images, query, masks):
    ims = [np.ascontiguousarray(x, np.uint8).reshape(-1, 32) for x in images]
    off = np.concatenate([[0], np.cumsum([len(x) for x in ims])]).astype(np.int32)
    codes = np.ascontiguousarray(np.concatenate(ims)) if off[-1] else np.zeros((1, 32), np.uint8)
    q = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
    m = None
    if masks is not None and len(masks):
        assert len(masks) == len(ims) and all(np.asarray(x).size == len(q) for x in masks)
        m = np.ascontiguousarray(np.stack([np.asarray(x).reshape(-1) != 0 for x in masks]), np.uint8).reshape(-1) if len(q) else np.zeros(1, np.uint8)
    return codes, off, len(ims), q if len(q) else np.zeros((1, 32), np.uint8), len(q), m


def collection_knn(images, query, k, masks=None):
    """knnMatch(query, matches, k, masks) after add(images), restated: per query (query_idx, train_idx, img_idx, distance) arrays."""
    codes, off, ni, q, nq, m = _pack(images, query, masks)
    kk = max(int(k), 1)
    n = np.zeros(max(nq, 1), np.int32)
    bufs = [np.zeros(max(nq * kk, 1), t) for t in (np.int32, np.int32, np.int32, np.float32)]
    rc = _orc().lbd_orc_collection_knn(_p(codes, C.c_uint8), _p(off, C.c_int32), ni, _p(q, C.c_uint8), nq, int(k), None if m is None else _p(m, C.c_uint8),
                                       _p(n, C.c_int32), _p(bufs[0], C.c_int32), _p(bufs[1], C.c_int32), _p(bufs[2], C.c_int32), _p(bufs[3], C.c_float))
    if rc < 0:
        raise ValueError("k must not be negative")
    return [tuple(b[i * kk:i * kk + n[i]].copy() for b in bufs) for i in range(nq)]


def collection_radius(images, query, max_distance, masks=None):
    """radiusMatch(query, matches, maxDistance, masks) after add(images), restated: per query (query_idx, train_idx, img_idx, distance)."""
    codes, off, ni, q, nq, m = _pack(images, query, masks)
    offs = np.zeros(nq + 1, np.int64)
    L = _orc()
    args = (_p(codes, C.c_uint8), _p(off, C.c_int32), ni, _p(q, C.c_uint8), nq, C.c_float(max_distance), None if m is None else _p(m, C.c_uint8),
            _p(offs, C.c_int64))
    total = L.lbd_orc_collection_radius(*args, None, None, None, None, C.c_int64(0))
    bufs = [np.zeros(max(total, 1), t) for t in (np.int32, np.int32, np.int32, np.float32)]
    L.lbd_orc_collection_radius(*args, _p(bufs[0], C.c_int32), _p(bufs[1], C.c_int32), _p(bufs[2], C.c_int32), _p(bufs[3], C.c_float), C.c_int64(total))
    return [tuple(b[offs[i]:offs[i + 1]].copy() for b in bufs) for i in range(nq)]


def collection_knn_lists(images, query, k, masks=None, compact=False):
    """The vector<vector<DMatch>> of knnMatch(query, matches, k, masks, compactResult): [] for an empty query set; with compactResult the
    lists left empty (by masks or by meeting nothing) are dropped."""
    if len(np.asarray(query).reshape(-1, 32)) == 0:
        return []
    per = collection_knn(images, query, k, masks)
    return [(i,) + per[i] for i in range(len(per)) if not (compact and len(per[i][0]) == 0)]


def collection_radius_lists(images, query, max_distance, masks=None, compact=False):
    if len(np.asarray(query).reshape(-1, 32)) == 0:
        return []
    per = collection_radius(images, query, max_distance, masks)
    return [(i,) + per[i] for i in range(len(per)) if not (compact and len(per[i][0]) == 0)]


def collection_match_list(images, query, masks=None):
    """match(query, matches, masks): the nearest code of each query kept when the mask of its image keeps the query, no fall-back ->
    (query_idx, train_idx, img_idx, distance) arrays, query order."""
    if len(np.asarray(query).reshape(-1, 32)) == 0:
        return tuple(np.zeros(0, t) for t in (np.int32, np.int32, np.int32, np.float32))
    per = collection_knn(images, query, 1, masks)
    return tuple(np.concatenate([x[j] for x in per]) for j in range(4))


def _ref_call(kind, images, query, k, max_distance, masks, compact):
    codes, off, ni, q, nq, m = _pack(images, query, masks)
    cap = max(nq * max(int(off[-1]), 1), 1)
    lq, ll = np.zeros(max(cap, nq, 1), np.int32), np.zeros(max(cap, nq, 1), np.int32)
    bufs = [np.zeros(cap, t) for t in (np.int32, np.int32, np.int32, np.float32)]
    n = _ref().ref_collection_query(kind, _p(codes, C.c_uint8), _p(off, C.c_int32), ni, _p(q, C.c_uint8), nq, int(k), C.c_float(max_distance),
                                    None if m is None else _p(m, C.c_uint8), int(bool(compact)), _p(lq, C.c_int32), _p(ll, C.c_int32),
                                    _p(bufs[0], C.c_int32), _p(bufs[1], C.c_int32), _p(bufs[2], C.c_int32), _p(bufs[3], C.c_float), cap)
    if n < 0:
        raise RuntimeError("reference collection matcher not run or failed (%d)" % n)
    out, o = [], 0
    for l in range(n):
        out.append((int(lq[l]),) + tuple(b[o:o + ll[l]].copy() for b in bufs))
        o += ll[l]
    return out


def ref_collection_knn(images, query, k, masks=None, compact=False):
    """The reference's OWN knnMatch(query, matches, k, masks, compactResult) after add(images), defined part only."""
    if len(np.asarray(query).reshape(-1, 32)) == 0:
        return []
    return _ref_call(1, images, query, k, 0.0, masks, compact)


def ref_collection_radius(images, query, max_distance, masks=None, compact=False):
    if len(np.asarray(query).reshape(-1, 32)) == 0:
        return []
    return _ref_call(2, images, query, 0, max_distance, masks, compact)


def ref_collection_match(images, query, masks=None):
    """The reference's OWN match(query, matches, masks) after add(images), defined part only -> (query_idx, train_idx, img_idx, distance)."""
    lists = _ref_call(0, images, query, 0, 0.0, masks, False)
    if not lists:
        return tuple(np.zeros(0, t) for t in (np.int32, np.int32, np.int32, np.float32))
    return tuple(np.concatenate([x[j] for x in lists]) for j in range(1, 5))


def ref_collection_time(kind, images, query, arg):
    """The reference's collection knnMatch (kind "knn", arg = k) or radiusMatch ("radius", arg = maxDistance) alone, nothing returned:
    for timing."""
    codes, off, ni, q, nq, _ = _pack(images, query, None)
    z = np.zeros(1, np.int32)
    _ref().ref_collection_query(1 if kind == "knn" else 2, _p(codes, C.c_uint8), _p(off, C.c_int32), ni, _p(q, C.c_uint8), nq,
                                int(arg) if kind == "knn" else 0, C.c_float(0.0 if kind == "knn" else arg), None, 0, _p(z, C.c_int32),
                                _p(z, C.c_int32), _p(z, C.c_int32), _p(z, C.c_int32), _p(z, C.c_int32), _p(z.view(np.float32), C.c_float), -1)
