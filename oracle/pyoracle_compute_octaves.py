"""BinaryDescriptor::compute on key lines of any octave that the caller gives, for the tests: the oracle's restatement (lbd_compute_octaves,
composed of pyoracle_octaves' descriptor pyramid and per-octave LBD) and the reference's own BinaryDescriptor (oracle/ref/
linelbd_compute_octaves_ref.cpp, compiled on demand where the reference checkout exists).  TEST INFRASTRUCTURE ONLY: the product package
cube_slam_b200 never imports it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.pyoracle import KEYLINE_DTYPE, _img_args, _p, lib
from oracle.pyoracle_octaves import OCTAVE_KEYLINE_DTYPE, REFERENCE, _REF_DEPS, descriptor_pyramid, lsd_gaussian_pyramid, sobel_u8

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_SRC = os.path.join(_HERE, "ref", "linelbd_compute_octaves_ref.cpp")
_REF_PATH = os.path.join(_HERE, "_ref", "liblinelbd_compute_octaves_ref.so")
_REF = None


def build_ref():
    """Compile oracle/_ref/liblinelbd_compute_octaves_ref.so from the reference checkout (flags of oracle/Makefile's liblinelbd_ref.so) when it
    is missing or older than its sources.  Without the checkout the file is used as it is, if there is one."""
    lib()                                                   # liboracle.so, which the wrapper links against
    if not os.path.exists(_REF_DEPS[0]):
        return _REF_PATH
    deps = _REF_DEPS + [_REF_SRC, os.path.join(_HERE, "ref", "minicv.hpp"), os.path.join(_HERE, "_build", "liboracle.so")]
    if os.path.exists(_REF_PATH) and all(os.path.getmtime(_REF_PATH) >= os.path.getmtime(d) for d in deps):
        return _REF_PATH
    os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
    fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(_REF_PATH))
    os.close(fd)
    try:
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-w",
                               "-I", os.path.join(_HERE, "ref", "fakecv"), "-I", os.path.join(REFERENCE, "line_lbd", "include"),
                               "-I", os.path.join(REFERENCE, "line_lbd", "libs"), "-o", tmp, _REF_SRC, "-L", os.path.join(_HERE, "_build"), "-loracle",
                               "-Wl,-rpath,$ORIGIN/../_build"])
        os.replace(tmp, _REF_PATH)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return _REF_PATH


def ref_available():
    return os.path.exists(build_ref())


def _ref_lib():
    global _REF
    if _REF is None:
        _REF = C.CDLL(build_ref())
        _REF.ref_lbd_compute_octaves.restype = C.c_int
    return _REF


def ref_lbd_compute_octaves(img, keylines, want_float=False):
    """The reference's OWN BinaryDescriptor::compute(image, keylines, descriptors[, returnFloatDescr]) on the given OCTAVE_KEYLINE_DTYPE
    records, in their order (oracle/ref/linelbd_octaves_ref.cpp: ref_lbd_compute_octaves) -> n x 32 uint8 (and n x 72 float32 with
    want_float).  Rows the reference does not write (all but the first of a repeated (class_id, octave) pair) are undefined.  The reference
    reads the first line of every class_id from 0 to the largest (computeLBD, binary_descriptor.cpp:1482-1490), so a list that skips a class_id
    crashes it: pass lists without gaps.  Raises RuntimeError with the reference's message when it throws."""
    img, w, h, ch = _img_args(img)
    kl = np.ascontiguousarray(keylines, OCTAVE_KEYLINE_DTYPE).reshape(-1)
    n = len(kl)
    desc = np.zeros((max(n, 1), 32), np.uint8)
    fdesc = np.zeros((max(n, 1), 72), np.float32)
    err = C.create_string_buffer(512)
    L = _ref_lib()
    rc = L.ref_lbd_compute_octaves(_p(img, C.c_uint8), w, h, ch, kl.ctypes.data_as(C.c_void_p), n, _p(desc, C.c_uint8),
                                   _p(fdesc, C.c_float) if want_float else None, err, len(err))
    if rc < 0:
        raise RuntimeError("ref_lbd_compute_octaves failed (%d): %s" % (rc, err.value.decode()))
    return (desc[:n], fdesc[:n]) if want_float else desc[:n]


def deepest_octave(w, h):
    """the deepest octave BinaryDescriptor::computeGaussianPyramid can build for a w x h image: pyrDown refuses a level of width or height 0"""
    k = 0
    while w // 2 > 0 and h // 2 > 0:
        w, h, k = w // 2, h // 2, k + 1
    return k


def pair_rows(keylines):
    """computeImpl's output map (binary_descriptor.cpp:655-693,750-788) -> {first row: last row} of every (class_id, octave) pair that more
    than one row shares: the first row receives the descriptor of the last"""
    first, last = {}, {}
    for i, (c, o) in enumerate(zip(keylines["class_id"].tolist(), keylines["octave"].tolist())):
        first.setdefault((c, o), i)
        last[(c, o)] = i
    return {first[k]: last[k] for k in first if first[k] != last[k]}


def lbd_compute_octaves(img, keylines):
    """BinaryDescriptor::compute on key lines of any octave, restated (binary_descriptor.cpp:587-790): the gray image, descriptor_pyramid of
    max(octave) + 1 levels, each key line described on the Sobel maps of its octave at its in-octave ends (lbd_oct_compute_maps), then the
    (class_id, octave) map of pair_rows.  -> n x 32 uint8; the rows the reference leaves unwritten hold their own descriptor.  Raises
    ValueError where the reference throws (an octave pyrDown cannot make) or is undefined (a negative class_id or octave)."""
    kl = np.ascontiguousarray(keylines, OCTAVE_KEYLINE_DTYPE).reshape(-1)
    desc = np.zeros((len(kl), 32), np.uint8)
    if not len(kl):
        return desc
    gray = lsd_gaussian_pyramid(img, 1)[0]
    h, w = gray.shape
    if (kl["class_id"] < 0).any() or (kl["octave"] < 0).any():
        raise ValueError("negative class_id or octave")
    if kl["octave"].max() > deepest_octave(w, h):
        raise ValueError("pyrDown destination size")
    dpyr = descriptor_pyramid(gray, int(kl["octave"].max()) + 1)
    for k, plane in enumerate(dpyr):
        rows = np.flatnonzero(kl["octave"] == k)
        if not len(rows):
            continue
        dx, dy = sobel_u8(plane)
        ko = np.zeros(len(rows), KEYLINE_DTYPE)
        for f in KEYLINE_DTYPE.names:
            ko[f] = kl[f][rows]
        ko["sx"], ko["sy"], ko["ex"], ko["ey"] = kl["s_oct_x"][rows], kl["s_oct_y"][rows], kl["e_oct_x"][rows], kl["e_oct_y"][rows]
        d = np.zeros((len(rows), 32), np.uint8)
        oh, ow = plane.shape
        lib().lbd_oct_compute_maps(_p(dx, C.c_int16), _p(dy, C.c_int16), ow, oh, ko.ctypes.data_as(C.c_void_p), len(ko), _p(d, C.c_uint8))
        desc[rows] = d
    for first, last in pair_rows(kl).items():
        desc[first] = desc[last]
    return desc
