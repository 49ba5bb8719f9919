"""Every octave of a multi-octave LSD line_lbd_detect, for the tests: the oracle's restatement (oracle/lbd_octaves_oracle.cpp in
liboracle.so, composed here with lsd_detect's raw segments per octave) and the reference's own class built with (numoctaves, octaveratio)
(oracle/ref/linelbd_octaves_ref.cpp, compiled on demand where the reference checkout exists).  TEST INFRASTRUCTURE ONLY: the product
package cube_slam_b200 never imports it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.pyoracle import KEYLINE_DTYPE, _img_args, _p, bgr2gray, lib, lsd_detect

_HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
_REF_SRC = os.path.join(_HERE, "ref", "linelbd_octaves_ref.cpp")
_REF_PATH = os.path.join(_HERE, "_ref", "liblinelbd_octaves_ref.so")
_REF_DEPS = [os.path.join(REFERENCE, "line_lbd", p) for p in ("libs/lsd.cpp", "libs/LSDDetector.cpp", "libs/binary_descriptor.cpp",
                                                                "class/line_lbd_allclass.cpp", "libs/binary_descriptor_matcher.cpp")]
_REF = None

OCTAVE_KEYLINE_DTYPE = np.dtype(KEYLINE_DTYPE.descr + [("s_oct_x", np.float32), ("s_oct_y", np.float32), ("e_oct_x", np.float32),
                                                        ("e_oct_y", np.float32), ("octave", np.int32), ("pad_", np.int32)])
assert OCTAVE_KEYLINE_DTYPE.itemsize == 64


def pyrdown(gray, dw, dh):
    """cv::pyrDown(gray, dst, Size(dw, dh)) on 8 bits (oracle/lbd_octaves_oracle.cpp: lbd_oct_pyrdown)"""
    gray = np.ascontiguousarray(gray, np.uint8)
    out = np.zeros((dh, dw), np.uint8)
    if lib().lbd_oct_pyrdown(_p(gray, C.c_uint8), gray.shape[1], gray.shape[0], _p(out, C.c_uint8), int(dw), int(dh)) != 0:
        raise ValueError("pyrDown: |2 * dst - src| > 2")
    return out


def gaussian5(gray):
    """cv::GaussianBlur(gray, dst, Size(5, 5), 1) on 8 bits (oracle/edl_oracle.cpp: edl_orc_gaussian5_u8)"""
    gray = np.ascontiguousarray(gray, np.uint8)
    out = np.zeros_like(gray)
    lib().edl_orc_gaussian5_u8(_p(gray, C.c_uint8), gray.shape[1], gray.shape[0], _p(out, C.c_uint8))
    return out


def sobel_u8(plane):
    """cv::Sobel to CV_16S, dx and dy, 3 x 3, of an 8-bit plane"""
    plane = np.ascontiguousarray(plane, np.uint8)
    dx, dy = np.zeros(plane.shape, np.int16), np.zeros(plane.shape, np.int16)
    lib().lbd_oct_sobel_u8(_p(plane, C.c_uint8), plane.shape[1], plane.shape[0], _p(dx, C.c_int16), _p(dy, C.c_int16))
    return dx, dy


def lsd_gaussian_pyramid(img, numoctaves):
    """LSDDetector::computeGaussianPyramid (LSDDetector.cpp:55-72) with scale 2: the gray frame, then pyrDown to (cols / 2, rows / 2)"""
    img = np.ascontiguousarray(img, np.uint8)
    pyr = [img if img.ndim == 2 else np.ascontiguousarray(bgr2gray(img))]
    for _ in range(1, numoctaves):
        h, w = pyr[-1].shape
        pyr.append(pyrdown(pyr[-1], w // 2, h // 2))
    return pyr


def descriptor_pyramid(gray, numoctaves):
    """BinaryDescriptor::computeGaussianPyramid (binary_descriptor.cpp:352-369): the blurred gray frame, then pyrDown per octave"""
    pyr = [gaussian5(gray)]
    for _ in range(1, numoctaves):
        h, w = pyr[-1].shape
        pyr.append(pyrdown(pyr[-1], w // 2, h // 2))
    return pyr


def _check_octaves(numoctaves, octaveratio):
    if numoctaves < 1:
        raise ValueError("numoctaves must be at least 1")
    if numoctaves > 1 and int(np.float32(octaveratio)) != 2:
        raise ValueError("pyrDown: |2 * dst - src| > 2 (octave ratio %g)" % octaveratio)


def lsd_octaves_raw(img, numoctaves, octaveratio=2.0, cap=8192):
    """detect_raw_lines of a detector with (numoctaves, octaveratio), LSD flavour (line_lbd_allclass.cpp:125-172, LSDDetector.cpp:176-250):
    -> one OCTAVE_KEYLINE_DTYPE array per octave.  LSD of each octave is lsd_detect's raw segments on the octave's image."""
    _check_octaves(numoctaves, octaveratio)
    pyr = lsd_gaussian_pyramid(img, numoctaves)
    h, w = pyr[0].shape
    out = []
    for k, plane in enumerate(pyr):
        raw = np.ascontiguousarray(lsd_detect(plane, 15.0, cap)["raw_lines"], np.float32)
        kl = np.zeros(max(len(raw), 1), OCTAVE_KEYLINE_DTYPE)
        oh, ow = plane.shape
        n = lib().lbd_oct_keylines(_p(raw, C.c_float), len(raw), k, ow, oh, w, h, kl.ctypes.data_as(C.c_void_p))
        out.append(kl[:n].copy())
    return out


def lsd_octaves_descrip(img, numoctaves, octaveratio=2.0, line_length_thres=15.0, cap=8192):
    """detect_descrip_lines_octaves (line_lbd_allclass.cpp:285-339) of the same detector -> ([key lines], [n x 32 descriptors]), one entry
    per octave: lineLength * (float)pow(octaveratio, octave) > line_length_thres, descriptors over the Sobel maps of the key line's octave
    at its in-octave ends, then start x <= end x and class_id within the octave."""
    raw = lsd_octaves_raw(img, numoctaves, octaveratio, cap)
    gray = lsd_gaussian_pyramid(img, 1)[0]
    dpyr = descriptor_pyramid(gray, numoctaves)
    kls, descs = [], []
    for k, kl in enumerate(raw):
        scale = np.float32(np.float32(octaveratio).astype(np.float64) ** k)
        kl = kl[kl["line_length"] * scale > np.float32(line_length_thres)].copy()
        dx, dy = sobel_u8(dpyr[k])
        ko = np.zeros(len(kl), KEYLINE_DTYPE)
        for f in KEYLINE_DTYPE.names:
            ko[f] = kl[f]
        ko["sx"], ko["sy"], ko["ex"], ko["ey"] = kl["s_oct_x"], kl["s_oct_y"], kl["e_oct_x"], kl["e_oct_y"]
        desc = np.zeros((len(kl), 32), np.uint8)
        if len(kl):
            oh, ow = dpyr[k].shape
            lib().lbd_oct_compute_maps(_p(dx, C.c_int16), _p(dy, C.c_int16), ow, oh, ko.ctypes.data_as(C.c_void_p), len(ko), _p(desc, C.c_uint8))
        PI = 3.14159265
        sw = kl["sx"] > kl["ex"]
        for a, b in (("sx", "ex"), ("sy", "ey"), ("s_oct_x", "e_oct_x"), ("s_oct_y", "e_oct_y")):
            t = kl[a][sw].copy()
            kl[a][sw] = kl[b][sw]
            kl[b][sw] = t
        ang = kl["angle"][sw].astype(np.float64)
        kl["angle"][sw] = np.where(ang > PI / 2, ang - PI, np.where(ang < -PI / 2, ang + PI, ang)).astype(np.float32)
        kl["class_id"] = np.arange(len(kl), dtype=np.int32)
        kls.append(kl)
        descs.append(desc)
    return kls, descs


def build_ref():
    """Compile oracle/_ref/liblinelbd_octaves_ref.so from the reference checkout (flags of oracle/Makefile's liblinelbd_ref.so) when it is
    missing or older than its sources.  Without the checkout the file is used as it is, if there is one."""
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
        _REF.ref_lsd_octaves.restype = C.c_int
    return _REF


def ref_lsd_octaves(img, numoctaves, octaveratio, line_length_thres=15.0, mode=2, cap=8192):
    """The reference's OWN line_lbd_detect(numoctaves, octaveratio) with use_LSD (oracle/ref/linelbd_octaves_ref.cpp: ref_lsd_octaves): mode 0
    detect_raw_lines(image, vector<vector<KeyLine>>), mode 1 detect_raw_lines(image, vector<KeyLine>) split by octave, mode 2
    detect_descrip_lines_octaves -> [OCTAVE_KEYLINE_DTYPE per octave] (mode 2: and [n x 32 descriptors]).  Raises RuntimeError when the
    reference throws."""
    img, w, h, ch = _img_args(img)
    L = _ref_lib()
    kl = np.zeros((numoctaves + 1, cap), OCTAVE_KEYLINE_DTYPE)
    desc = np.zeros((numoctaves + 1, cap, 32), np.uint8)
    cnt = np.zeros(numoctaves + 1, np.int32)
    n = L.ref_lsd_octaves(_p(img, C.c_uint8), w, h, ch, int(numoctaves), C.c_float(octaveratio), C.c_float(line_length_thres), int(mode),
                          kl.ctypes.data_as(C.c_void_p), _p(desc, C.c_uint8), _p(cnt, C.c_int32), cap)
    if n < 0:
        raise RuntimeError("ref_lsd_octaves failed (%d)" % n)
    kls = [kl[k, :cnt[k]].copy() for k in range(n)]
    return (kls, [desc[k, :cnt[k]].copy() for k in range(n)]) if mode == 2 else kls
