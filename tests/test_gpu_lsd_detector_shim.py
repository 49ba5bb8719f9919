"""The C++ drop-in for the reference's LSDDetector, RUN: shim/lsd_detector_b200.cpp compiled in place of line_lbd/libs/LSDDetector.cpp next to
the reference's other line_lbd sources, driven by shim/test/lsd_detector_shim_driver.cpp (oracle/_ref/libshim_lsd.so), against the same
sources with the reference's own LSDDetector.cpp and the same driver (oracle/_ref/libref_lsd_detector.so); both built by shim/test/Makefile
where the reference checkout exists.  Every KeyLine field is compared bit for bit, in order, for the three detect overloads, with masks,
pre-filled vectors, both values of opts.save_octave_line (and what the detector prints on std::cout), the input errors, the reference's own
line_lbd_detect running over the drop-in, two threads at once, and the Python mirror line_lbd_detect.lsd on the same cases."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = os.path.join(ROOT, "oracle", "_ref", "libshim_lsd.so")
REF = os.path.join(ROOT, "oracle", "_ref", "libref_lsd_detector.so")
FLAT, OCTAVES, VECTOR = 0, 1, 2
NO_ERROR, RUNTIME_ERROR, LENGTH_ERROR, OTHER_ERROR = 0, 1, 2, 3

# every KeyLine field as the driver returns it (lsdd_rec)
REC_DTYPE = np.dtype([("start_x", "<f4"), ("start_y", "<f4"), ("end_x", "<f4"), ("end_y", "<f4"), ("angle", "<f4"), ("line_length", "<f4"),
                      ("response", "<f4"), ("size", "<f4"), ("num_pixels", "<i4"), ("class_id", "<i4"), ("s_oct_x", "<f4"), ("s_oct_y", "<f4"),
                      ("e_oct_x", "<f4"), ("e_oct_y", "<f4"), ("octave", "<i4"), ("pt_x", "<f4"), ("pt_y", "<f4")])
FLAG_FALSE_MSG = "LSD line detector reset save octave lines to False  to match output !!!"
FLAG_TRUE_MSG = "LSD line detector reset save octave lines to True to match output !!!"
MASK_MSG = "Mask error while detecting lines: please check its dimensions and that data type is CV_8UC1"
MASKS_MSG = "Masks error while detecting lines: please check their dimensions and that data types are CV_8UC1"


class LsdMat(C.Structure):
    _fields_ = [("data", C.c_void_p), ("rows", C.c_int32), ("cols", C.c_int32), ("type", C.c_int32), ("step", C.c_int32)]


_DEPTH = {np.dtype(np.uint8): 0, np.dtype(np.int16): 3, np.dtype(np.float32): 5}


def lsd_mat(a, keep):
    """a numpy image (H x W or H x W x C, any row stride) as the driver's Mat descriptor; None an empty Mat"""
    if a is None:
        return LsdMat(None, 0, 0, 0, 0)
    a = np.asarray(a)
    if a.ndim == 3 and a.strides[1:] != (a.shape[2] * a.itemsize, a.itemsize) or a.ndim == 2 and a.strides[1] != a.itemsize:
        a = np.ascontiguousarray(a)
    keep.append(a)
    ch = 1 if a.ndim == 2 else a.shape[2]
    return LsdMat(a.ctypes.data, a.shape[0], a.shape[1], _DEPTH[a.dtype] + ((ch - 1) << 3), a.strides[0])


class Driver(object):
    """ctypes view of lsd_detector_shim_driver.cpp, in either build"""

    def __init__(self, path):
        L = self.L = C.CDLL(path)
        assert L.lsdd_rec_size() == REC_DTYPE.itemsize
        P = C.c_void_p
        L.lsdd_detect.argtypes = [C.c_int, P, C.c_int, P, C.c_int, C.c_int, C.c_int, P, P, P, C.c_int, P, P, C.c_int, C.c_int64, P, C.c_char_p, C.c_int]
        L.lsdd_threads.argtypes = [C.c_int, P, C.c_int, C.c_int, P, P, C.c_int64]
        L.lsdd_line_lbd.argtypes = [C.c_int, C.c_float, C.c_int, P, P, P, P, C.c_int, C.c_int64]

    @staticmethod
    def _lists(n, ll, recs):
        out, o = [], 0
        for l in range(n):
            out.append(recs[o:o + ll[l]].copy())
            o += ll[l]
        return out

    def detect(self, member, images, scale, num_octaves, masks=None, flag=False, pre=None, cap=1 << 18):
        """One detect call -> (lists, flag after, error kind, error text).  images: one image (FLAT / OCTAVES) or a list (VECTOR); masks:
        None (the default argument), one mask (FLAT / OCTAVES) or a list of masks, None entries being empty Mats; pre: the output vector's
        lists before the call (FLAT: one list)."""
        keep = []
        imgs = images if member == VECTOR else [images]
        ms = [] if masks is None else (masks if member == VECTOR else [masks])
        im = (LsdMat * max(len(imgs), 1))(*[lsd_mat(x, keep) for x in imgs])
        mm = (LsdMat * max(len(ms), 1))(*[lsd_mat(x, keep) for x in ms])
        pre = [] if pre is None else [np.ascontiguousarray(p, REC_DTYPE) for p in pre]
        pre_len = np.array([len(p) for p in pre] + [0], np.int32)
        pre_recs = np.ascontiguousarray(np.concatenate(pre + [np.zeros(1, REC_DTYPE)]))
        fl = np.array([int(bool(flag))], np.int32)
        cap_lists = max(len(imgs), len(pre), abs(num_octaves), 1) + 1
        ll = np.zeros(cap_lists, np.int32)
        recs = np.zeros(cap, REC_DTYPE)
        ek = np.zeros(1, np.int32)
        err = C.create_string_buffer(1024)
        n = self.L.lsdd_detect(member, im, len(imgs), mm, len(ms), int(scale), int(num_octaves), fl.ctypes.data, pre_len.ctypes.data, pre_recs.ctypes.data, len(pre),
                               ll.ctypes.data, recs.ctypes.data, cap_lists, cap, ek.ctypes.data, err, len(err))
        assert n >= 0, n
        return self._lists(n, ll, recs), bool(fl[0]), int(ek[0]), err.value.decode()

    def threads(self, images, num_octaves, repeat=1, cap=1 << 18):
        keep = []
        im = (LsdMat * len(images))(*[lsd_mat(x, keep) for x in images])
        ll = np.zeros(len(images), np.int32)
        recs = np.zeros(cap, REC_DTYPE)
        n = self.L.lsdd_threads(len(images), im, num_octaves, repeat, ll.ctypes.data, recs.ctypes.data, cap)
        assert n == len(images), n
        return self._lists(n, ll, recs)

    def line_lbd(self, num_octaves, member, image, line_length_thres=15.0, cap=1 << 18):
        """the reference's own line_lbd_detect(num_octaves, 2.0) with use_LSD: member 0 detect_raw_lines (flat), 1 detect_raw_lines (per
        octave), 2 detect_filter_lines (KeyLine), 3 detect_descrip_lines_octaves -> (lists, descriptors per list or None)"""
        keep = []
        m = lsd_mat(image, keep)
        cap_lists = max(num_octaves, 1) + 1
        ll = np.zeros(cap_lists, np.int32)
        recs = np.zeros(cap, REC_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = self.L.lsdd_line_lbd(num_octaves, float(line_length_thres), member, C.byref(m), ll.ctypes.data, recs.ctypes.data, desc.ctypes.data, cap_lists, cap)
        assert n >= 0, n
        lists = self._lists(n, ll, recs)
        if member != 3:
            return lists, None
        offs = np.concatenate([[0], np.cumsum(ll[:n])]).astype(int)
        return lists, [desc[offs[i]:offs[i + 1]].copy() for i in range(n)]


def same_lists(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (a, b) in enumerate(zip(got, want)):
        assert len(a) == len(b), (what, i, len(a), len(b))
        np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8), err_msg="%s list %d" % (what, i))


def run_both(shim, ref, member, images, scale, num_octaves, masks=None, flag=False, pre=None, same_text=True, what=""):
    """the same call on both libraries: the same lists, bit for bit, the same flag after, the same kind of exception and (same_text) its
    text.  Returns the shim's answer.  The reference's vector overload reads masks[i] and keylines[i] for every image, so the vector form is
    always given one mask (or empty Mat) and one list per image; the drop-in's answers to fewer are checked on their own (check_vector)."""
    if member == VECTOR:
        masks = [None] * len(images) if masks is None else masks
        pre = [np.zeros(0, REC_DTYPE)] * len(images) if pre is None else pre
    got = shim.detect(member, images, scale, num_octaves, masks, flag, pre)
    want = ref.detect(member, images, scale, num_octaves, masks, flag, pre)
    same_lists(got[0], want[0], what)
    assert got[1:3] == want[1:3], (what, got[1:], want[1:])
    if same_text:
        assert got[3] == want[3], (what, got[3], want[3])
    return got


# ---------------------------------------------------------------------------------------------------------------- inputs
def synthetic(w, h, gray, seed=0):
    import cv2
    from cube_slam_b200 import synthetic as S
    img = S.make_batch(w * 3 + h + seed, 1, 640, 480)[0][0]
    if (w, h) != (640, 480):
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
    return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if gray else img)


def box_mask(shape, boxes):
    """a CV_8UC1 mask that is 1 inside the 2-D boxes [x y w h prob] and 0 elsewhere"""
    m = np.zeros(shape[:2], np.uint8)
    for x, y, w, h, _ in boxes:
        x0, y0, x1, y1 = max(int(x), 0), max(int(y), 0), max(int(x + w), 0), max(int(y + h), 0)
        m[y0:y1, x0:x1] = 1
    return m


def random_mask(shape, rng, p=0.5):
    return (rng.random(shape[:2]) < p).astype(np.uint8) * rng.integers(1, 256, shape[:2], dtype=np.uint8)


def prefilled(rng, n, w, h, octave=0):
    """n key lines a caller might already hold: points inside a w x h frame, every field set"""
    r = np.zeros(n, REC_DTYPE)
    r["start_x"], r["end_x"] = rng.uniform(0, w - 1, n), rng.uniform(0, w - 1, n)
    r["start_y"], r["end_y"] = rng.uniform(0, h - 1, n), rng.uniform(0, h - 1, n)
    r["s_oct_x"], r["s_oct_y"], r["e_oct_x"], r["e_oct_y"] = r["start_x"], r["start_y"], r["end_x"], r["end_y"]
    r["angle"] = rng.uniform(-3, 3, n)
    r["line_length"] = rng.uniform(1, 100, n)
    r["response"] = rng.uniform(0, 1, n)
    r["num_pixels"] = rng.integers(1, 100, n)
    r["class_id"] = np.arange(n) + 1000
    r["octave"] = octave
    r["pt_x"], r["pt_y"] = (r["start_x"] + r["end_x"]) / 2, (r["start_y"] + r["end_y"]) / 2
    return r


def checkerboard_vga():
    """640 x 480 checkerboard of 10 px cells: about 2 850 LSD segments in octave 0, past the drop-in's first buffer of 2 048 per octave"""
    from test_oracle_ref_lsd import CHECKERBOARDS, checkerboard
    return checkerboard(*CHECKERBOARDS["vga_10px"])


def as_rec(kl):
    """OCTAVE_KEYLINE_DTYPE records (the Python mirror's) -> the driver's record (pt is the mid point of the two ends, as KeyLine::pt)"""
    r = np.zeros(len(kl), REC_DTYPE)
    for f in REC_DTYPE.names:
        if f not in ("pt_x", "pt_y"):
            r[f] = kl[f]
    r["pt_x"] = (kl["end_x"] + kl["start_x"]) / np.float32(2)
    r["pt_y"] = (kl["end_y"] + kl["start_y"]) / np.float32(2)
    return r


CONFIGS = [(2, 1), (2, 2), (2, 3), (1, 1), (3, 1)]   # (scale, numOctaves)


# ---------------------------------------------------------------------------------------------------------------- checks (GPU and host)
def check_frames(shim, ref, frames, configs=CONFIGS, mirror=None):
    """the flat and per-octave overloads, no mask, equal the reference's; the flat list is the octaves in order, class_id counts each
    octave's lines; every octave found lines; lbd.lsd (mirror) returns the same records"""
    for what, img in frames:
        for scale, K in configs:
            tag = "%s scale %d, %d octaves" % (what, scale, K)
            flat = run_both(shim, ref, FLAT, img, scale, K, what=tag + " flat")[0]
            octs = run_both(shim, ref, OCTAVES, img, scale, K, flag=True, what=tag + " per octave")[0]
            assert len(octs) == K and all(len(o) for o in octs), tag
            same_lists([np.concatenate(octs)], flat, tag + " flat is the octaves in order")
            for k, o in enumerate(octs):
                assert (o["octave"] == k).all() and (o["class_id"] == np.arange(len(o))).all(), tag
            if mirror is not None:
                same_lists([as_rec(p) for p in mirror.detect_octaves(img, scale, K)], octs, tag + " lbd.lsd")
                same_lists([as_rec(mirror.detect(img, scale, K))], flat, tag + " lbd.lsd flat")


def mask_cases(img, boxes, rng):
    shape = img.shape[:2]
    return [("no mask", None), ("all ones", np.ones(shape, np.uint8)), ("all zeros", np.zeros(shape, np.uint8)),
            ("boxes", box_mask(shape, boxes)), ("random", random_mask(shape, rng)), ("random sparse", random_mask(shape, rng, 0.05))]


def check_masks(shim, ref, img, boxes, rng, capfd=None, mirror=None, octaves=(1, 3)):
    """the single overloads with every mask case and pre-filled vectors: the mask rule over new and caller's lines, class_id gaps, the flag
    flips and the messages they print"""
    h, w = img.shape[:2]
    for K in octaves:
        for what, mask in mask_cases(img, boxes, rng):
            tag = "%s, %d octaves" % (what, K)
            pre = [prefilled(rng, 30, w, h)]
            for flag in (False, True):
                if capfd is not None:
                    capfd.readouterr()
                got = run_both(shim, ref, FLAT, img, 2, K, mask, flag=flag, pre=pre, what=tag + " flat")
                assert got[1] is False and got[2] == NO_ERROR
                if capfd is not None:
                    assert capfd.readouterr().out == (FLAG_FALSE_MSG + "\n") * (2 if flag else 0), tag
                    capfd.readouterr()
                # the per-octave overload: the caller's lists (as many as numOctaves, or more) are replaced
                pre_oct = [prefilled(rng, 5, w, h, k) for k in range(K + 1)]
                octs = run_both(shim, ref, OCTAVES, img, 2, K, mask, flag=flag, pre=pre_oct, what=tag + " per octave")[0]
                assert len(octs) == K
                if capfd is not None:
                    assert capfd.readouterr().out == (FLAG_TRUE_MSG + "\n") * (0 if flag else 2), tag
            flat = got[0][0]
            assert (flat[:30].view(np.uint8) == pre[0][:len(flat[:30])].view(np.uint8)).all() or mask is not None, tag
            if mask is not None and what != "all ones":
                full = shim.detect(FLAT, img, 2, K)[0][0]
                assert len(flat) - len(pre[0]) < len(full) or what == "boxes" and len(full) == 0, tag    # the mask removed lines
            if mirror is not None:
                same_lists([as_rec(p) for p in mirror.detect_octaves(img, 2, K, mask)], octs, tag + " lbd.lsd")
                new = shim.detect(FLAT, img, 2, K, mask)[0][0]
                same_lists([as_rec(mirror.detect(img, 2, K, mask))], [new], tag + " lbd.lsd flat")


def check_mask_errors(shim, ref, img, mirror=None):
    """a mask of the wrong size or type: the same exception and text in all three overloads; the vector overload's own text; the flag
    already flipped; nothing appended"""
    h, w = img.shape[:2]
    bad = [("wrong size", np.ones((h - 1, w), np.uint8)), ("wrong type", np.ones((h, w), np.int16)), ("3 channels", np.ones((h, w, 3), np.uint8))]
    pre = [prefilled(np.random.default_rng(5), 4, w, h)]
    for what, m in bad:
        got = run_both(shim, ref, FLAT, img, 2, 1, m, flag=True, pre=pre, what=what)
        assert got[1:] == (False, RUNTIME_ERROR, MASK_MSG), what
        same_lists(got[0], pre, what)
        got = run_both(shim, ref, OCTAVES, img, 2, 2, m, flag=False, pre=pre * 2, what=what)
        assert got[1:] == (True, RUNTIME_ERROR, MASK_MSG), what
        got = run_both(shim, ref, VECTOR, [img], 2, 1, [m], flag=True, pre=pre, what=what)
        assert got[1:] == (False, RUNTIME_ERROR, MASKS_MSG), what
        if mirror is not None:
            import cube_slam_b200 as cs
            with pytest.raises(cs.CubeSlamError, match="Mask error"):
                mirror.detect(img, 2, 1, m)
            with pytest.raises(cs.CubeSlamError, match="Masks error"):
                mirror.detect([img], 2, 1, [m])


def vector_case(frames, rng, n=40):
    """n images of the frames' sizes, gray and BGR interleaved, every third with a mask (random or all zeros), pre-filled lists"""
    import cv2
    imgs, masks, pre = [], [], []
    for i in range(n):
        img = frames[i % len(frames)]
        if (i // len(frames)) % 2:
            img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if img.ndim == 3 else cv2.cvtColor(img, cv2.COLOR_GRAY2BGR)
        imgs.append(np.ascontiguousarray(img))
        masks.append(None if i % 3 else (random_mask(img.shape, rng) if i % 2 else np.zeros(img.shape[:2], np.uint8)))
        pre.append(prefilled(rng, i % 4, img.shape[1], img.shape[0]))
    return imgs, masks, pre


def check_vector(shim, ref, frames, rng, K=2, n=40, mirror=None):
    """the vector overload: n images of several sizes, gray and BGR, some masked, appended to pre-filled lists; then a bad mask at
    position 7: images 0-6 appended, the rest untouched, the vector overload's message"""
    imgs, masks, pre = vector_case(frames, rng, n)
    got = run_both(shim, ref, VECTOR, imgs, 2, K, masks, flag=True, pre=pre, what="vector")
    assert got[1:] == (False, NO_ERROR, "")
    lists = got[0]
    assert all(len(lists[i]) > len(pre[i]) for i in range(n) if masks[i] is None)      # the unmasked images gained lines
    # defined here, undefined in the reference: fewer masks than images (the default empty vector too) leave the rest unmasked, and a
    # keylines vector shorter than the images grows to their number
    unmasked = shim.detect(VECTOR, imgs, 2, K, [None] * n)[0]
    same_lists(shim.detect(VECTOR, imgs, 2, K)[0], unmasked, "no masks")
    same_lists(shim.detect(VECTOR, imgs, 2, K, masks[:1])[0], [shim.detect(FLAT, imgs[0], 2, K, masks[0])[0][0]] + unmasked[1:], "one mask")
    short = shim.detect(VECTOR, imgs, 2, K, [None] * n, pre=pre[:3])[0]
    assert len(short) == n
    same_lists(short[3:], unmasked[3:], "keylines grown")
    if mirror is not None:
        py = mirror.detect(imgs, 2, K, masks)
        for i in range(n):
            new = lists[i][len(pre[i]):] if masks[i] is None else shim.detect(FLAT, imgs[i], 2, K, masks[i])[0][0]
            same_lists([as_rec(py[i])], [new], "lbd.lsd vector image %d" % i)
    bad = list(masks)
    bad[7] = np.ones((5, 5), np.uint8)
    got = run_both(shim, ref, VECTOR, imgs, 2, K, bad, pre=pre, what="bad mask at 7")
    assert got[1:] == (False, RUNTIME_ERROR, MASKS_MSG)
    for i in range(n):
        if i < 7:
            same_lists([got[0][i]], [lists[i]], "image %d appended" % i)
        else:
            same_lists([got[0][i]], [pre[i]], "image %d untouched" % i)
    # a bad image (16 bits) at position 3 stops it the same way
    bad_img = list(imgs)
    bad_img[3] = np.zeros(imgs[3].shape[:2], np.int16)
    got = run_both(shim, ref, VECTOR, bad_img, 2, K, pre=pre, what="16-bit image at 3")
    assert got[1:] == (False, RUNTIME_ERROR, "Error, depth image!= 0")


def check_roi(shim, ref, img):
    """an ROI of a larger frame (rows further apart than the ROI is wide): its lines are those of the same pixels in a frame of their own"""
    roi = img[37:37 + 301, 53:53 + 411]
    assert roi.strides[0] != roi.shape[1] * roi.itemsize * (roi.shape[2] if roi.ndim == 3 else 1)
    for K in (1, 2):
        got = run_both(shim, ref, FLAT, roi, 2, K, what="ROI %d octaves" % K)
        same_lists(got[0], shim.detect(FLAT, np.ascontiguousarray(roi), 2, K)[0], "ROI = its copy")
        assert len(got[0][0])
    imgs = [roi, np.ascontiguousarray(roi), roi]
    got = run_both(shim, ref, VECTOR, imgs, 2, 2, what="ROI in the vector overload")
    same_lists(got[0][:1], got[0][1:2])


def check_counts_and_depth(shim, ref, img, rng):
    """numOctaves 0: nothing detected, the flat overload still masks the caller's lines, the per-octave overload returns no list;
    numOctaves -1: std::length_error; a 16-bit image: "Error, depth image!= 0"; scale 3 with two octaves: std::runtime_error from pyrDown"""
    h, w = img.shape[:2]
    pre = [prefilled(rng, 40, w, h)]
    mask = random_mask(img.shape, rng, 0.3)
    got = run_both(shim, ref, FLAT, img, 2, 0, mask, pre=pre, what="0 octaves")
    assert got[2] == NO_ERROR and 0 < len(got[0][0]) < 40
    got = run_both(shim, ref, OCTAVES, img, 2, 0, pre=pre * 3, what="0 octaves per octave")
    assert got[0] == [] and got[2] == NO_ERROR
    got = run_both(shim, ref, VECTOR, [img, img], 2, 0, pre=pre * 2, what="0 octaves vector")
    same_lists(got[0], pre * 2)
    for member in (FLAT, OCTAVES):
        got = run_both(shim, ref, member, img, 2, -1, pre=pre, what="-1 octaves")
        assert got[2] == LENGTH_ERROR
        same_lists(got[0], pre)
        got = run_both(shim, ref, member, np.zeros((h, w), np.int16), 2, 1, pre=pre, what="16-bit")
        assert got[2:] == (RUNTIME_ERROR, "Error, depth image!= 0")
        got = run_both(shim, ref, member, img, 3, 2, pre=pre, same_text=False, what="scale 3, 2 octaves")
        assert got[2] == RUNTIME_ERROR
        same_lists(got[0], pre)
    got = run_both(shim, ref, VECTOR, [img, img], 2, -1, pre=pre * 2, what="-1 octaves vector")
    assert got[2] == LENGTH_ERROR


def check_outside_points_are_kept(shim, img):
    """defined here, undefined in the reference: a caller's line with an end point outside the mask keeps that point from reading 0"""
    h, w = img.shape[:2]
    pre = prefilled(np.random.default_rng(9), 4, w, h)
    pre["start_x"][0], pre["end_x"][0] = -5, w + 3          # both ends outside: kept
    pre["start_x"][1], pre["start_y"][1] = w + 1, h + 1      # one end outside, the other inside at a 0: kept
    pre["start_y"][2], pre["end_y"][2] = 2, 3                # both inside at a 0: erased
    pre["start_x"][3], pre["start_y"][3] = -0.5, -0.5        # (int) of -0.5 is 0: inside, at a 0; the other end too: erased
    got = shim.detect(FLAT, img, 2, 0, np.zeros((h, w), np.uint8), pre=[pre])
    same_lists(got[0], [pre[:2]])


def check_capacity(shim, ref):
    """a frame whose octave 0 holds more LSD segments than the drop-in's first buffer: answered in full, as by the reference"""
    board = checkerboard_vga()
    for K in (1, 2):
        got = run_both(shim, ref, FLAT, board, 2, K, what="checkerboard %d octaves" % K)
        assert got[2] == NO_ERROR and len(got[0][0]) > 2048


def check_line_lbd(shim, ref, img, octaves=(1, 2, 3)):
    """the reference's own line_lbd_detect(numoctaves, 2.0) with use_LSD, unchanged, over the drop-in: detect_raw_lines (both KeyLine
    overloads), detect_filter_lines and detect_descrip_lines_octaves (key lines and LBD descriptors) equal the all-reference build"""
    for K in octaves:
        for member in range(4):
            got, gd = shim.line_lbd(K, member, img)
            want, wd = ref.line_lbd(K, member, img)
            same_lists(got, want, "line_lbd_detect(%d) member %d" % (K, member))
            assert sum(map(len, got)), (K, member)
            if member == 3:
                for a, b in zip(gd, wd):
                    np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------- GPU tests
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def libs():
    if not (os.path.exists(SHIM) and os.path.exists(REF)):
        pytest.skip("oracle/_ref/libshim_lsd.so and libref_lsd_detector.so are built by build() where the reference checkout exists")
    shim, ref = Driver(SHIM), Driver(REF)
    shim.L.lsdd_cout_on()
    ref.L.lsdd_cout_on()
    return shim, ref


@pytest.fixture(scope="module")
def mirror():
    import cube_slam_b200 as cs
    return cs.line_lbd_detect(1, 1.0).lsd


def test_frames_octaves_and_scales(libs, mirror, fixture_a):
    """fixture A and synthetic VGA, odd-sized and KITTI-sized frames, BGR and gray; numOctaves 1-3 at scale 2, numOctaves 1 at scales 1, 3"""
    out = [("fixture A", fixture_a["img"])]
    for w, h in ((640, 480), (211, 97), (333, 251), (1242, 375)):
        for gray in (False, True):
            out.append(("%dx%d %s" % (w, h, "gray" if gray else "BGR"), synthetic(w, h, gray)))
    check_frames(*libs, out, mirror=mirror)


def test_fixture_b_every_frame_through_the_vector_overload(libs, fixture_b):
    """the 58 fixture-B frames in one vector call (one batch) at 1 and 3 octaves, each frame masked by its own 2-D boxes, against the
    reference's per-image loop; and each frame alone through the flat overload at 2 octaves"""
    shim, ref = libs
    imgs = [f[0] for f in fixture_b["frames"]]
    masks = [box_mask(f[0].shape, f[1]) if len(f[1]) else None for f in fixture_b["frames"]]
    for K in (1, 3):
        got = run_both(shim, ref, VECTOR, imgs, 2, K, what="fixture B, %d octaves" % K)
        assert all(len(l) for l in got[0])
        run_both(shim, ref, VECTOR, imgs, 2, K, masks, what="fixture B boxes, %d octaves" % K)
    check_frames(shim, ref, [("fixture B %d" % i, img) for i, img in enumerate(imgs)], configs=[(2, 2)])


def test_masks_prefilled_vectors_and_flags(libs, mirror, fixture_b, capfd):
    rng = np.random.default_rng(11)
    for i in (0, 17, 40):
        img, boxes = fixture_b["frames"][i]
        check_masks(*libs, img, boxes, rng, capfd=capfd, mirror=mirror)


def test_mask_errors(libs, mirror, fixture_a):
    check_mask_errors(*libs, fixture_a["img"], mirror=mirror)


def test_vector_overload_mixed_sizes_and_a_bad_mask(libs, mirror):
    frames = [synthetic(640, 480, False, 1), synthetic(333, 251, True, 2), synthetic(1242, 375, False, 3)]
    check_vector(*libs, frames, np.random.default_rng(12), K=2, n=40, mirror=mirror)


def test_roi(libs, fixture_a):
    check_roi(*libs, fixture_a["img"])


def test_octave_counts_depth_and_scale(libs, mirror, fixture_a):
    import cube_slam_b200 as cs
    check_counts_and_depth(*libs, fixture_a["img"], np.random.default_rng(13))
    check_outside_points_are_kept(libs[0], fixture_a["img"])
    img = fixture_a["img"]
    assert mirror.detect_octaves(img, 2, 0) == [] and len(mirror.detect(img, 2, 0)) == 0
    for args in ((img, 2, -1), (img, 3, 2), (np.zeros((40, 40), np.int16), 2, 1)):
        with pytest.raises(cs.CubeSlamError):
            mirror.detect(*args)


def test_textured_frame_overflows_the_first_buffer(libs, mirror):
    check_capacity(*libs)
    board = checkerboard_vga()
    flat = libs[0].detect(FLAT, board, 2, 1)[0]
    same_lists([as_rec(mirror.detect(board, 2, 1))], flat, "lbd.lsd checkerboard")


def test_smallest_octave_too_small(libs):
    """a 24 x 200 frame with 5 octaves: its octave 4 is 1 x 12, below what LSD's 0.8 scaling runs on.  The reference answers the lines of
    the other octaves (none in octave 4); the drop-in refuses with the C ABI's message"""
    shim, ref = libs
    img = np.ascontiguousarray(synthetic(640, 480, True)[:200, 100:124])
    want = ref.detect(OCTAVES, img, 2, 5, flag=True)
    assert want[2] == NO_ERROR and len(want[0]) == 5 and len(want[0][4]) == 0
    got = shim.detect(OCTAVES, img, 2, 5, flag=True)
    assert got[2] == RUNTIME_ERROR and "too small for LSD" in got[3]


def test_two_threads_at_once(libs, fixture_a):
    shim, ref = libs
    imgs = [fixture_a["img"], synthetic(640, 480, True, 4)]
    got = shim.threads(imgs, 2, repeat=3)
    for i, img in enumerate(imgs):
        same_lists([got[i]], ref.detect(FLAT, img, 2, 2)[0], "thread %d" % i)


def test_reference_line_lbd_detect_over_the_drop_in(libs, fixture_a):
    check_line_lbd(*libs, fixture_a["img"])
    check_line_lbd(*libs, synthetic(640, 480, True, 5), octaves=(2,))
