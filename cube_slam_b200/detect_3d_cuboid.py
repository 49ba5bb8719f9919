"""Host-side mirror of the reference's cuboid-detector interface, driving libcubeslam_b200.so.

Mirrors `class detect_3d_cuboid` / `class cuboid` (detect_3d_cuboid/include/detect_3d_cuboid/detect_3d_cuboid.h:15-80):
same member names, argument meaning and "print and continue" error behaviour, so that the parity tests
read like calls into the reference.  All numerical work is done by the CUDA library through its C ABI.
"""
import ctypes as C

import weakref

import numpy as np

from . import _lib
from ._lib import CUBOID_DTYPE, BatchStats, CuboidParams


class CubeSlamError(RuntimeError):
    pass


class cuboid(object):
    """class cuboid (detect_3d_cuboid.h:15-36) populated from one cs_cuboid_rec."""

    __slots__ = ("pos", "scale", "rotY", "box_config_type", "box_corners_2d", "box_corners_3d_world", "rect_detect_2d",
                 "edge_distance_error", "edge_angle_error", "normalized_error", "skew_ratio", "down_expand_height",
                 "camera_roll_delta", "camera_pitch_delta", "combined_score", "proposal_index", "height_sample_id")

    def __init__(self, rec):
        for name in self.__slots__:
            v = rec[name]
            setattr(self, name, v.copy() if isinstance(v, np.ndarray) else v.item())

    def print_cuboid(self):  # object_3d_util.cpp:28-39
        print("printing cuboids info....")
        print("pos   ", self.pos)
        print("scale   ", self.scale)
        print("rotY   ", self.rotY)
        print("box_config_type   ", self.box_config_type)
        print("box_corners_2d \n", self.box_corners_2d)
        print("box_corners_3d_world \n", self.box_corners_3d_world)


class cam_pose_infos(object):
    """struct cam_pose_infos (detect_3d_cuboid.h:39-51), the members callers read."""

    def __init__(self):
        self.transToWolrd = np.eye(4)
        self.Kalib = np.eye(3)
        self.euler_angle = np.zeros(3)
        self.KinvR = np.eye(3)
        self.camera_yaw = 0.0


class Context(object):
    """Owns one cs_ctx (one CUDA stream + device workspace).  One per host thread."""

    def __init__(self, device=0, max_width=1280, max_height=960, max_frames=1, max_boxes_per_frame=16, max_lines_per_frame=4096):
        self._dependents = weakref.WeakSet()   # objects holding library state made on this context (descriptor collections)
        self.L = _lib.load()
        self.h = self.L.cs_create(device, max_width, max_height, max_frames, max_boxes_per_frame, max_lines_per_frame)
        if not self.h:
            raise CubeSlamError("cs_create failed: no usable CUDA device %d (cube_slam_b200 has no CPU path)" % device)
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            for obj in list(getattr(self, "_dependents", ())):   # the C ABI wants them released before the context
                obj._release()
            self.L.cs_destroy(self.h)
            self.h = None

    def _depend(self, obj):
        """obj._release() frees what obj made on this context; close() calls it first"""
        self._dependents.add(obj)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc):
        if rc != 0:
            raise CubeSlamError("%s: %s" % (_lib.STATUS_NAMES.get(rc, rc), self.L.cs_last_error(self.h).decode()))

    # -- batch plumbing ------------------------------------------------------------------------
    @staticmethod
    def _pack(imgs, Ts, boxes_list, lines_list):
        imgs = np.ascontiguousarray(imgs, np.uint8)
        if imgs.ndim == 3:  # F x H x W gray
            F, H, W = imgs.shape
            ch = 1
        else:
            F, H, W, ch = imgs.shape
        Ts, boxes, box_off, lines, line_off = Context._pack_tables(F, Ts, boxes_list, lines_list)
        return imgs, F, H, W, ch, Ts, boxes, box_off, lines, line_off

    @staticmethod
    def _pack_tables(F, Ts, boxes_list, lines_list):
        Ts = np.ascontiguousarray(Ts, np.float64).reshape(F, 16)
        box_off = np.zeros(F + 1, np.int32)
        line_off = np.zeros(F + 1, np.int32)
        bl, ll = [], []
        for f in range(F):
            b = np.asarray(boxes_list[f], np.float64).reshape(-1, 5)
            l = np.asarray(lines_list[f], np.float64).reshape(-1, 4)
            bl.append(b)
            ll.append(l)
            box_off[f + 1] = box_off[f] + len(b)
            line_off[f + 1] = line_off[f] + len(l)
        boxes = np.ascontiguousarray(np.concatenate(bl) if bl else np.zeros((0, 5)))
        lines = np.ascontiguousarray(np.concatenate(ll) if ll else np.zeros((0, 4)))
        if len(boxes) == 0:
            boxes = np.zeros((1, 5))
        if len(lines) == 0:
            lines = np.zeros((1, 4))
        return Ts, boxes, box_off, lines, line_off

    def set_calibration(self, K):
        K = np.ascontiguousarray(K, np.float64).reshape(9)
        self.check(self.L.cs_set_calibration(self.h, _lib.ptr(K, C.c_double)))

    def upload(self, imgs, Ts, boxes_list, lines_list, params):
        imgs, F, H, W, ch, Ts, boxes, box_off, lines, line_off = self._pack(imgs, Ts, boxes_list, lines_list)
        self._n_obj = int(box_off[-1])
        self._topk = int(params.max_cuboid_num)
        self._box_off = box_off
        self.check(self.L.cs_batch_upload(self.h, imgs.ctypes.data, F, W, H, W * ch, ch, _lib.ptr(Ts, C.c_double),
                                          _lib.ptr(boxes, C.c_double), _lib.ptr(box_off, C.c_int32),
                                          _lib.ptr(lines, C.c_double), _lib.ptr(line_off, C.c_int32), C.byref(params)))

    def upload_online(self, imgs, Ts, boxes_list, line_params, params):
        """cs_batch_upload_online: no input lines, cs_batch_run detects them on the resident frames first."""
        F = len(imgs)
        imgs, F, H, W, ch, Ts, boxes, box_off, _, _ = self._pack(imgs, Ts, boxes_list, [np.zeros((0, 4))] * F)
        self._n_obj = int(box_off[-1])
        self._topk = int(params.max_cuboid_num)
        self._box_off = box_off
        self.check(self.L.cs_batch_upload_online(self.h, imgs.ctypes.data, F, W, H, W * ch, ch, _lib.ptr(Ts, C.c_double),
                                                 _lib.ptr(boxes, C.c_double), _lib.ptr(box_off, C.c_int32), C.byref(line_params), C.byref(params)))

    def upload_device(self, frames, Ts, boxes_list, lines_list, params, order="bgr", stream=None):
        """cs_batch_upload_device: upload() with frames already on the GPU -- any object with __cuda_array_interface__ (a torch CUDA tensor, a
        CuPy array), uint8, (N, H, W, 3) or (N, H, W), any strides.  order: "bgr" or "rgb".  stream: the stream the frames were written on
        (torch.cuda.Stream or raw handle; default: torch's current stream for a torch tensor, else the interface's, else the legacy default
        stream).  Returns without blocking the host; work queued on that stream afterwards waits until the library has read the frames."""
        fr = _lib.device_frames(frames, order, stream)
        F = fr.n_frames
        Ts, boxes, box_off, lines, line_off = self._pack_tables(F, Ts, boxes_list, lines_list)
        self._n_obj = int(box_off[-1])
        self._topk = int(params.max_cuboid_num)
        self._box_off = box_off
        self.check(self.L.cs_batch_upload_device(self.h, C.byref(fr), _lib.ptr(Ts, C.c_double), _lib.ptr(boxes, C.c_double),
                                                 _lib.ptr(box_off, C.c_int32), _lib.ptr(lines, C.c_double), _lib.ptr(line_off, C.c_int32),
                                                 C.byref(params)))

    def upload_online_device(self, frames, Ts, boxes_list, line_params, params, order="bgr", stream=None):
        """cs_batch_upload_online_device: upload_online() with frames already on the GPU (see upload_device)."""
        fr = _lib.device_frames(frames, order, stream)
        F = fr.n_frames
        Ts, boxes, box_off, _, _ = self._pack_tables(F, Ts, boxes_list, [np.zeros((0, 4))] * F)
        self._n_obj = int(box_off[-1])
        self._topk = int(params.max_cuboid_num)
        self._box_off = box_off
        self.check(self.L.cs_batch_upload_online_device(self.h, C.byref(fr), _lib.ptr(Ts, C.c_double), _lib.ptr(boxes, C.c_double),
                                                        _lib.ptr(box_off, C.c_int32), C.byref(line_params), C.byref(params)))

    # -- frames of different sizes and cameras ----------------------------------------------------
    @staticmethod
    def _pack_mixed(imgs, Ts, boxes_list, lines_list, K):
        """imgs: a list of H x W or H x W x 3 uint8 arrays of any sizes; K: None (the context's calibration), one 3 x 3 matrix or F x 3 x 3"""
        F = len(imgs)
        buf, views = _lib.pack_frames(imgs)
        Ts, boxes, box_off, lines, line_off = Context._pack_tables(F, Ts, boxes_list, lines_list)
        if K is not None:
            K = np.asarray(K, np.float64)
            K = np.ascontiguousarray(np.broadcast_to(K.reshape(3, 3), (F, 3, 3)) if K.size == 9 else K.reshape(F, 9)).reshape(F, 9)
        return buf, views, F, Ts, boxes, box_off, lines, line_off, K

    def _mixed_call(self, name, imgs, Ts, boxes_list, lines_list, line_params, params, K, out):
        buf, views, F, Ts, boxes, box_off, lines, line_off, K = self._pack_mixed(imgs, Ts, boxes_list, lines_list, K)
        n_obj, topk = int(box_off[-1]), int(params.max_cuboid_num)
        Kp = None if K is None else _lib.ptr(K, C.c_double)
        args = [self.h, buf.ctypes.data, views, F, Kp, _lib.ptr(Ts, C.c_double), _lib.ptr(boxes, C.c_double), _lib.ptr(box_off, C.c_int32)]
        args += [C.byref(line_params)] if line_params is not None else [_lib.ptr(lines, C.c_double), _lib.ptr(line_off, C.c_int32)]
        args.append(C.byref(params))
        if out:
            rec, counts = np.zeros((max(n_obj, 1), topk), CUBOID_DTYPE), np.zeros(max(n_obj, 1), np.int32)
            args += [rec.ctypes.data, _lib.ptr(counts, C.c_int32)]
        self.check(getattr(self.L, name)(*args))
        self._n_obj, self._topk, self._box_off = n_obj, topk, box_off
        return (rec[:n_obj], counts[:n_obj]) if out else None

    def upload_mixed(self, imgs, Ts, boxes_list, lines_list, params, K=None):
        """cs_batch_upload_mixed: upload() over a list of frames of any sizes, each with its own calibration (K: None, 3 x 3 or F x 3 x 3)."""
        self._mixed_call("cs_batch_upload_mixed", imgs, Ts, boxes_list, lines_list, None, params, K, False)

    def upload_online_mixed(self, imgs, Ts, boxes_list, line_params, params, K=None):
        """cs_batch_upload_online_mixed: upload_online() over a list of frames of any sizes and calibrations."""
        self._mixed_call("cs_batch_upload_online_mixed", imgs, Ts, boxes_list, [np.zeros((0, 4))] * len(imgs), line_params, params, K, False)

    def detect_batch_mixed(self, imgs, Ts, boxes_list, lines_list, params, K=None):
        """cs_detect_cuboids_batch_mixed: detect_batch_host() over a list of frames of any sizes and calibrations -> (records, counts)."""
        return self._mixed_call("cs_detect_cuboids_batch_mixed", imgs, Ts, boxes_list, lines_list, None, params, K, True)

    def detect_frames_mixed(self, imgs, Ts, boxes_list, line_params, params, K=None):
        """cs_detect_frames_batch_mixed: detect_frames_host() over a list of frames of any sizes and calibrations -> (records, counts)."""
        return self._mixed_call("cs_detect_frames_batch_mixed", imgs, Ts, boxes_list, [np.zeros((0, 4))] * len(imgs), line_params, params, K, True)

    def detect_frames_host(self, imgs, Ts, boxes_list, line_params, params, out=None, counts=None):
        """cs_detect_frames_batch: detect_filter_lines + detect_cuboid per frame, host buffers in / out."""
        F = len(imgs)
        imgs, F, H, W, ch, Ts, boxes, box_off, _, _ = self._pack(imgs, Ts, boxes_list, [np.zeros((0, 4))] * F)
        n_obj = int(box_off[-1])
        topk = int(params.max_cuboid_num)
        if out is None:
            out = np.zeros((max(n_obj, 1), topk), CUBOID_DTYPE)
            counts = np.zeros(max(n_obj, 1), np.int32)
        self.check(self.L.cs_detect_frames_batch(self.h, imgs.ctypes.data, F, W, H, W * ch, ch, _lib.ptr(Ts, C.c_double),
                                                 _lib.ptr(boxes, C.c_double), _lib.ptr(box_off, C.c_int32), C.byref(line_params),
                                                 C.byref(params), out.ctypes.data, _lib.ptr(counts, C.c_int32)))
        self._n_obj, self._topk, self._box_off = n_obj, topk, box_off
        return out[:n_obj], counts[:n_obj]

    def run(self):
        self.check(self.L.cs_batch_run(self.h))

    def run_async(self):
        self.check(self.L.cs_batch_run_async(self.h))

    def fetch(self):
        n = max(self._n_obj, 1)
        out = np.zeros((n, self._topk), CUBOID_DTYPE)
        counts = np.zeros(n, np.int32)
        self.check(self.L.cs_batch_fetch(self.h, out.ctypes.data, _lib.ptr(counts, C.c_int32)))
        return out[:self._n_obj], counts[:self._n_obj]

    def detect_batch_host(self, imgs, Ts, boxes_list, lines_list, params, out=None, counts=None):
        """cs_detect_cuboids_batch: host buffers in, host records out (H2D + kernels + D2H)."""
        imgs, F, H, W, ch, Ts, boxes, box_off, lines, line_off = self._pack(imgs, Ts, boxes_list, lines_list)
        n_obj = int(box_off[-1])
        topk = int(params.max_cuboid_num)
        if out is None:
            out = np.zeros((max(n_obj, 1), topk), CUBOID_DTYPE)
            counts = np.zeros(max(n_obj, 1), np.int32)
        self.check(self.L.cs_detect_cuboids_batch(self.h, imgs.ctypes.data, F, W, H, W * ch, ch, _lib.ptr(Ts, C.c_double),
                                                  _lib.ptr(boxes, C.c_double), _lib.ptr(box_off, C.c_int32),
                                                  _lib.ptr(lines, C.c_double), _lib.ptr(line_off, C.c_int32), C.byref(params),
                                                  out.ctypes.data, _lib.ptr(counts, C.c_int32)))
        self._n_obj, self._topk, self._box_off = n_obj, topk, box_off
        return out[:n_obj], counts[:n_obj]

    def stats(self):
        s = BatchStats()
        self.check(self.L.cs_batch_stats_get(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in BatchStats._fields_}

    def set_profiling(self, on=True):
        self.check(self.L.cs_set_profiling(self.h, int(on)))

    def stage_ms(self):
        out = {}
        for name in ("lsd", "gray", "canny", "hyst", "dt", "lines", "sweep", "fuse", "total"):
            v = C.c_float(0)
            self.check(self.L.cs_stage_ms(self.h, name.encode(), C.byref(v)))
            out[name] = v.value
        return out

    def stream(self):
        return self.L.cs_stream(self.h)

    def device_records(self):
        p = C.c_void_p()
        n = C.c_size_t()
        self.check(self.L.cs_batch_device_records(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def debug_roi(self, job, cap_px=1 << 21, cap_lines=256):
        roi = np.zeros(4, np.int32)
        self.check(self.L.cs_debug_roi(self.h, job, _lib.ptr(roi, C.c_int32), None, None, 0, None, 0, None, None))
        w, h = int(roi[2]), int(roi[3])
        canny = np.zeros(w * h, np.uint8)
        dist = np.zeros(w * h, np.float32)
        ml = np.zeros((cap_lines, 4))
        n_in = C.c_int32()
        n_m = C.c_int32()
        self.check(self.L.cs_debug_roi(self.h, job, _lib.ptr(roi, C.c_int32), _lib.ptr(canny, C.c_uint8), _lib.ptr(dist, C.c_float),
                                       w * h, _lib.ptr(ml, C.c_double), cap_lines, C.byref(n_in), C.byref(n_m)))
        return dict(roi=tuple(int(v) for v in roi), canny=canny.reshape(h, w), dist=dist.reshape(h, w),
                    n_lines_roi=n_in.value, n_lines_merged=n_m.value, merged_lines=ml[:n_m.value].copy())

    def debug_candidates(self, job):
        n = C.c_int32()
        self.check(self.L.cs_debug_candidates(self.h, job, C.byref(n), None, None, None, 0))
        valid = np.zeros(max(n.value, 1), np.uint8)
        de = np.zeros(max(n.value, 1))
        ae = np.zeros(max(n.value, 1))
        self.check(self.L.cs_debug_candidates(self.h, job, C.byref(n), _lib.ptr(valid, C.c_uint8), _lib.ptr(de, C.c_double),
                                              _lib.ptr(ae, C.c_double), n.value))
        return dict(n=n.value, valid=valid[:n.value], dist_err=de[:n.value], angle_err=ae[:n.value])


def cuboid_measurement(rec, cam_t, cam_q_xyzw, cam_euler_raw=None):
    """object_slam/src/main_obj.cpp:455-473,505: the cuboid record as a measurement in the camera frame.
    Returns (t[3], q_xyzw[4], scale[3], meas_quality).  cam_euler_raw = cam_pose_raw.euler_angle when roll / pitch were sampled."""
    L = _lib.load()
    rec = np.ascontiguousarray(np.asarray(rec).reshape(-1)[:1])
    t, q, s = np.zeros(3), np.zeros(4), np.zeros(3)
    qual = C.c_double()
    e = None if cam_euler_raw is None else _lib.ptr(np.ascontiguousarray(cam_euler_raw, np.float64), C.c_double)
    rc = L.cs_cuboid_measurement(rec.ctypes.data, _lib.ptr(np.ascontiguousarray(cam_t, np.float64), C.c_double),
                                 _lib.ptr(np.ascontiguousarray(cam_q_xyzw, np.float64), C.c_double), e, _lib.ptr(t, C.c_double),
                                 _lib.ptr(q, C.c_double), _lib.ptr(s, C.c_double), C.byref(qual))
    if rc != 0:
        raise CubeSlamError(_lib.STATUS_NAMES.get(rc, str(rc)))
    return t, q, s, qual.value


def cuboid_draw_edges(rec):
    """The 12 edges plot_image_with_cuboid draws for a cuboid record (object_3d_util.cpp:54-131): 12 x 8 int32 rows
    [x1 y1 x2 y2 B G R thickness]."""
    L = _lib.load()
    rec = np.ascontiguousarray(np.asarray(rec).reshape(-1)[:1])
    edges = np.zeros((12, 8), np.int32)
    rc = L.cs_cuboid_draw_edges(rec.ctypes.data, _lib.ptr(edges, C.c_int32))
    if rc != 0:
        raise CubeSlamError(_lib.STATUS_NAMES.get(rc, str(rc)))
    return edges


def plot_image_with_cuboid(plot_img, rec):
    """plot_image_with_cuboid (object_3d_util.cpp:126-131): draws the cuboid into plot_img in place with the reference's own call,
    cv::line(img, p1, p2, colour, thickness, CV_AA, 0)."""
    import cv2
    for x1, y1, x2, y2, b, g, r, th in cuboid_draw_edges(rec):
        cv2.line(plot_img, (int(x1), int(y1)), (int(x2), int(y2)), (int(b), int(g), int(r)), int(th), cv2.LINE_AA, 0)
    return plot_img


def default_params(**kw):
    p = CuboidParams()
    _lib.load().cs_default_cuboid_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class detect_3d_cuboid(object):
    """Drop-in mirror of `class detect_3d_cuboid` (detect_3d_cuboid.h:53-80).

    detect_cuboid(rgb_img, transToWolrd, obj_bbox_coors, edges) returns all_object_cuboids: a list (one
    ObjectSet per 2D box) of lists of `cuboid`, best first -- what the reference fills through its last
    reference argument (box_proposal_detail.cpp:56-57)."""

    def __init__(self, device=0, max_width=1280, max_height=960, max_boxes=64, max_lines=8192):
        self.cam_pose = cam_pose_infos()
        self.cam_pose_raw = cam_pose_infos()
        self.whether_plot_detail_images = False
        self.whether_plot_final_images = False
        self.whether_save_final_images = False
        self.cuboids_2d_img = None
        self.print_details = False
        self.consider_config_1 = True
        self.consider_config_2 = True
        self.whether_sample_cam_roll_pitch = False
        self.whether_sample_bbox_height = False
        self.max_cuboid_num = 1
        self.nominal_skew_ratio = 1.0
        self.max_cut_skew = 3.0
        self._ctx = Context(device, max_width, max_height, 1, max_boxes, max_lines)
        # the class mirror keeps the reference's semantics to the letter: with whether_sample_cam_roll_pitch, later boxes of a frame start
        # from the cam_pose the earlier ones left (cs_set_profiling bit 10, one pass per box rank; DESIGN.md section 2).  A frame with a
        # single box -- all object_slam ever passes -- takes the ordinary one-pass path either way.
        self._ctx.check(self._ctx.L.cs_set_profiling(self._ctx.h, 1024))
        self._K = None

    def params(self):
        return default_params(consider_config_1=int(self.consider_config_1), consider_config_2=int(self.consider_config_2),
                              whether_sample_cam_roll_pitch=int(self.whether_sample_cam_roll_pitch),
                              whether_sample_bbox_height=int(self.whether_sample_bbox_height),
                              max_cuboid_num=int(self.max_cuboid_num), nominal_skew_ratio=float(self.nominal_skew_ratio),
                              max_cut_skew=float(self.max_cut_skew))

    def set_calibration(self, Kalib):  # box_proposal_detail.cpp:36-40
        self._K = np.ascontiguousarray(Kalib, np.float64).reshape(3, 3)
        self.cam_pose.Kalib = self._K.copy()
        self._ctx.set_calibration(self._K)

    def set_cam_pose(self, transToWolrd):  # box_proposal_detail.cpp:42-54
        T = np.ascontiguousarray(transToWolrd, np.float64).reshape(4, 4)
        e = np.zeros(3)
        kr = np.zeros(9)
        rc = self._ctx.L.cs_cam_pose(_lib.ptr(self._K.reshape(9), C.c_double), _lib.ptr(T.reshape(16), C.c_double),
                                     _lib.ptr(e, C.c_double), _lib.ptr(kr, C.c_double))
        self._ctx.check(rc)
        self.cam_pose.transToWolrd = T.copy()
        self.cam_pose.euler_angle = e
        self.cam_pose.KinvR = kr.reshape(3, 3)
        self.cam_pose.camera_yaw = float(e[2])

    def detect_cuboid(self, rgb_img, transToWolrd, obj_bbox_coors, edges):
        if self._K is None:
            raise CubeSlamError("set_calibration has not been called")
        self.set_cam_pose(transToWolrd)
        raw = cam_pose_infos()
        raw.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.cam_pose.__dict__.items()})
        self.cam_pose_raw = raw
        boxes = np.asarray(obj_bbox_coors, np.float64).reshape(-1, 5)
        if len(boxes) == 0:  # empty bbox matrix => empty output (box_proposal_detail.cpp:71-72)
            return []
        img = np.ascontiguousarray(rgb_img, np.uint8)
        out, counts = self._ctx.detect_batch_host(img[None], np.asarray(transToWolrd, np.float64).reshape(1, 16), [boxes],
                                                  [np.asarray(edges, np.float64).reshape(-1, 4)], self.params())
        res = [[cuboid(out[i, k]) for k in range(counts[i])] for i in range(len(boxes))]
        if self.whether_save_final_images and img.ndim == 3:  # box_proposal_detail.cpp:541-556 (callers read cuboids_2d_img, main_obj.cpp:450)
            frame_all_cubes_img = img.copy()
            for i in range(len(boxes)):
                if counts[i]:
                    plot_image_with_cuboid(frame_all_cubes_img, out[i, 0])
            self.cuboids_2d_img = frame_all_cubes_img
        return res
