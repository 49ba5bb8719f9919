"""ctypes binding of libcubeslam_b200.so (the C ABI declared in include/cube_slam_b200.h).

The library is the product; there is no Python or CPU fallback.  If the shared object is missing or
no CUDA device is usable, loading / cs_create fails loudly.
"""
import ctypes as C
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcubeslam_b200.so")

CS_OK = 0
STATUS_NAMES = {0: "CS_OK", -1: "CS_ERR_INVALID_ARG", -2: "CS_ERR_CUDA", -3: "CS_ERR_CAPACITY",
                -4: "CS_ERR_NOT_PREPARED", -5: "CS_ERR_NCCL", -6: "CS_ERR_UNSUPPORTED"}


class CuboidParams(C.Structure):
    """cs_cuboid_params: detect_3d_cuboid's mode members + detect_cuboid's hard-coded locals."""
    _fields_ = [
        ("consider_config_1", C.c_int32), ("consider_config_2", C.c_int32),
        ("whether_sample_cam_roll_pitch", C.c_int32), ("whether_sample_bbox_height", C.c_int32),
        ("max_cuboid_num", C.c_int32), ("reweight_edge_distance", C.c_int32),
        ("whether_normalize_two_errors", C.c_int32), ("top_sample_count_override", C.c_int32),
        ("nominal_skew_ratio", C.c_double), ("max_cut_skew", C.c_double),
        ("vp12_edge_angle_thre", C.c_double), ("vp3_edge_angle_thre", C.c_double),
        ("shorted_edge_thre", C.c_double), ("weight_vp_angle", C.c_double), ("weight_skew_error", C.c_double),
        ("pre_merge_dist_thre", C.c_double), ("pre_merge_angle_thre", C.c_double),
        ("edge_length_threshold", C.c_double), ("canny_low", C.c_double), ("canny_high", C.c_double),
        ("yaw_half_range_deg", C.c_double), ("yaw_step_deg", C.c_double),
    ]


class LineParams(C.Structure):
    _fields_ = [("use_LSD", C.c_int32), ("numoctaves", C.c_int32), ("octaveratio", C.c_float),
                ("line_length_thres", C.c_float)]


class BatchStats(C.Structure):
    _fields_ = [("n_frames", C.c_int64), ("n_objects", C.c_int64), ("n_roi_jobs", C.c_int64),
                ("n_candidates", C.c_int64), ("n_valid", C.c_int64), ("n_kernel_launches", C.c_int64),
                ("roi_pixels", C.c_int64), ("n_lines_in", C.c_int64)]


# numpy view of cs_cuboid_rec (512 bytes)
CUBOID_DTYPE = np.dtype([
    ("pos", "f8", 3), ("scale", "f8", 3), ("rotY", "f8"), ("box_config_type", "f8", 2),
    ("box_corners_2d", "i4", (2, 8)), ("box_corners_3d_world", "f8", (3, 8)),
    ("rect_detect_2d", "f8", 4), ("edge_distance_error", "f8"), ("edge_angle_error", "f8"),
    ("normalized_error", "f8"), ("skew_ratio", "f8"), ("down_expand_height", "f8"),
    ("camera_roll_delta", "f8"), ("camera_pitch_delta", "f8"), ("combined_score", "f8"),
    ("proposal_index", "i4"), ("height_sample_id", "i4"), ("valid", "i4"), ("pad_", "i4"),
])

# numpy views of cs_keyline (40 bytes) and cs_dmatch (16 bytes)
KEYLINE_DTYPE = np.dtype([("start_x", "f4"), ("start_y", "f4"), ("end_x", "f4"), ("end_y", "f4"), ("angle", "f4"), ("line_length", "f4"),
                          ("response", "f4"), ("size", "f4"), ("num_pixels", "i4"), ("class_id", "i4")])
DMATCH_DTYPE = np.dtype([("query_idx", "i4"), ("train_idx", "i4"), ("img_idx", "i4"), ("distance", "f4")])
# numpy view of cs_keyline_octave (64 bytes): KEYLINE_DTYPE's fields, then the in-octave end points and the octave
OCTAVE_KEYLINE_DTYPE = np.dtype(KEYLINE_DTYPE.descr + [("s_oct_x", "f4"), ("s_oct_y", "f4"), ("e_oct_x", "f4"), ("e_oct_y", "f4"), ("octave", "i4"),
                                                        ("pad_", "i4")])

class DeviceFrames(C.Structure):
    """cs_device_frames: n_frames x height x width x channels bytes in device memory, byte strides."""
    _fields_ = [("data", C.c_void_p), ("n_frames", C.c_int32), ("height", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32),
                ("stride_frame", C.c_int64), ("stride_row", C.c_int64), ("stride_col", C.c_int64), ("stride_channel", C.c_int64),
                ("channel_order", C.c_int32), ("stream", C.c_void_p)]


ORDERS = {"bgr": 0, "rgb": 1}   # CS_ORDER_BGR, CS_ORDER_RGB


class FrameView(C.Structure):
    """cs_frame_view: one frame of a batch of frames of different sizes, `offset` bytes from the batch's base pointer."""
    _fields_ = [("offset", C.c_int64), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32), ("channels", C.c_int32)]


def pack_frames(imgs):
    """H x W gray or H x W x 3 uint8 images -> (one contiguous byte buffer, FrameView array) for the *_mixed calls"""
    views = (FrameView * len(imgs))()
    parts, off = [], 0
    for i, a in enumerate(imgs):
        a = np.ascontiguousarray(a, np.uint8)
        ch = 1 if a.ndim == 2 else a.shape[2]
        views[i].offset, views[i].height, views[i].width, views[i].channels = off, a.shape[0], a.shape[1], ch
        views[i].stride = a.shape[1] * ch
        parts.append(a.reshape(-1))
        off += a.size
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8), views


def _stream_handle(frames, stream):
    """cudaStream_t the producer wrote `frames` on: the given torch.cuda.Stream or raw handle; else torch's current stream for a torch tensor;
    else the `stream` entry of __cuda_array_interface__ (1: legacy default stream, 2: per-thread default stream); else the legacy default (0)."""
    if stream is not None:
        return int(getattr(stream, "cuda_stream", stream))
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(frames, torch.Tensor):
        return int(torch.cuda.current_stream(frames.device).cuda_stream)
    s = frames.__cuda_array_interface__.get("stream")
    if s is None or s == 1:
        return 0
    return int(s)       # 2 is cudaStreamPerThread's handle; any other value is a cudaStream_t


def device_frames(frames, order="bgr", stream=None):
    """The cs_device_frames of `frames`, any object with __cuda_array_interface__ (a torch CUDA tensor, a CuPy array) of dtype uint8 and shape
    (N, H, W, 3) or (N, H, W).  Strides come from the interface (None: C-contiguous).  Raises ValueError for another dtype or rank; everything
    about the memory itself is checked by the library (cs_check_device_frames)."""
    cai = getattr(frames, "__cuda_array_interface__", None)
    if cai is None:
        raise ValueError("frames must expose __cuda_array_interface__ (a CUDA tensor or array)")
    if np.dtype(cai["typestr"]) != np.uint8:
        raise ValueError("frames must be uint8, got %s" % cai["typestr"])
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) not in (3, 4):
        raise ValueError("frames must be (N, H, W, 3) or (N, H, W), got shape %s" % (shape,))
    strides = cai.get("strides")
    if strides is None:
        strides, acc = [], 1
        for n in reversed(shape):
            strides.insert(0, acc)
            acc *= n
    strides = [int(v) for v in strides]
    d = DeviceFrames()
    d.data = int(cai["data"][0])
    d.n_frames, d.height, d.width = shape[:3]
    d.channels = shape[3] if len(shape) == 4 else 1
    d.stride_frame, d.stride_row, d.stride_col = strides[:3]
    d.stride_channel = strides[3] if len(shape) == 4 else 0
    if isinstance(order, str):
        if order.lower() not in ORDERS:
            raise ValueError("order must be 'bgr' or 'rgb', got %r" % order)
        order = ORDERS[order.lower()]
    d.channel_order = int(order)      # an integer goes to the library as it is
    d.stream = _stream_handle(frames, stream) or None
    return d


_lib = None

EXPORTS = [
    "cs_abi_version", "cs_create", "cs_destroy", "cs_last_error", "cs_default_cuboid_params",
    "cs_default_line_params", "cs_set_calibration", "cs_cam_pose", "cs_cuboid_measurement", "cs_cuboid_measurement_orb", "cs_detect_cuboids", "cs_detect_cuboids_batch",
    "cs_batch_upload", "cs_batch_upload_online", "cs_detect_frames_batch", "cs_batch_run", "cs_batch_run_async", "cs_batch_fetch", "cs_batch_stats_get",
    "cs_batch_device_records", "cs_stream", "cs_stage_ms", "cs_set_profiling", "cs_debug_roi",
    "cs_debug_candidates", "cs_detect_lines", "cs_detect_lines_batch", "cs_debug_lsd", "cs_debug_lsd_stats", "cs_debug_lsd_prof", "cs_debug_atan2", "cs_atan2_host", "cs_cuboid_draw_edges", "cs_debug_edlines", "cs_debug_stage_offsets", "cs_comm_unique_id", "cs_comm_init",
    "cs_allgather_topk", "cs_allgather_wait", "cs_fetch_gathered",
    "cs_keylines_from_lines", "cs_lbd_compute", "cs_lbd_compute_batch", "cs_detect_descrip_lines", "cs_detect_descrip_lines_batch",
    "cs_match_line_descrip", "cs_match_line_descrip_batch", "cs_lbd_debug_prepare", "cs_lbd_debug_keylines_edl", "cs_debug_last_set_pose",
]
# frames already on the device (cs_ingest.cu).  They are bound where the library has them: a build of cs_context.cu alone, as the CPU test
# suite compiles it for the host, does not; build() checks that the product library has every name of EXPORTS.
DEVICE_FRAME_EXPORTS = ["cs_check_device_frames", "cs_batch_upload_device", "cs_batch_upload_online_device", "cs_detect_lines_batch_device"]
EXPORTS += DEVICE_FRAME_EXPORTS
# k-nearest-neighbour and radius matching of line descriptors (cs_lbd.cu), bound the same way
MATCHER_EXPORTS = ["cs_knn_match_line_descrip", "cs_knn_match_line_descrip_batch", "cs_radius_match_line_descrip", "cs_radius_match_line_descrip_batch"]
EXPORTS += MATCHER_EXPORTS
# matching against a device-resident collection of many images' codes (cs_lbd_collection.cu), bound the same way
COLLECTION_EXPORTS = ["cs_lbd_collection_create", "cs_lbd_collection_destroy", "cs_lbd_collection_add", "cs_lbd_collection_clear",
                      "cs_lbd_collection_size", "cs_lbd_collection_match", "cs_lbd_collection_knn_match", "cs_lbd_collection_radius_match"]
EXPORTS += COLLECTION_EXPORTS
# the LSD seed loop's defined-angle bit plane (cs_lsd.cu), bound the same way
LSD_DEBUG_EXPORTS = ["cs_debug_lsd_defb", "cs_debug_lsd_occupancy"]
EXPORTS += LSD_DEBUG_EXPORTS
# the line detectors' NFA on given (n, k, p) (cs_debug_math.cu), bound the same way: the host build of cs_context.cu that the CPU test suite
# compiles does not have it
NFA_DEBUG_EXPORTS = ["cs_debug_nfa"]
EXPORTS += NFA_DEBUG_EXPORTS
# the line descriptor's two calls on frames already on the device (cs_ingest.cu), bound the same way: the host builds of cs_lbd.cu that the
# CPU test suite compiles do not have them
LBD_DEVICE_FRAME_EXPORTS = ["cs_detect_descrip_lines_batch_device", "cs_lbd_compute_batch_device"]
EXPORTS += LBD_DEVICE_FRAME_EXPORTS
# every octave of a multi-octave LSD detector (cs_lbd_octaves.cu, cs_ingest.cu), bound the same way: the host builds of cs_lbd.cu and
# cs_context.cu that the CPU test suite compiles do not have them
OCTAVE_EXPORTS = ["cs_detect_raw_lines_octaves_batch", "cs_detect_descrip_lines_octaves_batch", "cs_detect_raw_lines_octaves_batch_device",
                  "cs_detect_descrip_lines_octaves_batch_device"]
EXPORTS += OCTAVE_EXPORTS
# descriptors of key lines the caller gives, of any octave (cs_lbd_octaves.cu, cs_ingest.cu), bound the same way
LBD_OCTAVE_EXPORTS = ["cs_lbd_compute_octaves_batch", "cs_lbd_compute_octaves_batch_device"]
EXPORTS += LBD_OCTAVE_EXPORTS
# batches of frames of different sizes (cs_lsd.cu, cs_lbd_octaves.cu), bound the same way
MIXED_EXPORTS = ["cs_detect_lines_batch_mixed", "cs_detect_raw_lines_octaves_batch_mixed", "cs_batch_upload_mixed", "cs_batch_upload_online_mixed",
                 "cs_detect_cuboids_batch_mixed", "cs_detect_frames_batch_mixed"]
EXPORTS += MIXED_EXPORTS


def load():
    """dlopen the product library; raises if it has not been built (python -m cube_slam_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise OSError("%s is missing: build it with `python -m cube_slam_b200.build` (needs nvcc); "
                      "cube_slam_b200 has no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i, d_p = C.c_void_p, C.c_int, C.POINTER(C.c_double)
    u8_p, i32_p, f_p = C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_float)
    L.cs_abi_version.restype = i
    L.cs_create.restype = vp
    L.cs_create.argtypes = [i] * 6
    L.cs_destroy.argtypes = [vp]
    L.cs_destroy.restype = None
    L.cs_last_error.restype = C.c_char_p
    L.cs_last_error.argtypes = [vp]
    L.cs_default_cuboid_params.argtypes = [C.POINTER(CuboidParams)]
    L.cs_default_line_params.argtypes = [C.POINTER(LineParams)]
    L.cs_set_calibration.argtypes = [vp, d_p]
    L.cs_cam_pose.argtypes = [d_p, d_p, d_p, d_p]
    L.cs_cuboid_measurement.argtypes = [vp, d_p, d_p, d_p, d_p, d_p, d_p, d_p]
    L.cs_cuboid_measurement_orb.argtypes = [vp, d_p, C.c_double, d_p, d_p, d_p, d_p]
    L.cs_detect_cuboids.argtypes = [vp, u8_p, i, i, i, i, d_p, d_p, i, d_p, i, C.POINTER(CuboidParams), vp, i32_p]
    L.cs_detect_cuboids_batch.argtypes = [vp, vp, i, i, i, i, i, d_p, d_p, i32_p, d_p, i32_p, C.POINTER(CuboidParams), vp, i32_p]
    L.cs_batch_upload.argtypes = [vp, vp, i, i, i, i, i, d_p, d_p, i32_p, d_p, i32_p, C.POINTER(CuboidParams)]
    L.cs_batch_upload_online.argtypes = [vp, vp, i, i, i, i, i, d_p, d_p, i32_p, C.POINTER(LineParams), C.POINTER(CuboidParams)]
    L.cs_detect_frames_batch.argtypes = [vp, vp, i, i, i, i, i, d_p, d_p, i32_p, C.POINTER(LineParams), C.POINTER(CuboidParams), vp, i32_p]
    L.cs_batch_run.argtypes = [vp]
    L.cs_batch_run_async.argtypes = [vp]
    L.cs_batch_fetch.argtypes = [vp, vp, i32_p]
    L.cs_batch_stats_get.argtypes = [vp, C.POINTER(BatchStats)]
    L.cs_batch_device_records.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.cs_stream.restype = vp
    L.cs_stream.argtypes = [vp]
    L.cs_stage_ms.argtypes = [vp, C.c_char_p, C.POINTER(C.c_float)]
    L.cs_set_profiling.argtypes = [vp, i]
    L.cs_debug_stage_offsets.argtypes = [vp, vp, f_p]
    L.cs_debug_roi.argtypes = [vp, i, i32_p, u8_p, f_p, i, d_p, i, i32_p, i32_p]
    L.cs_debug_candidates.argtypes = [vp, i, i32_p, u8_p, d_p, d_p, i]
    L.cs_detect_lines.argtypes = [vp, vp, i, i, i, i, C.POINTER(LineParams), f_p, i32_p]
    L.cs_detect_lines_batch.argtypes = [vp, vp, i, i, i, i, i, C.POINTER(LineParams), f_p, C.c_int32, i32_p]
    L.cs_debug_lsd.argtypes = [vp, i, i32_p, d_p, d_p, d_p, i32_p, i32_p, f_p, i32_p, i]
    L.cs_debug_lsd_stats.argtypes = [vp, i32_p, i32_p, i]
    L.cs_debug_lsd_prof.argtypes = [vp, C.POINTER(C.c_uint64), i]
    if hasattr(L, "cs_debug_lsd_defb"):
        L.cs_debug_lsd_defb.argtypes = [vp, i, C.POINTER(C.c_uint32), i32_p]
    if hasattr(L, "cs_debug_lsd_occupancy"):
        L.cs_debug_lsd_occupancy.argtypes = [vp, i32_p]
    L.cs_debug_atan2.argtypes = [vp, d_p, d_p, d_p, i]
    L.cs_atan2_host.argtypes = [C.c_double, C.c_double]
    L.cs_atan2_host.restype = C.c_double
    if hasattr(L, "cs_debug_nfa"):
        L.cs_debug_nfa.argtypes = [vp, i32_p, i32_p, d_p, C.c_double, i, d_p, i32_p, i]
    L.cs_cuboid_draw_edges.argtypes = [vp, i32_p]
    L.cs_debug_edlines.argtypes = [vp, i, u8_p, C.POINTER(C.c_int16), C.POINTER(C.c_int16), C.POINTER(C.c_int16), u8_p, i32_p, i32_p, u8_p, f_p, i32_p, i]
    L.cs_comm_unique_id.argtypes = [vp, C.c_char_p, u8_p]
    L.cs_comm_init.argtypes = [vp, C.c_char_p, u8_p, i, i]
    L.cs_allgather_topk.argtypes = [vp, i, C.POINTER(vp)]
    L.cs_allgather_wait.argtypes = [vp]
    L.cs_fetch_gathered.argtypes = [vp, vp, i]
    L.cs_keylines_from_lines.argtypes = [f_p, i, i, i, vp]
    L.cs_lbd_compute.argtypes = [vp, vp, i, i, i, i, vp, i, u8_p, f_p]
    L.cs_lbd_compute_batch.argtypes = [vp, vp, i, i, i, i, i, vp, i32_p, u8_p, f_p]
    L.cs_detect_descrip_lines.argtypes = [vp, vp, i, i, i, i, C.POINTER(LineParams), vp, u8_p, i32_p]
    L.cs_detect_descrip_lines_batch.argtypes = [vp, vp, i, i, i, i, i, C.POINTER(LineParams), vp, u8_p, C.c_int32, i32_p]
    L.cs_match_line_descrip.argtypes = [vp, u8_p, i, u8_p, i, C.c_float, vp, i32_p]
    L.cs_match_line_descrip_batch.argtypes = [vp, u8_p, i32_p, u8_p, i32_p, i, C.c_float, vp, i32_p]
    i64_p = C.POINTER(C.c_int64)
    if all(hasattr(L, n) for n in MATCHER_EXPORTS):
        L.cs_knn_match_line_descrip.argtypes = [vp, u8_p, i, u8_p, i, i, u8_p, vp, i32_p]
        L.cs_knn_match_line_descrip_batch.argtypes = [vp, u8_p, i32_p, u8_p, i32_p, i, i, u8_p, vp, i32_p]
        L.cs_radius_match_line_descrip.argtypes = [vp, u8_p, i, u8_p, i, C.c_float, u8_p, vp, C.c_int64, i64_p]
        L.cs_radius_match_line_descrip_batch.argtypes = [vp, u8_p, i32_p, u8_p, i32_p, i, C.c_float, u8_p, vp, C.c_int64, i64_p]
    if all(hasattr(L, n) for n in COLLECTION_EXPORTS):
        L.cs_lbd_collection_create.restype = vp
        L.cs_lbd_collection_create.argtypes = [vp]
        L.cs_lbd_collection_destroy.restype = None
        L.cs_lbd_collection_destroy.argtypes = [vp]
        L.cs_lbd_collection_add.argtypes = [vp, u8_p, i32_p, i]
        L.cs_lbd_collection_clear.argtypes = [vp]
        L.cs_lbd_collection_size.argtypes = [vp, i32_p, i64_p]
        L.cs_lbd_collection_match.argtypes = [vp, u8_p, i, u8_p, i, vp, i32_p]
        L.cs_lbd_collection_knn_match.argtypes = [vp, u8_p, i, i, u8_p, i, vp, i32_p]
        L.cs_lbd_collection_radius_match.argtypes = [vp, u8_p, i, C.c_float, u8_p, i, vp, C.c_int64, i64_p]
    L.cs_lbd_debug_prepare.argtypes = [vp, i, vp, f_p, f_p]
    L.cs_lbd_debug_keylines_edl.argtypes = [f_p, f_p, i, i, i, vp]
    L.cs_debug_last_set_pose.argtypes = [u8_p, d_p, d_p, i, i, i32_p]
    if all(hasattr(L, n) for n in DEVICE_FRAME_EXPORTS):
        df_p = C.POINTER(DeviceFrames)
        L.cs_check_device_frames.argtypes = [i, df_p]
        L.cs_batch_upload_device.argtypes = [vp, df_p, d_p, d_p, i32_p, d_p, i32_p, C.POINTER(CuboidParams)]
        L.cs_batch_upload_online_device.argtypes = [vp, df_p, d_p, d_p, i32_p, C.POINTER(LineParams), C.POINTER(CuboidParams)]
        L.cs_detect_lines_batch_device.argtypes = [vp, df_p, C.POINTER(LineParams), f_p, C.c_int32, i32_p]
    if all(hasattr(L, n) for n in LBD_DEVICE_FRAME_EXPORTS):
        df_p = C.POINTER(DeviceFrames)
        L.cs_detect_descrip_lines_batch_device.argtypes = [vp, df_p, C.POINTER(LineParams), vp, u8_p, C.c_int32, i32_p]
        L.cs_lbd_compute_batch_device.argtypes = [vp, df_p, vp, i32_p, u8_p, f_p]
    if all(hasattr(L, n) for n in OCTAVE_EXPORTS):
        df_p = C.POINTER(DeviceFrames)
        L.cs_detect_raw_lines_octaves_batch.argtypes = [vp, vp, i, i, i, i, i, C.POINTER(LineParams), vp, C.c_int32, i32_p]
        L.cs_detect_descrip_lines_octaves_batch.argtypes = [vp, vp, i, i, i, i, i, C.POINTER(LineParams), vp, u8_p, C.c_int32, i32_p]
        L.cs_detect_raw_lines_octaves_batch_device.argtypes = [vp, df_p, C.POINTER(LineParams), vp, C.c_int32, i32_p]
        L.cs_detect_descrip_lines_octaves_batch_device.argtypes = [vp, df_p, C.POINTER(LineParams), vp, u8_p, C.c_int32, i32_p]
    if all(hasattr(L, n) for n in LBD_OCTAVE_EXPORTS):
        L.cs_lbd_compute_octaves_batch.argtypes = [vp, vp, i, i, i, i, i, vp, i32_p, u8_p, f_p]
        L.cs_lbd_compute_octaves_batch_device.argtypes = [vp, C.POINTER(DeviceFrames), vp, i32_p, u8_p, f_p]
    if all(hasattr(L, n) for n in MIXED_EXPORTS):
        fv_p = C.POINTER(FrameView)
        L.cs_detect_lines_batch_mixed.argtypes = [vp, vp, fv_p, i, C.POINTER(LineParams), f_p, C.c_int32, i32_p]
        L.cs_detect_raw_lines_octaves_batch_mixed.argtypes = [vp, vp, fv_p, i, C.POINTER(LineParams), vp, C.c_int32, i32_p]
        cp_p, lp_p = C.POINTER(CuboidParams), C.POINTER(LineParams)
        L.cs_batch_upload_mixed.argtypes = [vp, vp, fv_p, i, d_p, d_p, d_p, i32_p, d_p, i32_p, cp_p]
        L.cs_batch_upload_online_mixed.argtypes = [vp, vp, fv_p, i, d_p, d_p, d_p, i32_p, lp_p, cp_p]
        L.cs_detect_cuboids_batch_mixed.argtypes = [vp, vp, fv_p, i, d_p, d_p, d_p, i32_p, d_p, i32_p, cp_p, vp, i32_p]
        L.cs_detect_frames_batch_mixed.argtypes = [vp, vp, fv_p, i, d_p, d_p, d_p, i32_p, lp_p, cp_p, vp, i32_p]
    for name in EXPORTS:
        if name in (DEVICE_FRAME_EXPORTS + MATCHER_EXPORTS + COLLECTION_EXPORTS + LSD_DEBUG_EXPORTS + NFA_DEBUG_EXPORTS + LBD_DEVICE_FRAME_EXPORTS
                    + OCTAVE_EXPORTS + LBD_OCTAVE_EXPORTS + MIXED_EXPORTS) and not hasattr(L, name):
            continue
        fn = getattr(L, name)
        if fn.restype is C.c_int and name not in ("cs_abi_version",):
            fn.restype = C.c_int
    _lib = L
    return L


def ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))
