/*
 * cube_slam_b200.h -- C ABI of the H100-native cuboid-proposal front end (libcubeslam_b200.so).
 *
 * Drop-in boundary for CubeSLAM's per-frame hot path.  Every entry point names the reference
 * interface it replaces (paths relative to the reference repository root).  Plain pointers and
 * sizes only; no C++/torch types.  All functions return CS_OK (0) or a negative cs_status; the
 * text of the last failure is available from cs_last_error().
 *
 * Threading contract (as the reference objects, SURVEY.md section 8b): one cs_ctx per host thread;
 * a context owns one CUDA stream plus its device workspace; calls are synchronous on return unless
 * the name ends in _async.
 */
#ifndef CUBE_SLAM_B200_H
#define CUBE_SLAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CS_ABI_VERSION 1

typedef enum cs_status {
    CS_OK = 0,
    CS_ERR_INVALID_ARG = -1,
    CS_ERR_CUDA = -2,          /* CUDA runtime failure or no usable sm_90 device */
    CS_ERR_CAPACITY = -3,      /* input exceeds the capacities given to cs_create */
    CS_ERR_NOT_PREPARED = -4,  /* run/fetch before a batch was uploaded */
    CS_ERR_NCCL = -5,
    CS_ERR_UNSUPPORTED = -6
} cs_status;

typedef struct cs_ctx cs_ctx;

/* Mode members of class detect_3d_cuboid (detect_3d_cuboid/include/detect_3d_cuboid/detect_3d_cuboid.h:65-79)
 * followed by the hard-coded locals of detect_cuboid() exposed with the reference's literals as
 * defaults (detect_3d_cuboid/src/box_proposal_detail.cpp:79-87,126-128,144,177-179,197). */
typedef struct cs_cuboid_params {
    int32_t consider_config_1;             /* detect_3d_cuboid.h:72, default 1 */
    int32_t consider_config_2;             /* :73, default 1 */
    int32_t whether_sample_cam_roll_pitch; /* :74, default 0 */
    int32_t whether_sample_bbox_height;    /* :75, default 0 */
    int32_t max_cuboid_num;                /* :77, default 1 */
    int32_t reweight_edge_distance;        /* box_proposal_detail.cpp:82, default 1 */
    int32_t whether_normalize_two_errors;  /* :85, default 1 */
    int32_t top_sample_count_override;     /* 0 = reference rule (:144-146); >0 = fixed count (BASELINE dense sweep) */
    double nominal_skew_ratio;             /* detect_3d_cuboid.h:78, default 1 */
    double max_cut_skew;                   /* :79, default 3 */
    double vp12_edge_angle_thre;           /* box_proposal_detail.cpp:79, default 15 (deg) */
    double vp3_edge_angle_thre;            /* :80, default 10 (deg) */
    double shorted_edge_thre;              /* :81, default 20 (px) */
    double weight_vp_angle;                /* :86, default 0.8 */
    double weight_skew_error;              /* :87, default 1.5 */
    double pre_merge_dist_thre;            /* :177, default 20 (px) */
    double pre_merge_angle_thre;           /* :178, default 5 (deg) */
    double edge_length_threshold;          /* :179, default 30 (px) */
    double canny_low;                      /* :197, default 80 */
    double canny_high;                     /* :197, default 200 */
    double yaw_half_range_deg;             /* :128, default 45 */
    double yaw_step_deg;                   /* :128, default 6 */
} cs_cuboid_params;

/* POD mirror of class cuboid (detect_3d_cuboid.h:15-36); matrices are row-major. */
typedef struct cs_cuboid_rec {
    double pos[3];
    double scale[3];
    double rotY;
    double box_config_type[2];
    int32_t box_corners_2d[16];       /* 2 x 8 */
    double box_corners_3d_world[24];  /* 3 x 8 */
    double rect_detect_2d[4];
    double edge_distance_error;
    double edge_angle_error;
    double normalized_error;
    double skew_ratio;
    double down_expand_height;
    double camera_roll_delta;
    double camera_pitch_delta;
    double combined_score;            /* normalized_error + skew penalty (box_proposal_detail.cpp:526) */
    int32_t proposal_index;           /* row in the reference's valid-proposal list of its height sample */
    int32_t height_sample_id;
    int32_t valid;                    /* 1 when this slot holds a cuboid */
    int32_t pad_;
} cs_cuboid_rec;

/* Members of class line_lbd_detect (line_lbd/include/line_lbd/line_lbd_allclass.h:22-31) and the
 * constants its two detectors are built with (line_lbd/libs/LSDDetector.cpp:173-183,205;
 * line_lbd/libs/binary_descriptor.cpp:1511-1522). */
typedef struct cs_line_params {
    int32_t use_LSD;            /* line_lbd_allclass.h:29; class default 0, object_slam sets 1 (main_obj.cpp:365) */
    int32_t numoctaves;         /* :26, default 1.  Any value >= 1 gives the same result in the octave-0 calls: only octave 0 survives
                                   filter_lines (:200-207) and detect_descrip_lines (:239,266), and octave 0 does not depend on the higher
                                   ones.  cs_detect_raw_lines_octaves_batch / cs_detect_descrip_lines_octaves_batch return every octave
                                   (LSD flavour, (int)octaveratio == 2 when numoctaves > 1) */
    float octaveratio;          /* :27, default 1 */
    float line_length_thres;    /* :30, class default 50, object_slam uses 15 */
} cs_line_params;

/* per-batch work counters (what BASELINE.json's metric counts) */
typedef struct cs_batch_stats {
    int64_t n_frames;
    int64_t n_objects;          /* 2D boxes */
    int64_t n_roi_jobs;         /* boxes x height samples */
    int64_t n_candidates;       /* enumerated (pose, yaw, top-x, config) tuples */
    int64_t n_valid;            /* proposals that reach box_edge_sum_dists == "scored cuboid proposals" */
    int64_t n_kernel_launches;  /* launches of this library's kernels in the last run */
    int64_t roi_pixels;         /* sum of dist-map ROI areas */
    int64_t n_lines_in;         /* input line segments over all frames */
} cs_batch_stats;

/* ---- life cycle ------------------------------------------------------------------------- */
int cs_abi_version(void);
/* Replaces constructing detect_3d_cuboid / line_lbd_detect objects (main_obj.cpp:354-366, Tracking.cc:242-244).
 * Capacities bound the device workspace; max_frames is the largest batch. */
cs_ctx *cs_create(int device, int max_width, int max_height, int max_frames, int max_boxes_per_frame,
                  int max_lines_per_frame);
void cs_destroy(cs_ctx *ctx);
const char *cs_last_error(const cs_ctx *ctx);
void cs_default_cuboid_params(cs_cuboid_params *p);
void cs_default_line_params(cs_line_params *p);

/* detect_3d_cuboid::set_calibration (box_proposal_detail.cpp:36-40); K row-major 3x3 */
int cs_set_calibration(cs_ctx *ctx, const double K[9]);

/* detect_3d_cuboid::set_cam_pose (box_proposal_detail.cpp:42-54) as a pure function: the ZYX Euler angles
 * (roll, pitch, yaw; cam_pose.euler_angle, read by callers as cam_pose_raw.euler_angle, main_obj.cpp:465) and
 * K*R^-1 of a camera-to-world transform.  Host-only, needs no context. */
int cs_cam_pose(const double K[9], const double T_wc[16], double euler_zyx[3], double KinvR[9]);

/* The step right after the path in object_slam (object_slam/src/main_obj.cpp:455-473,505): the best cuboid as a measurement in the
 * camera frame, cube_ground_value.transform_to(Twc) of g2o::cuboid (object_slam/include/object_slam/g2o_Object.h:36-41,127-133) with
 * g2o's SE3Quat algebra, and meas_quality = (1 - normalized_error + 0.5) / 2.  cam_t / cam_q_xyzw: the camera pose Twc as the
 * truth-pose file gives it (x y z qx qy qz qw); cam_euler_raw: cam_pose_raw.euler_angle when whether_sample_cam_roll_pitch was on
 * (the measurement is then taken in the frame of the sampled roll / pitch), else NULL.  Host-only, needs no context. */
int cs_cuboid_measurement(const cs_cuboid_rec *rec, const double cam_t[3], const double cam_q_xyzw[4], const double cam_euler_raw[3],
                          double meas_t[3], double meas_q_xyzw[4], double meas_scale[3], double *meas_quality);

/* The same step in orb_object_slam (orb_object_slam/src/Tracking.cc:1636-1647,1680-1687): the camera pose comes as a 4x4 camera-to-ground
 * matrix (Converter::toSE3Quat), meas_quality = (60 - clamp(z, 10, 30)) / 40, times the 2-D box confidence when that is positive. */
int cs_cuboid_measurement_orb(const cs_cuboid_rec *rec, const double T_cam_to_ground[16], double box_confidence, double meas_t[3],
                              double meas_q_xyzw[4], double meas_scale[3], double *meas_quality);

/* ---- cuboid proposals ------------------------------------------------------------------- */
/* detect_3d_cuboid::detect_cuboid (box_proposal_detail.cpp:56-557; header detect_3d_cuboid.h:62-63)
 * for ONE frame with HOST buffers.  img: H x stride bytes, channels 3 (BGR) or 1; T_wc row-major 4x4;
 * boxes N x 5 [x y w h prob] 0-based; lines M x 4 [x1 y1 x2 y2];
 * out: N x topk records (topk = params->max_cuboid_num); out_counts: N. */
int cs_detect_cuboids(cs_ctx *ctx, const uint8_t *img, int width, int height, int stride, int channels,
                      const double T_wc[16], const double *boxes, int n_boxes, const double *lines, int n_lines,
                      const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts);

/* The same call over a batch of frames (host buffers).  Frames are images of identical size laid out
 * back to back (frame f at imgs + f*height*stride).  box_offsets/line_offsets have n_frames+1 entries
 * (CSR); out holds box_offsets[n_frames] x topk records. */
int cs_detect_cuboids_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride,
                            int channels, const double *T_wc /* n_frames x 16 */, const double *boxes,
                            const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                            const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts);

/* The whole per-frame front end of object_slam's online mode in one call (object_slam/src/main_obj.cpp:424-450):
 * line_lbd_detect::detect_filter_lines on every frame, its n x 4 float output widened to double, then detect_cuboid.
 * Lines never leave the device.  Host buffers in, host records out. */
int cs_detect_frames_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                           const double *T_wc, const double *boxes, const int32_t *box_offsets,
                           const cs_line_params *line_params, const cs_cuboid_params *params, cs_cuboid_rec *out,
                           int32_t *out_counts);

/* Device-resident variant used by the throughput benchmark: upload once, run many times, fetch.
 * Reuse of the caller's buffers: cs_batch_upload and cs_batch_upload_online copy imgs (and every table) on the context's stream and wait
 * for that stream before they return, so imgs may be overwritten or freed as soon as the call returns, whether it is pageable or pinned
 * host memory.  The wait also covers work still queued on this context (a cs_batch_run_async not yet fetched): an upload to a context
 * with a batch in flight returns only when that batch has finished.  A pipeline that overlaps copies with kernels therefore keeps one
 * context per batch in flight. */
int cs_batch_upload(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                    const double *T_wc, const double *boxes, const int32_t *box_offsets, const double *lines,
                    const int32_t *line_offsets, const cs_cuboid_params *params);
/* same, online mode: no input lines, cs_batch_run detects them first (as cs_detect_frames_batch) */
int cs_batch_upload_online(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                           const double *T_wc, const double *boxes, const int32_t *box_offsets,
                           const cs_line_params *line_params, const cs_cuboid_params *params);

/* ---- frames already in GPU memory ---------------------------------------------------------------------------------------------------- */
/* A batch of frames that lives on the device, described as n_frames x height x width x channels bytes with byte strides, so that any strided
 * view is one descriptor: packed NHWC, planar NCHW (a permute(0, 2, 3, 1) view), a crop (a slice), every other frame (t[::2]), the first
 * three channels of BGRA / RGBA (t[..., :3]).  channels 3 is BGR or RGB (channel_order), channels 1 is gray.  The library copies the view
 * into its own packed buffer (pitch width * channels, BGR or gray) on the device -- one device-to-device copy when the view is already
 * packed BGR or gray, else the kernel k_ingest_frames -- and everything after that is the host path's code.
 * Stream order both ways, without a host block: the copy waits for the work queued on `stream` before the call, and work queued on `stream`
 * after the call (overwriting or freeing the frames) waits for the copy. */
#define CS_ORDER_BGR 0
#define CS_ORDER_RGB 1
typedef struct cs_device_frames {
    const uint8_t *data;                     /* device (or managed) memory on the context's device: byte (0, 0, 0, 0) of the view */
    int32_t n_frames, height, width, channels; /* channels 1 or 3 */
    int64_t stride_frame, stride_row, stride_col, stride_channel; /* bytes, >= 0 (stride_channel is ignored when channels == 1) */
    int32_t channel_order;                   /* CS_ORDER_BGR or CS_ORDER_RGB; ignored when channels == 1 */
    void *stream;                            /* cudaStream_t the producer wrote the frames on; NULL = the legacy default stream */
} cs_device_frames;

/* Host-only check of a descriptor, made by the three calls below before they enqueue anything: CS_ERR_INVALID_ARG when the pointer is not
 * device or managed memory on `device`, a stride is negative, channels is not 1 or 3, the order is unknown, or the last byte the view
 * touches lies outside the pointer's allocation.  The text of a failure is what cs_last_error(NULL) returns on the calling thread. */
int cs_check_device_frames(int device, const cs_device_frames *frames);
/* cs_batch_upload / cs_batch_upload_online with the frames taken from the device.  Poses, boxes and lines stay host buffers, as in the
 * host forms.  Returns once the copy is enqueued on the context stream; cs_batch_run[_async], cs_batch_fetch, cs_batch_device_records and
 * cs_allgather_topk then work as after the host forms. */
int cs_batch_upload_device(cs_ctx *ctx, const cs_device_frames *frames, const double *T_wc, const double *boxes, const int32_t *box_offsets,
                           const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params);
int cs_batch_upload_online_device(cs_ctx *ctx, const cs_device_frames *frames, const double *T_wc, const double *boxes,
                                  const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params);
/* cs_detect_lines_batch on device frames.  The frames go to the line detector's own buffer, as the host form's do, never to the one a batch
 * uploaded to the context reads from.  Synchronous, like the host form. */
int cs_detect_lines_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const cs_line_params *params, float *lines_xyxy,
                                 int32_t max_lines_per_frame, int32_t *n_lines /* n_frames */);
/* cs_detect_descrip_lines_batch (below) on device frames: the same outputs -- host key lines, host 32-byte descriptors, frame f's slots at
 * f * max_lines_per_frame -- the same checks (numoctaves >= 1, capacity) and the same error statuses and messages.  The frames go to the
 * detector's own buffer (LSD or EDLines, after use_LSD), as in cs_detect_lines_batch_device.  Synchronous. */
struct cs_keyline; /* defined with the line descriptors below */
int cs_detect_descrip_lines_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const cs_line_params *params, struct cs_keyline *keylines,
                                         uint8_t *desc32, int32_t max_lines_per_frame, int32_t *n_lines /* n_frames */);
/* cs_lbd_compute_batch (below) on device frames: the key lines and their CSR stay host buffers, desc72 is optional.  With no key line at all
 * it returns CS_OK after the descriptor check, as the host form does.  The frames go to the EDLines detector's buffer.  Synchronous. */
int cs_lbd_compute_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const struct cs_keyline *keylines,
                                const int32_t *keyline_offsets /* n_frames + 1 */, uint8_t *desc32, float *desc72);

int cs_batch_run(cs_ctx *ctx);                       /* host-side sampling tables + every kernel; synchronous */
int cs_batch_run_async(cs_ctx *ctx);                 /* same, returns after enqueueing on the context stream */
int cs_batch_fetch(cs_ctx *ctx, cs_cuboid_rec *out, int32_t *out_counts);
int cs_batch_stats_get(cs_ctx *ctx, cs_batch_stats *stats);
/* device pointer of the record buffer ([n_objects] x topk cs_cuboid_rec) and its size in bytes */
int cs_batch_device_records(cs_ctx *ctx, void **dev_ptr, size_t *n_bytes);
/* raw CUDA stream of the context (cudaStream_t) so callers can time with events on it */
void *cs_stream(cs_ctx *ctx);
/* milliseconds spent in the named stage of the last cs_batch_run ("lsd","gray","canny","hyst","dt","lines","sweep","fuse","total") */
int cs_stage_ms(cs_ctx *ctx, const char *stage, float *ms);
/* bit 0: per-stage CUDA-event timing (adds event records only; the chain then stays on one stream).  Debug / A-B switches:
 * bit 3 CTA-wide selection kernel (k_fuse_rank) for every box, bit 4 no high-priority
 * stream for the distance transform -> sweep -> selection tail, bit 5 raster-scan distance transform (one kernel) instead of the cone form,
 * bit 6 cone-form distance transform reading the edge bits from global memory (the path of ROIs whose bit plane exceeds 96 KB),
 * bit 7 the line detectors' round-1 kernels (EDLines: routing and fitting on the pixel maps, one thread per frame) instead of the walk-graph
 * / warp-per-chain ones (the LSD seed loop has one form since the ordered-speculation kernel was measured and removed),
 * bit 8 byte-load staging in the line detectors' tile kernels (A/B of TMA).  Bits 2 and 9 are accepted and ignored: they once selected
 * kernel variants whose results were bit-identical to the default kernels', so callers that still pass them get the same output.
 * Mode switch, bit 10: with whether_sample_cam_roll_pitch the reference derives the yaw samples of box k + 1 of a frame from the
 * cam_pose box k left behind (box_proposal_detail.cpp:126-128 after :237,485) -- an ulp away from the raw pose's, which decides between 15
 * and 16 yaw samples.  By default every box starts from the raw pose (boxes independent, one pass); with bit 10
 * cs_detect_cuboids[_batch] runs one pass per box rank and carries the pose exactly as the reference does (DESIGN.md section 2). */
int cs_set_profiling(cs_ctx *ctx, int enable);
/* tests: which pose hypothesis the reference's cam_pose holds after one height sample of a box in roll / pitch-sampling mode, from the
 * candidate records of that job (valid flag, distance error, angle error, enumeration order, pose-major).  Host-only, needs no context. */
int cs_debug_last_set_pose(const uint8_t *valid, const double *dist_err, const double *angle_err, int n_cand, int n_pose, int32_t *pose_out);

/* debug: when several contexts run concurrently with profiling on, the offsets (ms) of the 8 stage starts and the end of ctx's last run
 * from the start of ref's last run -- a timeline of how the batches in flight overlap (tools/timeline.py) */
int cs_debug_stage_offsets(cs_ctx *ctx, cs_ctx *ref, float offsets_ms[9]);

/* debug/inspection: copy intermediate per-ROI results of the last run back to the host.
 * job = ROI job index (object-major, height-sample-minor). Any pointer may be NULL. */
int cs_debug_roi(cs_ctx *ctx, int job, int32_t roi_xywh[4], uint8_t *canny, float *dist, int cap_px,
                 double *merged_lines, int cap_lines, int32_t *n_lines_roi, int32_t *n_lines_merged);
int cs_debug_candidates(cs_ctx *ctx, int job, int32_t *n_candidates, uint8_t *valid, double *dist_err,
                        double *angle_err, int cap);

/* ---- line segments ---------------------------------------------------------------------- */
/* line_lbd_detect::detect_filter_lines(const cv::Mat&, cv::Mat&) (line_lbd/class/line_lbd_allclass.cpp:216-221):
 * detect (LSD or EDLines) -> keep octave 0 and length > line_length_thres -> n x 4 float [x1 y1 x2 y2].
 * lines_xyxy has room for *n_inout segments; on return *n_inout is the number written. */
int cs_detect_lines(cs_ctx *ctx, const uint8_t *img, int width, int height, int stride, int channels,
                    const cs_line_params *params, float *lines_xyxy, int32_t *n_inout);
int cs_detect_lines_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride,
                          int channels, const cs_line_params *params, float *lines_xyxy, int32_t max_lines_per_frame,
                          int32_t *n_lines /* n_frames */);

/* One frame of a batch of frames of different sizes: `height` rows of `stride` bytes starting `offset` bytes from the batch's base pointer,
 * each row `width` pixels of `channels` (1 = gray, 3 = BGR) bytes. */
typedef struct cs_frame_view {
    int64_t offset;
    int32_t width, height, stride, channels;
} cs_frame_view;

/* cs_detect_lines_batch over host frames of different sizes and channel counts: frame f is imgs + views[f].offset; its segments go to
 * lines_xyxy + f * max_lines_per_frame * 4, n_lines[f] of them -- what cs_detect_lines_batch returns for that frame alone.  LSD runs the
 * whole list as one batch; EDLines (use_LSD == 0) runs one batch per (width, height, channels) group.  Every argument is checked before
 * anything is enqueued: null pointers, n_frames <= 0, an empty size, channels other than 1 or 3, stride < width * channels and (LSD) a frame
 * too small for LSD are CS_ERR_INVALID_ARG naming the frame; more segments than max_lines_per_frame is CS_ERR_CAPACITY naming the frame.
 * Synchronous. */
int cs_detect_lines_batch_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params,
                                float *lines_xyxy, int32_t max_lines_per_frame, int32_t *n_lines /* n_frames */);

/* The cuboid calls over host frames of different sizes, channel counts and cameras: frame f is imgs + views[f].offset (cs_frame_view), with
 * calibration K + 9 f (K: n_frames x 9 row-major, one per frame; NULL = the context's, cs_set_calibration).  Poses, boxes, lines and their
 * CSRs are the one-size forms'.  Each frame's records and counts are byte for byte what the one-size call (cs_detect_cuboids_batch,
 * cs_detect_frames_batch) returns for that frame alone with its K set by cs_set_calibration; records stay in box order.
 * After either upload, cs_batch_run[_async], cs_batch_fetch, cs_batch_stats_get, cs_batch_device_records, cs_debug_roi / cs_debug_candidates
 * and cs_allgather_topk work as after the one-size forms.  The frames are packed into the context's buffer (rows without padding); a 3-channel
 * frame's gray plane is made by one table-driven launch over every such frame, a gray frame is read in place.  Online: LSD runs the whole list
 * as one batch (a candidate-buffer overflow fails the batch at fetch with CS_ERR_CAPACITY, as in the one-size online batch; cs_debug_lsd
 * refuses afterwards), EDLines one batch per (width, height, channels) group.  cs_detect_cuboids_batch_mixed honours cs_set_profiling bit 10.
 * Refused on the host before anything is enqueued, naming the frame: the frame checks of cs_detect_lines_batch_mixed (CS_ERR_INVALID_ARG); a
 * frame larger than cs_create's max_width x max_height (CS_ERR_CAPACITY); a K entry that is not finite or a K of zero determinant
 * (CS_ERR_INVALID_ARG); and online, a frame outside the detector's sizes, with cs_detect_lines_batch_mixed's messages.  K == NULL without
 * cs_set_calibration is CS_ERR_INVALID_ARG.  The uploads wait for the context stream as cs_batch_upload does; the detect calls are
 * synchronous. */
int cs_batch_upload_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                          const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                          const cs_cuboid_params *params);
int cs_batch_upload_online_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                 const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params);
int cs_detect_cuboids_batch_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                  const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                                  const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts);
int cs_detect_frames_batch_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                 const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params,
                                 cs_cuboid_rec *out, int32_t *out_counts);

/* inspection of the last cs_detect_lines[_batch] run (tests): intermediate images of one frame; any pointer may be NULL.  It and
 * cs_debug_lsd_defb read one-size LSD batches only: after a mixed-size call or an octave call (LSD over planes of several sizes) they return
 * CS_ERR_UNSUPPORTED. */
int cs_debug_lsd(cs_ctx *ctx, int frame, int32_t scaled_wh[2], double *scaled, double *modgrad, double *angles, int32_t *list,
                 int32_t *list_len, float *raw_lines, int32_t *n_raw, int cap_raw);
/* diagnostics of the last LSD run's seed loop: stats4 is kept for ABI stability and reads zero (it described the ordered-speculation kernel
 * that round 2 measured and removed); redo[f] = 1: the frame went through the one-warp-per-frame kernel, as every frame does now */
int cs_debug_lsd_stats(cs_ctx *ctx, int32_t *stats4, int32_t *redo, int n_frames);
/* clock64 cycles the seed-loop warps spent per phase since the last reset (diagnostics; tools/time_lines.py): {region_grow, region2rect,
 * refine, raster scan for seeds (the seed loop outside the per-seed pipeline), used-map re-reads after a grow (a count), seeds grown, whole
 * kernel summed over CTAs, region pixels, seeds whose region list outgrew its shared-memory part (LSD_SEQ_SCAP entries), and seven unused
 * slots}; only runs made while profiling is enabled (cs_set_profiling bit 0) count */
int cs_debug_lsd_prof(cs_ctx *ctx, uint64_t *out16, int reset);
/* resources of the LSD seed loop (k_lsd_grow_seq, out14[0..6]) and front end (k_lsd_front, out14[7..13]) on the context's device, each
 * {registers per thread, local memory bytes per thread, static shared bytes, dynamic shared bytes per launch, threads per CTA, CTAs an SM
 * holds at that launch configuration (cudaOccupancyMaxActiveBlocksPerMultiprocessor), preferred shared-memory carveout in percent} */
int cs_debug_lsd_occupancy(cs_ctx *ctx, int32_t *out14);
/* the last LSD run's "angle defined" bit plane of one frame, as the seed loop scans it: bit x & 31 of word y * words_per_row + x / 32 of the
 * scaled image, words_per_row = ceil(W / 32); bits holds H * words_per_row words; either pointer may be NULL */
int cs_debug_lsd_defb(cs_ctx *ctx, int frame, uint32_t *bits, int32_t *words_per_row);
/* same for the EDLines flavour (use_LSD = 0): EDLineDetector's maps (binary_descriptor.cpp:1617-1666: blurred image, dxImg_, dyImg_,
 * gImgWO_ / 4, dirImg_), the anchors in scan order as y * width + x, the edge map after smart routing, the segments before the length filter */
int cs_debug_edlines(cs_ctx *ctx, int frame, uint8_t *blur, int16_t *dx, int16_t *dy, int16_t *g, uint8_t *dir, int32_t *anchors,
                     int32_t *n_anchors, uint8_t *edge, float *raw_lines, int32_t *n_raw, int cap_raw);

/* ---- line descriptors and matching (SURVEY.md section 8 row f4: the rest of class line_lbd_detect) -------------------------------------- */
/* The KeyLine fields callers and the descriptor read (line_lbd/include/line_lbd/line_descriptor/descriptor.hpp:104-172) for octave 0, where
 * startPoint == sPointInOctave; KeyLine::pt is the mid point of the two ends, KeyLine::octave is 0. */
typedef struct cs_keyline {
    float start_x, start_y, end_x, end_y; /* startPointX / Y, endPointX / Y */
    float angle;                          /* KeyLine::angle: EDLines' lineDirection_, LSD's atan2(dy, dx) (LSDDetector.cpp:244) */
    float line_length;                    /* KeyLine::lineLength */
    float response;                       /* lineLength / max(width, height) */
    float size;                           /* (endX - startX) * (endY - startY) */
    int32_t num_pixels;                   /* KeyLine::numOfPixels: the length of the descriptor's support region */
    int32_t class_id;                     /* position in the list this call returns (0 .. n-1) */
} cs_keyline;
/* cv::DMatch as match_line_descrip returns it */
typedef struct cs_dmatch {
    int32_t query_idx, train_idx, img_idx;
    float distance;
} cs_dmatch;

/* KeyLine fields of the LSD flavour from n x 4 segment rows, e.g. cs_detect_lines' output (LSDDetector::detectImpl,
 * line_lbd/libs/LSDDetector.cpp:226-250: length, cv::LineIterator pixel count, angle, size, response).  Host-only, needs no context.
 * (line_lbd_detect::get_line_descriptors goes through mat_to_keylines, line_lbd_allclass.cpp:68-108, which reads KeyLine fields before it
 * sets them and leaves class_id / octave unset in what it returns: undefined in the reference.  This is the defined equivalent.) */
int cs_keylines_from_lines(const float *lines_xyxy, int n, int width, int height, cs_keyline *out);

/* BinaryDescriptor::compute(image, keylines, descriptors[, returnFloatDescr]) (line_lbd/libs/binary_descriptor.cpp:587-592, computeImpl
 * :603-790, computeSobel :352-398, computeLBD :1146-1509) as line_lbd_detect calls it: row i of desc32 (n x 32 bytes) is the binary LBD
 * descriptor of key line i; desc72 (optional, n x 72 floats) the float descriptor it is made from.  Reads start / end point, angle and
 * num_pixels of each key line.  The batch form takes frames laid out back to back and a CSR of key lines per frame. */
int cs_lbd_compute(cs_ctx *ctx, const uint8_t *img, int width, int height, int stride, int channels, const cs_keyline *keylines, int n,
                   uint8_t *desc32, float *desc72);
int cs_lbd_compute_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                         const cs_keyline *keylines, const int32_t *keyline_offsets /* n_frames + 1 */, uint8_t *desc32, float *desc72);

/* line_lbd_detect::detect_descrip_lines(gray_img, keylines_out, line_descrips) (line_lbd/class/line_lbd_allclass.cpp:253-272): detect
 * (LSD or EDLines), describe, keep octave 0 and lineLength > line_length_thres.  keylines / desc32 have room for *n_inout lines (batch:
 * max_lines_per_frame per frame, frame f at f * max_lines_per_frame); on return *n_inout (n_lines[f]) is the number kept.  The Mat
 * overload (:224-250, no length filter) is the same call with line_length_thres = -1; detect_descrip_lines_octaves (:285-339) for one
 * octave is this call followed by the start / end swap of :321-330 on the host (shim/line_lbd_b200.cpp, cube_slam_b200/line_lbd.py). */
int cs_detect_descrip_lines(cs_ctx *ctx, const uint8_t *img, int width, int height, int stride, int channels, const cs_line_params *params,
                            cs_keyline *keylines, uint8_t *desc32, int32_t *n_inout);
int cs_detect_descrip_lines_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                  const cs_line_params *params, cs_keyline *keylines, uint8_t *desc32, int32_t max_lines_per_frame,
                                  int32_t *n_lines /* n_frames */);

/* Every octave of a multi-octave LSD detector (use_LSD = 1): the KeyLine of octave k with both pairs of end points.  kl.start / end are the
 * points in the input frame (the in-octave points times 2^k), kl.response and kl.num_pixels are measured on the octave image, kl.class_id is
 * the position in the octave's list.  KeyLine::pt is the mid point of kl's two ends. */
typedef struct cs_keyline_octave {
    cs_keyline kl;
    float s_oct_x, s_oct_y, e_oct_x, e_oct_y; /* sPointInOctaveX / Y, ePointInOctaveX / Y */
    int32_t octave;                           /* KeyLine::octave */
    int32_t pad_;
} cs_keyline_octave;

/* line_lbd_detect::detect_raw_lines(gray, vector<KeyLine>&) and its vector<vector<KeyLine>> overload (line_lbd_allclass.cpp:125-172) for a
 * detector built with numoctaves octaves, LSD flavour (LSDDetector.cpp:55-72,176-250): octave 0 is the gray frame, octave k is cv::pyrDown of
 * octave k - 1 to (w / 2, h / 2); LSD runs on every octave; a segment's ends are clamped to its octave, scaled by 2^k and dropped when both
 * lie within 10 px of the same border of the input frame.  Octave k of frame f is written at keylines + (f * numoctaves + k) *
 * max_lines_per_octave, n_lines[f * numoctaves + k] of them (n_lines holds n_frames * numoctaves counts).  max_lines_per_octave bounds the
 * segments LSD finds in one octave, before the border test.
 * Errors: use_LSD == 0 is CS_ERR_UNSUPPORTED (EDLines groups its octaves differently); numoctaves < 1, or numoctaves > 1 with
 * (int)octaveratio != 2 (pyrDown only halves an image: |2 * dst - src| <= 2), or a smallest octave too small for LSD is CS_ERR_INVALID_ARG;
 * more segments than max_lines_per_octave in an octave is CS_ERR_CAPACITY, naming the frame and the octave.  Synchronous. */
int cs_detect_raw_lines_octaves_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                      const cs_line_params *params, cs_keyline_octave *keylines, int32_t max_lines_per_octave,
                                      int32_t *n_lines /* n_frames * numoctaves */);
/* cs_detect_raw_lines_octaves_batch over host frames of different sizes and channel counts (cs_frame_view, as in cs_detect_lines_batch_mixed):
 * slot (f, k) and n_lines[f * numoctaves + k] hold what cs_detect_raw_lines_octaves_batch returns for frame f alone.  The pyramids of every
 * frame are built one level per launch, and LSD runs once over every octave of every frame.  The same refusals, naming the frame, and the
 * frame checks of cs_detect_lines_batch_mixed, all before anything is enqueued; CS_ERR_CAPACITY names the frame and the octave.  Synchronous. */
int cs_detect_raw_lines_octaves_batch_mixed(cs_ctx *ctx, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params,
                                            cs_keyline_octave *keylines, int32_t max_lines_per_octave, int32_t *n_lines /* n_frames * numoctaves */);
/* line_lbd_detect::detect_descrip_lines_octaves(gray, keylines_out, line_descrips) (line_lbd_allclass.cpp:285-339) for the same detector:
 * the key lines above whose lineLength * (float)pow(octaveratio, octave) > line_length_thres, with start x <= end x (both pairs of ends
 * swapped and the angle folded into [-pi/2, pi/2] where needed), class_id the position in the octave's kept list, and their 32-byte LBD
 * descriptors (binary_descriptor.cpp:603-790), read from the Sobel maps of the key line's octave at its in-octave ends before the swap.  The
 * descriptor's pyramid is its own: GaussianBlur(5 x 5, sigma 1) of the gray frame, then pyrDown per octave, then Sobel 3 x 3.  Slots, counts,
 * checks and errors as cs_detect_raw_lines_octaves_batch; desc32 slot (f, k) starts at row (f * numoctaves + k) * max_lines_per_octave. */
int cs_detect_descrip_lines_octaves_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                          const cs_line_params *params, cs_keyline_octave *keylines, uint8_t *desc32,
                                          int32_t max_lines_per_octave, int32_t *n_lines /* n_frames * numoctaves */);
/* the two calls above on frames already in GPU memory (cs_device_frames): the same outputs, checks and errors; the frames go to the EDLines
 * detector's own buffer, as in cs_lbd_compute_batch_device.  Synchronous. */
int cs_detect_raw_lines_octaves_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const cs_line_params *params, cs_keyline_octave *keylines,
                                             int32_t max_lines_per_octave, int32_t *n_lines);
int cs_detect_descrip_lines_octaves_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const cs_line_params *params,
                                                 cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines);

/* BinaryDescriptor::compute(image, keylines, descriptors[, returnFloatDescr]) (binary_descriptor.cpp:587-790, computeSobel :352-398,
 * computeLBD :1146-1509) on key lines the caller gives, of any octave: the usual line_descriptor pattern of describing what LSDDetector::detect
 * returned, after the caller kept, reordered or edited it.  One call per frame of the reference, frame f with keylines[keyline_offsets[f] ..
 * keyline_offsets[f + 1]) in any order:
 *   - a 3-channel frame is converted to gray (cvtColor BGR2GRAY; the device form follows channel_order);
 *   - the pyramid has max(octave) + 1 levels: GaussianBlur(5 x 5, sigma 1) of the gray frame, then pyrDown to (cols / 2, rows / 2) per level,
 *     a 3 x 3 CV_16S Sobel of each -- the descriptor pyramid of cs_detect_descrip_lines_octaves_batch;
 *   - key line i is described on the maps of its octave, bounded by that octave's width and height, from s_oct_* / e_oct_*, kl.angle and
 *     kl.num_pixels; kl.start_* / end_* are not read;
 *   - rows follow the reference's (class_id, octave) map: when several rows share a pair, the first of them gets the descriptor of the last of
 *     them in list order.  The reference never writes the pair's other rows; here each gets its own descriptor.  The reference also reads the
 *     first line of every class_id from 0 to the largest (:1482-1490) and crashes on a list that skips one, e.g. a filtered subset of a
 *     detector's list; here such a list is described row by row like any other.
 * desc32 has room for keyline_offsets[n_frames] rows of 32 bytes, desc72 (optional) for as many rows of 72 floats.  A frame without key lines
 * writes nothing (the reference prints "keypoint list is empty" and returns).  Errors, all found before anything is enqueued:
 * CS_ERR_INVALID_ARG for a negative class_id or octave (undefined in the reference) and for an octave beyond the pyramid pyrDown can make of
 * the frame (a level of width or height 0, where the reference throws), each naming the frame and the row within it.  Frames of different
 * depths may share a batch.  C++ code that calls the reference's lbd->compute keeps the reference's (INTEGRATION.md section 2).  Synchronous. */
int cs_lbd_compute_octaves_batch(cs_ctx *ctx, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                 const cs_keyline_octave *keylines, const int32_t *keyline_offsets /* n_frames + 1 */, uint8_t *desc32,
                                 float *desc72 /* optional */);
/* the same on frames already in GPU memory (cs_device_frames); the key lines and their CSR stay host buffers; the frames go to the EDLines
 * detector's own buffer, as in cs_lbd_compute_batch_device.  Synchronous. */
int cs_lbd_compute_octaves_batch_device(cs_ctx *ctx, const cs_device_frames *frames, const cs_keyline_octave *keylines,
                                        const int32_t *keyline_offsets, uint8_t *desc32, float *desc72);

/* line_lbd_detect::match_line_descrip(query, train, good_matches, matching_dist_thres) (line_lbd_allclass.cpp:341-356) over
 * BinaryDescriptorMatcher::match (line_lbd/libs/binary_descriptor_matcher.cpp:196-262): for every query descriptor the train descriptor
 * at the smallest Hamming distance -- of several, the one the reference's multi-index hash meets first -- kept when distance < thres.
 * matches has room for n_query entries; they come in query order.  Two cases the reference leaves undefined are defined here: a nearest
 * code further than 128 bits away (its trainIdx is never written there) reports train_idx -1, and a query none of whose bytes is within 4
 * bits of any train code's (the hash never visits anything) yields no match, as in the reference.
 * The batch form matches n_pairs independent (query set, train set) pairs given as CSRs of 32-byte rows: pair p's matches start at
 * matches[query_offsets[p]], n_matches[p] of them. */
int cs_match_line_descrip(cs_ctx *ctx, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, float matching_dist_thres,
                          cs_dmatch *matches, int32_t *n_matches);
int cs_match_line_descrip_batch(cs_ctx *ctx, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32,
                                const int32_t *train_offsets, int n_pairs, float matching_dist_thres, cs_dmatch *matches, int32_t *n_matches);

/* BinaryDescriptorMatcher::knnMatch(query, train, matches, k, mask, compactResult) and radiusMatch(query, train, matches, maxDistance, mask,
 * compactResult) (line_lbd/libs/binary_descriptor_matcher.cpp:264-341, 431-507) -- the pairwise forms, as line_lbd_detect::bdm offers them.
 * A query's answer comes in the order of the reference's multi-index hash (distance first, then the order the hash meets equally near codes,
 * as in cs_match_line_descrip): knn the first k codes, radius every code at distance <= max_distance (note <=, where match_line_descrip
 * keeps distance < thres).  query_idx / train_idx count within the pair, img_idx is 0.  What the reference leaves undefined is defined here:
 *   - only codes the hash meets count (a code none of whose 32 bytes is within 4 bits of the query's is never met), so a query may get
 *     fewer than k entries -- the reference returns k with uninitialised ones;
 *   - a code in the answer further than 128 bits away reports train_idx -1 (the reference never writes its trainIdx), distance as it is;
 *   - an empty query or train set gives no entries (the reference prints and returns); k = 0 gives none; k < 0 is CS_ERR_INVALID_ARG.
 * query_mask (NULL: every query; else one byte per query, 0 = skip) follows the reference's mask: a skipped query gets no entries.  Whether
 * such a query shows as an empty list (compactResult) is the caller's view of n_per_query / match_offsets.
 * Every pair's train set holds at most CS_LBD_KNN_MAX_TRAIN = 16384 codes (the sorting kernel stages a query's keys in 128 KB of shared
 * memory); a larger one is CS_ERR_CAPACITY.
 * knn: matches has room for n_queries x k entries; query i's n_per_query[i] entries start at matches[i * k] (the rest of its row is left as
 * it is).  k <= 2, what a ratio test asks for, takes a kernel of its own that keeps the two best in registers.
 * radius: the entries of query i are matches[match_offsets[i] .. match_offsets[i + 1]), query after query, in matches[0 .. max_matches).
 * When they do not fit the call returns CS_ERR_CAPACITY with match_offsets (n_queries + 1) filled, so match_offsets[n_queries] is the
 * size to call again with. */
int cs_knn_match_line_descrip(cs_ctx *ctx, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, int k, const uint8_t *query_mask,
                              cs_dmatch *matches, int32_t *n_per_query);
int cs_knn_match_line_descrip_batch(cs_ctx *ctx, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32,
                                    const int32_t *train_offsets, int n_pairs, int k, const uint8_t *query_mask, cs_dmatch *matches,
                                    int32_t *n_per_query);
int cs_radius_match_line_descrip(cs_ctx *ctx, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, float max_distance,
                                 const uint8_t *query_mask, cs_dmatch *matches, int64_t max_matches, int64_t *match_offsets);
int cs_radius_match_line_descrip_batch(cs_ctx *ctx, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32,
                                       const int32_t *train_offsets, int n_pairs, float max_distance, const uint8_t *query_mask,
                                       cs_dmatch *matches, int64_t max_matches, int64_t *match_offsets);

/* The collection forms of BinaryDescriptorMatcher ("from one image to a set", line_lbd/libs/binary_descriptor_matcher.cpp:70-104 add / train /
 * clear, :126-193 match, :344-428 knnMatch, :510-595 radiusMatch): one query set against the codes of many images -- a keyframe map for
 * relocalisation or loop closure -- that stay on the device between queries.
 * A collection is created on a context and uses its device and stream; several collections may share one context.  Destroy every
 * collection before its context (cs_lbd_collection_destroy reads the context).  clear() forgets every image and returns the collection's
 * device memory (its codes and scratch buffers); the collection stays usable.  It holds fewer than 2^31 codes in all (CS_ERR_CAPACITY beyond), otherwise only device memory bounds it;
 * there is no per-image or per-call cap on its size.
 * add: n_images images whose codes are codes32[image_offsets[i] .. image_offsets[i + 1]) (32-byte rows, image_offsets has n_images + 1
 * entries starting at 0), appended after what is there; uploaded on the context stream, synchronous.  The reference's train() is implied:
 * the queries search everything added since creation or the last clear.
 * The answers are the pairwise answers (cs_knn_match_line_descrip etc.) over the concatenation of every image added, in the same order:
 *   - train_idx is the GLOBAL row in that concatenation (the reference's choice, not OpenCV's usual row within its image);
 *   - img_idx is the image of the row as the reference's add() records it: an image of 0 codes followed by images starting at the same row
 *     owns that row (std::map::insert keeps the first), so a later non-empty image's matches report the empty image's index, and that
 *     index selects the mask;
 *   - masks (NULL: none; else n_masks = the number of images, mask i at masks + i * n_query, one byte per query, 0 = skip) filter entries
 *     after the selection: an entry survives when the mask of its image keeps its query.  match does not fall back to the next nearest code
 *     when the nearest one's image masks the query: that query gets no match.  n_masks other than the number of images (or nonzero
 *     without masks) is CS_ERR_INVALID_ARG.
 * Where the reference is undefined this is defined:
 *   - a query meets fewer than k codes, or none at all: fewer entries, no match (as the pairwise forms);
 *   - an entry further than D = 128 bits away reports train_idx -1 and img_idx -1 (its trainIdx is never written there); with masks such
 *     entries are dropped, as there is no image mask to consult;
 *   - a second query after more add()s (the reference re-populates its hash with rows restarting at 0, and a second collection
 *     radiusMatch runs with setK(0)): every query answers as the reference's first query after all the add()s since creation or clear().
 * An empty collection or query set gives no entries; k = 0 gives none; k < 0 is CS_ERR_INVALID_ARG.
 * Output layouts and the radius protocol are the pairwise ones: knn writes query i's n_per_query[i] entries at matches[i * k]; match writes
 * its matches in query order, *n_matches of them (room for n_query); radius writes query i's entries at matches[match_offsets[i] ..
 * match_offsets[i + 1]) and returns CS_ERR_CAPACITY with match_offsets (n_query + 1) filled when they exceed max_matches. */
typedef struct cs_lbd_collection cs_lbd_collection;
cs_lbd_collection *cs_lbd_collection_create(cs_ctx *ctx); /* NULL when ctx is NULL */
void cs_lbd_collection_destroy(cs_lbd_collection *coll);
int cs_lbd_collection_add(cs_lbd_collection *coll, const uint8_t *codes32, const int32_t *image_offsets, int n_images);
int cs_lbd_collection_clear(cs_lbd_collection *coll);
int cs_lbd_collection_size(const cs_lbd_collection *coll, int32_t *n_images, int64_t *n_codes);
int cs_lbd_collection_match(cs_lbd_collection *coll, const uint8_t *query32, int n_query, const uint8_t *masks, int n_masks, cs_dmatch *matches,
                            int32_t *n_matches);
int cs_lbd_collection_knn_match(cs_lbd_collection *coll, const uint8_t *query32, int n_query, int k, const uint8_t *masks, int n_masks,
                                cs_dmatch *matches, int32_t *n_per_query);
int cs_lbd_collection_radius_match(cs_lbd_collection *coll, const uint8_t *query32, int n_query, float max_distance, const uint8_t *masks,
                                   int n_masks, cs_dmatch *matches, int64_t max_matches, int64_t *match_offsets);

/* tests: what the host side hands the descriptor kernel -- per key line {mid x, mid y, cos, sin, length, frame} (6 x 4 bytes) -- and the
 * two Gaussian weight tables F_g (63) and F_l (21) as floats (binary_descriptor.cpp:140-179).  Host-only, needs no context. */
int cs_lbd_debug_prepare(const cs_keyline *keylines, int n, void *lines24, float *coef_g63, float *coef_l21);
/* tests: the key lines cs_detect_descrip_lines assembles for the EDLines flavour from what the detector kernels leave per kept segment --
 * the ordered end points and extra2 = {lineDirection_, numOfPixels as an integer's bits} (binary_descriptor.cpp:526-545).  Host-only. */
int cs_lbd_debug_keylines_edl(const float *lines_xyxy, const float *extra2, int n, int width, int height, cs_keyline *out);

/* How the reference draws a detected cuboid (plot_image_with_cuboid, detect_3d_cuboid/src/object_3d_util.cpp:54-131, called with
 * whether_save_final_images / whether_plot_final_images, box_proposal_detail.cpp:541-556): its 12 edges in the reference's order, each
 * {x1, y1, x2, y2, B, G, R, thickness}; the caller rasterises them with cv::line(..., CV_AA) exactly as the reference does
 * (visible edges thick, hidden ones thin; red / green / blue per vanishing-point family).  Host-only, needs no context. */
int cs_cuboid_draw_edges(const cs_cuboid_rec *rec, int32_t edges[12][8]);

/* The atan2 of the cuboid stage's angle-error chain (merge_break_lines, VP_support_edge_infos, box_edge_alignment_angle_error;
 * object_3d_util.cpp:167-172,321,392,480) is defined arithmetically (cube_slam_b200/csrc/cs_pmath.h: IEEE + - * / only, within 1 ulp of
 * glibc's) so that it rounds the same on the host, on the device and in the test oracle.  cs_debug_atan2 evaluates it on the device,
 * cs_atan2_host on the host (tests). */
int cs_debug_atan2(cs_ctx *ctx, const double *y, const double *x, double *out, int n);
double cs_atan2_host(double y, double x);

/* The number-of-false-alarms test both line detectors end with (cube_slam_b200/csrc/cs_nfa.cuh: lsd.cpp's nfa with lsd_first_term = 1,
 * descriptor.hpp's with 0), evaluated on the device by one warp per (n[i], k[i], p[i]) with the log_gamma table the detectors use (tests):
 * out_value[i] the NFA, out_break[i] the i at which the binomial tail's loop stopped (n + 1: it ran to the end; -1: an early return or the
 * underflow branch). */
int cs_debug_nfa(cs_ctx *ctx, const int32_t *n, const int32_t *k, const double *p, double logNT, int lsd_first_term, double *out_value,
                 int32_t *out_break, int count);

/* ---- multi-GPU -------------------------------------------------------------------------- */
/* Frames shard across ranks; the only exchange is one all-gather of the top-K record buffers.
 * No reference counterpart (the reference is single process); see BASELINE.json north_star. */
int cs_comm_unique_id(cs_ctx *ctx, const char *nccl_library_path, uint8_t id_out[128]);
int cs_comm_init(cs_ctx *ctx, const char *nccl_library_path, const uint8_t id[128], int world_size, int rank);
/* all-gather recs_per_rank records from every rank's record buffer into gathered (DEVICE pointer owned by the
 * context, returned through *gathered_dev; world_size x recs_per_rank records).
 * The collective runs on a stream of its own, ordered after the work queued on the context so far; the context's next batch only waits
 * for it where it overwrites the record buffer.  cs_fetch_gathered waits for it; anything else a caller queues on the context stream and
 * wants ordered behind the gather (a timing event, its own copy of *gathered_dev) goes after cs_allgather_wait (a stream-level wait, the
 * host does not block). */
int cs_allgather_topk(cs_ctx *ctx, int recs_per_rank, void **gathered_dev);
int cs_allgather_wait(cs_ctx *ctx);
int cs_fetch_gathered(cs_ctx *ctx, cs_cuboid_rec *out, int n_records);

#ifdef __cplusplus
}
#endif
#endif /* CUBE_SLAM_B200_H */
