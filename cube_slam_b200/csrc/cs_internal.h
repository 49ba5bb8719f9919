/* cs_internal.h -- structures shared by the host orchestration and the sm_90a kernels. */
#ifndef CS_INTERNAL_H
#define CS_INTERNAL_H

#include <stdint.h>

#include <vector>

#include "../../include/cube_slam_b200.h"

#define CS_MAX_YAW 512        /* yaw samples per object (reference default 16; dense sweep 181) */
#define CS_MAX_POSE 32        /* roll x pitch samples (reference 5 x 5) */
#define CS_MAX_TOPK 32        /* upper bound of max_cuboid_num handled on device */
#define CS_LINE_CAP 1024      /* lines of one frame that fall inside one ROI (shared-memory resident) */
#define CS_MAXL_OUT 256       /* merged lines kept per ROI */
#define CS_SM_COUNT 132       /* H100 SXM: the grid-stride kernels launch at most a small multiple of this many CTAs */

/* One camera pose hypothesis: detect_3d_cuboid::cam_pose after set_cam_pose
 * (box_proposal_detail.cpp:42-54) plus the ground plane in the sensor frame (:100,238). */
struct CsPose {
    double KinvR[9];
    double T[16];
    double ground[4];
    double roll, pitch;
    double camera_yaw; /* cam_pose.camera_yaw re-derived through the quaternion */
};

/* Per-frame constants */
struct CsFrame {
    double invK[9];
    double euler_raw[3];
    int32_t pose_off;  /* first CsPose of this frame; pose 0 == raw pose when sampling is off */
    int32_t n_pose;
    int32_t yaw_off;   /* first yaw sample of this frame in the yaw table */
    int32_t n_yaw;
    int32_t line_off;  /* CSR into the batch line array */
    int32_t n_lines;
};

/* One (2D box, height sample) ROI job: box_proposal_detail.cpp:107-163 evaluated on the host. */
struct CsJob {
    int32_t frame;
    int32_t obj;        /* global object index */
    int32_t hs;         /* height-sample id */
    int32_t left, top, right;           /* left_x_raw, top_y_raw, right_x_raw */
    int32_t width_raw, height_raw;
    int32_t down_expand, down_y_expan;
    int32_t roi_l, roi_t, roi_r, roi_b; /* dist-map ROI corners (inclusive box test uses these) */
    int32_t roi_w, roi_h;               /* width_expan_distmap, height_expan_distmap */
    int32_t n_top, top_lo, top_hi, top_step, top_override;
    int32_t n_cand;                     /* n_pose * n_yaw * n_top * 2 */
    int32_t tile_off;                   /* first canny tile of this job (prefix over jobs) */
    int32_t tiles_x;
    int32_t bw;                         /* 32-bit words per bit-plane row, ceil(roi_w / 32) */
    int32_t dpitch;                     /* row pitch of the dist map in floats (roi_w rounded up to 4) */
    int32_t gray_pitch;                 /* row pitch (bytes) of the frame's gray plane */
    int64_t gray_off;                   /* byte (roi_l, roi_t) of the frame's gray plane, from the batch's frame buffer */
    int64_t bit_off;                    /* offset (words) of this ROI's two bordered bit planes */
    int64_t px_off;                     /* offset (floats) of this ROI's dist map, multiple of 16 */
    int64_t cand_off;                   /* offset into the candidate record arenas */
    double diag;                        /* obj_diaglength_expan */
};

struct CsObj {
    int32_t frame;
    int32_t job_off, n_jobs;
    int32_t left, top, width_raw, height_raw;
};


/* narrow view of the context for the other translation units (the struct itself lives in cs_context.cu) */
#ifdef __CUDACC__
#include <cuda_runtime.h>
cudaStream_t cs_ctx_stream(cs_ctx *c);
#endif
int cs_ctx_device(cs_ctx *c);
int cs_ctx_fail(cs_ctx *c, int code, const char *fmt, ...);
void **cs_ctx_lsd_slot(cs_ctx *c);          /* owned by cs_lsd.cu */
void cs_lsd_destroy(void *state);           /* called from cs_destroy */
int cs_lsd_run_device(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int w, int h, int stride, int channels, float line_length_thres, int cap,
                      const float **d_lines, const int32_t **d_counts);
void cs_ctx_count_launches(cs_ctx *c, int64_t n);
int cs_ctx_seq_lines(cs_ctx *c);            /* cs_set_profiling bit 7; read by cs_edlines.cu only */
int cs_ctx_profiling(cs_ctx *c);            /* cs_set_profiling bit 0 */
int cs_ctx_use_tma(cs_ctx *c);              /* cs_set_profiling bit 8 clear */
void **cs_ctx_edl_slot(cs_ctx *c);          /* owned by cs_edlines.cu */
void cs_edl_destroy(void *state);           /* called from cs_destroy */
/* EDLines flavour of detect_filter_lines: frames on the device (or host, copied in) -> filtered float32 segments + counts in HBM */
int cs_edl_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
               int cap, const float **d_lines, const int32_t **d_counts);

/* the same run, also keeping per kept segment what the descriptor needs of its key line (binary_descriptor.cpp:526-540): d_extra holds
 * cap x 2 floats per frame, {KeyLine::angle (lineDirection_), KeyLine::numOfPixels as an integer's bits}, parallel to d_lines */
int cs_edl_run_keylines(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels,
                        float line_length_thres, int cap, const float **d_lines, const int32_t **d_counts, const float **d_extra,
                        const int16_t **d_dx, const int16_t **d_dy /* the detector's own Sobel maps, the ones the descriptor reads */);
/* BinaryDescriptor::computeSobel for octave 0 (binary_descriptor.cpp:352-398: GaussianBlur 5 x 5 sigma 1, Sobel 3 x 3 to 16S) = the front
 * end of the EDLines detector: the two int16 maps of every frame, in HBM, owned by the EDLines workspace */
int cs_edl_sobel_maps(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels,
                      const int16_t **d_dx, const int16_t **d_dy);
/* LSD flavour of detect_filter_lines from host frames (the body of cs_detect_lines_batch's LSD branch): filtered segments + counts in HBM */
int cs_lsd_run_host(cs_ctx *c, const uint8_t *imgs, int n_frames, int w, int h, int stride, int channels, float line_length_thres, int cap,
                    const float **d_lines, const int32_t **d_counts, const uint8_t **d_frames);
/* the same synchronous run on host frames or on frames already in the LSD frame buffer; d_frames: the frames the run read, in HBM */
int cs_lsd_run_sync(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
                    int cap, const float **d_lines, const int32_t **d_counts, const uint8_t **d_frames);
/* The line detectors' error words: 16 bytes in HBM per workspace, cleared at the start of every run (and of cs_edl_sobel_maps), set by
 * their kernels.  LSD: [0] 4 = a frame had more candidate rectangles than the hand-off buffer holds ([1]: the largest such count, [2]: the
 * buffer's size per frame), 8 = a TMA tile copy of the front end did not complete.  EDLines: [0] 1 = more anchors in a frame than
 * w * h / 5 + 1, 8 = a TMA tile copy of the front end did not complete.  The workspaces behind cs_ctx_lsd_slot / cs_ctx_edl_slot begin
 * with a CsLineHead, so the batch path finds the word without a call into the detectors.  The synchronous entry points read it back with
 * their results and fail precisely instead of returning wrong segments with CS_OK. */
struct CsLineHead {
    int32_t *d_err; /* the error word of the workspace's runs (device memory; null before the first run) */
};
static inline const int32_t *cs_line_err_word(void *workspace) { return workspace ? ((const CsLineHead *)workspace)->d_err : nullptr; }
static inline int cs_lsd_check_err(cs_ctx *c, const int32_t err[4])
{
    if (err[0] & 8) return cs_ctx_fail(c, CS_ERR_CUDA, "a TMA tile copy of the LSD front end did not complete");
    if (err[0] & 4)
        return cs_ctx_fail(c, CS_ERR_CAPACITY, "a frame has %d LSD candidate regions, more than the %d per frame the candidate buffer held", err[1], err[2]);
    return CS_OK;
}
static inline int cs_edl_check_err(cs_ctx *c, const int32_t err[4])
{
    if (err[0] & 8) return cs_ctx_fail(c, CS_ERR_CUDA, "a TMA tile copy of the EDLines front-end kernel did not complete");
    if (err[0] & 1) return cs_ctx_fail(c, CS_ERR_CAPACITY, "a frame has more EDLines anchors than w * h / 5 + 1");
    return CS_OK;
}
void **cs_ctx_lbd_slot(cs_ctx *c);          /* owned by cs_lbd.cu */

/* frames already on the device (cs_ingest.cu) */
int cs_ctx_store_device_batch(cs_ctx *c, int n_frames, int width, int height, int channels, const double *T_wc, const double *boxes,
                              const int32_t *box_offsets, const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params,
                              const cs_line_params *online, uint8_t **d_img);
void cs_ctx_mark_prepared(cs_ctx *c);
void cs_set_frames_error(const char *msg);  /* what cs_last_error(NULL) reports after a failed cs_check_device_frames */
/* the line detectors' own frame buffers (the ones cs_detect_lines_batch copies host frames into), grown to `bytes`; null on failure */
uint8_t *cs_lsd_frame_buffer(cs_ctx *c, size_t bytes);
uint8_t *cs_edl_frame_buffer(cs_ctx *c, size_t bytes);
/* the body of cs_detect_lines_batch after its argument checks, on host frames or on frames already on the device; with views (LSD only), on
 * frames of different sizes on the device at imgs + views[f].offset; frame_index: the caller's numbers of the frames, for the messages */
int cs_detect_lines_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int width, int height, int stride, int channels,
                        const cs_line_params *params, float *lines_xyxy, int32_t max_lines_per_frame, int32_t *n_lines,
                        const cs_frame_view *views = nullptr, const int32_t *frame_index = nullptr);
/* ---- batches of frames of different sizes (cs_lsd.cu) */
/* the host checks of a frame table (cs_detect_lines_batch_mixed's), each failure naming the frame */
int cs_check_frame_views(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames);
/* the line detectors' size checks of a frame table (cs_detect_lines_batch_mixed's, each failure naming the frame): LSD's smallest frame and
 * batch size, EDLines' size bounds, numoctaves >= 1 */
int cs_check_line_frames(cs_ctx *c, const cs_frame_view *views, int n_frames, const cs_line_params *params);
/* bytes of the frames packed back to back without row padding, and the copy of host frames into that layout; `packed` their views there */
size_t cs_packed_frames_bytes(const cs_frame_view *views, int n_frames);
int cs_pack_host_frames(cs_ctx *c, uint8_t *d_dst, const uint8_t *imgs, const cs_frame_view *views, int n_frames, std::vector<cs_frame_view> &packed);
/* cs_lsd_run_sync on device frames of different sizes, frame f at d_imgs + views[f].offset: one LSD run over all of them; the raw segments
 * (cs_lsd_raw_segments) and the filtered ones at cap per frame, in HBM.  cs_debug_lsd and cs_debug_lsd_defb refuse after such a run. */
#define CS_LSD_MAX_MIXED_FRAMES 33554431 /* frames (or octave planes) of one mixed LSD run: 64 validation CTAs each in a grid's x (2^31 - 1) */
int cs_lsd_run_mixed_sync(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, float line_length_thres, int cap,
                          const float **d_lines, const int32_t **d_counts);
/* the same run enqueued only (the online cuboid batch, cs_mixed.cu): no host sync, no rerun; *d_err is the run's error word, a candidate
 * overflow shows there */
int cs_lsd_run_mixed_device(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, float line_length_thres, int cap,
                            const float **d_lines, const int32_t **d_counts, const int32_t **d_err);
/* One plane of a table-driven 8-bit conversion over frames of any sizes: its source (sw x sh, rows of sstride bytes, ch channels) and its
 * destination (dw x dh, packed), and px0, the pixels of the table's earlier planes (cs_launch_gray_tab, cs_lbd_octaves.cu). */
struct OctPlane {
    int64_t src, dst, px0;
    int32_t sw, sh, sstride, ch, dw, dh, pad_;
};
void cs_lbd_destroy(void *state);           /* called from cs_destroy */
/* what a synchronous detector run of the descriptor path leaves in HBM: the kept segments and their counts (cap per frame); EDLines: the
 * {direction, numOfPixels} pairs and the Sobel maps the descriptor reads; LSD: the frames the detector read, for the Sobel maps */
struct CsDetectedLines {
    const float *lines = nullptr, *extra = nullptr;
    const int32_t *counts = nullptr;
    const int16_t *dx = nullptr, *dy = nullptr;
    const uint8_t *lsd_frames = nullptr;
};
/* the body of cs_detect_descrip_lines_batch after detection (cs_lbd.cu): key lines filled on the host, descriptors, the per-frame slots;
 * `stride` is the row pitch of d.lsd_frames */
int cs_lbd_describe_detected(cs_ctx *c, const CsDetectedLines &d, bool use_LSD, int n_frames, int width, int height, int stride, int channels,
                             cs_keyline *keylines, uint8_t *desc32, int32_t max_lines_per_frame, int32_t *n_lines);
/* cs_lbd_compute_batch's key-line arguments: the CSR checked, *n its total; 0 = nothing to describe (no output touched) */
int cs_lbd_check_given(cs_ctx *c, int n_frames, const cs_keyline *keylines, const int32_t *keyline_offsets, const uint8_t *desc32, int *n);
/* the body of cs_lbd_compute_batch after its checks, on host frames or on frames already on the device (packed rows of `stride` bytes) */
int cs_lbd_compute_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int width, int height, int stride, int channels,
                       const cs_keyline *keylines, const int32_t *keyline_offsets, uint8_t *desc32, float *desc72);

/* ---- every octave of a multi-octave LSD detector (cs_lbd_octaves.cu) */
/* the raw segments of the last LSD run (accepted candidates in seed order, before the key-line filter): max_lines_per_frame x 4 floats per
 * frame, and per frame their count (> the capacity when they did not fit) -- in HBM, until the next run (cs_lsd.cu) */
void cs_lsd_raw_segments(cs_ctx *c, const float **d_raw, const int32_t **d_nraw);
/* LSDDetector::detect's KeyLine fill (LSDDetector.cpp:205-250) for one LSD segment `raw` of octave `octave` (an ow x oh image, 2^octave =
 * `scale`) of a w x h input frame: false when the border test drops it (cs_lbd.cu) */
bool cs_keyline_from_lsd_octave(const float *raw, float scale, int ow, int oh, int w, int h, int octave, int class_id, cs_keyline_octave &o);
/* the 32-byte descriptors of n key lines, line i of frame frame[i] of the n_frames x h x w Sobel maps d_dx / d_dy, to the host, and the
 * 72-float descriptors when desc72 is not NULL (cs_lbd.cu) */
int cs_lbd_describe_keylines(cs_ctx *c, const cs_keyline *keylines, const int32_t *frame, int n, const int16_t *d_dx, const int16_t *d_dy, int w,
                             int h, uint8_t *desc32, float *desc72);
/* the body of the octave calls after their argument checks, on packed frames (rows of `stride` bytes) already on the device */
int cs_lsd_octaves_run(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int width, int height, int stride, int channels, const cs_line_params *params,
                       bool describe, cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines);
/* cs_lbd_compute_octaves_batch's checks of its key lines (the frames are checked by the caller): the CSR, class_id and octave >= 0, every
 * octave within the pyramid pyrDown can make of a width x height frame; *n the total, 0 = nothing to describe (no output touched) */
int cs_lbd_octaves_check_given(cs_ctx *c, int n_frames, int width, int height, const cs_keyline_octave *keylines, const int32_t *keyline_offsets,
                               const uint8_t *desc32, int *n);
/* its body after the checks, on packed frames (rows of `stride` bytes) already on the device */
int cs_lbd_compute_octaves_run(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int width, int height, int stride, int channels,
                               const cs_keyline_octave *keylines, const int32_t *keyline_offsets, uint8_t *desc32, float *desc72);
/* the octave calls' checks of params and max_lines_per_octave (the frames are checked by the caller); frame >= 0: the frame the size
 * message names */
int cs_lsd_octaves_check(cs_ctx *c, int width, int height, const cs_line_params *params, const void *keylines, const void *desc32, bool describe,
                         int32_t max_lines_per_octave, const int32_t *n_lines, int frame = -1);
/* cs_lsd_octaves_run on frames of any sizes already on the device, frame f at d_imgs + views[f].offset (describe: frames of one size) */
int cs_lsd_octaves_run_views(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params, bool describe,
                             cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines);

#endif
