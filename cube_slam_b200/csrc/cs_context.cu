/*
 * cs_context.cu -- the C ABI of libcubeslam_b200.so: context, batch orchestration, host<->device.
 *
 * Host work per batch is O(frames + boxes): the camera-pose tables, the sample grids and the
 * per-box ROI job descriptors of detect_cuboid (box_proposal_detail.cpp:59-60,99-163,215-226);
 * everything per pixel / per line / per proposal runs in the CUDA kernels.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "cs_carried.h"
#include "cs_host_pose.h"
#include "cs_internal.h"
#include "cs_kernels.h"

namespace {

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

enum Stage { ST_LSD, ST_GRAY, ST_CANNY, ST_HYST, ST_DT, ST_LINES, ST_SWEEP, ST_FUSE, ST_COUNT };
const char *kStageNames[ST_COUNT] = {"lsd", "gray", "canny", "hyst", "dt", "lines", "sweep", "fuse"};

}  // namespace

struct cs_ctx {
    int device = 0;
    int max_w = 0, max_h = 0, max_frames = 0, max_boxes = 0, max_lines = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    double K[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    bool have_K = false;

    /* current batch (host copies of the small inputs) */
    bool prepared = false;
    int n_frames = 0, w = 0, h = 0, stride = 0, channels = 0; /* a one-size batch's frames (0 for a batch of mixed sizes) */
    /* per frame, for every batch: where it lies in d_img, its calibration (9 doubles) and its gray plane (bytes from d_img, rows of
     * views[f].width bytes: the frame itself when it is packed gray, else a plane after the frames that the gray stage fills) */
    std::vector<cs_frame_view> views;
    std::vector<double> Ks;
    std::vector<int64_t> gray_off;
    int64_t gray_base = 0;             /* where the converted gray planes start in d_img */
    /* a batch of mixed sizes: its stages (cs_mixed.cu), the table of its frames to convert to gray, and its frames in d_img order */
    const CsMixedStages *mixed = nullptr;
    std::vector<OctPlane> gray_tab;
    int64_t gray_tab_px = 0;
    std::vector<int32_t> order;
    cs_cuboid_params prm;
    std::vector<double> h_T, h_boxes, h_lines;
    std::vector<int32_t> h_box_off, h_line_off;
    int topk = 1;
    bool online_lines = false; /* lines come from the line detector run on the uploaded frames */
    cs_line_params line_prm;
    int online_cap = 1024;
    const int32_t *d_online_counts = nullptr; /* per-frame segment counts of the last online run (device) */

    /* host tables built by build_tables() */
    std::vector<CsFrame> frames;
    std::vector<CsPose> poses;
    std::vector<double> yaws;
    std::vector<CsJob> jobs;
    std::vector<CsObj> objs;
    std::vector<int4> sweep_blocks4; /* warp sweep: (job, pose, first yaw, yaws in block) */
    int max_n_cand = 0;
    int use_cta_select = 0; /* debug: force the CTA-wide selection kernel (k_fuse_rank) for every box */
    std::vector<int32_t> dt_ids, tile_job;
    int dt_class_off[CS_DT_CLASSES + 1] = {0}, dt_class_plane_words[CS_DT_CLASSES] = {0};
    int64_t total_px = 0, total_cand = 0, total_bits = 0;
    int n_tiles = 0, max_plane_words = 0, max_dpitch = 0;
    int use_raster_dt = 0; /* A/B: two-pass raster-scan distance transform instead of the cone form */
    bool use_tma = true;       /* tile kernels of the line detectors: interior tiles staged by the copy engine (cp.async.bulk.tensor); bit 8 of cs_set_profiling turns it off */
    cudaStream_t stream2 = nullptr; /* side stream: the line kernel runs beside the image chain */
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    /* the skinny, latency-bound tail of the chain (distance transform -> sweep -> selection: a few warps per SM, long dependent chains) runs on
     * a high-priority stream: with several batches in flight its blocks are dispatched ahead of another batch's machine-filling
     * gray / Canny grids instead of queueing behind them */
    cudaStream_t stream_hi = nullptr;
    cudaEvent_t ev_mid = nullptr, ev_done = nullptr, ev_dt_fork = nullptr, ev_dt_join = nullptr;
    cudaEvent_t ev_ingest_in = nullptr, ev_ingest_out = nullptr; /* device frames (cs_ingest.cu): producer stream -> context stream -> producer stream */
    int use_prio = 1;
    int seq_lines = 0;     /* A/B: EDLines' round-1 routing and fitting kernels (cs_edlines.cu) */

    /* device buffers (grow only) */
    DevBuf d_img, d_lines, d_frames, d_poses, d_yaws, d_jobs, d_objs, d_blocks4, d_dtids, d_tilejob;
    DevBuf d_bits, d_dist, d_mlines, d_lcounts, d_err;
    DevBuf d_cvalid, d_cdist, d_cangle, d_cskew, d_vlist, d_key, d_idx, d_flag, d_keep, d_norm, d_score, d_jcounts;
    DevBuf d_out, d_outcnt, d_gather, d_send;
    DevBuf d_graytab, d_order, d_online_lines, d_online_nl; /* a batch of mixed sizes: gray table, d_img order, EDLines' per-frame slots */
    void *pinned = nullptr;
    size_t pinned_cap = 0;

    /* profiling */
    bool profiling = false;
    cudaEvent_t ev[ST_COUNT + 1] = {nullptr};
    cudaEvent_t ev_total[2] = {nullptr, nullptr};
    float stage_ms[ST_COUNT] = {0};
    float total_ms = 0;
    bool stage_valid = false;
    int64_t launches = 0;
    cs_batch_stats stats;

    void *lsd_state = nullptr; /* line-detector workspace (cs_lsd.cu) */
    void *edl_state = nullptr; /* EDLines workspace (cs_edlines.cu) */
    void *lbd_state = nullptr; /* descriptor / matcher workspace (cs_lbd.cu) */
    /* cs_set_profiling bit 10: later boxes of a roll / pitch-sampled frame start from the camera pose the reference leaves behind
     * (detect_batch_carried); yaw_override[f] is the cam_pose.camera_yaw a pass derives its yaw samples from (NaN: the raw pose's) */
    bool carry_cam_pose = false;
    std::vector<double> yaw_override;
    int64_t line_launches = 0;

    /* NCCL (loaded at run time) */
    void *nccl_lib = nullptr;
    void *nccl_comm = nullptr;
    /* the all-gather runs on a stream of its own (cs_nccl_impl.inc): a rank that reaches a batch's gather before its peer must not hold
     * up the kernels of the context's next batch, only that batch's final write of the record buffer */
    cudaStream_t gather_stream = nullptr;
    cudaEvent_t ev_gather_ready = nullptr, ev_gather_done = nullptr;
    bool gather_pending = false;
    int world = 1, rank = 0;
};

#include "cs_nccl.h"

cudaStream_t cs_ctx_stream(cs_ctx *c) { return c->stream; }
int cs_ctx_device(cs_ctx *c) { return c->device; }
void **cs_ctx_lsd_slot(cs_ctx *c) { return &c->lsd_state; }
int cs_ctx_seq_lines(cs_ctx *c) { return c->seq_lines; }
int cs_ctx_profiling(cs_ctx *c) { return c->profiling ? 1 : 0; }
int cs_ctx_use_tma(cs_ctx *c) { return c->use_tma ? 1 : 0; }
void **cs_ctx_edl_slot(cs_ctx *c) { return &c->edl_state; }
void **cs_ctx_lbd_slot(cs_ctx *c) { return &c->lbd_state; }
void cs_ctx_count_launches(cs_ctx *c, int64_t n) { c->line_launches += n; }
void cs_ctx_ingest_events(cs_ctx *c, cudaEvent_t *in, cudaEvent_t *out)
{
    *in = c->ev_ingest_in;
    *out = c->ev_ingest_out;
}
/* the message of the calling thread's last failed cs_check_device_frames (no context to hold it); cs_last_error(NULL) returns it */
static thread_local std::string t_frames_err;
void cs_set_frames_error(const char *msg) { t_frames_err = msg ? msg : ""; }
int cs_ctx_fail(cs_ctx *c, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    return code;
}

namespace {

int fail(cs_ctx *c, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    return code;
}

#define CS_CUDA(c, call)                                                                              \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) return fail((c), CS_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
    } while (0)

int ensure(cs_ctx *c, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return CS_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    const size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) return fail(c, CS_ERR_CUDA, "cudaMalloc(%zu): %s", want, cudaGetErrorString(e));
    b.cap = want;
    return CS_OK;
}

template <class T>
int upload(cs_ctx *c, DevBuf &b, const std::vector<T> &v)
{
    const size_t bytes = sizeof(T) * v.size();
    int rc = ensure(c, b, std::max<size_t>(bytes, 16));
    if (rc) return rc;
    if (bytes) CS_CUDA(c, cudaMemcpyAsync(b.p, v.data(), bytes, cudaMemcpyHostToDevice, c->stream));
    return CS_OK;
}

/* Host evaluation of box_proposal_detail.cpp:59-60,99-163,215-226 for the whole batch. */
int build_tables(cs_ctx *c)
{
    const cs_cuboid_params &p = c->prm;
    const int F = c->n_frames;
    c->frames.assign(F, CsFrame());
    c->poses.clear();
    c->yaws.clear();
    c->jobs.clear();
    c->objs.clear();
    c->sweep_blocks4.clear();
    c->max_n_cand = 0;
    c->total_px = 0;
    c->total_cand = 0;
    c->total_bits = 0;
    c->n_tiles = 0;
    c->max_plane_words = 0;
    c->max_dpitch = 0;

    for (int f = 0; f < F; f++) {
        CsFrame &fr = c->frames[f];
        const int img_width = c->views[f].width, img_height = c->views[f].height;
        const double *K = &c->Ks[(size_t)f * 9];
        cshost::invert3(K, fr.invK);
        const double *T = &c->h_T[(size_t)f * 16];
        CsPose raw;
        cshost::make_pose(K, T, &raw, fr.euler_raw);
        fr.pose_off = (int32_t)c->poses.size();
        if (p.whether_sample_cam_roll_pitch) {
            /* :215-226, :233-239 */
            std::vector<double> rolls, pitches;
            cshost::linespace_d(fr.euler_raw[0] - 6.0 / 180.0 * M_PI, fr.euler_raw[0] + 6.0 / 180.0 * M_PI, 3.0 / 180.0 * M_PI, rolls);
            cshost::linespace_d(fr.euler_raw[1] - 6.0 / 180.0 * M_PI, fr.euler_raw[1] + 6.0 / 180.0 * M_PI, 3.0 / 180.0 * M_PI, pitches);
            if ((int)(rolls.size() * pitches.size()) > CS_MAX_POSE) return fail(c, CS_ERR_CAPACITY, "too many roll/pitch samples");
            for (double r : rolls)
                for (double q : pitches) {
                    double Tn[16], Rn[9];
                    std::memcpy(Tn, T, sizeof(Tn));
                    cshost::euler_to_rot(r, q, fr.euler_raw[2], Rn);
                    for (int i = 0; i < 3; i++)
                        for (int j = 0; j < 3; j++) Tn[i * 4 + j] = Rn[i * 3 + j];
                    CsPose ps;
                    cshost::make_pose(K, Tn, &ps, nullptr);
                    ps.roll = r; /* the sampled values are what the reference records (:453) */
                    ps.pitch = q;
                    c->poses.push_back(ps);
                }
        } else {
            raw.roll = fr.euler_raw[0];
            raw.pitch = fr.euler_raw[1];
            c->poses.push_back(raw);
        }
        fr.n_pose = (int32_t)c->poses.size() - fr.pose_off;
        /* :126-128 */
        const double cam_yaw = ((size_t)f < c->yaw_override.size() && !std::isnan(c->yaw_override[f])) ? c->yaw_override[f] : raw.camera_yaw;
        const double yaw_init = cam_yaw - 90.0 / 180.0 * M_PI;
        std::vector<double> ys;
        cshost::linespace_d(yaw_init - p.yaw_half_range_deg / 180.0 * M_PI, yaw_init + p.yaw_half_range_deg / 180.0 * M_PI,
                            p.yaw_step_deg / 180.0 * M_PI, ys);
        if ((int)ys.size() > CS_MAX_YAW) return fail(c, CS_ERR_CAPACITY, "too many yaw samples (%zu)", ys.size());
        fr.yaw_off = (int32_t)(c->yaws.size() / 3); /* entries of {yaw, cos, sin}: the reference takes both from libm on the host (object_3d_util.cpp:604-606,44) */
        fr.n_yaw = (int32_t)ys.size();
        for (double yv : ys) {
            c->yaws.push_back(yv);
            c->yaws.push_back(std::cos(yv));
            c->yaws.push_back(std::sin(yv));
        }
        fr.line_off = c->h_line_off[f];
        fr.n_lines = c->h_line_off[f + 1] - c->h_line_off[f];

        for (int b = c->h_box_off[f]; b < c->h_box_off[f + 1]; b++) {
            const double *bb = &c->h_boxes[(size_t)b * 5];
            /* :107-112 */
            const int left_x_raw = (int)bb[0], top_y_raw = (int)bb[1];
            const int obj_width_raw = (int)bb[2], obj_height_raw = (int)bb[3];
            const int right_x_raw = (int)(left_x_raw + bb[2]);
            CsObj ob;
            ob.frame = f;
            ob.job_off = (int32_t)c->jobs.size();
            ob.left = left_x_raw;
            ob.top = top_y_raw;
            ob.width_raw = obj_width_raw;
            ob.height_raw = obj_height_raw;
            /* :114-123 */
            int hs_list[3], n_hs = 0;
            hs_list[n_hs++] = 0;
            if (p.whether_sample_bbox_height) {
                int r = std::max(std::min(20, obj_height_raw - 90), 20);
                r = std::min(r, img_height - top_y_raw - obj_height_raw - 1);
                if (r > 10) hs_list[n_hs++] = (int)std::round(r / 2);
                hs_list[n_hs++] = r;
            }
            for (int hs = 0; hs < n_hs; hs++) {
                CsJob jb;
                std::memset(&jb, 0, sizeof(jb));
                jb.frame = f;
                jb.obj = b;
                jb.hs = hs;
                jb.left = left_x_raw;
                jb.top = top_y_raw;
                jb.right = right_x_raw;
                jb.width_raw = obj_width_raw;
                jb.height_raw = obj_height_raw;
                jb.down_expand = hs_list[hs];
                const int obj_height_expan = obj_height_raw + jb.down_expand;
                jb.down_y_expan = top_y_raw + obj_height_expan;
                jb.diag = std::sqrt((double)(obj_width_raw * obj_width_raw + obj_height_expan * obj_height_expan)); /* :141 */
                /* :144-146 */
                jb.top_lo = left_x_raw + 5;
                jb.top_hi = right_x_raw - 5;
                if (p.top_sample_count_override > 0) {
                    jb.top_override = 1;
                    jb.top_step = 1;
                    jb.n_top = (jb.top_hi >= jb.top_lo) ? p.top_sample_count_override : 0;
                } else {
                    jb.top_step = (int)std::round(std::min(20, obj_width_raw / 10));
                    jb.n_top = cshost::linespace_count_i(jb.top_lo, jb.top_hi, jb.top_step);
                }
                /* :155-161 */
                const int e = std::min(std::max(std::min(20, obj_width_raw - 100), 10), std::max(std::min(20, obj_height_expan - 100), 10));
                jb.roi_l = std::max(0, left_x_raw - e);
                jb.roi_r = std::min(img_width - 1, right_x_raw + e);
                jb.roi_t = std::max(0, top_y_raw - e);
                jb.roi_b = std::min(img_height - 1, jb.down_y_expan + e);
                jb.roi_w = jb.roi_r - jb.roi_l;
                jb.roi_h = jb.roi_b - jb.roi_t;
                if (jb.roi_w <= 0 || jb.roi_h <= 0 || jb.roi_l + jb.roi_w > img_width || jb.roi_t + jb.roi_h > img_height || jb.roi_l >= img_width ||
                    jb.roi_t >= img_height)
                    return fail(c, CS_ERR_INVALID_ARG, "frame %d box %d: empty or out-of-image ROI", f, b - c->h_box_off[f]);
                if (cs_dt_class_of(jb.roi_w) < 0) return fail(c, CS_ERR_CAPACITY, "ROI wider than %d px", 32 * 64);
                if (jb.roi_h > 255 * 32) return fail(c, CS_ERR_CAPACITY, "ROI taller than %d px", 255 * 32); /* tile-row table packs the row in 8 bits */
                jb.n_cand = fr.n_pose * fr.n_yaw * jb.n_top * 2;
                jb.bw = (jb.roi_w + 31) / 32;
                jb.dpitch = (jb.roi_w + 3) & ~3;
                jb.gray_pitch = img_width;
                jb.gray_off = c->gray_off[f] + (int64_t)jb.roi_t * img_width + jb.roi_l;
                jb.px_off = c->total_px;
                c->total_px += ((int64_t)jb.dpitch * jb.roi_h + 15) / 16 * 16;
                jb.bit_off = c->total_bits;
                const int plane_words = (jb.roi_h + 2) * (jb.bw + 2);
                c->total_bits += 2 * (int64_t)plane_words;
                c->max_plane_words = std::max(c->max_plane_words, plane_words);
                c->max_dpitch = std::max(c->max_dpitch, jb.dpitch);
                jb.cand_off = c->total_cand;
                c->total_cand += jb.n_cand;
                jb.tile_off = c->n_tiles;
                jb.tiles_x = (jb.roi_w + 31) / 32;
                c->n_tiles += jb.tiles_x * ((jb.roi_h + 31) / 32);
                const int job_id = (int)c->jobs.size();
                for (int ps = 0; ps < fr.n_pose; ps++) {
                    const int ypb = cs_sweep_warp_yaws();
                    for (int y0 = 0; y0 < fr.n_yaw; y0 += ypb) c->sweep_blocks4.push_back(make_int4(job_id, ps, y0, std::min(ypb, fr.n_yaw - y0)));
                }
                c->max_n_cand = std::max(c->max_n_cand, jb.n_cand);
                c->jobs.push_back(jb);
            }
            ob.n_jobs = (int32_t)c->jobs.size() - ob.job_off;
            c->objs.push_back(ob);
        }
    }
    /* distance-transform order: jobs grouped by width class so neighbouring CTAs share an instantiation */
    c->tile_job.clear();
    c->tile_job.reserve(c->n_tiles);
    for (size_t j = 0; j < c->jobs.size(); j++) {
        const int rows = (c->jobs[j].roi_h + 31) / 32; /* one NMS block per row of tiles: (job << 8) | tile_y */
        for (int ty = 0; ty < rows; ty++) c->tile_job.push_back((int32_t)((j << 8) | ty));
    }
    /* distance transform work list: by width class, the tallest ROI of a class first (its dependency chain is the longest) */
    c->dt_ids.clear();
    for (int cls = 0; cls < CS_DT_CLASSES; cls++) {
        c->dt_class_off[cls] = (int)c->dt_ids.size();
        c->dt_class_plane_words[cls] = 0;
        for (size_t j = 0; j < c->jobs.size(); j++)
            if (cs_dt_class_of(c->jobs[j].roi_w) == cls) {
                c->dt_ids.push_back((int32_t)j);
                c->dt_class_plane_words[cls] = std::max(c->dt_class_plane_words[cls], (c->jobs[j].roi_h + 2) * (c->jobs[j].bw + 2));
            }
        std::stable_sort(c->dt_ids.begin() + c->dt_class_off[cls], c->dt_ids.end(),
                         [&](int32_t a, int32_t b) { return c->jobs[a].roi_h > c->jobs[b].roi_h; });
    }
    c->dt_class_off[CS_DT_CLASSES] = (int)c->dt_ids.size();
    return CS_OK;
}

int alloc_work(cs_cuboid_params &, cs_ctx *c)
{
    int rc;
    const size_t px = (size_t)std::max<int64_t>(c->total_px, 16), cand = (size_t)std::max<int64_t>(c->total_cand, 16);
    const size_t nj = std::max<size_t>(c->jobs.size(), 1), no = std::max<size_t>(c->objs.size(), 1);
    if ((rc = ensure(c, c->d_bits, (size_t)std::max<int64_t>(c->total_bits, 16) * 4))) return rc;
    if ((rc = ensure(c, c->d_dist, px * 4))) return rc;
    if ((rc = ensure(c, c->d_mlines, nj * CS_MAXL_OUT * 7 * sizeof(double)))) return rc;
    if ((rc = ensure(c, c->d_lcounts, nj * 2 * 4))) return rc;
    if ((rc = ensure(c, c->d_err, 32))) return rc; /* words 0-3: the cuboid stage's flags; 4-7: the line detector's error word */
    if ((rc = ensure(c, c->d_cvalid, cand))) return rc;
    if ((rc = ensure(c, c->d_cdist, cand * 8))) return rc;
    if ((rc = ensure(c, c->d_cangle, cand * 8))) return rc;
    if ((rc = ensure(c, c->d_cskew, cand * 8))) return rc;
    if ((rc = ensure(c, c->d_vlist, cand * 4))) return rc;
    if ((rc = ensure(c, c->d_key, cand * 2 * 8))) return rc;
    if ((rc = ensure(c, c->d_idx, cand * 2 * 4))) return rc;
    if ((rc = ensure(c, c->d_flag, cand))) return rc;
    if ((rc = ensure(c, c->d_keep, cand * 4))) return rc;
    if ((rc = ensure(c, c->d_norm, cand * 8))) return rc;
    if ((rc = ensure(c, c->d_score, cand * 8))) return rc;
    if ((rc = ensure(c, c->d_jcounts, nj * 2 * 4))) return rc;
    if ((rc = ensure(c, c->d_out, no * c->topk * sizeof(cs_cuboid_rec)))) return rc;
    if ((rc = ensure(c, c->d_outcnt, no * 4))) return rc;
    return CS_OK;
}

/* Host tables (sample grids, pose hypotheses, ROI job descriptors) depend only on the batch's poses, boxes and
 * parameters: they are built and uploaded once per batch, at upload time, with the images. */
int prepare_tables(cs_ctx *c)
{
    int rc;
    if ((rc = build_tables(c))) return rc;
    if ((rc = alloc_work(c->prm, c))) return rc;
    if ((rc = upload(c, c->d_frames, c->frames))) return rc;
    if ((rc = upload(c, c->d_poses, c->poses))) return rc;
    if ((rc = upload(c, c->d_yaws, c->yaws))) return rc;
    if ((rc = upload(c, c->d_jobs, c->jobs))) return rc;
    if ((rc = upload(c, c->d_objs, c->objs))) return rc;
    if ((rc = upload(c, c->d_blocks4, c->sweep_blocks4))) return rc;
    if ((rc = upload(c, c->d_dtids, c->dt_ids))) return rc;
    if ((rc = upload(c, c->d_tilejob, c->tile_job))) return rc;
    if (c->mixed && ((rc = upload(c, c->d_graytab, c->gray_tab)) || (rc = upload(c, c->d_order, c->order)))) return rc;
    return CS_OK;
}

int run_batch(cs_ctx *c, bool sync)
{
    if (!c->prepared) return fail(c, CS_ERR_NOT_PREPARED, "no batch uploaded");
    int rc;
    cudaStream_t st = c->stream;
    c->launches = 0;
    if (c->profiling) cudaEventRecord(c->ev_total[0], st);
    CS_CUDA(c, cudaMemsetAsync(c->d_err.p, 0, 32, st));

    const int n_jobs = (int)c->jobs.size(), n_objs = (int)c->objs.size();
    uint8_t *d_img = (uint8_t *)c->d_img.p;
    auto mark = [&](int s) {
        if (c->profiling) cudaEventRecord(c->ev[s], st);
    };
    const float *d_lines_f32 = nullptr;
    const int32_t *d_nlines = nullptr;
    mark(ST_LSD);
    const int64_t line_launches_before = c->line_launches; /* the line detectors count their own kernels (cs_ctx_count_launches) */
    if (c->online_lines && c->mixed) {
        const CsMixedLines m = {d_img, c->views.data(), c->order.data(), (const int32_t *)c->d_order.p, c->n_frames, c->online_cap, &c->line_prm,
                                (float *)c->d_online_lines.p, (int32_t *)c->d_online_nl.p, (int32_t *)c->d_err.p + 4};
        if ((rc = c->mixed->lines(c, m, &d_lines_f32, &d_nlines))) return rc;
    } else if (c->online_lines) { /* line_lbd_detect::detect_filter_lines on the resident frames (object_slam main_obj.cpp:428) */
        if (c->line_prm.use_LSD) {
            if ((rc = cs_lsd_run_device(c, (const uint8_t *)c->d_img.p, c->n_frames, c->w, c->h, c->stride, c->channels, c->line_prm.line_length_thres,
                                        c->online_cap, &d_lines_f32, &d_nlines)))
                return rc;
        } else if ((rc = cs_edl_run(c, (const uint8_t *)c->d_img.p, true, c->n_frames, c->w, c->h, c->stride, c->channels,
                                    c->line_prm.line_length_thres, c->online_cap, &d_lines_f32, &d_nlines)))
            return rc;
        /* the detector's error word beside the cuboid stage's flags, so that fetch reads both with its one copy (no host sync here) */
        const int32_t *line_err = cs_line_err_word(*(c->line_prm.use_LSD ? cs_ctx_lsd_slot(c) : cs_ctx_edl_slot(c)));
        CS_CUDA(c, cudaMemcpyAsync((int32_t *)c->d_err.p + 4, line_err, 16, cudaMemcpyDeviceToDevice, st));
    }
    c->launches += c->line_launches - line_launches_before;
    c->d_online_counts = d_nlines;
    /* fork: the per-ROI line selection / merging only needs the lines and the job table */
    cudaEventRecord(c->ev_fork, st);
    cudaStreamWaitEvent(c->stream2, c->ev_fork, 0);
    cs_launch_roi_lines((const CsJob *)c->d_jobs.p, n_jobs, (const CsFrame *)c->d_frames.p, (const double *)c->d_lines.p, d_lines_f32, d_nlines,
                        c->online_cap, (double *)c->d_mlines.p, (int32_t *)c->d_lcounts.p, (int32_t *)c->d_err.p, c->prm.pre_merge_dist_thre,
                        c->prm.pre_merge_angle_thre, c->prm.edge_length_threshold, c->stream2, &c->launches);
    cudaEventRecord(c->ev_join, c->stream2);
    mark(ST_GRAY);
    if (c->mixed)
        c->mixed->gray(d_img, (const OctPlane *)c->d_graytab.p, (int)c->gray_tab.size(), c->gray_tab_px, d_img, st, &c->launches);
    else if (!c->gray_tab.empty()) /* one size: every frame or none has a plane of its own, back to back from gray_base */
        cs_launch_gray(d_img, d_img + c->gray_base, c->n_frames, c->w, c->h, c->stride, c->channels, st, &c->launches);
    mark(ST_CANNY);
    int low = (int)std::floor(std::min(c->prm.canny_low, c->prm.canny_high)), high = (int)std::floor(std::max(c->prm.canny_low, c->prm.canny_high));
    cs_launch_canny(d_img, 0, 0, (const CsJob *)c->d_jobs.p, n_jobs, (const int32_t *)c->d_tilejob.p, (int)c->tile_job.size(), (uint32_t *)c->d_bits.p,
                    (size_t)c->total_bits * 4, low, high, st, &c->launches);
    mark(ST_HYST);
    cs_launch_hyst((const CsJob *)c->d_jobs.p, n_jobs, (uint32_t *)c->d_bits.p, c->max_plane_words, st, &c->launches);
    mark(ST_DT);
    const bool tail_hi = c->use_prio && !c->profiling;
    if (tail_hi) { /* hand the rest of the chain to the high-priority stream */
        cudaEventRecord(c->ev_mid, st);
        st = c->stream_hi;
        cudaStreamWaitEvent(st, c->ev_mid, 0);
    }
    cs_launch_dt((const CsJob *)c->d_jobs.p, (const int32_t *)c->d_dtids.p, n_jobs, c->max_dpitch, c->dt_class_off, c->dt_class_plane_words, (const uint32_t *)c->d_bits.p,
                 (float *)c->d_dist.p, c->use_raster_dt, st, c->stream2, c->ev_dt_fork, c->ev_dt_join, &c->launches);
    mark(ST_LINES);
    cudaStreamWaitEvent(st, c->ev_join, 0); /* join */
    mark(ST_SWEEP);
    cs_launch_sweep_warp((const CsJob *)c->d_jobs.p, (const CsFrame *)c->d_frames.p, (const CsPose *)c->d_poses.p, (const double *)c->d_yaws.p,
                         (const int4 *)c->d_blocks4.p, (int)c->sweep_blocks4.size(), (const double *)c->d_mlines.p, (const int32_t *)c->d_lcounts.p,
                         (const float *)c->d_dist.p, (uint8_t *)c->d_cvalid.p, (double *)c->d_cdist.p, (double *)c->d_cangle.p, (double *)c->d_cskew.p, &c->prm,
                         st, &c->launches);
    mark(ST_FUSE);
    /* the previous batch's all-gather (its own stream) may still be reading the record buffer: only this point has to wait for it */
    if (c->gather_pending) cudaStreamWaitEvent(st, c->ev_gather_done, 0);
    /* record slots past a box's count must read valid = 0 on the device too (the all-gather ships the whole buffer) */
    if (n_objs > 0) CS_CUDA(c, cudaMemsetAsync(c->d_out.p, 0, (size_t)n_objs * c->topk * sizeof(cs_cuboid_rec), st));
    if (!c->use_cta_select && c->max_n_cand <= cs_fuse_warp_cap())
        cs_launch_fuse_warp((const CsObj *)c->d_objs.p, n_objs, (const CsJob *)c->d_jobs.p, (const CsFrame *)c->d_frames.p, (const CsPose *)c->d_poses.p,
                            (const double *)c->d_yaws.p, (const uint8_t *)c->d_cvalid.p, (const double *)c->d_cdist.p, (const double *)c->d_cangle.p,
                            (const double *)c->d_cskew.p, (int32_t *)c->d_vlist.p, (int32_t *)c->d_keep.p, (double *)c->d_norm.p, (double *)c->d_score.p, (int32_t *)c->d_jcounts.p,
                            (cs_cuboid_rec *)c->d_out.p, (int32_t *)c->d_outcnt.p, c->topk, &c->prm, st, &c->launches);
    else
        cs_launch_fuse((const CsObj *)c->d_objs.p, n_objs, (const CsJob *)c->d_jobs.p, (const CsFrame *)c->d_frames.p, (const CsPose *)c->d_poses.p,
                       (const double *)c->d_yaws.p, (const uint8_t *)c->d_cvalid.p, (const double *)c->d_cdist.p, (const double *)c->d_cangle.p,
                       (int32_t *)c->d_vlist.p, (uint64_t *)c->d_key.p, (uint32_t *)c->d_idx.p, (uint8_t *)c->d_flag.p, (int32_t *)c->d_keep.p,
                       (double *)c->d_norm.p, (double *)c->d_score.p, (int32_t *)c->d_jcounts.p, (cs_cuboid_rec *)c->d_out.p, (int32_t *)c->d_outcnt.p,
                       c->topk, &c->prm, st, &c->launches);
    mark(ST_COUNT);
    if (tail_hi) { /* everything queued on the context stream after this run is ordered behind the tail */
        cudaEventRecord(c->ev_done, st);
        st = c->stream;
        cudaStreamWaitEvent(st, c->ev_done, 0);
    }
    if (c->profiling) cudaEventRecord(c->ev_total[1], st);
    CS_CUDA(c, cudaGetLastError());
    c->stage_valid = false;
    if (sync) {
        CS_CUDA(c, cudaStreamSynchronize(st));
        if (c->profiling) {
            for (int s = 0; s < ST_COUNT; s++) cudaEventElapsedTime(&c->stage_ms[s], c->ev[s], c->ev[s + 1]);
            cudaEventElapsedTime(&c->total_ms, c->ev_total[0], c->ev_total[1]);
            c->stage_valid = true;
        }
    }
    return CS_OK;
}

/* The batch: frame f at imgs + views[f].offset (rows of views[f].stride bytes), copied to d_img as it lies; calibration K + 9 f (K null: the
 * context's, cs_set_calibration).  imgs null: the caller fills d_img itself -- device frames (cs_ingest.cu), packed host frames of mixed sizes
 * (cs_mixed.cu) -- and then marks the batch prepared.  mixed: the stages of a batch of mixed sizes, its frames in d_img in the order `order`
 * (null: one size; `one` then holds its width, height, stride and channels, else zeros).  Gray planes: a packed gray frame is its own; every
 * other frame's plane follows the frames in d_img, 256-byte aligned.  A refusal before anything is stored leaves the previous batch as it was;
 * the batch is prepared only once its tables are built. */
int store_frames(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const CsMixedStages *mixed,
                 const int32_t *order, const int one[4], const double *T_wc, const double *boxes, const int32_t *box_offsets, const double *lines,
                 const int32_t *line_offsets, const cs_cuboid_params *params, const cs_line_params *online)
{
    std::vector<int32_t> zero_off;
    if (online) { /* no input lines: CSR of zeros */
        zero_off.assign((size_t)std::max(n_frames, 0) + 1, 0);
        line_offsets = zero_off.data();
        lines = nullptr;
    }
    if (!views || n_frames <= 0 || !T_wc || !box_offsets || !line_offsets || !params) return fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (!K && !c->have_K) return fail(c, CS_ERR_INVALID_ARG, "cs_set_calibration has not been called");
    if (params->max_cuboid_num < 1 || params->max_cuboid_num > CS_MAX_TOPK)
        return fail(c, CS_ERR_CAPACITY, "max_cuboid_num must be in [1,%d]", CS_MAX_TOPK);
    if (n_frames > c->max_frames) return fail(c, CS_ERR_CAPACITY, "batch exceeds cs_create capacities");
    for (int f = 0; f < n_frames; f++)
        if (views[f].width > c->max_w || views[f].height > c->max_h)
            return fail(c, CS_ERR_CAPACITY, "frame %d: %d x %d exceeds cs_create's %d x %d", f, views[f].width, views[f].height, c->max_w, c->max_h);
    if (box_offsets[0] != 0 || line_offsets[0] != 0) /* records, counts and jobs are indexed from 0: a CSR slice must be rebased by the caller */
        return fail(c, CS_ERR_INVALID_ARG, "box_offsets[0] and line_offsets[0] must be 0");
    for (int f = 0; f < n_frames; f++) {
        if (box_offsets[f + 1] < box_offsets[f] || line_offsets[f + 1] < line_offsets[f]) return fail(c, CS_ERR_INVALID_ARG, "offsets must be non-decreasing");
        if (box_offsets[f + 1] - box_offsets[f] > c->max_boxes) return fail(c, CS_ERR_CAPACITY, "frame %d: more than %d boxes", f, c->max_boxes);
        if (line_offsets[f + 1] - line_offsets[f] > c->max_lines) return fail(c, CS_ERR_CAPACITY, "frame %d: more than %d lines", f, c->max_lines);
    }
    const int nb = box_offsets[n_frames], nl = line_offsets[n_frames];
    if ((nb > 0 && !boxes) || (nl > 0 && !lines)) return fail(c, CS_ERR_INVALID_ARG, "null boxes/lines");
    c->prepared = false;
    c->w = one[0];
    c->h = one[1];
    c->stride = one[2];
    c->channels = one[3];
    c->online_lines = online != nullptr;
    if (online) {
        if (online->numoctaves < 1) return fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1"); /* > 1: same lines, see cs_detect_lines_batch */
        c->line_prm = *online;
        c->online_cap = std::max(64, std::min(c->max_lines > 0 ? c->max_lines : 1024, 4096));
    }
    c->n_frames = n_frames;
    c->prm = *params;
    c->topk = params->max_cuboid_num;
    c->h_T.assign(T_wc, T_wc + (size_t)n_frames * 16);
    c->h_boxes.assign(boxes, boxes + (size_t)nb * 5);
    if (nl) c->h_lines.assign(lines, lines + (size_t)nl * 4); else c->h_lines.clear();
    c->h_box_off.assign(box_offsets, box_offsets + n_frames + 1);
    c->h_line_off.assign(line_offsets, line_offsets + n_frames + 1);
    c->views.assign(views, views + n_frames);
    c->Ks.resize((size_t)n_frames * 9);
    for (int f = 0; f < n_frames; f++) std::memcpy(&c->Ks[(size_t)f * 9], K ? K + (size_t)f * 9 : c->K, 9 * sizeof(double));
    c->mixed = mixed;
    c->order.resize((size_t)n_frames);
    for (int f = 0; f < n_frames; f++) c->order[f] = order ? order[f] : f;
    int64_t img_bytes = 0;
    for (int f = 0; f < n_frames; f++) img_bytes = std::max(img_bytes, views[f].offset + (int64_t)views[f].height * views[f].stride);
    c->gray_base = (img_bytes + 255) & ~(int64_t)255;
    c->gray_off.resize((size_t)n_frames);
    c->gray_tab.clear();
    c->gray_tab_px = 0;
    for (int f = 0; f < n_frames; f++) {
        const cs_frame_view &v = views[f];
        if (v.channels == 1 && v.stride == v.width) { /* packed gray: the frame is its gray plane */
            c->gray_off[f] = v.offset;
            continue;
        }
        OctPlane P;
        std::memset(&P, 0, sizeof P);
        P.src = v.offset;
        P.dst = c->gray_off[f] = c->gray_base + c->gray_tab_px;
        P.px0 = c->gray_tab_px;
        P.sw = P.dw = v.width;
        P.sh = P.dh = v.height;
        P.sstride = v.stride;
        P.ch = v.channels;
        c->gray_tab.push_back(P);
        c->gray_tab_px += (int64_t)v.width * v.height;
    }
    int rc;
    if ((rc = ensure(c, c->d_img, (size_t)(c->gray_base + c->gray_tab_px) + 64))) return rc;
    if ((rc = ensure(c, c->d_lines, std::max<size_t>((size_t)nl * 4 * sizeof(double), 64)))) return rc;
    if (mixed && online && !online->use_LSD && ((rc = ensure(c, c->d_online_lines, (size_t)n_frames * c->online_cap * 16)) ||
                                                (rc = ensure(c, c->d_online_nl, (size_t)n_frames * 4))))
        return rc;
    if (imgs) CS_CUDA(c, cudaMemcpyAsync(c->d_img.p, imgs, (size_t)img_bytes, cudaMemcpyHostToDevice, c->stream));
    if (nl) CS_CUDA(c, cudaMemcpyAsync(c->d_lines.p, lines, (size_t)nl * 4 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    if ((rc = prepare_tables(c))) return rc;
    c->prepared = imgs != nullptr;
    return CS_OK;
}

/* a batch of frames of one size, frame f at imgs + f * height * stride (device_frames: the caller fills d_img, cs_ingest.cu) */
int store_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                const cs_cuboid_params *params, const cs_line_params *online = nullptr, bool device_frames = false)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if ((!imgs && !device_frames) || n_frames <= 0 || width <= 0 || height <= 0 || !T_wc || !box_offsets || (!line_offsets && !online) || !params)
        return fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3");
    if (stride < width * channels) return fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    if (!c->have_K) return fail(c, CS_ERR_INVALID_ARG, "cs_set_calibration has not been called");
    if (params->max_cuboid_num < 1 || params->max_cuboid_num > CS_MAX_TOPK)
        return fail(c, CS_ERR_CAPACITY, "max_cuboid_num must be in [1,%d]", CS_MAX_TOPK);
    if (width > c->max_w || height > c->max_h || n_frames > c->max_frames) return fail(c, CS_ERR_CAPACITY, "batch exceeds cs_create capacities");
    std::vector<cs_frame_view> views((size_t)n_frames);
    for (int f = 0; f < n_frames; f++) views[f] = cs_frame_view{(int64_t)f * height * stride, width, height, stride, channels};
    const int one[4] = {width, height, stride, channels};
    return store_frames(c, device_frames ? nullptr : imgs, views.data(), n_frames, nullptr, nullptr, nullptr, one, T_wc, boxes, box_offsets, lines,
                        line_offsets, params, online);
}

int fetch(cs_ctx *c, cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c->prepared) return fail(c, CS_ERR_NOT_PREPARED, "no batch uploaded");
    const size_t no = c->objs.size();
    if (no == 0) return CS_OK;
    if (out) CS_CUDA(c, cudaMemcpyAsync(out, c->d_out.p, no * c->topk * sizeof(cs_cuboid_rec), cudaMemcpyDeviceToHost, c->stream));
    if (out_counts) CS_CUDA(c, cudaMemcpyAsync(out_counts, c->d_outcnt.p, no * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    int32_t words[8] = {0, 0, 0, 0, 0, 0, 0, 0}; /* one copy: the cuboid stage's flags and the line detector's error word */
    CS_CUDA(c, cudaMemcpyAsync(words, c->d_err.p, sizeof words, cudaMemcpyDeviceToHost, c->stream));
    CS_CUDA(c, cudaStreamSynchronize(c->stream));
    const int32_t err = words[0], *line_err = words + 4;
    if (c->online_lines) { /* the line detector's own word first: its overflow also shows as a segment count past online_cap (err & 4) */
        /* a candidate overflow is not re-run here (that would need a host sync in the batch path): the batch fails; a synchronous
         * cs_detect_lines_batch on the same context grows the buffer for later batches */
        const int rc = c->line_prm.use_LSD ? cs_lsd_check_err(c, line_err) : cs_edl_check_err(c, line_err);
        if (rc) return rc;
    }
    if (err & 1) return fail(c, CS_ERR_CAPACITY, "more than %d line segments inside one ROI", CS_LINE_CAP);
    if (err & 2) return fail(c, CS_ERR_CAPACITY, "more than %d merged segments inside one ROI", CS_MAXL_OUT);
    if (err & 4) return fail(c, CS_ERR_CAPACITY, "the line detector found more than %d segments in a frame (raise max_lines_per_frame)", c->online_cap);
    if (err & 8) return fail(c, CS_ERR_CUDA, "a TMA tile copy of the Canny kernel did not complete");
    if (out && out_counts) { /* slots past the count are not cuboids */
        for (size_t o = 0; o < no; o++)
            for (int k = out_counts[o]; k < c->topk; k++) std::memset(&out[o * c->topk + k], 0, sizeof(cs_cuboid_rec));
    }
    return CS_OK;
}

/* Which camera pose hypothesis the reference's cam_pose holds when it is done with one height sample of a box in roll / pitch-sampling
 * mode: the sampling loop leaves the last hypothesis (box_proposal_detail.cpp:230-239), then the loop over the kept proposals
 * (:479-487) sets the pose of each one in turn and so leaves the LAST kept proposal's -- last in good_proposal_ids, which
 * fuse_normalize_scores_v2 (object_3d_util.cpp:495-527) fills either with the ascending intersection of the two "best 2/3" sets or, when
 * the angle errors saturate at the cut, with the distance-sorted prefix.  valid / dist / angle: the candidate records of the job in
 * enumeration order (pose-major), as the sweep kernels leave them; ties rank by index, NaN last (the rule the selection kernels use). */
int last_set_pose(const uint8_t *valid, const double *dist, const double *angle, int n_cand, int n_pose)
{
    if (n_pose <= 0) return 0;
    std::vector<int> vidx;
    for (int i = 0; i < n_cand; i++)
        if (valid[i]) vidx.push_back(i);
    const int n = (int)vidx.size();
    if (n == 0 || n_cand % n_pose != 0) return n_pose - 1;
    const int per_pose = n_cand / n_pose;
    auto prefix = [&](const double *v, std::vector<int> &idx, int top_k) {
        std::partial_sort(idx.begin(), idx.begin() + top_k, idx.end(), [&](int a, int b) {
            const double va = v[vidx[a]], vb = v[vidx[b]];
            const bool na = std::isnan(va), nb = std::isnan(vb);
            if (na || nb) return (!na && nb) || (na == nb && a < b);
            return va < vb || (va == vb && a < b);
        });
    };
    int last; /* position in the valid list of the last kept proposal */
    if (n > 4) {
        const int breaking_num = (int)std::round(float(n) / 3.0 * 2.0);
        std::vector<int> ds(n), as;
        for (int i = 0; i < n; i++) ds[i] = i;
        as = ds;
        prefix(dist, ds, breaking_num);
        prefix(angle, as, breaking_num);
        if (angle[vidx[as[breaking_num - 1]]] > angle[vidx[as[breaking_num - 2]]]) {
            std::vector<char> in_d(n, 0);
            for (int i = 0; i < breaking_num - 1; i++) in_d[ds[i]] = 1;
            last = -1;
            for (int i = 0; i < breaking_num - 1; i++)
                if (in_d[as[i]]) last = std::max(last, as[i]);
            if (last < 0) return n_pose - 1; /* empty intersection: no kept proposal, the sampling loop's last pose stands */
        } else
            last = ds[breaking_num - 2];
    } else
        last = n - 1;
    return vidx[last] / per_pose;
}

/* cs_detect_cuboids_batch when cs_set_profiling bit 10 is set, roll / pitch sampling is on and some frame carries more than one box.
 * The reference works through the boxes of a frame in order and derives box k + 1's yaw samples from the cam_pose box k left behind
 * (box_proposal_detail.cpp:126-128 after :237,485): the re-derived camera yaw is the raw one give or take an ulp, and because
 * linespace(yaw - 45 deg, yaw + 45 deg, 6 deg) spans exactly 15 steps, that ulp decides between 15 and 16 yaw samples
 * (tests/test_sampling_deviation.py).  So: one pass per box rank.  Pass r runs the rank-r box of every frame that has one through the
 * ordinary kernels, with the frame's yaw samples derived from the pose pass r - 1 left; then the candidate records of each box's last
 * height sample come back and the host works out which hypothesis the reference's cam_pose would hold (last_set_pose).  Boxes of one
 * frame are sequential by definition here; frames (and the boxes of one rank) still run side by side. */
int detect_batch_carried(cs_ctx *c, const CsStoreBoxes &store, int n_frames, const double *boxes, const int32_t *box_offsets, const cs_cuboid_params *params,
                         cs_cuboid_rec *out, int32_t *out_counts)
{
    std::vector<uint8_t> h_valid;
    std::vector<double> h_dist, h_angle;
    /* one pass (cs_carried.h): the ordinary kernels over the rank-r boxes, then -- unless it is the last pass -- the candidate records of
     * each box's last height sample come back and the host works out which hypothesis the reference's cam_pose would hold */
    auto run_pass = [&](const double *sub_boxes, const int32_t *sub_off, const std::vector<double> &cam_yaw, cs_cuboid_rec *recs, int32_t *counts,
                        std::vector<double> *yaw_left) -> int {
        c->yaw_override = cam_yaw;
        int rc = store(sub_boxes, sub_off); /* the caller's batch with this pass's boxes */
        c->yaw_override.clear(); /* the override belongs to this pass only */
        if (rc) return rc;
        if ((rc = run_batch(c, false))) return rc;
        if ((rc = fetch(c, recs, counts))) return rc;
        if (!yaw_left) return CS_OK;
        const size_t nc = (size_t)c->total_cand;
        h_valid.resize(std::max<size_t>(nc, 1));
        h_dist.resize(std::max<size_t>(nc, 1));
        h_angle.resize(std::max<size_t>(nc, 1));
        if (nc && (cudaMemcpyAsync(h_valid.data(), c->d_cvalid.p, nc, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
                   cudaMemcpyAsync(h_dist.data(), c->d_cdist.p, nc * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
                   cudaMemcpyAsync(h_angle.data(), c->d_cangle.p, nc * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
                   cudaStreamSynchronize(c->stream) != cudaSuccess))
            return fail(c, CS_ERR_CUDA, "candidate record copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        for (size_t o = 0; o < c->objs.size(); o++) { /* every height sample starts with the sampling loop: the last one decides */
            const CsObj &ob = c->objs[o];
            const CsFrame &fr = c->frames[ob.frame];
            int hyp = fr.n_pose - 1;
            if (ob.n_jobs > 0) {
                const CsJob &jb = c->jobs[(size_t)ob.job_off + ob.n_jobs - 1];
                hyp = last_set_pose(h_valid.data() + jb.cand_off, h_dist.data() + jb.cand_off, h_angle.data() + jb.cand_off, jb.n_cand, fr.n_pose);
            }
            (*yaw_left)[ob.frame] = c->poses[(size_t)fr.pose_off + hyp].camera_yaw;
        }
        return CS_OK;
    };
    const int rc = cs_carried_passes(n_frames, boxes, box_offsets, params->max_cuboid_num, out, out_counts, run_pass);
    c->yaw_override.clear();
    return rc;
}

}  // namespace

/* cs_batch_upload[_online]_device (cs_ingest.cu): everything of the host forms but the frames, which the caller copies into *d_img (packed
 * rows, pitch width * channels) on the context stream and then marks the batch prepared */
int cs_ctx_store_device_batch(cs_ctx *c, int n_frames, int width, int height, int channels, const double *T_wc, const double *boxes,
                              const int32_t *box_offsets, const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params,
                              const cs_line_params *online, uint8_t **d_img)
{
    const int rc = store_batch(c, nullptr, n_frames, width, height, width * channels, channels, T_wc, boxes, box_offsets, lines, line_offsets, params,
                               online, true);
    if (rc) return rc;
    *d_img = (uint8_t *)c->d_img.p;
    return CS_OK;
}
void cs_ctx_mark_prepared(cs_ctx *c) { c->prepared = true; }

/* cs_mixed.cu's ways in: a batch of frames of mixed sizes, already checked, packed in d_img at `packed` in the order `order` */
int cs_ctx_store_mixed_batch(cs_ctx *c, const cs_frame_view *packed, const int32_t *order, int n_frames, const double *K, const double *T_wc,
                             const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                             const cs_cuboid_params *params, const cs_line_params *online, const CsMixedStages *stages, uint8_t **d_img)
{
    const int none[4] = {0, 0, 0, 0};
    const int rc = store_frames(c, nullptr, packed, n_frames, K, stages, order, none, T_wc, boxes, box_offsets, lines, line_offsets, params, online);
    if (rc) return rc;
    *d_img = (uint8_t *)c->d_img.p;
    return CS_OK;
}
/* whether cs_detect_cuboids_batch[_mixed] takes the carried-pose passes (cs_set_profiling bit 10 with sampled roll / pitch and a frame of
 * several boxes), and those passes with `store` storing the caller's batch with a pass's boxes */
bool cs_ctx_carries_pose(cs_ctx *c, const cs_cuboid_params *params, const int32_t *box_offsets, int n_frames, const cs_cuboid_rec *out,
                         const int32_t *out_counts)
{
    if (!(c->carry_cam_pose && params && params->whether_sample_cam_roll_pitch && box_offsets && out && out_counts && n_frames > 0)) return false;
    for (int f = 0; f < n_frames; f++)
        if (box_offsets[f + 1] - box_offsets[f] > 1) return true;
    return false;
}
int cs_ctx_detect_carried(cs_ctx *c, const CsStoreBoxes &store, int n_frames, const double *boxes, const int32_t *box_offsets,
                          const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts)
{
    return detect_batch_carried(c, store, n_frames, boxes, box_offsets, params, out, out_counts);
}

/* ============================================================================================ C ABI */
extern "C" {

int cs_abi_version(void) { return CS_ABI_VERSION; }

void cs_default_cuboid_params(cs_cuboid_params *p)
{
    if (!p) return;
    std::memset(p, 0, sizeof(*p));
    p->consider_config_1 = 1;
    p->consider_config_2 = 1;
    p->whether_sample_cam_roll_pitch = 0;
    p->whether_sample_bbox_height = 0;
    p->max_cuboid_num = 1;
    p->reweight_edge_distance = 1;
    p->whether_normalize_two_errors = 1;
    p->top_sample_count_override = 0;
    p->nominal_skew_ratio = 1;
    p->max_cut_skew = 3;
    p->vp12_edge_angle_thre = 15;
    p->vp3_edge_angle_thre = 10;
    p->shorted_edge_thre = 20;
    p->weight_vp_angle = 0.8;
    p->weight_skew_error = 1.5;
    p->pre_merge_dist_thre = 20;
    p->pre_merge_angle_thre = 5;
    p->edge_length_threshold = 30;
    p->canny_low = 80;
    p->canny_high = 200;
    p->yaw_half_range_deg = 45;
    p->yaw_step_deg = 6;
}

void cs_default_line_params(cs_line_params *p)
{
    if (!p) return;
    p->use_LSD = 0;          /* line_lbd_allclass.cpp:121 */
    p->numoctaves = 1;       /* line_lbd_allclass.h:25 */
    p->octaveratio = 1.f;
    p->line_length_thres = 50; /* line_lbd_allclass.cpp:122 */
}

cs_ctx *cs_create(int device, int max_width, int max_height, int max_frames, int max_boxes_per_frame, int max_lines_per_frame)
{
    if (max_width <= 0 || max_height <= 0 || max_frames <= 0 || max_boxes_per_frame < 0 || max_lines_per_frame < 0) return nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
        fprintf(stderr, "cube_slam_b200: no usable CUDA device %d (found %d); this library has no CPU path\n", device, n_dev);
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    cs_ctx *c = new cs_ctx();
    c->device = device;
    c->max_w = max_width;
    c->max_h = max_height;
    c->max_frames = max_frames;
    c->max_boxes = max_boxes_per_frame;
    c->max_lines = max_lines_per_frame;
    std::memset(&c->stats, 0, sizeof(c->stats));
    cs_default_cuboid_params(&c->prm);
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete c;
        return nullptr;
    }
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi); /* numerically lower = higher priority */
    cudaStreamCreateWithPriority(&c->stream2, cudaStreamNonBlocking, prio_hi);
    cudaStreamCreateWithPriority(&c->stream_hi, cudaStreamNonBlocking, prio_hi);
    cudaEventCreateWithFlags(&c->ev_mid, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_dt_fork, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_dt_join, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_ingest_in, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&c->ev_ingest_out, cudaEventDisableTiming);
    for (int s = 0; s <= ST_COUNT; s++) cudaEventCreate(&c->ev[s]);
    cudaEventCreate(&c->ev_total[0]);
    cudaEventCreate(&c->ev_total[1]);
    return c;
}

void cs_destroy(cs_ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    cs_nccl_teardown(c);
    if (c->lsd_state) cs_lsd_destroy(c->lsd_state);
    if (c->edl_state) cs_edl_destroy(c->edl_state);
    if (c->lbd_state) cs_lbd_destroy(c->lbd_state);
    DevBuf *all[] = {&c->d_img,   &c->d_graytab, &c->d_order, &c->d_online_lines, &c->d_online_nl, &c->d_lines,  &c->d_frames, &c->d_poses,   &c->d_yaws, &c->d_jobs, &c->d_objs,
                     &c->d_blocks4, &c->d_dtids, &c->d_tilejob, &c->d_bits, &c->d_dist, &c->d_mlines, &c->d_lcounts, &c->d_err,
                     &c->d_cvalid, &c->d_cdist, &c->d_cangle, &c->d_cskew, &c->d_vlist,  &c->d_key,     &c->d_idx,  &c->d_flag, &c->d_keep,  &c->d_norm,
                     &c->d_score,  &c->d_jcounts, &c->d_out,  &c->d_outcnt, &c->d_gather, &c->d_send};
    for (DevBuf *b : all)
        if (b->p) cudaFree(b->p);
    if (c->pinned) cudaFreeHost(c->pinned);
    for (int s = 0; s <= ST_COUNT; s++)
        if (c->ev[s]) cudaEventDestroy(c->ev[s]);
    cudaEventDestroy(c->ev_total[0]);
    cudaEventDestroy(c->ev_total[1]);
    cudaEventDestroy(c->ev_fork);
    cudaEventDestroy(c->ev_join);
    cudaEventDestroy(c->ev_ingest_in);
    cudaEventDestroy(c->ev_ingest_out);
    cudaStreamDestroy(c->stream2);
    cudaStreamDestroy(c->stream_hi);
    if (c->gather_stream) cudaStreamDestroy(c->gather_stream);
    if (c->ev_gather_ready) cudaEventDestroy(c->ev_gather_ready);
    if (c->ev_gather_done) cudaEventDestroy(c->ev_gather_done);
    cudaEventDestroy(c->ev_mid);
    cudaEventDestroy(c->ev_dt_fork);
    cudaEventDestroy(c->ev_dt_join);
    cudaEventDestroy(c->ev_done);
    cudaStreamDestroy(c->stream);
    delete c;
}

const char *cs_last_error(const cs_ctx *c)
{
    if (c) return c->err.c_str();
    return t_frames_err.empty() ? "null context (cs_create failed: no CUDA device?)" : t_frames_err.c_str();
}

int cs_set_calibration(cs_ctx *c, const double K[9])
{
    if (!c || !K) return CS_ERR_INVALID_ARG;
    std::memcpy(c->K, K, sizeof(c->K));
    c->have_K = true;
    return CS_OK;
}

int cs_cam_pose(const double K[9], const double T_wc[16], double euler_zyx[3], double KinvR[9])
{
    if (!K || !T_wc) return CS_ERR_INVALID_ARG;
    CsPose ps;
    double e[3];
    cshost::make_pose(K, T_wc, &ps, e);
    if (euler_zyx) std::memcpy(euler_zyx, e, sizeof(e));
    if (KinvR) std::memcpy(KinvR, ps.KinvR, sizeof(ps.KinvR));
    return CS_OK;
}

int cs_cuboid_measurement(const cs_cuboid_rec *rec, const double cam_t[3], const double cam_q_xyzw[4], const double cam_euler_raw[3],
                          double meas_t[3], double meas_q_xyzw[4], double meas_scale[3], double *meas_quality)
{
    if (!rec || !cam_t || !cam_q_xyzw || !meas_t || !meas_q_xyzw) return CS_ERR_INVALID_ARG;
    double e[3];
    const double *en = nullptr;
    if (cam_euler_raw) { /* main_obj.cpp:465-471: the pose the winning proposal was generated with */
        e[0] = cam_euler_raw[0] + rec->camera_roll_delta;
        e[1] = cam_euler_raw[1] + rec->camera_pitch_delta;
        e[2] = cam_euler_raw[2];
        en = e;
    }
    cshost::cuboid_measurement(rec->pos, rec->rotY, cam_t, cam_q_xyzw, en, meas_t, meas_q_xyzw);
    if (meas_scale) std::memcpy(meas_scale, rec->scale, 3 * sizeof(double));
    if (meas_quality) *meas_quality = (1 - rec->normalized_error + 0.5) / 2; /* main_obj.cpp:505 */
    return CS_OK;
}

int cs_cuboid_measurement_orb(const cs_cuboid_rec *rec, const double T_cam_to_ground[16], double box_confidence, double meas_t[3],
                              double meas_q_xyzw[4], double meas_scale[3], double *meas_quality)
{
    if (!rec || !T_cam_to_ground || !meas_t || !meas_q_xyzw) return CS_ERR_INVALID_ARG;
    /* Converter::toSE3Quat(cv::Mat 4x4): SE3Quat(R, t) -> Quaterniond(R), normalised */
    const double R[9] = {T_cam_to_ground[0], T_cam_to_ground[1], T_cam_to_ground[2], T_cam_to_ground[4], T_cam_to_ground[5],
                         T_cam_to_ground[6], T_cam_to_ground[8], T_cam_to_ground[9], T_cam_to_ground[10]};
    const double t[3] = {T_cam_to_ground[3], T_cam_to_ground[7], T_cam_to_ground[11]};
    double q[4];
    cshost::quat_of_rotation(R, q);
    cshost::cuboid_measurement(rec->pos, rec->rotY, t, q, nullptr, meas_t, meas_q_xyzw);
    if (meas_scale) std::memcpy(meas_scale, rec->scale, 3 * sizeof(double));
    if (meas_quality) { /* Tracking.cc:1680-1687 */
        const double obj_cam_dist = std::min(std::max(meas_t[2], 10.0), 30.0);
        double quality = (60.0 - obj_cam_dist) / 40.0;
        if (box_confidence > 0) quality *= box_confidence;
        *meas_quality = quality;
    }
    return CS_OK;
}

int cs_batch_upload(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                    const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                    const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(c->device);
    int rc = store_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, boxes, box_offsets, lines, line_offsets, params);
    if (rc) return rc;
    CS_CUDA(c, cudaStreamSynchronize(c->stream));
    return CS_OK;
}

int cs_batch_upload_online(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                           const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!line_params) return fail(c, CS_ERR_INVALID_ARG, "null line params");
    cudaSetDevice(c->device);
    int rc = store_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, boxes, box_offsets, nullptr, nullptr, params, line_params);
    if (rc) return rc;
    CS_CUDA(c, cudaStreamSynchronize(c->stream));
    return CS_OK;
}

int cs_detect_frames_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                           const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params,
                           cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!line_params) return fail(c, CS_ERR_INVALID_ARG, "null line params");
    cudaSetDevice(c->device);
    int rc = store_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, boxes, box_offsets, nullptr, nullptr, params, line_params);
    if (rc) return rc;
    if ((rc = run_batch(c, false))) return rc;
    return fetch(c, out, out_counts);
}

int cs_batch_run(cs_ctx *c)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(c->device);
    return run_batch(c, true);
}

int cs_batch_run_async(cs_ctx *c)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(c->device);
    return run_batch(c, false);
}

int cs_batch_fetch(cs_ctx *c, cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(c->device);
    return fetch(c, out, out_counts);
}

int cs_detect_cuboids_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                            const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                            const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(c->device);
    if (cs_ctx_carries_pose(c, params, box_offsets, n_frames, out, out_counts))
        return detect_batch_carried(
            c,
            [&](const double *sub_boxes, const int32_t *sub_off) {
                return store_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, sub_boxes, sub_off, lines, line_offsets, params);
            },
            n_frames, boxes, box_offsets, params, out, out_counts);
    int rc = store_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, boxes, box_offsets, lines, line_offsets, params);
    if (rc) return rc;
    if ((rc = run_batch(c, false))) return rc;
    return fetch(c, out, out_counts);
}

/* tests: last_set_pose on caller-given candidate records (host-only, needs no context) */
int cs_debug_last_set_pose(const uint8_t *valid, const double *dist_err, const double *angle_err, int n_cand, int n_pose, int32_t *pose_out)
{
    if (!valid || !dist_err || !angle_err || n_cand < 0 || n_pose <= 0 || !pose_out) return CS_ERR_INVALID_ARG;
    *pose_out = last_set_pose(valid, dist_err, angle_err, n_cand, n_pose);
    return CS_OK;
}

int cs_detect_cuboids(cs_ctx *c, const uint8_t *img, int width, int height, int stride, int channels, const double T_wc[16], const double *boxes,
                      int n_boxes, const double *lines, int n_lines, const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts)
{
    if (n_boxes < 0 || n_lines < 0) return c ? fail(c, CS_ERR_INVALID_ARG, "negative count") : CS_ERR_INVALID_ARG;
    const int32_t bo[2] = {0, n_boxes}, lo[2] = {0, n_lines};
    static const double dummy[5] = {0, 0, 0, 0, 0};
    if (n_boxes == 0) { /* empty bbox matrix => empty output (box_proposal_detail.cpp:71-72) */
        return CS_OK;
    }
    return cs_detect_cuboids_batch(c, img, 1, width, height, stride, channels, T_wc, boxes, bo, n_lines ? lines : dummy, lo, params, out, out_counts);
}

int cs_batch_stats_get(cs_ctx *c, cs_batch_stats *s)
{
    if (!c || !s) return CS_ERR_INVALID_ARG;
    if (!c->prepared) return fail(c, CS_ERR_NOT_PREPARED, "no batch uploaded");
    cudaSetDevice(c->device);
    std::memset(s, 0, sizeof(*s));
    s->n_frames = c->n_frames;
    s->n_objects = (int64_t)c->objs.size();
    s->n_roi_jobs = (int64_t)c->jobs.size();
    s->n_candidates = c->total_cand;
    s->n_kernel_launches = c->launches;
    s->n_lines_in = c->h_line_off.empty() ? 0 : c->h_line_off.back();
    for (const CsJob &j : c->jobs) s->roi_pixels += (int64_t)j.roi_w * j.roi_h;
    if (!c->jobs.empty()) {
        std::vector<int32_t> jc(c->jobs.size() * 2);
        CS_CUDA(c, cudaMemcpyAsync(jc.data(), c->d_jcounts.p, jc.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CS_CUDA(c, cudaStreamSynchronize(c->stream));
        for (size_t j = 0; j < c->jobs.size(); j++) s->n_valid += jc[j * 2];
    }
    if (c->online_lines && c->d_online_counts && c->n_frames > 0) { /* segments the line detector handed to the cuboid stage */
        std::vector<int32_t> nl(c->n_frames);
        CS_CUDA(c, cudaMemcpyAsync(nl.data(), c->d_online_counts, nl.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CS_CUDA(c, cudaStreamSynchronize(c->stream));
        s->n_lines_in = 0;
        for (int32_t v : nl) s->n_lines_in += v;
    }
    c->stats = *s;
    return CS_OK;
}

int cs_batch_device_records(cs_ctx *c, void **dev_ptr, size_t *n_bytes)
{
    if (!c || !dev_ptr || !n_bytes) return CS_ERR_INVALID_ARG;
    if (!c->prepared) return fail(c, CS_ERR_NOT_PREPARED, "no batch uploaded");
    *dev_ptr = c->d_out.p;
    *n_bytes = c->objs.size() * c->topk * sizeof(cs_cuboid_rec);
    return CS_OK;
}

void *cs_stream(cs_ctx *c) { return c ? (void *)c->stream : nullptr; }

int cs_set_profiling(cs_ctx *c, int enable)
{
    if (!c) return CS_ERR_INVALID_ARG;
    c->profiling = (enable & 1) != 0;
    c->use_raster_dt = ((enable & 32) ? 1 : 0) | ((enable & 64) ? 2 : 0); /* bit 5: raster-scan distance transform kernel; bit 6: cone form, bits from global */
    c->use_prio = (enable & 16) == 0;      /* bit 4: keep the whole chain on one stream (no high-priority tail) */
    c->seq_lines = (enable & 128) != 0;    /* bit 7: EDLines' round-1 kernels (routing and fitting on the pixel maps, one thread per frame); LSD does not read it */
    c->use_tma = (enable & 256) == 0;      /* bit 8: the line detectors' tile kernels stage every tile with byte loads (A/B of the TMA path) */
    c->use_cta_select = (enable & 8) != 0; /* bit 3: CTA-wide selection kernel (k_fuse_rank) for every box instead of k_fuse_warp */
    c->carry_cam_pose = (enable & 1024) != 0; /* bit 10: cs_detect_cuboids[_batch] carries the reference's cam_pose from box to box of a sampled frame */
    return CS_OK;
}

int cs_stage_ms(cs_ctx *c, const char *stage, float *ms)
{
    if (!c || !stage || !ms) return CS_ERR_INVALID_ARG;
    if (!c->stage_valid) return fail(c, CS_ERR_NOT_PREPARED, "no profiled synchronous run");
    if (!strcmp(stage, "total")) {
        *ms = c->total_ms;
        return CS_OK;
    }
    for (int s = 0; s < ST_COUNT; s++)
        if (!strcmp(stage, kStageNames[s])) {
            *ms = c->stage_ms[s];
            return CS_OK;
        }
    return fail(c, CS_ERR_INVALID_ARG, "unknown stage %s", stage);
}

/* timeline of the last profiled run of `c`: milliseconds from the start of the last profiled run of `ref` to each stage mark of `c`
 * (9 values: the 8 stage starts in kStageNames order and the end).  Both runs must have completed. */
int cs_debug_stage_offsets(cs_ctx *c, cs_ctx *ref, float *offsets_ms)
{
    if (!c || !ref || !offsets_ms) return CS_ERR_INVALID_ARG;
    if (!c->profiling || !ref->profiling) return fail(c, CS_ERR_NOT_PREPARED, "profiling must be enabled on both contexts");
    cudaSetDevice(c->device);
    for (int s = 0; s <= ST_COUNT; s++)
        if (cudaEventElapsedTime(&offsets_ms[s], ref->ev_total[0], c->ev[s]) != cudaSuccess) {
            cudaGetLastError();
            return fail(c, CS_ERR_CUDA, "stage event %d not recorded or not complete", s);
        }
    return CS_OK;
}

int cs_debug_roi(cs_ctx *c, int job, int32_t roi_xywh[4], uint8_t *canny, float *dist, int cap_px, double *merged_lines, int cap_lines,
                 int32_t *n_lines_roi, int32_t *n_lines_merged)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!c->prepared || job < 0 || job >= (int)c->jobs.size()) return fail(c, CS_ERR_INVALID_ARG, "bad job index");
    cudaSetDevice(c->device);
    const CsJob &jb = c->jobs[job];
    const int npx = jb.roi_w * jb.roi_h;
    if (roi_xywh) {
        roi_xywh[0] = jb.roi_l;
        roi_xywh[1] = jb.roi_t;
        roi_xywh[2] = jb.roi_w;
        roi_xywh[3] = jb.roi_h;
    }
    CS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (canny && cap_px >= npx) {
        const int bwp = jb.bw + 2;
        std::vector<uint32_t> plane((size_t)(jb.roi_h + 2) * bwp);
        CS_CUDA(c, cudaMemcpy(plane.data(), (uint32_t *)c->d_bits.p + jb.bit_off, plane.size() * 4, cudaMemcpyDeviceToHost));
        for (int y = 0; y < jb.roi_h; y++)
            for (int x = 0; x < jb.roi_w; x++) canny[(size_t)y * jb.roi_w + x] = ((plane[(size_t)(y + 1) * bwp + 1 + (x >> 5)] >> (x & 31)) & 1u) ? 255 : 0;
    }
    if (dist && cap_px >= npx)
        CS_CUDA(c, cudaMemcpy2D(dist, (size_t)jb.roi_w * 4, (float *)c->d_dist.p + jb.px_off, (size_t)jb.dpitch * 4, (size_t)jb.roi_w * 4, jb.roi_h,
                                cudaMemcpyDeviceToHost));
    int32_t cnt[2];
    CS_CUDA(c, cudaMemcpy(cnt, (int32_t *)c->d_lcounts.p + job * 2, 8, cudaMemcpyDeviceToHost));
    if (n_lines_roi) *n_lines_roi = cnt[0];
    if (n_lines_merged) *n_lines_merged = cnt[1];
    if (merged_lines) {
        std::vector<double> tmp((size_t)CS_MAXL_OUT * 7);
        CS_CUDA(c, cudaMemcpy(tmp.data(), (double *)c->d_mlines.p + (size_t)job * CS_MAXL_OUT * 7, tmp.size() * 8, cudaMemcpyDeviceToHost));
        for (int i = 0; i < std::min(cnt[1], cap_lines); i++)
            for (int k = 0; k < 4; k++) merged_lines[i * 4 + k] = tmp[(size_t)k * CS_MAXL_OUT + i];
    }
    return CS_OK;
}

int cs_debug_candidates(cs_ctx *c, int job, int32_t *n_candidates, uint8_t *valid, double *dist_err, double *angle_err, int cap)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!c->prepared || job < 0 || job >= (int)c->jobs.size()) return fail(c, CS_ERR_INVALID_ARG, "bad job index");
    cudaSetDevice(c->device);
    const CsJob &jb = c->jobs[job];
    if (n_candidates) *n_candidates = jb.n_cand;
    const int n = std::min(cap, jb.n_cand);
    CS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (valid && n) CS_CUDA(c, cudaMemcpy(valid, (uint8_t *)c->d_cvalid.p + jb.cand_off, n, cudaMemcpyDeviceToHost));
    if (dist_err && n) CS_CUDA(c, cudaMemcpy(dist_err, (double *)c->d_cdist.p + jb.cand_off, (size_t)n * 8, cudaMemcpyDeviceToHost));
    if (angle_err && n) CS_CUDA(c, cudaMemcpy(angle_err, (double *)c->d_cangle.p + jb.cand_off, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return CS_OK;
}

} /* extern "C" */

#include "cs_nccl_impl.inc"
