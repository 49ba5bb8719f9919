/* tests/host_core/context_emu.cpp -- cube_slam_b200/csrc/cs_context.cu ITSELF (the host orchestration of the cuboid stage: batch storage,
 * sample tables, the launch sequence, fetch, and the carried-pose pass loop of cs_set_profiling bit 10) compiled for the host, with the
 * kernel launchers of the other translation units replaced by one stand-in that answers from the CPU ORACLE: when the last stage of a
 * batch is "launched", every box's records and the candidate records of its last height sample are filled in from orc_detect_cuboid,
 * which is told -- through orc_set_first_box_cam_yaw -- the camera yaw the library's own yaw table for that frame was derived from (found
 * by regenerating the table from the raw pose and from each pose hypothesis and comparing bits).  So the test around this file checks the
 * library's real code for: which boxes go into which pass, the per-pass yaw override reaching build_tables, the job / candidate offsets
 * the host reads the records back through, last_set_pose, the pose table lookup and the scatter of the results.  Test infrastructure,
 * never shipped.  g++ -std=c++20 -I tests/host_core/fake_cuda ... cs_host_pose.cpp, linked against oracle/_build/liboracle.so. */
#include <cuda_runtime.h> /* tests/host_core/fake_cuda */

#define cs_create cs_create_in_library /* wrapped below: the stand-in launchers need to know which context is running */
#include "../../cube_slam_b200/csrc/cs_context.cu"
#undef cs_create

#include "../../oracle/orc_api.h"

extern "C" void orc_set_first_box_cam_yaw(double yaw);
static_assert(sizeof(orc_cuboid) == sizeof(cs_cuboid_rec), "one record layout");

static cs_ctx *g_cur = nullptr;
static int g_mismatch = 0; /* bit 0: no camera yaw reproduces the frame's yaw table; bit 1: candidate count differs from the oracle's */

/* ---- the other translation units' symbols cs_context.cu refers to */
void cs_lsd_destroy(void *) {}
void cs_edl_destroy(void *) {}
void cs_lbd_destroy(void *) {}
int cs_lsd_run_device(cs_ctx *c, const uint8_t *, int, int, int, int, int, float, int, const float **, const int32_t **) { return cs_ctx_fail(c, CS_ERR_UNSUPPORTED, "no line detector in this emulation"); }
int cs_edl_run(cs_ctx *c, const uint8_t *, bool, int, int, int, int, int, float, int, const float **, const int32_t **) { return cs_ctx_fail(c, CS_ERR_UNSUPPORTED, "no line detector in this emulation"); }
const int cs_dt_class_width[CS_DT_CLASSES] = {128, 256, 384, 512, 640, 1024, 2048};
int cs_dt_class_of(int roi_w)
{
    for (int i = 0; i < CS_DT_CLASSES; i++)
        if (roi_w <= cs_dt_class_width[i]) return i;
    return -1;
}
int cs_fuse_warp_cap(void) { return 1024; }
int cs_sweep_warp_yaws(void) { return 4; }

static void fill_from_oracle(cs_ctx *c)
{
    const int topk = c->topk;
    orc_params p;
    orc_default_params(&p);
    const cs_cuboid_params &q = c->prm;
    p.consider_config_1 = q.consider_config_1;
    p.consider_config_2 = q.consider_config_2;
    p.whether_sample_cam_roll_pitch = q.whether_sample_cam_roll_pitch;
    p.whether_sample_bbox_height = q.whether_sample_bbox_height;
    p.max_cuboid_num = q.max_cuboid_num;
    p.nominal_skew_ratio = q.nominal_skew_ratio;
    p.max_cut_skew = q.max_cut_skew;
    p.top_sample_count_override = q.top_sample_count_override;
    p.yaw_half_range_deg = q.yaw_half_range_deg;
    p.yaw_step_deg = q.yaw_step_deg;
    uint8_t *cv = (uint8_t *)c->d_cvalid.p;
    double *cd = (double *)c->d_cdist.p, *ca = (double *)c->d_cangle.p;
    cs_cuboid_rec *out = (cs_cuboid_rec *)c->d_out.p;
    int32_t *outcnt = (int32_t *)c->d_outcnt.p;
    std::memset(c->d_err.p, 0, 16);
    for (size_t o = 0; o < c->objs.size(); o++) {
        const CsObj &ob = c->objs[o];
        const int f = ob.frame;
        const CsFrame &fr = c->frames[f];
        /* which camera yaw was this frame's yaw table derived from? */
        double used = std::nan("");
        bool found = false;
        for (int cand = -1; cand < fr.n_pose && !found; cand++) {
            CsPose raw;
            double eu[3];
            cshost::make_pose(c->K, &c->h_T[(size_t)f * 16], &raw, eu);
            const double cam_yaw = cand < 0 ? raw.camera_yaw : c->poses[(size_t)fr.pose_off + cand].camera_yaw;
            const double yaw_init = cam_yaw - 90.0 / 180.0 * M_PI;
            std::vector<double> ys;
            cshost::linespace_d(yaw_init - q.yaw_half_range_deg / 180.0 * M_PI, yaw_init + q.yaw_half_range_deg / 180.0 * M_PI, q.yaw_step_deg / 180.0 * M_PI, ys);
            if ((int)ys.size() != fr.n_yaw) continue;
            bool same = true;
            for (int k = 0; k < fr.n_yaw && same; k++) same = std::memcmp(&ys[k], &c->yaws[(size_t)(fr.yaw_off + k) * 3], 8) == 0;
            if (same) {
                found = true;
                used = cand < 0 ? std::nan("") : cam_yaw;
            }
        }
        if (!found) g_mismatch |= 1;
        orc_set_first_box_cam_yaw(used);
        const int last_hs = ob.n_jobs - 1;
        std::vector<double> rows((size_t)(1 << 17) * 9);
        std::vector<int32_t> cidx((size_t)1 << 17);
        orc_trace tr;
        std::memset(&tr, 0, sizeof tr);
        tr.want_object = 0;
        tr.want_height_sample = last_hs;
        tr.rows = rows.data();
        tr.cand_index = cidx.data();
        tr.cap_valid = 1 << 17;
        int cnt = 0;
        const uint8_t *img = (const uint8_t *)c->d_img.p + (size_t)f * c->h * c->stride;
        orc_detect_cuboid(img, c->w, c->h, c->stride, c->channels, c->K, &c->h_T[(size_t)f * 16], &c->h_boxes[o * 5], 1,
                          c->h_lines.data() + (size_t)c->h_line_off[f] * 4, c->h_line_off[f + 1] - c->h_line_off[f], &p, topk, (orc_cuboid *)&out[o * topk], &cnt, nullptr,
                          nullptr, &tr);
        outcnt[o] = cnt;
        if (ob.n_jobs > 0) {
            const CsJob &jb = c->jobs[(size_t)ob.job_off + last_hs];
            if (tr.n_candidates != jb.n_cand) g_mismatch |= 2;
            for (int i = 0; i < jb.n_cand; i++) cv[jb.cand_off + i] = 0;
            for (int i = 0; i < tr.n_valid && i < tr.cap_valid; i++) {
                const int64_t ci = jb.cand_off + cidx[i];
                cv[ci] = 1;
                cd[ci] = rows[(size_t)i * 9 + 4];
                ca[ci] = rows[(size_t)i * 9 + 5];
            }
        }
    }
    orc_set_first_box_cam_yaw(std::nan(""));
}

/* the launchers: every stage is a no-op except the last one of the chain */
void cs_launch_gray(const uint8_t *, uint8_t *, int, int, int, int, int, cudaStream_t, int64_t *) {}
void cs_launch_canny(const uint8_t *, int, int, const CsJob *, int, const int32_t *, int, uint32_t *, size_t, int, int, cudaStream_t, int64_t *) {}
void cs_launch_hyst(const CsJob *, int, uint32_t *, int, cudaStream_t, int64_t *) {}
void cs_launch_dt(const CsJob *, const int32_t *, int, int, const int *, const int *, const uint32_t *, float *, int, cudaStream_t, cudaStream_t, cudaEvent_t, cudaEvent_t,
                  int64_t *)
{
}
void cs_launch_roi_lines(const CsJob *, int, const CsFrame *, const double *, const float *, const int32_t *, int, double *, int32_t *, int32_t *, double, double, double,
                         cudaStream_t, int64_t *)
{
}
void cs_launch_sweep_warp(const CsJob *, const CsFrame *, const CsPose *, const double *, const int4 *, int, const double *, const int32_t *, const float *, uint8_t *,
                          double *, double *, double *, const cs_cuboid_params *, cudaStream_t, int64_t *)
{
}
void cs_launch_fuse(const CsObj *, int, const CsJob *, const CsFrame *, const CsPose *, const double *, const uint8_t *, const double *, const double *, int32_t *, uint64_t *,
                    uint32_t *, uint8_t *, int32_t *, double *, double *, int32_t *, cs_cuboid_rec *, int32_t *, int, const cs_cuboid_params *, cudaStream_t, int64_t *)
{
    fill_from_oracle(g_cur);
}
void cs_launch_fuse_warp(const CsObj *, int, const CsJob *, const CsFrame *, const CsPose *, const double *, const uint8_t *, const double *, const double *, const double *,
                         int32_t *, int32_t *, double *, double *, int32_t *, cs_cuboid_rec *, int32_t *, int, const cs_cuboid_params *, cudaStream_t, int64_t *)
{
    fill_from_oracle(g_cur);
}

/* entry points for the test */
extern "C" int emu_detect_cuboids_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const double *T_wc,
                                        const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                                        const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts)
{
    g_cur = c;
    g_mismatch = 0;
    return cs_detect_cuboids_batch(c, imgs, n_frames, width, height, stride, channels, T_wc, boxes, box_offsets, lines, line_offsets, params, out, out_counts);
}
extern "C" int emu_mismatch(void) { return g_mismatch; }

/* cs_create as the Python mirror calls it: the library's own, plus a note of the context for the stand-in launchers (one context at a time) */
extern "C" cs_ctx *cs_create(int device, int max_width, int max_height, int max_frames, int max_boxes_per_frame, int max_lines_per_frame)
{
    g_cur = cs_create_in_library(device, max_width, max_height, max_frames, max_boxes_per_frame, max_lines_per_frame);
    g_mismatch = 0;
    return g_cur;
}
