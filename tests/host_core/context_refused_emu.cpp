/* tests/host_core/context_refused_emu.cpp -- cube_slam_b200/csrc/cs_context.cu compiled for the host (as context_emu.cpp does), with launchers
 * that record what they are asked to read and write instead of running anything: the gray conversion's frames and planes, and every Canny
 * ROI's gray bytes, each checked against the batch's frame buffer.  The test around it uploads a batch, has later uploads refused, and runs
 * again: the run must still be the prepared batch's, inside its buffer.  Test infrastructure, never shipped.
 * g++ -std=c++20 -I tests/host_core/fake_cuda ... cs_host_pose.cpp */
#include <cuda_runtime.h> /* tests/host_core/fake_cuda */

#define cs_create cs_create_in_library
#include "../../cube_slam_b200/csrc/cs_context.cu"
#undef cs_create

static cs_ctx *g_cur = nullptr;
/* {gray launches, gray reads or writes outside d_img, Canny launches, Canny ROIs outside d_img, last gray n, w, h, stride, channels} */
static int64_t g_rec[9];

static bool inside(const void *p, int64_t bytes)
{
    const uint8_t *b = (const uint8_t *)g_cur->d_img.p, *q = (const uint8_t *)p;
    return bytes >= 0 && q >= b && q + bytes <= b + g_cur->d_img.cap;
}

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

void cs_launch_gray(const uint8_t *src, uint8_t *dst, int n, int w, int h, int stride, int ch, cudaStream_t, int64_t *)
{
    g_rec[0]++;
    if (!inside(src, (int64_t)n * h * stride) || !inside(dst, (int64_t)n * w * h)) g_rec[1]++;
    g_rec[4] = n, g_rec[5] = w, g_rec[6] = h, g_rec[7] = stride, g_rec[8] = ch;
}
void cs_launch_canny(const uint8_t *base, int, int, const CsJob *jobs, int n_jobs, const int32_t *, int, uint32_t *, size_t, int, int, cudaStream_t, int64_t *)
{
    g_rec[2]++;
    for (int j = 0; j < n_jobs; j++)
        if (!inside(base + jobs[j].gray_off, (int64_t)(jobs[j].roi_h - 1) * jobs[j].gray_pitch + jobs[j].roi_w)) g_rec[3]++;
}
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
}
void cs_launch_fuse_warp(const CsObj *, int, const CsJob *, const CsFrame *, const CsPose *, const double *, const uint8_t *, const double *, const double *, const double *,
                         int32_t *, int32_t *, double *, double *, int32_t *, cs_cuboid_rec *, int32_t *, int, const cs_cuboid_params *, cudaStream_t, int64_t *)
{
}

extern "C" cs_ctx *cs_create(int device, int max_width, int max_height, int max_frames, int max_boxes_per_frame, int max_lines_per_frame)
{
    return g_cur = cs_create_in_library(device, max_width, max_height, max_frames, max_boxes_per_frame, max_lines_per_frame);
}
extern "C" void emu_record(int64_t out[9]) { std::memcpy(out, g_rec, sizeof g_rec); }
/* the mixed uploads' store step (cs_mixed.cu), frames packed back to back in call order; the frames themselves are not copied */
extern "C" int emu_store_mixed(cs_ctx *c, const cs_frame_view *packed, int n_frames, const double *T_wc, const double *boxes, const int32_t *box_offsets,
                               const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params)
{
    static const CsMixedStages stages = {nullptr, nullptr};
    std::vector<int32_t> order((size_t)std::max(n_frames, 0));
    for (int f = 0; f < n_frames; f++) order[f] = f;
    uint8_t *d_img = nullptr;
    return cs_ctx_store_mixed_batch(c, packed, order.data(), n_frames, nullptr, T_wc, boxes, box_offsets, lines, line_offsets, params, nullptr, &stages, &d_img);
}
