/* cs_mixed.cu -- the cuboid batch over frames of different sizes and cameras (include/cube_slam_b200.h: cs_batch_upload_mixed,
 * cs_batch_upload_online_mixed, cs_detect_cuboids_batch_mixed, cs_detect_frames_batch_mixed).
 *
 * The cuboid stage is per frame already: every frame carries its own invK and every pose its own K * R^-1, and the ROI jobs carry their
 * frame's gray plane (CsJob::gray_off / gray_pitch).  What a batch of mixed sizes adds is here:
 *   - the host checks, every one before anything is enqueued, each naming the frame;
 *   - the layout of d_img: the frames packed back to back in call order (EDLines online: its size groups one after the other, each group
 *     256-byte aligned), then the gray planes of the 3-channel frames (cs_context.cu: store_frames);
 *   - the two stages run_batch runs differently (CsMixedStages): the gray planes in one table-driven launch (cs_launch_gray_tab), and the
 *     online line detector -- LSD over every frame as one run (cs_lsd_run_mixed_device), EDLines one run per size group, each group's
 *     segments scattered to the batch's per-frame slots by k_edl_scatter.  Neither waits on the host.
 * Records, counts and everything after the upload are the one-size path's: run, fetch, stats, the debug reads and the all-gather. */
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "cs_internal.h"
#include "cs_kernels.h"

namespace {

/* one EDLines size group's segments (slot j of its run) into the batch's slot of frame order[j], and the group's error word ORed into the
 * batch's.  One CTA per frame of the group. */
__global__ void __launch_bounds__(256) k_edl_scatter(const float4 *__restrict__ src, const int32_t *__restrict__ src_n, const int32_t *__restrict__ order,
                                                      int cap, float4 *__restrict__ dst, int32_t *__restrict__ dst_n, const int32_t *__restrict__ err,
                                                      int32_t *__restrict__ err4)
{
    const int j = blockIdx.x, f = order[j];
    const int n = src_n[j], m = min(n, cap); /* a count past cap is passed on: the ROI line kernel reports it (fetch: CS_ERR_CAPACITY) */
    for (int i = threadIdx.x; i < m; i += blockDim.x) dst[(size_t)f * cap + i] = src[(size_t)j * cap + i];
    if (threadIdx.x == 0) {
        dst_n[f] = n;
        if (j == 0)
            for (int k = 0; k < 4; k++)
                if (err[k]) atomicOr(&err4[k], err[k]);
    }
}

bool same_size(const cs_frame_view &a, const cs_frame_view &b) { return a.width == b.width && a.height == b.height && a.channels == b.channels; }

/* CsMixedStages::lines: enqueued only, like the one-size online run */
int mixed_lines(cs_ctx *c, const CsMixedLines &m, const float **d_lines, const int32_t **d_counts)
{
    cudaStream_t st = cs_ctx_stream(c);
    int rc;
    if (m.prm->use_LSD) {
        const int32_t *err = nullptr;
        if ((rc = cs_lsd_run_mixed_device(c, m.d_img, m.views, m.n_frames, m.prm->line_length_thres, m.cap, d_lines, d_counts, &err))) return rc;
        if (cudaMemcpyAsync(m.d_err4, err, 16, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "LSD error word copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        return CS_OK;
    }
    for (int g0 = 0; g0 < m.n_frames;) { /* a group: frames order[g0 .. g1), back to back in d_img */
        const cs_frame_view &v = m.views[m.order[g0]];
        int g1 = g0 + 1;
        while (g1 < m.n_frames && same_size(m.views[m.order[g1]], v)) g1++;
        const float *gl = nullptr;
        const int32_t *gn = nullptr;
        if ((rc = cs_edl_run(c, m.d_img + v.offset, true, g1 - g0, v.width, v.height, v.stride, v.channels, m.prm->line_length_thres, m.cap, &gl, &gn)))
            return rc;
        k_edl_scatter<<<g1 - g0, 256, 0, st>>>((const float4 *)gl, gn, m.d_order + g0, m.cap, (float4 *)m.d_lines, m.d_counts,
                                               cs_line_err_word(*cs_ctx_edl_slot(c)), m.d_err4);
        cs_ctx_count_launches(c, 1);
        g0 = g1;
    }
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "EDLines scatter launch failed");
    *d_lines = m.d_lines;
    *d_counts = m.d_counts;
    return CS_OK;
}

const CsMixedStages kStages = {cs_launch_gray_tab, mixed_lines};

/* the refusals of the mixed calls that the batch store does not make itself (it checks capacities, parameters and the CSRs) */
int check_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const cs_line_params *online)
{
    int rc;
    if ((rc = cs_check_frame_views(c, imgs, views, n_frames))) return rc;
    if (K)
        for (int f = 0; f < n_frames; f++) {
            const double *k = K + (size_t)f * 9;
            for (int i = 0; i < 9; i++)
                if (!std::isfinite(k[i])) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: K[%d] = %g is not finite", f, i, k[i]);
            const double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6]);
            if (det == 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: K has a zero determinant", f);
        }
    if (online && (rc = cs_check_line_frames(c, views, n_frames, online))) return rc;
    return CS_OK;
}

/* where the frames go in d_img: order = the frames in d_img order, groups = its runs that are packed with one copy each; packed = the
 * frames' views there (frame order) */
void layout(const cs_frame_view *views, int n_frames, bool by_size, std::vector<int32_t> &order, std::vector<int> &groups,
            std::vector<cs_frame_view> &packed)
{
    order.clear();
    groups.clear();
    if (!by_size) {
        for (int f = 0; f < n_frames; f++) order.push_back(f);
        groups.push_back(0);
    } else { /* EDLines runs one batch per (width, height, channels): its groups in order of first appearance, frames in call order */
        std::vector<char> done((size_t)n_frames, 0);
        for (int f0 = 0; f0 < n_frames; f0++) {
            if (done[f0]) continue;
            groups.push_back((int)order.size());
            for (int f = f0; f < n_frames; f++)
                if (!done[f] && same_size(views[f], views[f0])) {
                    order.push_back(f);
                    done[f] = 1;
                }
        }
    }
    groups.push_back(n_frames);
    packed.assign(views, views + n_frames);
    int64_t off = 0;
    for (size_t g = 0; g + 1 < groups.size(); g++) {
        off = (off + 255) & ~(int64_t)255; /* a group starts aligned, as a frame buffer of its own would (the EDLines front end's TMA path) */
        for (int i = groups[g]; i < groups[g + 1]; i++) {
            cs_frame_view &v = packed[order[i]];
            v.offset = off;
            v.stride = v.width * v.channels;
            off += (int64_t)v.stride * v.height;
        }
    }
}

/* the body of the two uploads: check, store the tables, pack the frames into d_img, mark the batch prepared (nothing waits here) */
int store_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc, const double *boxes,
                const int32_t *box_offsets, const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params, const cs_line_params *online)
{
    int rc;
    if ((rc = check_mixed(c, imgs, views, n_frames, K, online))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    std::vector<int32_t> order;
    std::vector<int> groups;
    std::vector<cs_frame_view> packed, part, got;
    layout(views, n_frames, online && !online->use_LSD, order, groups, packed);
    uint8_t *d_img = nullptr;
    if ((rc = cs_ctx_store_mixed_batch(c, packed.data(), order.data(), n_frames, K, T_wc, boxes, box_offsets, lines, line_offsets, params, online, &kStages,
                                       &d_img)))
        return rc;
    for (size_t g = 0; g + 1 < groups.size(); g++) {
        part.clear();
        for (int i = groups[g]; i < groups[g + 1]; i++) part.push_back(views[order[i]]);
        if ((rc = cs_pack_host_frames(c, d_img + packed[order[groups[g]]].offset, imgs, part.data(), (int)part.size(), got))) return rc;
    }
    cs_ctx_mark_prepared(c);
    return CS_OK;
}

int detect_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc, const double *boxes,
                 const int32_t *box_offsets, const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params, const cs_line_params *online,
                 cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!online && cs_ctx_carries_pose(c, params, box_offsets, n_frames, out, out_counts))
        return cs_ctx_detect_carried(
            c,
            [&](const double *sub_boxes, const int32_t *sub_off) {
                return store_mixed(c, imgs, views, n_frames, K, T_wc, sub_boxes, sub_off, lines, line_offsets, params, nullptr);
            },
            n_frames, boxes, box_offsets, params, out, out_counts);
    int rc;
    if ((rc = store_mixed(c, imgs, views, n_frames, K, T_wc, boxes, box_offsets, lines, line_offsets, params, online))) return rc;
    if ((rc = cs_batch_run_async(c))) return rc;
    return cs_batch_fetch(c, out, out_counts);
}

}  // namespace

extern "C" {

int cs_batch_upload_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                          const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc;
    if ((rc = store_mixed(c, imgs, views, n_frames, K, T_wc, boxes, box_offsets, lines, line_offsets, params, nullptr))) return rc;
    if (cudaStreamSynchronize(cs_ctx_stream(c)) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "upload: %s", cudaGetErrorString(cudaGetLastError()));
    return CS_OK;
}

int cs_batch_upload_online_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                 const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!line_params) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null line params");
    int rc;
    if ((rc = store_mixed(c, imgs, views, n_frames, K, T_wc, boxes, box_offsets, nullptr, nullptr, params, line_params))) return rc;
    if (cudaStreamSynchronize(cs_ctx_stream(c)) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "upload: %s", cudaGetErrorString(cudaGetLastError()));
    return CS_OK;
}

int cs_detect_cuboids_batch_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                  const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                                  const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c) return CS_ERR_INVALID_ARG;
    return detect_mixed(c, imgs, views, n_frames, K, T_wc, boxes, box_offsets, lines, line_offsets, params, nullptr, out, out_counts);
}

int cs_detect_frames_batch_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const double *K, const double *T_wc,
                                 const double *boxes, const int32_t *box_offsets, const cs_line_params *line_params, const cs_cuboid_params *params,
                                 cs_cuboid_rec *out, int32_t *out_counts)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!line_params) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null line params");
    return detect_mixed(c, imgs, views, n_frames, K, T_wc, boxes, box_offsets, nullptr, nullptr, params, line_params, out, out_counts);
}

} /* extern "C" */
