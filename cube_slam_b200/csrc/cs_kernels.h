/* cs_kernels.h -- launcher prototypes of the sm_90a kernels (one .cu per stage group). */
#ifndef CS_KERNELS_H
#define CS_KERNELS_H

#include <cuda_runtime.h>
#include <stdint.h>

#include "cs_internal.h"

/* One shared-memory carveout for every kernel of the chain: kernels of several batches share the SMs, and an SM only changes its
 * L1 / shared split when it is idle.  75 % shared (a preference: a kernel that needs more shared memory still gets it).  H100, c3
 * headline with 12 batches in flight: 8.75 ms per step at 75 % shared, 9.06 with the driver's per-kernel choice. */
#define CS_SMEM_CARVEOUT_PCT 75
/* Function attributes are per device: CS_ONCE_PER_DEVICE(body) runs body until it has completed once on the current device (the flag word
 * is a bit per device ordinal: contexts on several devices / host threads may launch the same kernel).  The bit is set only AFTER the body
 * has run, so a thread that finds it set knows the attribute is in place before its launch.  Threads that arrive together all run the body;
 * every body sets constants, so running it twice does no harm.  (Setting the bit first would let a second thread skip the body and launch
 * with more than 48 KB of dynamic shared memory before the first thread had raised the limit.) */
#include <atomic>
#include <functional>
static inline unsigned long long cs_device_bit()
{
    int dev = 0;
    cudaGetDevice(&dev);
    return 1ull << (dev & 63);
}
#define CS_ONCE_PER_DEVICE(...)                                    \
    do {                                                           \
        static std::atomic<unsigned long long> once_flags_{0};     \
        const unsigned long long once_bit_ = cs_device_bit();      \
        if ((once_flags_.load() & once_bit_) == 0) {               \
            __VA_ARGS__;                                           \
            once_flags_.fetch_or(once_bit_);                       \
        }                                                          \
    } while (0)
/* let a kernel use as much dynamic shared memory as the device offers beyond its static allocation (the opt-in limit, 227 KB on H100) */
template <typename K>
static inline void cs_allow_max_dynamic_smem(K kernel)
{
    cudaFuncAttributes a;
    int dev = 0, optin = 0;
    if (cudaFuncGetAttributes(&a, kernel) != cudaSuccess || cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return;
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)a.sharedSizeBytes);
}
#define CS_APPLY_CARVEOUT(kernel) \
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, CS_SMEM_CARVEOUT_PCT))

#define CS_DT_CLASSES 7
extern const int cs_dt_class_width[CS_DT_CLASSES];
int cs_dt_class_of(int roi_w);

void cs_launch_gray(const uint8_t *d_img, uint8_t *d_gray, int n_frames, int w, int h, int stride, int channels, cudaStream_t st,
                    int64_t *launches);
/* cvtColor of frames of any sizes, one launch over the plane table d_tab[0 .. n) (total: its pixels); sources at d_img + src, destinations at
 * d_dst + dst -- the arithmetic of cs_launch_gray (cs_lbd_octaves.cu: k_oct_gray_tab) */
void cs_launch_gray_tab(const uint8_t *d_img, const OctPlane *d_tab, int n, int64_t total, uint8_t *d_dst, cudaStream_t st, int64_t *launches);
/* ROI j reads its gray plane at d_base + jobs[j].gray_off, rows of jobs[j].gray_pitch bytes, so frames of any sizes share a launch.  The two
 * ints after d_base are not read: they keep the parameter list the host build of cs_context.cu in the CPU tests stubs by signature. */
void cs_launch_canny(const uint8_t *d_base, int, int, const CsJob *d_jobs, int n_jobs, const int32_t *d_tile_job, int n_tiles, uint32_t *d_bits,
                     size_t bits_bytes, int low, int high, cudaStream_t st, int64_t *launches);
void cs_launch_hyst(const CsJob *d_jobs, int n_jobs, uint32_t *d_bits, int max_plane_words, cudaStream_t st, int64_t *launches);
void cs_launch_dt(const CsJob *d_jobs, const int32_t *d_ids, int n_jobs, int max_dpitch, const int *class_off, const int *class_plane_words,
                  const uint32_t *d_bits, float *d_dist, int raster_or_flags, cudaStream_t st, cudaStream_t st_side, cudaEvent_t ev_fork,
                  cudaEvent_t ev_join, int64_t *launches);
void cs_launch_roi_lines(const CsJob *d_jobs, int n_jobs, const CsFrame *d_frames, const double *d_lines, const float *d_lines_f32,
                         const int32_t *d_n_lines_dev, int f32_pitch, double *d_out_lines,
                         int32_t *d_out_counts, int32_t *d_err, double dist_thre, double angle_thre_deg, double len_thre, cudaStream_t st,
                         int64_t *launches);
void cs_launch_fuse(const CsObj *d_objs, int n_objs, const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw,
                    const uint8_t *c_valid, const double *c_dist, const double *c_angle, int32_t *w_vlist, uint64_t *w_key, uint32_t *w_idx,
                    uint8_t *w_flag, int32_t *w_keep, double *w_norm, double *w_score, int32_t *job_counts, cs_cuboid_rec *d_out,
                    int32_t *d_out_counts, int topk, const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches);

void cs_launch_sweep_warp(const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw, const int4 *d_blocks4,
                          int n_blocks, const double *d_mlines, const int32_t *d_line_counts, const float *d_dist, uint8_t *c_valid,
                          double *c_dist, double *c_angle, double *c_skew, const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches);
void cs_launch_fuse_warp(const CsObj *d_objs, int n_objs, const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw,
                         const uint8_t *c_valid, const double *c_dist, const double *c_angle, const double *c_skew, int32_t *w_vlist, int32_t *w_keep,
                         double *w_norm, double *w_score, int32_t *job_counts, cs_cuboid_rec *d_out, int32_t *d_out_counts, int topk,
                         const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches);
int cs_fuse_warp_cap(void);
int cs_sweep_warp_yaws(void);

/* A batch of frames of different sizes (cs_mixed.cu) hands run_batch the two stages it runs differently, as functions: cs_context.cu is also
 * compiled alone for the host by the CPU tests (tests/host_core/context_emu.cpp), so it names no function of the line detectors or of the
 * table-driven gray kernel. */
struct CsMixedLines {
    const uint8_t *d_img;        /* the batch's frame buffer */
    const cs_frame_view *views;  /* host, frame order: where each frame lies in d_img */
    const int32_t *order;        /* host: the frames in the order they lie in d_img (EDLines: its size groups one after the other) */
    const int32_t *d_order;      /* the same on the device */
    int n_frames, cap;           /* cap: segments per frame slot */
    const cs_line_params *prm;
    float *d_lines;              /* n_frames x cap x 4 floats and n_frames counts: the slots EDLines' groups are scattered to */
    int32_t *d_counts;
    int32_t *d_err4;             /* the batch's line-detector error word (4 ints, zeroed by run_batch) */
};
struct CsMixedStages {
    void (*gray)(const uint8_t *d_img, const OctPlane *d_tab, int n, int64_t total, uint8_t *d_dst, cudaStream_t st, int64_t *launches);
    /* enqueues the online line detector over every frame: segments and counts per frame slot, its error word in d_err4 */
    int (*lines)(cs_ctx *c, const CsMixedLines &m, const float **d_lines, const int32_t **d_counts);
};
/* cs_mixed.cu's ways into the batch (cs_context.cu): store a checked batch of mixed sizes whose frames the caller then packs into *d_img at
 * `packed`, in the order `order`, before it marks the batch prepared (cs_ctx_mark_prepared); and the carried-pose passes of
 * cs_set_profiling bit 10 over any store step (a pass stores the caller's batch with its own boxes, CSR sub_off) */
int cs_ctx_store_mixed_batch(cs_ctx *c, const cs_frame_view *packed, const int32_t *order, int n_frames, const double *K, const double *T_wc,
                             const double *boxes, const int32_t *box_offsets, const double *lines, const int32_t *line_offsets,
                             const cs_cuboid_params *params, const cs_line_params *online, const CsMixedStages *stages, uint8_t **d_img);
typedef std::function<int(const double *sub_boxes, const int32_t *sub_off)> CsStoreBoxes;
bool cs_ctx_carries_pose(cs_ctx *c, const cs_cuboid_params *params, const int32_t *box_offsets, int n_frames, const cs_cuboid_rec *out,
                         const int32_t *out_counts);
int cs_ctx_detect_carried(cs_ctx *c, const CsStoreBoxes &store, int n_frames, const double *boxes, const int32_t *box_offsets,
                          const cs_cuboid_params *params, cs_cuboid_rec *out, int32_t *out_counts);

#endif
