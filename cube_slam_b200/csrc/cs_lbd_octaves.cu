/* cs_lbd_octaves.cu -- every octave of a multi-octave LSD line_lbd_detect: the image pyramids, LSD per octave, the key lines and their LBD
 * descriptors (include/cube_slam_b200.h: cs_detect_raw_lines_octaves_batch, cs_detect_descrip_lines_octaves_batch); and the LBD descriptors of
 * key lines of any octave that the caller gives (cs_lbd_compute_octaves_batch).
 *
 * Replaces   line_lbd/class/line_lbd_allclass.cpp:125-172,285-339   detect_raw_lines (both KeyLine overloads), detect_descrip_lines_octaves
 *            line_lbd/libs/LSDDetector.cpp:55-72,176-250             computeGaussianPyramid, detect: LSD per octave, KeyLine fill
 *            line_lbd/libs/binary_descriptor.cpp:352-398             computeGaussianPyramid + computeSobel for every octave
 *            line_lbd/libs/binary_descriptor.cpp:587-790             BinaryDescriptor::compute / computeImpl on given key lines of any octave
 *
 *   k_oct_gray      cvtColor of the frames (the fixed-point arithmetic of k_lsd_front / k_ed_front): octave 0 of the LSD pyramid
 *   k_oct_pyrdown   cv::pyrDown on 8-bit planes: the separable 1-4-6-4-1 kernel at the even source positions, BORDER_REFLECT_101, one
 *                   rounding (sum + 128) >> 8 (oracle/ref/minicv.hpp states it and pins it to cv2)
 *   k_oct_blur5     GaussianBlur(5 x 5, sigma 1) of the gray plane: OpenCV's fixed-point kernel (14 62 104 62 14) in both directions, one
 *                   rounding (sum + 32768) >> 16 -- what k_ed_front computes -- the base of the descriptor's pyramid
 *   k_oct_sobel     3 x 3 Sobel to int16 (BORDER_REFLECT_101) of the descriptor's pyramid, octaves >= 1; octave 0's maps come from
 *                   cs_edl_sobel_maps, as for the one-octave descriptor
 *   k_oct_gray_tab / k_oct_pyrdown_tab   the same two on frames of any sizes, one launch per level over every frame (OctPlane table)
 * One thread per output pixel over the whole batch; every plane is a few hundred KB, bound by its bytes.  LSD runs once over every octave of
 * every frame (cs_lsd_run_mixed_sync: a batch of planes of different sizes); the raw segments go to the host in one copy, where the key lines
 * are filled and filtered (cs_keyline_from_lsd_octave, cs_lbd.cu), and the descriptors are computed per octave by the one-octave descriptor
 * kernel. */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <unordered_map>
#include <utility>
#include <vector>

#include "cs_internal.h"
#include "cs_kernels.h" /* cs_launch_gray_tab */
#include "cs_lbd_core.h" /* CS_LBD_BYTES, CS_LBD_DESC */

namespace {

__device__ __forceinline__ int oct_reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = (p < 0) ? -p : 2 * n - 2 - p;
    return p;
}

__global__ void __launch_bounds__(256) k_oct_gray(const uint8_t *__restrict__ img, int n_frames, int w, int h, int stride, int channels,
                                                  uint8_t *__restrict__ gray)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint8_t *row = img + ((size_t)f * h + y) * stride;
        if (channels == 3) {
            const uint8_t *q = row + 3 * x;
            gray[p] = (uint8_t)((q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15);
        } else
            gray[p] = row[x];
    }
}

__global__ void __launch_bounds__(256) k_oct_pyrdown(const uint8_t *__restrict__ src, int n_frames, int sw, int sh, uint8_t *__restrict__ dst, int dw,
                                                     int dh)
{
    const int64_t total = (int64_t)n_frames * dw * dh;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)dw * dh);
        const int r = (int)(p - f * (int64_t)dw * dh);
        const int y = r / dw, x = r - y * dw;
        const uint8_t *s = src + (size_t)f * sw * sh;
        const int k[5] = {1, 4, 6, 4, 1};
        int xs[5];
#pragma unroll
        for (int i = 0; i < 5; i++) xs[i] = oct_reflect101(2 * x + i - 2, sw);
        uint32_t a = 0;
#pragma unroll
        for (int j = 0; j < 5; j++) {
            const uint8_t *row = s + (size_t)oct_reflect101(2 * y + j - 2, sh) * sw;
            uint32_t t = 0;
#pragma unroll
            for (int i = 0; i < 5; i++) t += k[i] * (uint32_t)row[xs[i]];
            a += k[j] * t;
        }
        dst[p] = (uint8_t)((a + 128u) >> 8);
    }
}

/* One plane of a level of the LSD pyramids of frames of any sizes is an OctPlane (cs_internal.h); one launch per level covers every frame. */

/* the plane of the level that output pixel p belongs to: the last one whose px0 is <= p */
__device__ __forceinline__ int oct_plane_of(const OctPlane *__restrict__ tab, int n, int64_t p)
{
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].px0 <= p)
            lo = mid;
        else
            hi = mid - 1;
    }
    return lo;
}

/* k_oct_gray over frames of any sizes: octave 0 of every frame's pyramid; the gray planes of a cuboid batch of mixed sizes
 * (cs_launch_gray_tab) */
__global__ void __launch_bounds__(256) k_oct_gray_tab(const uint8_t *__restrict__ img, const OctPlane *__restrict__ tab, int n, int64_t total,
                                                      uint8_t *__restrict__ pyr)
{
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const OctPlane &P = tab[oct_plane_of(tab, n, p)];
        const int r = (int)(p - P.px0);
        const int y = r / P.dw, x = r - y * P.dw;
        const uint8_t *row = img + P.src + (size_t)y * P.sstride;
        if (P.ch == 3) {
            const uint8_t *q = row + 3 * x;
            pyr[P.dst + r] = (uint8_t)((q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15);
        } else
            pyr[P.dst + r] = row[x];
    }
}

/* k_oct_pyrdown over frames of any sizes: one level of every frame's pyramid from the level above it, both in pyr */
__global__ void __launch_bounds__(256) k_oct_pyrdown_tab(const OctPlane *__restrict__ tab, int n, int64_t total, uint8_t *__restrict__ pyr)
{
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const OctPlane &P = tab[oct_plane_of(tab, n, p)];
        const int r = (int)(p - P.px0);
        const int y = r / P.dw, x = r - y * P.dw;
        const uint8_t *s = pyr + P.src;
        const int sw = P.sw, sh = P.sh;
        const int k[5] = {1, 4, 6, 4, 1};
        int xs[5];
#pragma unroll
        for (int i = 0; i < 5; i++) xs[i] = oct_reflect101(2 * x + i - 2, sw);
        uint32_t a = 0;
#pragma unroll
        for (int j = 0; j < 5; j++) {
            const uint8_t *row = s + (size_t)oct_reflect101(2 * y + j - 2, sh) * sw;
            uint32_t t = 0;
#pragma unroll
            for (int i = 0; i < 5; i++) t += k[i] * (uint32_t)row[xs[i]];
            a += k[j] * t;
        }
        pyr[P.dst + r] = (uint8_t)((a + 128u) >> 8);
    }
}

__global__ void __launch_bounds__(256) k_oct_blur5(const uint8_t *__restrict__ src, int n_frames, int w, int h, uint8_t *__restrict__ dst)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint8_t *s = src + (size_t)f * w * h;
        const int k[5] = {14, 62, 104, 62, 14};
        int xs[5];
#pragma unroll
        for (int i = 0; i < 5; i++) xs[i] = oct_reflect101(x + i - 2, w);
        uint32_t a = 0;
#pragma unroll
        for (int j = 0; j < 5; j++) {
            const uint8_t *row = s + (size_t)oct_reflect101(y + j - 2, h) * w;
            uint32_t t = 0;
#pragma unroll
            for (int i = 0; i < 5; i++) t += k[i] * (uint32_t)row[xs[i]];
            a += k[j] * t;
        }
        dst[p] = (uint8_t)((a + 32768u) >> 16);
    }
}

__global__ void __launch_bounds__(256) k_oct_sobel(const uint8_t *__restrict__ src, int n_frames, int w, int h, int16_t *__restrict__ dxo,
                                                   int16_t *__restrict__ dyo)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint8_t *b = src + (size_t)f * w * h;
        const int ym = oct_reflect101(y - 1, h), yp = oct_reflect101(y + 1, h), xm = oct_reflect101(x - 1, w), xp = oct_reflect101(x + 1, w);
        const int a00 = b[(size_t)ym * w + xm], a01 = b[(size_t)ym * w + x], a02 = b[(size_t)ym * w + xp];
        const int a10 = b[(size_t)y * w + xm], a12 = b[(size_t)y * w + xp];
        const int a20 = b[(size_t)yp * w + xm], a21 = b[(size_t)yp * w + x], a22 = b[(size_t)yp * w + xp];
        dxo[p] = (int16_t)((a02 + 2 * a12 + a22) - (a00 + 2 * a10 + a20));
        dyo[p] = (int16_t)((a20 + 2 * a21 + a22) - (a00 + 2 * a01 + a02));
    }
}

inline unsigned grid_for(int64_t n) { return (unsigned)std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), CS_SM_COUNT * 32); }

/* device scratch of one call, returned to the stream-ordered pool when the call ends */
struct Scratch {
    void *p = nullptr;
    cudaStream_t st;
    explicit Scratch(cudaStream_t s) : st(s) {}
    ~Scratch()
    {
        if (p) cudaFreeAsync(p, st);
    }
};

/* octave sizes: octave k is octave k - 1 halved with integer division (Size(cols / scale, rows / scale), scale 2) */
void octave_sizes(int w, int h, int K, std::vector<int> &ow, std::vector<int> &oh)
{
    ow.assign((size_t)K, w);
    oh.assign((size_t)K, h);
    for (int k = 1; k < K; k++) {
        ow[k] = ow[k - 1] / 2;
        oh[k] = oh[k - 1] / 2;
    }
}

/* the descriptor's pyramid (BinaryDescriptor::computeSobel, binary_descriptor.cpp:352-398) of n_frames gray frames: the blurred frame, then
 * pyrDown per octave into blur (octave k of frame f at off[k] + f * ow[k] * oh[k]); the Sobel maps of octaves k0 .. K - 1 into dx / dy, octave
 * k at off[k] - off[k0].  2K - k0 launches. */
void descriptor_pyramid(cudaStream_t st, const uint8_t *gray, int F, const std::vector<int> &ow, const std::vector<int> &oh, const std::vector<size_t> &off,
                        int K, int k0, uint8_t *blur, int16_t *dx, int16_t *dy)
{
    k_oct_blur5<<<grid_for((int64_t)off[1]), 256, 0, st>>>(gray, F, ow[0], oh[0], blur);
    for (int k = 1; k < K; k++)
        k_oct_pyrdown<<<grid_for((int64_t)(off[k + 1] - off[k])), 256, 0, st>>>(blur + off[k - 1], F, ow[k - 1], oh[k - 1], blur + off[k], ow[k], oh[k]);
    for (int k = k0; k < K; k++)
        k_oct_sobel<<<grid_for((int64_t)(off[k + 1] - off[k])), 256, 0, st>>>(blur + off[k], F, ow[k], oh[k], dx + (off[k] - off[k0]), dy + (off[k] - off[k0]));
}

}  // namespace

void cs_launch_gray_tab(const uint8_t *d_img, const OctPlane *d_tab, int n, int64_t total, uint8_t *d_dst, cudaStream_t st, int64_t *launches)
{
    if (n <= 0 || total <= 0) return;
    k_oct_gray_tab<<<grid_for(total), 256, 0, st>>>(d_img, d_tab, n, total, d_dst);
    (*launches)++;
}

int cs_lsd_octaves_check(cs_ctx *c, int width, int height, const cs_line_params *params, const void *keylines, const void *desc32, bool describe,
                         int32_t max_lines_per_octave, const int32_t *n_lines, int frame)
{
    if (!params || !keylines || (describe && !desc32) || !n_lines || max_lines_per_octave <= 0)
        return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (!params->use_LSD)
        return cs_ctx_fail(c, CS_ERR_UNSUPPORTED, "the octave calls are provided for the LSD flavour (use_LSD = 1): EDLines groups its octaves differently");
    const int K = params->numoctaves;
    if (K < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1");
    /* the reference passes the float ratio to an int scale (line_lbd_allclass.cpp:140); cv::pyrDown takes only |2 * dst - src| <= 2 */
    if (K > 1 && !(params->octaveratio >= 2.0f && params->octaveratio < 3.0f))
        return cs_ctx_fail(c, CS_ERR_INVALID_ARG,
                           "numoctaves > 1 needs (int)octaveratio == 2 (got %g): cv::pyrDown makes an octave of (w / scale, h / scale) only when "
                           "|2 * dst - src| <= 2",
                           (double)params->octaveratio);
    std::vector<int> ow, oh;
    octave_sizes(width, height, K, ow, oh);
    if (std::lrint(ow[K - 1] * 0.8) < 2 || std::lrint(oh[K - 1] * 0.8) < 2 || width > 32767 || height > 32767) {
        if (frame >= 0)
            return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: octave %d of a %d x %d frame is %d x %d: too small for LSD", frame, K - 1, width, height,
                               ow[K - 1], oh[K - 1]);
        return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "octave %d of a %d x %d frame is %d x %d: too small for LSD", K - 1, width, height, ow[K - 1], oh[K - 1]);
    }
    return CS_OK;
}

/* the octave calls' body on frames of any sizes on the device, frame f at d_imgs + views[f].offset.  The gray pyramids of every frame, level
 * after level (K launches); then ONE LSD run over the F x K planes, and the key lines filled on the host from one copy of the raw segments.
 * describe: frames of one size only (the descriptor's pyramid, descriptor_pyramid, is laid out for one size). */
int cs_lsd_octaves_run_views(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params, bool describe,
                             cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines)
{
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    const int F = n_frames, K = params->numoctaves, cap = max_lines_per_octave;
    if ((int64_t)F * K > CS_LSD_MAX_MIXED_FRAMES) /* before anything is enqueued: LSD runs the F x K planes as one batch */
        return cs_ctx_fail(c, CS_ERR_CAPACITY, "%d frames x %d octaves: more than the %d planes one LSD run takes", F, K, CS_LSD_MAX_MIXED_FRAMES);
    /* plane (k, f): octave k of frame f, of size pw x ph, at pyr + poff; planes level after level, frame after frame -- for frames of one size,
     * octave k of frame f lies at off[k] + f * ow[k] * oh[k], the layout descriptor_pyramid reads */
    const size_t NP = (size_t)F * K;
    std::vector<int> pw(NP), ph(NP);
    std::vector<OctPlane> tab(NP);
    std::vector<cs_frame_view> planes(NP);
    std::vector<int64_t> level_px((size_t)K, 0);
    size_t total = 0;
    for (int k = 0; k < K; k++)
        for (int f = 0; f < F; f++) {
            const size_t q = (size_t)k * F + f, qa = q - F; /* qa: the plane above, octave k - 1 of the same frame */
            pw[q] = k ? pw[qa] / 2 : views[f].width;    /* Size(cols / scale, rows / scale), scale 2 */
            ph[q] = k ? ph[qa] / 2 : views[f].height;
            OctPlane &P = tab[q];
            memset(&P, 0, sizeof P);
            P.dst = (int64_t)total;
            P.dw = pw[q];
            P.dh = ph[q];
            P.px0 = level_px[k];
            if (k == 0) {
                P.src = views[f].offset;
                P.sw = views[f].width;
                P.sh = views[f].height;
                P.sstride = views[f].stride;
                P.ch = views[f].channels;
            } else {
                P.src = tab[qa].dst;
                P.sw = pw[qa];
                P.sh = ph[qa];
                P.sstride = pw[qa];
                P.ch = 1;
            }
            planes[q].offset = (int64_t)total;
            planes[q].width = planes[q].stride = pw[q];
            planes[q].height = ph[q];
            planes[q].channels = 1;
            level_px[k] += (int64_t)pw[q] * ph[q];
            total += (size_t)pw[q] * ph[q];
        }

    /* the LSD pyramids, in the LSD detector's frame buffer (LSD reads its planes from there); their table in scratch until the call ends */
    uint8_t *pyr = cs_lsd_frame_buffer(c, total);
    if (!pyr) return CS_ERR_CUDA;
    Scratch d_tab(st);
    if (cudaMallocAsync(&d_tab.p, NP * sizeof(OctPlane), st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMallocAsync(%zu) failed for the pyramid table", NP * sizeof(OctPlane));
    if (cudaMemcpyAsync(d_tab.p, tab.data(), NP * sizeof(OctPlane), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the pyramid table failed");
    const OctPlane *dt = (const OctPlane *)d_tab.p;
    k_oct_gray_tab<<<grid_for(level_px[0]), 256, 0, st>>>(d_imgs, dt, F, level_px[0], pyr);
    for (int k = 1; k < K; k++) k_oct_pyrdown_tab<<<grid_for(level_px[k]), 256, 0, st>>>(dt + (size_t)k * F, F, level_px[k], pyr);
    cs_ctx_count_launches(c, K);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "pyramid kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));

    /* LSD once over every plane; its raw segments to the host in one copy, then the KeyLine fill, octave after octave */
    const float *d_lines, *d_raw;
    const int32_t *d_counts, *d_nraw;
    int rc;
    if ((rc = cs_lsd_run_mixed_sync(c, pyr, planes.data(), (int)NP, params->line_length_thres, cap, &d_lines, &d_counts))) return rc;
    cs_lsd_raw_segments(c, &d_raw, &d_nraw);
    std::vector<float> raw(NP * cap * 4);
    std::vector<int32_t> nraw(NP);
    if (cudaMemcpyAsync(nraw.data(), d_nraw, NP * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(raw.data(), d_raw, raw.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "LSD segment copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    std::vector<cs_keyline_octave> all(NP * cap);
    std::vector<int32_t> cnt(NP, 0);
    for (int k = 0; k < K; k++) {
        const float scale = (float)(1 << k);
        for (int f = 0; f < F; f++) {
            const size_t q = (size_t)k * F + f;
            if (nraw[q] > cap)
                return cs_ctx_fail(c, CS_ERR_CAPACITY, "frame %d, octave %d: %d LSD segments exceed max_lines_per_octave = %d", f, k, nraw[q], cap);
            cs_keyline_octave *o = &all[((size_t)f * K + k) * cap];
            int n = 0;
            for (int i = 0; i < nraw[q]; i++)
                if (cs_keyline_from_lsd_octave(&raw[(q * cap + i) * 4], scale, pw[q], ph[q], views[f].width, views[f].height, k, n, o[n])) n++;
            cnt[(size_t)f * K + k] = n;
        }
    }
    if (!describe) {
        for (size_t s = 0; s < cnt.size(); s++) {
            n_lines[s] = cnt[s];
            if (cnt[s]) memcpy(keylines + s * cap, &all[s * cap], (size_t)cnt[s] * sizeof(cs_keyline_octave));
        }
        return CS_OK;
    }

    const int width = views[0].width, height = views[0].height;
    std::vector<int> ow, oh;
    octave_sizes(width, height, K, ow, oh);
    std::vector<size_t> off((size_t)K + 1, 0); /* plane k of every frame at off[k], frame f at off[k] + f * ow[k] * oh[k] */
    for (int k = 0; k < K; k++) off[k + 1] = off[k] + (size_t)F * ow[k] * oh[k];

    /* detect_descrip_lines_octaves' filter (:312-317): lineLength * (float)pow((float)octaveratio, octave) > line_length_thres */
    size_t n_kept = 0;
    std::vector<int32_t> kept_cnt(cnt.size(), 0);
    for (int f = 0; f < F; f++)
        for (int k = 0; k < K; k++) {
            const float octave_scale = (float)std::pow(params->octaveratio, k);
            const size_t s = (size_t)f * K + k;
            cs_keyline_octave *o = &all[s * cap];
            int n = 0;
            for (int i = 0; i < cnt[s]; i++)
                if (o[i].kl.line_length * octave_scale > params->line_length_thres) o[n++] = o[i];
            kept_cnt[s] = n;
            n_kept += n;
        }
    for (size_t s = 0; s < cnt.size(); s++) n_lines[s] = kept_cnt[s];
    if (n_kept) {
        /* the descriptor's pyramid: blurred octave 0, pyrDown per octave, Sobel of octaves >= 1 (octave 0's maps: cs_edl_sobel_maps) */
        Scratch tmp(st);
        const size_t hi = off[K] - off[1];
        if (cudaMallocAsync(&tmp.p, off[K] + hi * 4 + 16, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMallocAsync(%zu) failed for the descriptor pyramid", off[K] + hi * 4 + 16);
        uint8_t *blur = (uint8_t *)tmp.p;
        int16_t *sob = (int16_t *)(((uintptr_t)(blur + off[K]) + 15) & ~(uintptr_t)15); /* dx of octave k at 2 * (off[k] - off[1]), dy after all dx */
        descriptor_pyramid(st, pyr, F, ow, oh, off, K, 1, blur, sob, sob + hi);
        cs_ctx_count_launches(c, 2 * K - 1);
        if (cudaGetLastError() != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "descriptor pyramid kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        std::vector<cs_keyline> lines;
        std::vector<int32_t> frame;
        std::vector<uint8_t> packed;
        for (int k = 0; k < K; k++) {
            lines.clear();
            frame.clear();
            for (int f = 0; f < F; f++) {
                const size_t s = (size_t)f * K + k;
                for (int i = 0; i < kept_cnt[s]; i++) {
                    const cs_keyline_octave &o = all[s * cap + i];
                    cs_keyline kl = o.kl; /* computeLBD reads the in-octave ends, numOfPixels and angle (binary_descriptor.cpp:1207-1250) */
                    kl.start_x = o.s_oct_x;
                    kl.start_y = o.s_oct_y;
                    kl.end_x = o.e_oct_x;
                    kl.end_y = o.e_oct_y;
                    lines.push_back(kl);
                    frame.push_back(f);
                }
            }
            if (lines.empty()) continue;
            const int16_t *d_dx, *d_dy;
            int rc;
            if (k == 0) {
                if ((rc = cs_edl_sobel_maps(c, pyr, true, F, width, height, width, 1, &d_dx, &d_dy))) return rc;
            } else {
                d_dx = sob + (off[k] - off[1]);
                d_dy = sob + hi + (off[k] - off[1]);
            }
            packed.resize(lines.size() * 32);
            if ((rc = cs_lbd_describe_keylines(c, lines.data(), frame.data(), (int)lines.size(), d_dx, d_dy, ow[k], oh[k], packed.data(), nullptr)))
                return rc;
            size_t row = 0;
            for (int f = 0; f < F; f++) {
                const size_t s = (size_t)f * K + k;
                if (kept_cnt[s]) memcpy(desc32 + s * cap * 32, &packed[row * 32], (size_t)kept_cnt[s] * 32);
                row += kept_cnt[s];
            }
        }
    }
    /* :319-330: start x <= end x (both pairs of ends swapped, the angle folded by normalize_to_PI in double), class_id within the octave */
    const double PI = 3.14159265; /* line_lbd_allclass.cpp:19 */
    for (size_t s = 0; s < cnt.size(); s++)
        for (int i = 0; i < kept_cnt[s]; i++) {
            cs_keyline_octave o = all[s * cap + i];
            if (o.kl.start_x > o.kl.end_x) {
                std::swap(o.kl.start_x, o.kl.end_x);
                std::swap(o.kl.start_y, o.kl.end_y);
                std::swap(o.s_oct_x, o.e_oct_x);
                std::swap(o.s_oct_y, o.e_oct_y);
                const float a = o.kl.angle;
                if (a > PI / 2)
                    o.kl.angle = (float)(a - PI);
                else if (a < -PI / 2)
                    o.kl.angle = (float)(a + PI);
            }
            o.kl.class_id = i;
            keylines[s * cap + i] = o;
        }
    return CS_OK;
}

int cs_lsd_octaves_run(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int width, int height, int stride, int channels, const cs_line_params *params,
                       bool describe, cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines)
{
    std::vector<cs_frame_view> views((size_t)n_frames);
    for (int f = 0; f < n_frames; f++) views[f] = cs_frame_view{(int64_t)f * height * stride, width, height, stride, channels};
    return cs_lsd_octaves_run_views(c, d_imgs, views.data(), n_frames, params, describe, keylines, desc32, max_lines_per_octave, n_lines);
}

/* ---- BinaryDescriptor::compute on key lines the caller gives, of any octave (cs_lbd_compute_octaves_batch[_device]) */
int cs_lbd_octaves_check_given(cs_ctx *c, int n_frames, int width, int height, const cs_keyline_octave *keylines, const int32_t *keyline_offsets,
                               const uint8_t *desc32, int *n)
{
    *n = 0;
    if (!keyline_offsets || keyline_offsets[0] != 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "keyline_offsets must start at 0");
    for (int f = 0; f < n_frames; f++)
        if (keyline_offsets[f + 1] < keyline_offsets[f]) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "keyline_offsets must not decrease");
    if (keyline_offsets[n_frames] == 0) return CS_OK; /* "Error: keypoint list is empty": descriptors left as they are (:618-622) */
    if (!keylines || !desc32) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null key lines or output");
    /* the deepest octave whose pyramid computeGaussianPyramid can build: pyrDown refuses a level of width or height 0 */
    int deepest = 0;
    for (int w = width, h = height; w / 2 > 0 && h / 2 > 0; w /= 2, h /= 2) deepest++;
    for (int f = 0; f < n_frames; f++)
        for (int i = keyline_offsets[f]; i < keyline_offsets[f + 1]; i++) {
            const cs_keyline_octave &o = keylines[i];
            if (o.kl.class_id < 0 || o.octave < 0)
                return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d, row %d: class_id %d and octave %d must not be negative", f, i - keyline_offsets[f],
                                   o.kl.class_id, o.octave);
            if (o.octave > deepest)
                return cs_ctx_fail(c, CS_ERR_INVALID_ARG,
                                   "frame %d, row %d: octave %d is beyond the pyramid of a %d x %d frame, whose octave %d is %d x %d: pyrDown cannot "
                                   "make an octave of width or height 0",
                                   f, i - keyline_offsets[f], o.octave, width, height, deepest, width >> deepest, height >> deepest);
        }
    *n = keyline_offsets[n_frames];
    return CS_OK;
}

int cs_lbd_compute_octaves_run(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int width, int height, int stride, int channels,
                               const cs_keyline_octave *keylines, const int32_t *keyline_offsets, uint8_t *desc32, float *desc72)
{
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    const int F = n_frames, n = keyline_offsets[F];
    /* one pyramid as deep as the deepest frame's: the levels a frame does not read do not change its bytes */
    int K = 0;
    for (int i = 0; i < n; i++) K = std::max(K, keylines[i].octave + 1);
    std::vector<int> ow, oh;
    octave_sizes(width, height, K, ow, oh);
    std::vector<size_t> off((size_t)K + 1, 0);
    for (int k = 0; k < K; k++) off[k + 1] = off[k] + (size_t)F * ow[k] * oh[k];

    /* gray frames, the blurred pyramid, and the Sobel maps of every octave (computeSobel(image, max octave + 1), :632-633) */
    Scratch tmp(st);
    const size_t bytes = off[1] + off[K] + 16 + off[K] * 4;
    if (cudaMallocAsync(&tmp.p, bytes, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMallocAsync(%zu) failed for the descriptor pyramid", bytes);
    uint8_t *gray = (uint8_t *)tmp.p, *blur = gray + off[1];
    int16_t *dx = (int16_t *)(((uintptr_t)(blur + off[K]) + 15) & ~(uintptr_t)15), *dy = dx + off[K];
    k_oct_gray<<<grid_for((int64_t)off[1]), 256, 0, st>>>(d_imgs, F, width, height, stride, channels, gray);
    descriptor_pyramid(st, gray, F, ow, oh, off, K, 0, blur, dx, dy);
    cs_ctx_count_launches(c, 2 * K + 1);
    if (cudaGetLastError() != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "descriptor pyramid kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));

    /* computeLBD per key line on its octave's maps at its in-octave ends (:1207-1250); one launch per octave over every frame */
    std::vector<cs_keyline> lines;
    std::vector<int32_t> frame, row;
    std::vector<uint8_t> packed;
    std::vector<float> fpacked;
    for (int k = 0; k < K; k++) {
        lines.clear();
        frame.clear();
        row.clear();
        for (int f = 0; f < F; f++)
            for (int i = keyline_offsets[f]; i < keyline_offsets[f + 1]; i++) {
                const cs_keyline_octave &o = keylines[i];
                if (o.octave != k) continue;
                cs_keyline kl = o.kl;
                kl.start_x = o.s_oct_x;
                kl.start_y = o.s_oct_y;
                kl.end_x = o.e_oct_x;
                kl.end_y = o.e_oct_y;
                lines.push_back(kl);
                frame.push_back(f);
                row.push_back(i);
            }
        if (lines.empty()) continue;
        packed.resize(lines.size() * CS_LBD_BYTES);
        if (desc72) fpacked.resize(lines.size() * CS_LBD_DESC);
        int rc;
        if ((rc = cs_lbd_describe_keylines(c, lines.data(), frame.data(), (int)lines.size(), dx + (off[k] - off[0]), dy + (off[k] - off[0]), ow[k], oh[k],
                                           packed.data(), desc72 ? fpacked.data() : nullptr)))
            return rc;
        for (size_t j = 0; j < row.size(); j++) {
            memcpy(desc32 + (size_t)row[j] * CS_LBD_BYTES, &packed[j * CS_LBD_BYTES], CS_LBD_BYTES);
            if (desc72) memcpy(desc72 + (size_t)row[j] * CS_LBD_DESC, &fpacked[j * CS_LBD_DESC], CS_LBD_DESC * sizeof(float));
        }
    }

    /* the output map (:655-693, :750-788): the row of a (class_id, octave) pair is the first row that has it, and the rows of the pair are
     * written there in list order, so it ends with the last one's descriptor; the other rows of the pair keep their own */
    std::unordered_map<uint64_t, std::pair<int, int>> first_last;
    for (int f = 0; f < F; f++) {
        first_last.clear();
        for (int i = keyline_offsets[f]; i < keyline_offsets[f + 1]; i++) {
            const uint64_t key = ((uint64_t)(uint32_t)keylines[i].kl.class_id << 32) | (uint32_t)keylines[i].octave;
            auto it = first_last.emplace(key, std::make_pair(i, i)).first;
            it->second.second = i;
        }
        for (const auto &e : first_last) {
            const int first = e.second.first, last = e.second.second;
            if (first == last) continue;
            memcpy(desc32 + (size_t)first * CS_LBD_BYTES, desc32 + (size_t)last * CS_LBD_BYTES, CS_LBD_BYTES);
            if (desc72) memcpy(desc72 + (size_t)first * CS_LBD_DESC, desc72 + (size_t)last * CS_LBD_DESC, CS_LBD_DESC * sizeof(float));
        }
    }
    return CS_OK;
}

namespace {

int octaves_host(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const cs_line_params *params,
                 bool describe, cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!imgs || n_frames <= 0 || width <= 0 || height <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3");
    if (stride < width * channels) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    int rc;
    if ((rc = cs_lsd_octaves_check(c, width, height, params, keylines, desc32, describe, max_lines_per_octave, n_lines))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const size_t bytes = (size_t)n_frames * height * stride;
    uint8_t *buf = cs_edl_frame_buffer(c, bytes);
    if (!buf) return CS_ERR_CUDA;
    if (cudaMemcpyAsync(buf, imgs, bytes, cudaMemcpyHostToDevice, cs_ctx_stream(c)) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames failed");
    return cs_lsd_octaves_run(c, buf, n_frames, width, height, stride, channels, params, describe, keylines, desc32, max_lines_per_octave, n_lines);
}

}  // namespace

extern "C" {

int cs_detect_raw_lines_octaves_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                      const cs_line_params *params, cs_keyline_octave *keylines, int32_t max_lines_per_octave, int32_t *n_lines)
{
    return octaves_host(c, imgs, n_frames, width, height, stride, channels, params, false, keylines, nullptr, max_lines_per_octave, n_lines);
}

int cs_detect_descrip_lines_octaves_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                          const cs_line_params *params, cs_keyline_octave *keylines, uint8_t *desc32, int32_t max_lines_per_octave,
                                          int32_t *n_lines)
{
    return octaves_host(c, imgs, n_frames, width, height, stride, channels, params, true, keylines, desc32, max_lines_per_octave, n_lines);
}

int cs_detect_raw_lines_octaves_batch_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params,
                                            cs_keyline_octave *keylines, int32_t max_lines_per_octave, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc;
    if ((rc = cs_check_frame_views(c, imgs, views, n_frames))) return rc;
    for (int f = 0; f < n_frames; f++)
        if ((rc = cs_lsd_octaves_check(c, views[f].width, views[f].height, params, keylines, nullptr, false, max_lines_per_octave, n_lines, f))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    /* the frames go to the EDLines buffer: the LSD buffer takes the pyramids */
    uint8_t *buf = cs_edl_frame_buffer(c, cs_packed_frames_bytes(views, n_frames));
    if (!buf) return CS_ERR_CUDA;
    std::vector<cs_frame_view> packed;
    if ((rc = cs_pack_host_frames(c, buf, imgs, views, n_frames, packed))) return rc;
    return cs_lsd_octaves_run_views(c, buf, packed.data(), n_frames, params, false, keylines, nullptr, max_lines_per_octave, n_lines);
}

int cs_lbd_compute_octaves_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                 const cs_keyline_octave *keylines, const int32_t *keyline_offsets, uint8_t *desc32, float *desc72)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!imgs || n_frames <= 0 || width <= 0 || height <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3");
    if (stride < width * channels) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    int rc, n = 0;
    if ((rc = cs_lbd_octaves_check_given(c, n_frames, width, height, keylines, keyline_offsets, desc32, &n)) || n == 0) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const size_t bytes = (size_t)n_frames * height * stride;
    uint8_t *buf = cs_edl_frame_buffer(c, bytes);
    if (!buf) return CS_ERR_CUDA;
    if (cudaMemcpyAsync(buf, imgs, bytes, cudaMemcpyHostToDevice, cs_ctx_stream(c)) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames failed");
    return cs_lbd_compute_octaves_run(c, buf, n_frames, width, height, stride, channels, keylines, keyline_offsets, desc32, desc72);
}

}  // extern "C"
