/*
 * cs_edlines.cu -- line_lbd_detect::detect_filter_lines, EDLines flavour (use_LSD = false, the class default), for sm_90a.
 *
 * Replaces, for one octave:
 *   BinaryDescriptor::detectImpl / OctaveKeyLines      line_lbd/libs/binary_descriptor.cpp:483-585,792-886,1060-1141
 *   EDLineDetector::EdgeDrawing                        line_lbd/libs/binary_descriptor.cpp:1579-2377
 *   EDLineDetector::EDline / LeastSquaresLineFit_ / LineValidation_      :2379-2870
 *   nfa / log_gamma                                    line_lbd/include/line_lbd/line_descriptor/descriptor.hpp:680-830
 *
 * Streaming stages (thread per pixel, integer-exact):
 *   k_ed_hblur / k_ed_vblur   cvtColor + cv::GaussianBlur(8U, 5x5, sigma 1) == fixed-point kernel (14,62,104,62,14)/256, one final rounding
 *   k_ed_maps                 Sobel 3x3 (REFLECT_101), |dx|+|dy| thresholded at 81 then /4 (round half to even), direction map
 *   k_ed_anchors              anchors in the reference's column-major scan order (x outer, y inner, stride 2) by an ordered block compaction
 * Sequential stage:
 *   k_ed_route_fit            smart routing of the anchors in order (each chain claims pixels first come, first served), chain assembly,
 *                             least-squares line fitting with extension, NFA validation: one warp per frame, lane 0 walks (the walk is a
 *                             pointer chase through the gradient map; order defines the result).  Frames run in parallel.
 */
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "cs_internal.h"
#include "cs_nfa.cuh"
#include "cs_tma.cuh"

#define ED_PI 3.14159265358979323846
#define ED_LN10 2.30258509299404568402
#define ED_HORIZONTAL 255
#define ED_UP 1
#define ED_RIGHT 2
#define ED_DOWN 3
#define ED_LEFT 4
#define ED_TRYTIME 6
#define ED_SKIP 2
#define ED_MINLEN 15
#define ED_FITERR 1.6

namespace {

__device__ __forceinline__ int ed_reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = (p < 0) ? -p : 2 * n - 2 - p;
    return p;
}

__global__ void __launch_bounds__(256) k_ed_hblur(const uint8_t *__restrict__ img, int n_frames, int w, int h, int stride, int channels,
                                                  uint16_t *__restrict__ tmp)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint8_t *row = img + ((size_t)f * h + y) * stride;
        const int k[5] = {14, 62, 104, 62, 14};
        uint32_t s = 0;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            const int xx = ed_reflect101(x + i - 2, w);
            uint32_t g;
            if (channels == 3) {
                const uint8_t *q = row + 3 * xx;
                g = (q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15;
            } else
                g = row[xx];
            s += k[i] * g;
        }
        tmp[p] = (uint16_t)s; /* <= 255 * 256 */
    }
}

__global__ void __launch_bounds__(256) k_ed_vblur(const uint16_t *__restrict__ tmp, int n_frames, int w, int h, uint8_t *__restrict__ blur)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint16_t *base = tmp + (size_t)f * w * h;
        const int k[5] = {14, 62, 104, 62, 14};
        uint32_t s = 0;
#pragma unroll
        for (int j = 0; j < 5; j++) s += k[j] * (uint32_t)base[(size_t)ed_reflect101(y + j - 2, h) * w + x];
        blur[p] = (uint8_t)((s + 32768u) >> 16);
    }
}

__global__ void __launch_bounds__(256) k_ed_maps(const uint8_t *__restrict__ blur, int n_frames, int w, int h, int16_t *__restrict__ dxo,
                                                 int16_t *__restrict__ dyo, int16_t *__restrict__ go, uint8_t *__restrict__ diro)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int r = (int)(p - f * (int64_t)w * h);
        const int y = r / w, x = r - y * w;
        const uint8_t *b = blur + (size_t)f * w * h;
        const int ym = ed_reflect101(y - 1, h), yp = ed_reflect101(y + 1, h), xm = ed_reflect101(x - 1, w), xp = ed_reflect101(x + 1, w);
        const int a00 = b[(size_t)ym * w + xm], a01 = b[(size_t)ym * w + x], a02 = b[(size_t)ym * w + xp];
        const int a10 = b[(size_t)y * w + xm], a12 = b[(size_t)y * w + xp];
        const int a20 = b[(size_t)yp * w + xm], a21 = b[(size_t)yp * w + x], a22 = b[(size_t)yp * w + xp];
        const int gx = (a02 + 2 * a12 + a22) - (a00 + 2 * a10 + a20);
        const int gy = (a20 + 2 * a21 + a22) - (a00 + 2 * a01 + a02);
        const int ax = abs(gx), ay = abs(gy), sum = ax + ay;
        const int s = (sum > 81) ? sum : 0; /* threshold(TOZERO, gradienThreshold_ + 1) */
        const int q = s >> 2, rr = s & 3;
        dxo[p] = (int16_t)gx;
        dyo[p] = (int16_t)gy;
        go[p] = (int16_t)(rr < 2 ? q : (rr == 3 ? q + 1 : q + (q & 1))); /* `mat / 4`: round half to even */
        diro[p] = (ax < ay) ? ED_HORIZONTAL : 0;
    }
}

/* cvtColor + GaussianBlur + Sobel + gradient / direction maps in one pass over 64 x 32 tiles (the three kernels above, fused: the frame is
 * read once, 3 bytes per pixel, and nothing intermediate goes to HBM).  Tiles work in virtual coordinates: position v outside the image
 * stands for pixel reflect101(v), which is what BORDER_REFLECT_101 means for the blur and, because the blur kernel is symmetric and the
 * sums are integers, also for the Sobel taps on the blurred image. */
#define EDF_TW 64
#define EDF_TH 32
#define EDF_BOXW 240 /* 3 * (EDF_TW + 6) = 210 bytes of BGR + up to 15 of alignment slack (a TMA box starts at a multiple of 16 bytes), a multiple of 16 */
template <bool kTma>
__global__ void __launch_bounds__(256) k_ed_front(const __grid_constant__ CUtensorMap tmap, const uint8_t *__restrict__ img, int w, int h, int stride,
                                                  int channels, uint8_t *__restrict__ blur, int16_t *__restrict__ dxo, int16_t *__restrict__ dyo,
                                                  int16_t *__restrict__ go, uint8_t *__restrict__ diro, int32_t *__restrict__ err_flag)
{
    __shared__ uint8_t s_gray[EDF_TH + 6][EDF_TW + 8];
    __shared__ uint16_t s_h[EDF_TH + 6][EDF_TW + 4];
    __shared__ uint8_t s_blur[EDF_TH + 2][EDF_TW + 4];
    __shared__ __align__(128) uint8_t s_rgb[kTma ? (EDF_TH + 6) * EDF_BOXW : 16]; /* kTma: BGR bytes of an interior tile, fetched by the copy engine */
    __shared__ __align__(8) unsigned long long s_bar;
    const int f = blockIdx.z, x0 = blockIdx.x * EDF_TW, y0 = blockIdx.y * EDF_TH, tid = threadIdx.x;
    const uint8_t *frame = img + (size_t)f * h * stride;
    const bool interior = kTma && x0 - 3 >= 0 && x0 + EDF_TW + 3 <= w - 1 && y0 - 3 >= 0 && y0 + EDF_TH + 3 <= h - 1;
    if (interior) {
        if (tid == 0) cs_mbar_init(&s_bar);
        __syncthreads();
        const int bx = 3 * (x0 - 3), boff = bx & 15; /* the box starts at a multiple of 16 bytes */
        if (tid == 0) cs_tma_load_2d(&tmap, s_rgb, &s_bar, bx - boff, f * h + y0 - 3, (EDF_TH + 6) * EDF_BOXW);
        if (!cs_mbar_wait(&s_bar, 0) && tid == 0) atomicOr(err_flag, 8);
        for (int i = tid; i < (EDF_TH + 6) * (EDF_TW + 6); i += 256) {
            const int r = i / (EDF_TW + 6), c = i - r * (EDF_TW + 6);
            const uint8_t *q = &s_rgb[r * EDF_BOXW + boff + 3 * c];
            s_gray[r][c] = (uint8_t)((q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15);
        }
    } else
        /* gray, halo 3 */
        for (int i = tid; i < (EDF_TH + 6) * (EDF_TW + 6); i += 256) {
            const int r = i / (EDF_TW + 6), c = i - r * (EDF_TW + 6);
            const int yy = ed_reflect101(y0 - 3 + r, h), xx = ed_reflect101(x0 - 3 + c, w);
            const uint8_t *q = frame + (size_t)yy * stride;
            uint32_t g;
            if (channels == 3) {
                q += 3 * xx;
                g = (q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15;
            } else
                g = q[xx];
            s_gray[r][c] = (uint8_t)g;
        }
    __syncthreads();
    /* horizontal pass, columns -1 .. TW (halo 1), rows -3 .. TH + 2 */
    for (int i = tid; i < (EDF_TH + 6) * (EDF_TW + 2); i += 256) {
        const int r = i / (EDF_TW + 2), c = i - r * (EDF_TW + 2);
        const uint8_t *q = &s_gray[r][c]; /* virtual x = x0 - 1 + c, taps at -2 .. +2 -> gray columns c .. c + 4 */
        s_h[r][c] = (uint16_t)(14u * q[0] + 62u * q[1] + 104u * q[2] + 62u * q[3] + 14u * q[4]);
    }
    __syncthreads();
    /* vertical pass + the one rounding, rows -1 .. TH */
    for (int i = tid; i < (EDF_TH + 2) * (EDF_TW + 2); i += 256) {
        const int r = i / (EDF_TW + 2), c = i - r * (EDF_TW + 2);
        const uint32_t t = 14u * s_h[r][c] + 62u * s_h[r + 1][c] + 104u * s_h[r + 2][c] + 62u * s_h[r + 3][c] + 14u * s_h[r + 4][c];
        s_blur[r][c] = (uint8_t)((t + 32768u) >> 16);
    }
    __syncthreads();
    for (int i = tid; i < EDF_TH * EDF_TW; i += 256) {
        const int r = i / EDF_TW, c = i - r * EDF_TW;
        const int x = x0 + c, y = y0 + r;
        if (x >= w || y >= h) continue;
        const int a00 = s_blur[r][c], a01 = s_blur[r][c + 1], a02 = s_blur[r][c + 2];
        const int a10 = s_blur[r + 1][c], a11 = s_blur[r + 1][c + 1], a12 = s_blur[r + 1][c + 2];
        const int a20 = s_blur[r + 2][c], a21 = s_blur[r + 2][c + 1], a22 = s_blur[r + 2][c + 2];
        const int gx = (a02 + 2 * a12 + a22) - (a00 + 2 * a10 + a20);
        const int gy = (a20 + 2 * a21 + a22) - (a00 + 2 * a01 + a02);
        const int ax = abs(gx), ay = abs(gy), sum = ax + ay;
        const int sv = (sum > 81) ? sum : 0; /* threshold(TOZERO, gradienThreshold_ + 1) */
        const int q = sv >> 2, rr = sv & 3;
        const size_t p = ((size_t)f * h + y) * w + x;
        blur[p] = (uint8_t)a11;
        dxo[p] = (int16_t)gx;
        dyo[p] = (int16_t)gy;
        go[p] = (int16_t)(rr < 2 ? q : (rr == 3 ? q + 1 : q + (q & 1))); /* `mat / 4`: round half to even */
        diro[p] = (ax < ay) ? ED_HORIZONTAL : 0;
    }
}

/* Anchors (binary_descriptor.cpp:1640-1666: x = 1, 3, ... outer, y = 1, 3, ... inner) in two steps: k_ed_anchor_flags tests every candidate
 * and keeps, per candidate column, a bit per candidate row (rows across the bits of 32-bit words) and the column's count; k_ed_anchor_list
 * scans the column counts of a frame and lets one warp per column write its anchors in row order. */
__global__ void __launch_bounds__(256) k_ed_anchor_flags(const int16_t *__restrict__ g_all, const uint8_t *__restrict__ dir_all, int w, int h, int nw, int nh,
                                                         int nhw, uint32_t *__restrict__ abits, int32_t *__restrict__ colcnt)
{
    /* block: 32 candidate rows (one word) x 8 warps of 32 candidate columns; lane = column so that g is read along rows */
    __shared__ uint32_t s_t[8][32];
    const int f = blockIdx.z, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int wi = (blockIdx.x * 8 + wid) * 32 + lane; /* candidate column */
    const int hw = blockIdx.y;                        /* word of candidate rows */
    const int16_t *g = g_all + (size_t)f * w * h;
    const uint8_t *dir = dir_all + (size_t)f * w * h;
    uint32_t word = 0;
    for (int b = 0; b < 32; b++) {
        const int hi = hw * 32 + b;
        bool a = false;
        if (wi < nw && hi < nh) {
            const int idx = (1 + 2 * hi) * w + 1 + 2 * wi;
            const int gv = g[idx];
            if (dir[idx] == ED_HORIZONTAL)
                a = (gv >= g[idx - w] + 8) && (gv >= g[idx + w] + 8);
            else
                a = (gv >= g[idx - 1] + 8) && (gv >= g[idx + 1] + 8);
        }
        word |= a ? (1u << b) : 0u;
    }
    (void)s_t;
    if (wi < nw) {
        abits[((size_t)f * nw + wi) * nhw + hw] = word;
        if (word) atomicAdd(&colcnt[(size_t)f * (nw + 1) + wi], __popc(word));
    }
}

__global__ void __launch_bounds__(1024) k_ed_anchor_list(int w, int nw, int nhw, const uint32_t *__restrict__ abits, int32_t *__restrict__ colcnt,
                                                         int32_t *__restrict__ anchors_all, int32_t *__restrict__ n_anchors, int cap)
{
    __shared__ int s_w[32];
    __shared__ int s_base;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int32_t *cc = colcnt + (size_t)f * (nw + 1);
    int32_t *out = anchors_all + (size_t)f * cap;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int b = 0; b < nw; b += 1024) { /* exclusive scan of the column counts, in place */
        const int i = b + tid;
        const int v = i < nw ? cc[i] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        int off = s_base;
        for (int k = 0; k < wid; k++) off += s_w[k];
        if (i < nw) cc[i] = off + inc - v;
        __syncthreads();
        if (tid == 1023) s_base = off + inc;
        __syncthreads();
    }
    if (tid == 0) {
        cc[nw] = s_base;
        n_anchors[f] = s_base;
    }
    __syncthreads();
    /* one warp per column: lane = word of rows */
    for (int wi = wid; wi < nw; wi += 32) {
        int off = cc[wi];
        if (cc[wi + 1] == off) continue;
        const uint32_t *col = abits + ((size_t)f * nw + wi) * nhw;
        for (int w0 = 0; w0 < nhw; w0 += 32) {
            const uint32_t word = (w0 + lane < nhw) ? col[w0 + lane] : 0u;
            int inc = __popc(word);
            const int mine = inc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            int slot = off + inc - mine;
            uint32_t m = word;
            while (m) {
                const int b = __ffs(m) - 1;
                m &= m - 1;
                const int hi = (w0 + lane) * 32 + b;
                if (slot < cap) out[slot] = (1 + 2 * hi) * w + 1 + 2 * wi;
                slot++;
            }
            off += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
}

/* anchors, reference scan order: for w = 1, 3, ...: for h = 1, 3, ... (binary_descriptor.cpp:1640-1666) */
__global__ void __launch_bounds__(256) k_ed_anchors(const int16_t *__restrict__ g_all, const uint8_t *__restrict__ dir_all, int w, int h,
                                                    int32_t *__restrict__ anchors_all, int32_t *__restrict__ n_anchors, int cap)
{
    __shared__ int s_warp[8];
    __shared__ int s_total;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int16_t *g = g_all + (size_t)f * w * h;
    const uint8_t *dir = dir_all + (size_t)f * w * h;
    int32_t *out = anchors_all + (size_t)f * cap;
    const int nw = (w - 2 + 1) / 2, nh = (h - 2 + 1) / 2; /* w = 1,3,..,<= w-2 ; h likewise */
    if (tid == 0) s_total = 0;
    __syncthreads();
    const int total = nw * nh;
    for (int base = 0; base < total; base += 256) {
        const int i = base + tid;
        bool a = false;
        int idx = 0;
        if (i < total) {
            const int wi = i / nh, hi = i - wi * nh;
            const int x = 1 + 2 * wi, y = 1 + 2 * hi;
            idx = y * w + x;
            const int gv = g[idx];
            if (dir[idx] == ED_HORIZONTAL)
                a = (gv >= g[idx - w] + 8) && (gv >= g[idx + w] + 8);
            else
                a = (gv >= g[idx - 1] + 8) && (gv >= g[idx + 1] + 8);
        }
        const unsigned m = __ballot_sync(0xffffffffu, a);
        if (lane == 0) s_warp[wid] = __popc(m);
        __syncthreads();
        int off = s_total;
        for (int k = 0; k < wid; k++) off += s_warp[k];
        if (a) {
            const int slot = off + __popc(m & ((1u << lane) - 1u));
            if (slot < cap) out[slot] = idx;
        }
        __syncthreads();
        if (tid == 0) {
            int t = s_total;
            for (int k = 0; k < 8; k++) t += s_warp[k];
            s_total = t;
        }
        __syncthreads();
    }
    if (tid == 0) n_anchors[f] = s_total;
}

/* ---------------------------------------------------------------------------------------- sequential stage */
struct EdFrame {
    int W, H;
    const int16_t *dx, *dy, *g;
    const uint8_t *dir;
    uint8_t *edge;
    float ATA[4], ATV[2];
    double logNT;
    const double *lgam; /* log_gamma of small integers (cs_nfa.cuh), or nullptr */
};

__device__ __forceinline__ uint32_t ed_pack(int x, int y) { return (uint32_t)x | ((uint32_t)y << 16); }
__device__ __forceinline__ int ed_x(uint32_t p) { return (int)(p & 0xffffu); }
__device__ __forceinline__ int ed_y(uint32_t p) { return (int)(p >> 16); }

/* one smart-routing walk; appends packed pixels to out[*n] */
__device__ void ed_walk(EdFrame &F, int x, int y, int lastDirection, uint32_t *out, unsigned &n, unsigned cap, int &lastX, int &lastY)
{
    const int W = F.W, H = F.H;
    int idx = y * W + x;
    while (F.g[idx] > 0 && !F.edge[idx]) {
        F.edge[idx] = 1;
        if (n < cap) out[n] = ed_pack(x, y);
        n++;
        int shouldGo = 0;
        if (F.dir[idx] == ED_HORIZONTAL) {
            if (lastDirection == ED_UP || lastDirection == ED_DOWN) shouldGo = (x > lastX) ? ED_RIGHT : ED_LEFT;
            lastX = x;
            lastY = y;
            if (lastDirection == ED_RIGHT || shouldGo == ED_RIGHT) {
                if (x == W - 1 || y == 0 || y == H - 1) break;
                const uint8_t g1 = (uint8_t)F.g[idx - W + 1], g2 = (uint8_t)F.g[idx + 1], g3 = (uint8_t)F.g[idx + W + 1];
                if (g1 >= g2 && g1 >= g3) {
                    x = x + 1;
                    y = y - 1;
                } else if (g3 >= g2 && g3 >= g1) {
                    x = x + 1;
                    y = y + 1;
                } else
                    x = x + 1;
                lastDirection = ED_RIGHT;
            } else if (lastDirection == ED_LEFT || shouldGo == ED_LEFT) {
                if (x == 0 || y == 0 || y == H - 1) break;
                const uint8_t g1 = (uint8_t)F.g[idx - W - 1], g2 = (uint8_t)F.g[idx - 1], g3 = (uint8_t)F.g[idx + W - 1];
                if (g1 >= g2 && g1 >= g3) {
                    x = x - 1;
                    y = y - 1;
                } else if (g3 >= g2 && g3 >= g1) {
                    x = x - 1;
                    y = y + 1;
                } else
                    x = x - 1;
                lastDirection = ED_LEFT;
            }
        } else {
            if (lastDirection == ED_RIGHT || lastDirection == ED_LEFT) shouldGo = (y > lastY) ? ED_DOWN : ED_UP;
            lastX = x;
            lastY = y;
            if (lastDirection == ED_DOWN || shouldGo == ED_DOWN) {
                if (x == 0 || x == W - 1 || y == H - 1) break;
                const uint8_t g1 = (uint8_t)F.g[idx + W + 1], g2 = (uint8_t)F.g[idx + W], g3 = (uint8_t)F.g[idx + W - 1];
                if (g1 >= g2 && g1 >= g3) {
                    x = x + 1;
                    y = y + 1;
                } else if (g3 >= g2 && g3 >= g1) {
                    x = x - 1;
                    y = y + 1;
                } else
                    y = y + 1;
                lastDirection = ED_DOWN;
            } else if (lastDirection == ED_UP || shouldGo == ED_UP) {
                if (x == 0 || x == W - 1 || y == 0) break;
                const uint8_t g1 = (uint8_t)F.g[idx - W + 1], g2 = (uint8_t)F.g[idx - W], g3 = (uint8_t)F.g[idx - W - 1];
                if (g1 >= g2 && g1 >= g3) {
                    x = x + 1;
                    y = y - 1;
                } else if (g3 >= g2 && g3 >= g1) {
                    x = x - 1;
                    y = y - 1;
                } else
                    y = y - 1;
                lastDirection = ED_UP;
            }
        }
        idx = y * W + x;
    }
}

__device__ __forceinline__ bool ed_double_equal(double a, double b)
{
    if (a == b) return true;
    const double abs_diff = fabs(a - b);
    const double aa = fabs(a), bb = fabs(b);
    double abs_max = (aa > bb) ? aa : bb;
    if (abs_max < DBL_MIN) abs_max = DBL_MIN;
    return (abs_diff / abs_max) <= (100.0 * DBL_EPSILON);
}
__device__ double ed_log_gamma(double x)
{
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
    double b = 0.0;
    for (int n = 0; n < 7; n++) {
        a -= log(x + (double)n);
        b += q[n] * pow(x, (double)n);
    }
    return a + log(b);
}
__device__ double ed_nfa(int n, int k, double p, double logNT)
{
    const double tolerance = 0.1;
    if (n == 0 || k == 0) return -logNT;
    if (n == k) return -logNT - (double)n * log10(p);
    const double p_term = p / (1.0 - p);
    const double log1term = ed_log_gamma((double)n + 1.0) - ed_log_gamma((double)k + 1.0) - ed_log_gamma((double)(n - k) + 1.0) + (double)k * log(p) +
                            (double)(n - k) * log(1.0 - p);
    double term = exp(log1term);
    if (ed_double_equal(term, 0.0)) {
        if ((double)k > (double)n * p) return -log1term / ED_LN10 - logNT;
        return -logNT;
    }
    double bin_tail = term;
    for (int i = k + 1; i <= n; i++) {
        const double bin_term = (double)(n - i + 1) / (double)i;
        const double mult_term = bin_term * p_term;
        term *= mult_term;
        bin_tail += term;
        if (bin_term < 1.0) {
            const double err = term * ((1.0 - pow(mult_term, (double)(n - i + 1))) / (1.0 - mult_term) - 1.0);
            if (err < tolerance * fabs(-log10(bin_tail) - logNT) * bin_tail) break;
        }
    }
    return -log10(bin_tail) - logNT;
}

/* LeastSquaresLineFit_, first overload (:2628-2714).  Sums of products of small integers are exact in double; OpenCV's float gemm
 * accumulates in double and rounds once to float. */
__device__ double ed_fit_initial(EdFrame &F, const uint32_t *pts, unsigned offsetS, double *eq)
{
    const bool horiz = F.dir[ed_y(pts[offsetS]) * F.W + ed_x(pts[offsetS])] == ED_HORIZONTAL;
    double suu = 0, su = 0, suv = 0, sv = 0;
    for (int i = 0; i < ED_MINLEN; i++) {
        const uint32_t p = pts[offsetS + i];
        const double u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
        suu += u * u;
        su += u;
        suv += u * v;
        sv += v;
    }
    F.ATA[0] = (float)suu;
    F.ATA[1] = (float)su;
    F.ATA[2] = (float)su;
    F.ATA[3] = (float)(double)ED_MINLEN;
    F.ATV[0] = (float)suv;
    F.ATV[1] = (float)sv;
    const double coef = 1.0 / ((double)F.ATA[0] * (double)F.ATA[3] - (double)F.ATA[1] * (double)F.ATA[2]);
    eq[0] = coef * ((double)F.ATA[3] * (double)F.ATV[0] - (double)F.ATA[1] * (double)F.ATV[1]);
    eq[1] = coef * ((double)F.ATA[0] * (double)F.ATV[1] - (double)F.ATA[2] * (double)F.ATV[0]);
    double fitError = 0;
    for (int i = 0; i < ED_MINLEN; i++) {
        const uint32_t p = pts[offsetS + i];
        const double u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
        const double c = v - u * eq[0] - eq[1];
        fitError += c * c;
    }
    return sqrt(fitError);
}

/* second overload (:2716-2787) */
__device__ void ed_fit_update(EdFrame &F, const uint32_t *pts, unsigned offsetS, unsigned newOffsetS, unsigned offsetE, double *eq)
{
    const int length = (int)offsetE - (int)offsetS, newLength = (int)offsetE - (int)newOffsetS;
    if (length <= 0 || newLength <= 0) return;
    const bool horiz = F.dir[ed_y(pts[offsetS]) * F.W + ed_x(pts[offsetS])] == ED_HORIZONTAL;
    double suu = 0, su = 0, suv = 0, sv = 0;
    for (unsigned i = newOffsetS; i < offsetE; i++) {
        const uint32_t p = pts[i];
        const double u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
        suu += u * u;
        su += u;
        suv += u * v;
        sv += v;
    }
    F.ATA[0] = F.ATA[0] + (float)suu;
    F.ATA[1] = F.ATA[1] + (float)su;
    F.ATA[2] = F.ATA[2] + (float)su;
    F.ATA[3] = F.ATA[3] + (float)(double)newLength;
    F.ATV[0] = F.ATV[0] + (float)suv;
    F.ATV[1] = F.ATV[1] + (float)sv;
    const double coef = 1.0 / ((double)F.ATA[0] * (double)F.ATA[3] - (double)F.ATA[1] * (double)F.ATA[2]);
    eq[0] = coef * ((double)F.ATA[3] * (double)F.ATV[0] - (double)F.ATA[1] * (double)F.ATV[1]);
    eq[1] = coef * ((double)F.ATA[0] * (double)F.ATV[1] - (double)F.ATA[2] * (double)F.ATV[0]);
}

/* LineValidation_ (:2789-2870) */
__device__ bool ed_validate(EdFrame &F, const uint32_t *pts, unsigned offsetS, unsigned offsetE, const double *lineEqu, float &direction)
{
    const int n = (int)offsetE - (int)offsetS;
    int meanGradientX = 0, meanGradientY = 0;
    for (int i = 0; i < n; i++) {
        const uint32_t p = pts[offsetS + i];
        const int index = ed_y(p) * F.W + ed_x(p);
        meanGradientX += F.dx[index];
        meanGradientY += F.dy[index];
    }
    const double ddx = fabs(lineEqu[1]), ddy = fabs(lineEqu[0]);
    if (meanGradientX == 0 && meanGradientY == 0) return false;
    if (meanGradientX > 0 && meanGradientY >= 0) direction = (float)atan2(-ddy, ddx);
    if (meanGradientX <= 0 && meanGradientY > 0) direction = (float)atan2(ddy, ddx);
    if (meanGradientX < 0 && meanGradientY <= 0) direction = (float)atan2(ddy, -ddx);
    if (meanGradientX >= 0 && meanGradientY < 0) direction = (float)atan2(-ddy, -ddx);
    if (fabs((double)direction) < 0.15 || ED_PI - fabs((double)direction) < 0.15) {
        if (fabs(lineEqu[2]) < 10 || fabs((double)F.H - fabs(lineEqu[2])) < 10) return false;
    }
    if (fabs(fabs((double)direction) - ED_PI * 0.5) < 0.15) {
        if (fabs(lineEqu[2]) < 10 || fabs((double)F.W - fabs(lineEqu[2])) < 10) return false;
    }
    int k = 0;
    for (int i = 0; i < n; i++) {
        const uint32_t p = pts[offsetS + i];
        const int index = ed_y(p) * F.W + ed_x(p);
        const double pd = atan2(-(double)F.dx[index], (double)F.dy[index]);
        const double dis = fabs((double)direction - pd);
        if (fabs(2 * ED_PI - dis) < 0.392699 || dis < 0.392699) k++;
    }
    return ed_nfa(n, k, 0.125, F.logNT) > 0;
}

/* routing + fitting for one frame by lane 0 of a warp */
__global__ void __launch_bounds__(32) k_ed_route_fit(int W, int H, const int16_t *__restrict__ dx_all, const int16_t *__restrict__ dy_all,
                                                     const int16_t *__restrict__ g_all, const uint8_t *__restrict__ dir_all,
                                                     uint8_t *__restrict__ edge_all, const int32_t *__restrict__ anchors_all,
                                                     const int32_t *__restrict__ n_anchors, int anchor_cap, uint32_t *__restrict__ scratch_all,
                                                     size_t scratch_per_frame, double logNT, float line_length_thres, float *__restrict__ raw_all,
                                                     int32_t *__restrict__ n_raw_all, float *__restrict__ out_all, int32_t *__restrict__ n_out_all,
                                                     int cap, int32_t *__restrict__ err_flag, const int32_t *__restrict__ redo,
                                                     float *__restrict__ klx_all /* optional: cap x {direction, numOfPixels} per frame */)
{
    if (threadIdx.x != 0) return;
    const int f = blockIdx.x;
    if (!redo[f]) return;
    const size_t npx = (size_t)W * H;
    EdFrame F;
    F.W = W;
    F.H = H;
    F.dx = dx_all + f * npx;
    F.dy = dy_all + f * npx;
    F.g = g_all + f * npx;
    F.dir = dir_all + f * npx;
    F.edge = edge_all + f * npx;
    F.logNT = logNT;
    F.lgam = nullptr;
    for (int i = 0; i < 4; i++) F.ATA[i] = 0;
    F.ATV[0] = F.ATV[1] = 0;
    const unsigned P = (unsigned)(npx / 5), maxEdges = P / 20;
    uint32_t *scratch = scratch_all + (size_t)f * scratch_per_frame;
    uint32_t *fP = scratch;                 /* first parts   [P]        */
    uint32_t *sP = fP + P;                  /* second parts  [P]        */
    uint32_t *fS = sP + P;                  /* [maxEdges + 2]           */
    uint32_t *sS = fS + maxEdges + 2;       /* [maxEdges + 2]           */
    uint32_t *chain = sS + maxEdges + 2;    /* assembled chains [2P]    */
    uint32_t *sId = chain + 2 * P;          /* [maxEdges + 2]           */
    uint32_t *lpt = sId + maxEdges + 2;     /* line pixels [2P]         */
    float *raw = raw_all + (size_t)f * cap * 4;
    float *out = out_all + (size_t)f * cap * 4;
    n_raw_all[f] = 0;
    n_out_all[f] = 0;

    const int32_t *anchors = anchors_all + (size_t)f * anchor_cap;
    const int na = n_anchors[f];
    if (na > anchor_cap || (unsigned)na > P) { /* reference: "anchor size is larger than its maximal size" -> no lines */
        if (na > anchor_cap) atomicOr(err_flag, 1);
        return;
    }
    unsigned nF = 0, nS = 0, nE = 0;
    int lastX = 0, lastY = 0;
    for (int i = 0; i < na; i++) {
        const int idx = anchors[i];
        if (F.edge[idx]) continue;
        const int y = idx / W, x = idx - y * W;
        const unsigned f0 = nF, s0 = nS;
        if (F.dir[idx] == ED_HORIZONTAL) {
            ed_walk(F, x, y, ED_RIGHT, fP, nF, P, lastX, lastY);
            F.edge[idx] = 0;
            ed_walk(F, x, y, ED_LEFT, sP, nS, P, lastX, lastY);
        } else {
            ed_walk(F, x, y, ED_DOWN, fP, nF, P, lastX, lastY);
            F.edge[idx] = 0;
            ed_walk(F, x, y, ED_UP, sP, nS, P, lastX, lastY);
        }
        if ((int)(nF - f0) + (int)(nS - s0) < ED_MINLEN + 1) {
            nF = f0;
            nS = s0;
        } else {
            if (nE <= maxEdges) {
                fS[nE] = f0;
                sS[nE] = s0;
            }
            nE++;
        }
    }
    if (nE > maxEdges || nF > P || nS > P) return; /* reference prints "Edge drawing Error" and detects nothing */
    fS[nE] = nF;
    sS[nE] = nS;
    /* chain assembly: first part reversed, then the second part without the anchor */
    unsigned nc = 0;
    for (unsigned e = 0; e < nE; e++) {
        sId[e] = nc;
        for (int t = (int)fS[e + 1] - 1; t >= (int)fS[e]; t--) chain[nc++] = fP[t];
        for (int t = (int)sS[e] + 1; t < (int)sS[e + 1]; t++) chain[nc++] = sP[t];
    }
    sId[nE] = nc;
    if (nE == 0) return;

    int n_raw = 0, n_out = 0;
    double lineFitErr = 0, eq[2] = {0, 0};
    unsigned offL = 0, newOffsetS = 0;
    float direction = 0;
    for (unsigned edgeID = 0; edgeID < nE; edgeID++) {
        unsigned S = sId[edgeID];
        const unsigned Eend = sId[edgeID + 1];
        while (Eend > S + ED_MINLEN) {
            while (Eend > S + ED_MINLEN) {
                lineFitErr = ed_fit_initial(F, chain, S, eq);
                if (lineFitErr <= ED_FITERR) break;
                S += ED_SKIP;
            }
            if (lineFitErr > ED_FITERR) break;
            const unsigned lineStart = offL;
            double coef1 = 0;
            bool bExtended = true, bFirstTry = true;
            int numOfOutlier, tryTimes = 0;
            const bool horiz = F.dir[ed_y(chain[S]) * W + ed_x(chain[S])] == ED_HORIZONTAL;
            while (bExtended) {
                tryTimes++;
                if (bFirstTry) {
                    bFirstTry = false;
                    for (int i = 0; i < ED_MINLEN; i++) lpt[offL++] = chain[S++];
                } else
                    ed_fit_update(F, lpt, lineStart, newOffsetS, offL, eq);
                coef1 = horiz ? 1 / sqrt(eq[0] * eq[0] + 1) : 1 / sqrt(1 + eq[0] * eq[0]);
                numOfOutlier = 0;
                newOffsetS = offL;
                while (Eend > S) {
                    const uint32_t p = chain[S];
                    const double d = horiz ? fabs(eq[0] * (double)ed_x(p) - (double)ed_y(p) + eq[1]) * coef1
                                           : fabs((double)ed_x(p) - eq[0] * (double)ed_y(p) - eq[1]) * coef1;
                    lpt[offL++] = p;
                    S++;
                    if (d > ED_FITERR) {
                        numOfOutlier++;
                        if (numOfOutlier > 3) break;
                    } else
                        numOfOutlier = 0;
                }
                offL -= numOfOutlier;
                S -= numOfOutlier;
                if (!(offL - newOffsetS > 0 && tryTimes < ED_TRYTIME)) bExtended = false;
            }
            double lineEqu[3];
            if (horiz) {
                lineEqu[0] = eq[0] * coef1;
                lineEqu[1] = -1 * coef1;
                lineEqu[2] = eq[1] * coef1;
            } else {
                lineEqu[0] = 1 * coef1;
                lineEqu[1] = -eq[0] * coef1;
                lineEqu[2] = -eq[1] * coef1;
            }
            if (ed_validate(F, lpt, lineStart, offL, lineEqu, direction)) {
                const double a1 = lineEqu[1] * lineEqu[1], a2 = lineEqu[0] * lineEqu[0], a3 = lineEqu[0] * lineEqu[1];
                const double a4 = lineEqu[2] * lineEqu[0], a5 = lineEqu[2] * lineEqu[1];
                unsigned Px = ed_x(lpt[lineStart]), Py = ed_y(lpt[lineStart]);
                const float s1 = (float)(a1 * Px - a3 * Py - a4), s2 = (float)(a2 * Py - a3 * Px - a5);
                Px = ed_x(lpt[offL - 1]);
                Py = ed_y(lpt[offL - 1]);
                const float e1 = (float)(a1 * Px - a3 * Py - a4), e2 = (float)(a2 * Py - a3 * Px - a5);
                /* OctaveKeyLines: length and start / end ordering (:862-886,1069-1139) */
                float fdx = fabsf(s1 - e1), fdy = fabsf(s2 - e2);
                const float lineLength = sqrtf(fdx * fdx + fdy * fdy);
                fdx = e1 - s1;
                fdy = e2 - s2;
                bool sw = false;
                const double dr = (double)direction;
                if (dr >= -0.75 * ED_PI && dr < -0.25 * ED_PI && fdy > 0) sw = true;
                if (dr >= -0.25 * ED_PI && dr < 0.25 * ED_PI && fdx < 0) sw = true;
                if (dr >= 0.25 * ED_PI && dr < 0.75 * ED_PI && fdy < 0) sw = true;
                if (((dr >= 0.75 * ED_PI && dr < ED_PI) || (dr >= -ED_PI && dr < -0.75 * ED_PI)) && fdx > 0) sw = true;
                const float sx = sw ? e1 : s1, sy = sw ? e2 : s2, ex = sw ? s1 : e1, ey = sw ? s2 : e2;
                if (n_raw < cap) {
                    raw[4 * n_raw + 0] = sx;
                    raw[4 * n_raw + 1] = sy;
                    raw[4 * n_raw + 2] = ex;
                    raw[4 * n_raw + 3] = ey;
                }
                n_raw++;
                if (lineLength > line_length_thres) {
                    if (n_out < cap) {
                        out[4 * n_out + 0] = sx;
                        out[4 * n_out + 1] = sy;
                        out[4 * n_out + 2] = ex;
                        out[4 * n_out + 3] = ey;
                        if (klx_all) { /* KeyLine::angle = lineDirection_, KeyLine::numOfPixels = the fitted line's pixels (:1073-1077) */
                            float *kx = klx_all + ((size_t)f * cap + n_out) * 2;
                            kx[0] = direction;
                            kx[1] = __int_as_float((int)(offL - lineStart));
                        }
                    }
                    n_out++;
                }
            } else
                offL = lineStart;
        }
    }
    n_raw_all[f] = n_raw;
    n_out_all[f] = n_out;
}

/* ---------------------------------------------------------------------------------------- the same, restructured for the GPU
 *
 * Smart routing is a pointer chase: which pixel a walk visits next depends only on the gradient map (never on other walks), other
 * walks only decide where it STOPS (first pixel that is already an edge pixel).  So the walk graph is built once, in parallel:
 *   k_ed_rowcount / k_ed_rowscan / k_ed_nodes   pixels with g > 0 become nodes, numbered in raster order (ordered compaction)
 *   k_ed_next                                   per node the two moves its direction class allows (0: right / down, 1: left / up, for a
 *                                               horizontal-edge resp. vertical-edge pixel): the chosen neighbour's node id, or TERM when
 *                                               the walk would leave the image or step on a pixel with g = 0, plus one bit: which of
 *                                               the TARGET's two moves the walk takes next (lastDirection / shouldGo resolved here)
 *   k_ed_route                                  one CTA per frame copies the graph into shared memory (4 bytes + 2 bits per node) and
 *                                               ONE thread replays the anchors in order; a step is one shared-memory load, not a
 *                                               handful of dependent L2 gathers.  Frames whose graph does not fit walk it in HBM.
 *   k_ed_fit                                    chains are independent of each other: one warp per chain assembles it (first part
 *                                               reversed + second part) and runs the fit / extension / validation loop with the
 *                                               lanes trying start offsets, testing 32 chain points per step and counting aligned
 *                                               gradient directions in parallel; every floating-point sum keeps the reference order
 *                                               (the integer-valued sums of the normal equations are exact in any order)
 *   k_ed_emit                                   segments in chain order (ordered compaction)
 */
#define ED_TERM 0x3fffffffu
#define ED_PLUS 0x40000000u
#define ED_SM_TERM 0x7fffu
#define ED_SM_ANCHORS 8192 /* anchor node ids k_ed_route keeps in shared memory (16 bits each) */

__global__ void __launch_bounds__(256) k_ed_rowcount(const int16_t *__restrict__ g_all, int w, int h, int n_frames, int32_t *__restrict__ rowcnt)
{
    /* one warp per (frame, row) */
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int f = warp / h, y = warp - f * h;
    if (f >= n_frames) return;
    const int16_t *row = g_all + ((size_t)f * h + y) * w;
    int n = 0;
    for (int x = lane; x < w; x += 32) n += row[x] > 0 ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (lane == 0) rowcnt[(size_t)f * (h + 1) + y] = n;
}

/* exclusive scan of the row counts of one frame, in place; rowcnt[f][h] = number of nodes */
__global__ void __launch_bounds__(1024) k_ed_rowscan(int h, int32_t *__restrict__ rowcnt)
{
    __shared__ int s_w[32];
    __shared__ int s_base;
    int32_t *rc = rowcnt + (size_t)blockIdx.x * (h + 1);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int b = 0; b < h; b += 1024) {
        const int i = b + tid;
        const int v = i < h ? rc[i] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        int off = s_base;
        for (int k = 0; k < wid; k++) off += s_w[k];
        if (i < h) rc[i] = off + inc - v;
        __syncthreads();
        if (tid == 1023) s_base = off + inc;
        __syncthreads();
    }
    if (tid == 0) rc[h] = s_base;
}

/* node ids in raster order: pid[pixel] (only pixels with g > 0 are ever looked up), packed coordinates and the direction class per node */
__global__ void __launch_bounds__(256) k_ed_nodes(const int16_t *__restrict__ g_all, const uint8_t *__restrict__ dir_all, int w, int h, int n_frames,
                                                  const int32_t *__restrict__ rowoff, uint32_t *__restrict__ pid_all, uint32_t *__restrict__ xy_all,
                                                  uint8_t *__restrict__ flags_all, size_t node_cap)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int f = warp / h, y = warp - f * h;
    if (f >= n_frames) return;
    const size_t rowbase = ((size_t)f * h + y) * w;
    int base = rowoff[(size_t)f * (h + 1) + y];
    for (int x0 = 0; x0 < w; x0 += 32) {
        const int x = x0 + lane;
        const bool on = x < w && g_all[rowbase + x] > 0;
        const unsigned m = __ballot_sync(0xffffffffu, on);
        if (on) {
            const int id = base + __popc(m & ((1u << lane) - 1u));
            pid_all[rowbase + x] = (uint32_t)id;
            if ((size_t)id < node_cap) {
                xy_all[(size_t)f * node_cap + id] = ed_pack(x, y);
                flags_all[(size_t)f * node_cap + id] = dir_all[rowbase + x] == ED_HORIZONTAL ? 1 : 0;
            }
        }
        base += __popc(m);
    }
}

/* the two moves of every node (EdgeDrawing's neighbour choice, binary_descriptor.cpp:1713-1862) and the node id of every anchor */
__global__ void __launch_bounds__(256) k_ed_next(const int16_t *__restrict__ g_all, int w, int h, int n_frames, const int32_t *__restrict__ rowoff,
                                                 const uint32_t *__restrict__ pid_all, const uint32_t *__restrict__ xy_all,
                                                 const uint8_t *__restrict__ flags_all, size_t node_cap, uint2 *__restrict__ next_all,
                                                 const int32_t *__restrict__ anchors_all, const int32_t *__restrict__ n_anchors, int anchor_cap,
                                                 uint32_t *__restrict__ anchor_nid)
{
    const int f = blockIdx.y;
    const size_t npx = (size_t)w * h;
    const int16_t *g = g_all + f * npx;
    const uint32_t *pid = pid_all + f * npx;
    const int n = min(rowoff[(size_t)f * (h + 1) + h], (int)node_cap);
    for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
        const uint32_t p = xy_all[(size_t)f * node_cap + id];
        const int x = ed_x(p), y = ed_y(p), idx = y * w + x;
        const bool horiz = flags_all[(size_t)f * node_cap + id] & 1;
        uint32_t e[2];
#pragma unroll
        for (int k = 0; k < 2; k++) {
            /* k = 0: right (horizontal class) / down; k = 1: left / up */
            int nx = x, ny = y;
            bool term;
            if (horiz) {
                const int sx = k == 0 ? 1 : -1;
                term = (k == 0 ? x == w - 1 : x == 0) || y == 0 || y == h - 1;
                if (!term) {
                    const uint8_t g1 = (uint8_t)g[idx - w + sx], g2 = (uint8_t)g[idx + sx], g3 = (uint8_t)g[idx + w + sx];
                    nx = x + sx;
                    if (g1 >= g2 && g1 >= g3)
                        ny = y - 1;
                    else if (g3 >= g2 && g3 >= g1)
                        ny = y + 1;
                }
            } else {
                const int sy = k == 0 ? 1 : -1;
                term = x == 0 || x == w - 1 || (k == 0 ? y == h - 1 : y == 0);
                if (!term) {
                    const uint8_t g1 = (uint8_t)g[idx + sy * w + 1], g2 = (uint8_t)g[idx + sy * w], g3 = (uint8_t)g[idx + sy * w - 1];
                    ny = y + sy;
                    if (g1 >= g2 && g1 >= g3)
                        nx = x + 1;
                    else if (g3 >= g2 && g3 >= g1)
                        nx = x - 1;
                }
            }
            uint32_t v = ED_TERM;
            if (!term && g[ny * w + nx] > 0) {
                const uint32_t t = pid[ny * w + nx];
                if (t < ED_TERM && (size_t)t < node_cap) {
                    /* which of the target's two moves the walk takes there: the same direction when the target is of the same class;
                     * otherwise shouldGo (:1722,1785): right / down when x, resp. y, grew on this step, left / up when not */
                    const bool t_horiz = flags_all[(size_t)f * node_cap + t] & 1;
                    const int sel = (t_horiz == horiz) ? k : ((horiz ? ny > y : nx > x) ? 0 : 1);
                    v = t | (sel ? ED_PLUS : 0u);
                }
            }
            e[k] = v;
        }
        next_all[(size_t)f * node_cap + id] = make_uint2(e[0], e[1]);
    }
    const int na = min(n_anchors[f], anchor_cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x)
        anchor_nid[(size_t)f * anchor_cap + i] = pid[anchors_all[(size_t)f * anchor_cap + i]];
}

/* how the walker reads the graph: shared-memory copy (15-bit ids) or HBM */
struct EdNavShared {
    uint32_t *w;      /* per node: move 0 in the low half, move 1 in the high half: id (15 bits) | next selector << 15 */
    uint32_t *edge;   /* bit per node */
    __device__ __forceinline__ bool is_edge(uint32_t id) const { return (edge[id >> 5] >> (id & 31)) & 1u; }
    __device__ __forceinline__ void set_edge(uint32_t id) const { edge[id >> 5] |= 1u << (id & 31); }
    __device__ __forceinline__ void clr_edge(uint32_t id) const { edge[id >> 5] &= ~(1u << (id & 31)); }
    __device__ __forceinline__ bool move(uint32_t id, int &k, uint32_t &to) const
    {
        const uint32_t e = (w[id] >> (16 * k)) & 0xffffu;
        to = e & 0x7fffu;
        k = (int)(e >> 15);
        return to != ED_SM_TERM;
    }
};
struct EdNavGlobal {
    const uint2 *nx;
    uint8_t *fl; /* bit 0 direction class, bit 1 edge */
    __device__ __forceinline__ bool is_edge(uint32_t id) const { return fl[id] & 2; }
    __device__ __forceinline__ void set_edge(uint32_t id) const { fl[id] |= 2; }
    __device__ __forceinline__ void clr_edge(uint32_t id) const { fl[id] &= ~2; }
    __device__ __forceinline__ bool move(uint32_t id, int &k, uint32_t &to) const
    {
        const uint2 v = nx[id];
        const uint32_t e = k ? v.y : v.x;
        to = e & ED_TERM;
        k = (e & ED_PLUS) ? 1 : 0;
        return to != ED_TERM;
    }
};

/* one smart-routing walk over the graph, starting with move k of node cur; appends node ids to out[n...] */
template <typename Nav>
__device__ __forceinline__ void ed_walk_graph(const Nav &N, uint32_t cur, int k, uint32_t *__restrict__ out, unsigned &n, unsigned cap)
{
    while (!N.is_edge(cur)) {
        N.set_edge(cur);
        if (n < cap) out[n] = cur;
        n++;
        uint32_t to;
        if (!N.move(cur, k, to)) break;
        cur = to;
    }
}

template <typename Nav, typename AnchorT>
__device__ void ed_route_frame(const Nav &N, const AnchorT *__restrict__ anchor_nid, int na, unsigned P, unsigned maxEdges, uint32_t *fP, uint32_t *sP,
                               uint32_t *fS, uint32_t *sS, uint32_t *sId, int32_t *hdr)
{
    unsigned nF = 0, nS = 0, nE = 0, nc = 0;
    for (int i = 0; i < na; i++) {
        const uint32_t a = anchor_nid[i];
        if (N.is_edge(a)) continue;
        const unsigned f0 = nF, s0 = nS;
        ed_walk_graph(N, a, 0, fP, nF, P); /* right (horizontal-edge pixel) / down */
        N.clr_edge(a);
        ed_walk_graph(N, a, 1, sP, nS, P); /* left / up */
        if ((int)(nF - f0) + (int)(nS - s0) < ED_MINLEN + 1) {
            nF = f0;
            nS = s0;
        } else {
            if (nE <= maxEdges) {
                fS[nE] = f0;
                sS[nE] = s0;
                sId[nE] = nc;
            }
            nc += (nF - f0) + (nS - s0) - 1;
            nE++;
        }
    }
    const bool bad = nE > maxEdges || nF > P || nS > P; /* the reference prints "Edge drawing Error" and detects nothing */
    if (!bad) {
        fS[nE] = nF;
        sS[nE] = nS;
        sId[nE] = nc;
    }
    hdr[0] = bad ? 0 : (int32_t)nE;
}

/* per-frame scratch layout (uint32 words) shared by the routing, fitting and emission kernels */
struct EdScratch {
    uint32_t *fP, *sP, *fS, *sS, *chain, *sId, *segcnt;
    float *seg; /* 4 floats per temporary segment + 1 flag word, slot = chain offset / ED_MINLEN + k */
    int32_t *hdr;
};
__host__ __device__ inline size_t ed_scratch_words(unsigned P, unsigned maxEdges)
{
    return (size_t)P * 2 + (size_t)(maxEdges + 2) * 4 + (size_t)P * 2 + ((size_t)2 * P / ED_MINLEN + 2) * 5 + 64;
}
__device__ __forceinline__ EdScratch ed_scratch_of(uint32_t *base, unsigned P, unsigned maxEdges)
{
    EdScratch s;
    s.hdr = (int32_t *)base;
    s.fP = base + 16;
    s.sP = s.fP + P;
    s.fS = s.sP + P;
    s.sS = s.fS + maxEdges + 2;
    s.sId = s.sS + maxEdges + 2;
    s.segcnt = s.sId + maxEdges + 2;
    s.chain = s.segcnt + maxEdges + 2;
    s.seg = (float *)(s.chain + 2 * (size_t)P);
    return s;
}

__global__ void __launch_bounds__(128) k_ed_route(int W, int H, const int32_t *__restrict__ rowoff, const uint2 *__restrict__ next_all,
                                                  uint8_t *__restrict__ flags_all, size_t node_cap, const uint32_t *__restrict__ anchor_nid_all,
                                                  const int32_t *__restrict__ n_anchors, int anchor_cap, uint32_t *__restrict__ scratch_all,
                                                  size_t scratch_per_frame, int sm_nodes, int32_t *__restrict__ err_flag, int32_t *__restrict__ redo,
                                                  int force_seq)
{
    extern __shared__ uint32_t s_dyn[];
    const int f = blockIdx.x, tid = threadIdx.x;
    const size_t npx = (size_t)W * H;
    const unsigned P = (unsigned)(npx / 5), maxEdges = P / 20;
    EdScratch S = ed_scratch_of(scratch_all + (size_t)f * scratch_per_frame, P, maxEdges);
    const int n_all = rowoff[(size_t)f * (H + 1) + H];
    const int na = n_anchors[f];
    if (tid == 0) {
        S.hdr[0] = 0;
        redo[f] = (force_seq || (size_t)n_all > node_cap) ? 1 : 0; /* more nodes than the graph arrays hold: the pixel-map kernel redoes the frame */
    }
    if (force_seq || (size_t)n_all > node_cap) return;
    if (na > anchor_cap || (unsigned)na > P) { /* reference: "anchor size is larger than its maximal size" -> no lines */
        if (tid == 0 && na > anchor_cap) atomicOr(err_flag, 1);
        return;
    }
    const uint2 *nx = next_all + (size_t)f * node_cap;
    uint8_t *fl = flags_all + (size_t)f * node_cap;
    const uint32_t *anchor_nid = anchor_nid_all + (size_t)f * anchor_cap;
    if (n_all <= sm_nodes && n_all < (int)ED_SM_TERM) {
        EdNavShared N;
        N.w = s_dyn;
        N.edge = s_dyn + sm_nodes;
        uint16_t *s_anchor = (uint16_t *)(N.edge + (sm_nodes + 31) / 32);
        for (int i = tid; i < n_all; i += blockDim.x) {
            const uint2 v = nx[i];
            const uint32_t a = (v.x & ED_TERM) == ED_TERM ? ED_SM_TERM : ((v.x & 0x7fffu) | ((v.x & ED_PLUS) ? 0x8000u : 0u));
            const uint32_t b = (v.y & ED_TERM) == ED_TERM ? ED_SM_TERM : ((v.y & 0x7fffu) | ((v.y & ED_PLUS) ? 0x8000u : 0u));
            N.w[i] = a | (b << 16);
        }
        for (int i = tid; i < (n_all + 31) / 32; i += blockDim.x) N.edge[i] = 0;
        const bool anchors_staged = na <= ED_SM_ANCHORS;
        if (anchors_staged)
            for (int i = tid; i < na; i += blockDim.x) s_anchor[i] = (uint16_t)anchor_nid[i];
        __syncthreads();
        if (tid == 0) {
            if (anchors_staged)
                ed_route_frame(N, (const uint16_t *)s_anchor, na, P, maxEdges, S.fP, S.sP, S.fS, S.sS, S.sId, S.hdr);
            else
                ed_route_frame(N, anchor_nid, na, P, maxEdges, S.fP, S.sP, S.fS, S.sS, S.sId, S.hdr);
        }
        __syncthreads();
        for (int i = tid; i < n_all; i += blockDim.x) fl[i] = (uint8_t)((fl[i] & 1) | (N.is_edge(i) ? 2 : 0)); /* the edge map, for inspection */
    } else if (tid == 0) {
        EdNavGlobal N;
        N.nx = nx;
        N.fl = fl;
        ed_route_frame(N, anchor_nid, na, P, maxEdges, S.fP, S.sP, S.fS, S.sS, S.sId, S.hdr);
    }
}

/* inspection: the edge map of one frame from the node flags */
__global__ void __launch_bounds__(256) k_ed_edge_map(const uint32_t *__restrict__ xy, const uint8_t *__restrict__ fl, int n, int w, uint8_t *__restrict__ edge)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (fl[i] & 2)) edge[ed_y(xy[i]) * w + ed_x(xy[i])] = 1;
}

/* ---- fitting, one warp per chain */
struct EdFit {
    float ATA[4], ATV[2];
    double eq[2];
};

/* LeastSquaresLineFit_, first overload (:2628-2714), on one lane */
__device__ __forceinline__ double ed_fit_initial_lane(const uint32_t *__restrict__ pts, bool horiz, EdFit &T)
{
    double suu = 0, su = 0, suv = 0, sv = 0;
    for (int i = 0; i < ED_MINLEN; i++) {
        const uint32_t p = pts[i];
        const double u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
        suu += u * u;
        su += u;
        suv += u * v;
        sv += v;
    }
    T.ATA[0] = (float)suu;
    T.ATA[1] = (float)su;
    T.ATA[2] = (float)su;
    T.ATA[3] = (float)(double)ED_MINLEN;
    T.ATV[0] = (float)suv;
    T.ATV[1] = (float)sv;
    const double coef = 1.0 / ((double)T.ATA[0] * (double)T.ATA[3] - (double)T.ATA[1] * (double)T.ATA[2]);
    T.eq[0] = coef * ((double)T.ATA[3] * (double)T.ATV[0] - (double)T.ATA[1] * (double)T.ATV[1]);
    T.eq[1] = coef * ((double)T.ATA[0] * (double)T.ATV[1] - (double)T.ATA[2] * (double)T.ATV[0]);
    double fitError = 0;
    for (int i = 0; i < ED_MINLEN; i++) {
        const uint32_t p = pts[i];
        const double u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
        const double c = v - u * T.eq[0] - T.eq[1];
        fitError += c * c;
    }
    return sqrt(fitError);
}

__device__ __forceinline__ long long ed_warp_sum_ll(long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int ed_warp_sum_i(int v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

/* the chain [S, Eend) of one edge -> segments; every lane returns the same counts.  seg: 5 words per temporary slot. */
__device__ void ed_fit_chain(const EdFrame &F, const uint32_t *__restrict__ chain, unsigned S, const unsigned Eend, float line_length_thres, float *seg,
                             float *segx /* optional: 2 floats per temporary slot, {direction, numOfPixels} */, int &n_raw, int &n_kept)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, W = F.W;
    n_raw = 0;
    n_kept = 0;
    while (Eend > S + ED_MINLEN) {
        /* first start offset S, S + 2, S + 4, ... whose 15-point fit is good enough: 32 offsets at a time */
        EdFit T;
        bool found = false;
        bool horiz = false;
        while (Eend > S + ED_MINLEN) {
            const unsigned Sl = S + ED_SKIP * lane;
            const bool valid = Eend > Sl + ED_MINLEN;
            double err = 1e300;
            bool hz = false;
            if (valid) {
                const uint32_t p0 = chain[Sl];
                hz = F.dir[ed_y(p0) * W + ed_x(p0)] == ED_HORIZONTAL;
                err = ed_fit_initial_lane(chain + Sl, hz, T);
            }
            const unsigned good = __ballot_sync(FULL, valid && err <= ED_FITERR);
            const int nvalid = __popc(__ballot_sync(FULL, valid));
            if (good) {
                const int fl = __ffs(good) - 1;
                S += ED_SKIP * fl;
#pragma unroll
                for (int k = 0; k < 4; k++) T.ATA[k] = __shfl_sync(FULL, T.ATA[k], fl);
                T.ATV[0] = __shfl_sync(FULL, T.ATV[0], fl);
                T.ATV[1] = __shfl_sync(FULL, T.ATV[1], fl);
                T.eq[0] = __shfl_sync(FULL, T.eq[0], fl);
                T.eq[1] = __shfl_sync(FULL, T.eq[1], fl);
                horiz = __shfl_sync(FULL, (int)hz, fl) != 0;
                found = true;
                break;
            }
            S += ED_SKIP * nvalid;
        }
        if (!found) break;
        const unsigned lineStart = S;
        double coef1 = 0;
        bool bExtended = true, bFirstTry = true;
        int tryTimes = 0;
        unsigned newOffsetS = 0;
        while (bExtended) {
            tryTimes++;
            if (bFirstTry) {
                bFirstTry = false;
                S += ED_MINLEN;
            } else {
                /* second overload (:2716-2787) over the points [newOffsetS, S): integer-valued sums, exact in any order */
                const int newLength = (int)S - (int)newOffsetS;
                if ((int)S - (int)lineStart > 0 && newLength > 0) {
                    long long suu = 0, su = 0, suv = 0, sv = 0;
                    for (unsigned i = newOffsetS + lane; i < S; i += 32) {
                        const uint32_t p = chain[i];
                        const long long u = horiz ? ed_x(p) : ed_y(p), v = horiz ? ed_y(p) : ed_x(p);
                        suu += u * u;
                        su += u;
                        suv += u * v;
                        sv += v;
                    }
                    suu = ed_warp_sum_ll(suu);
                    su = ed_warp_sum_ll(su);
                    suv = ed_warp_sum_ll(suv);
                    sv = ed_warp_sum_ll(sv);
                    T.ATA[0] = T.ATA[0] + (float)(double)suu;
                    T.ATA[1] = T.ATA[1] + (float)(double)su;
                    T.ATA[2] = T.ATA[2] + (float)(double)su;
                    T.ATA[3] = T.ATA[3] + (float)(double)newLength;
                    T.ATV[0] = T.ATV[0] + (float)(double)suv;
                    T.ATV[1] = T.ATV[1] + (float)(double)sv;
                    const double coef = 1.0 / ((double)T.ATA[0] * (double)T.ATA[3] - (double)T.ATA[1] * (double)T.ATA[2]);
                    T.eq[0] = coef * ((double)T.ATA[3] * (double)T.ATV[0] - (double)T.ATA[1] * (double)T.ATV[1]);
                    T.eq[1] = coef * ((double)T.ATA[0] * (double)T.ATV[1] - (double)T.ATA[2] * (double)T.ATV[0]);
                }
            }
            coef1 = 1 / sqrt(T.eq[0] * T.eq[0] + 1);
            int numOfOutlier = 0;
            newOffsetS = S;
            /* extension: stop after the 4th consecutive outlier */
            while (Eend > S) {
                const unsigned i = S + lane;
                const bool valid = i < Eend;
                bool outl = false;
                if (valid) {
                    const uint32_t p = chain[i];
                    const double d = horiz ? fabs(T.eq[0] * (double)ed_x(p) - (double)ed_y(p) + T.eq[1]) * coef1
                                           : fabs((double)ed_x(p) - T.eq[0] * (double)ed_y(p) - T.eq[1]) * coef1;
                    outl = d > ED_FITERR;
                }
                const unsigned m = __ballot_sync(FULL, outl);
                const int nvalid = __popc(__ballot_sync(FULL, valid));
                /* bits 0..3: the outliers carried in (the most recent one at bit 3), bits 4..: this chunk */
                const unsigned long long M = ((unsigned long long)m << 4) | (unsigned long long)(((1u << numOfOutlier) - 1u) << (4 - numOfOutlier));
                const unsigned long long R4 = M & (M << 1) & (M << 2) & (M << 3);
                const unsigned long long hit = R4 >> 4; /* bit l: the 4th consecutive outlier is chunk point l */
                if (hit) {
                    const int l = __ffsll((long long)hit) - 1;
                    S += l + 1;
                    numOfOutlier = 4;
                    break;
                }
                /* no break in this chunk: outliers trailing its last valid point */
                int t = 0;
                while (t < 4 && t < nvalid + 4 && ((M >> (nvalid + 3 - t)) & 1ull)) t++;
                numOfOutlier = t;
                S += nvalid;
            }
            S -= numOfOutlier;
            if (!((int)S - (int)newOffsetS > 0 && tryTimes < ED_TRYTIME)) bExtended = false;
        }
        double lineEqu[3];
        if (horiz) {
            lineEqu[0] = T.eq[0] * coef1;
            lineEqu[1] = -1 * coef1;
            lineEqu[2] = T.eq[1] * coef1;
        } else {
            lineEqu[0] = 1 * coef1;
            lineEqu[1] = -T.eq[0] * coef1;
            lineEqu[2] = -T.eq[1] * coef1;
        }
        /* LineValidation_ (:2789-2870) over chain[lineStart, S) */
        const int n = (int)S - (int)lineStart;
        int mgx = 0, mgy = 0;
        for (int i = lane; i < n; i += 32) {
            const uint32_t p = chain[lineStart + i];
            const int index = ed_y(p) * W + ed_x(p);
            mgx += F.dx[index];
            mgy += F.dy[index];
        }
        mgx = ed_warp_sum_i(mgx);
        mgy = ed_warp_sum_i(mgy);
        bool ok = !(mgx == 0 && mgy == 0);
        float direction = 0;
        if (ok) {
            const double ddx = fabs(lineEqu[1]), ddy = fabs(lineEqu[0]);
            if (mgx > 0 && mgy >= 0) direction = (float)atan2(-ddy, ddx);
            if (mgx <= 0 && mgy > 0) direction = (float)atan2(ddy, ddx);
            if (mgx < 0 && mgy <= 0) direction = (float)atan2(ddy, -ddx);
            if (mgx >= 0 && mgy < 0) direction = (float)atan2(-ddy, -ddx);
            if (fabs((double)direction) < 0.15 || ED_PI - fabs((double)direction) < 0.15) {
                if (fabs(lineEqu[2]) < 10 || fabs((double)F.H - fabs(lineEqu[2])) < 10) ok = false;
            }
            if (ok && fabs(fabs((double)direction) - ED_PI * 0.5) < 0.15) {
                if (fabs(lineEqu[2]) < 10 || fabs((double)F.W - fabs(lineEqu[2])) < 10) ok = false;
            }
        }
        if (ok) {
            int k = 0;
            for (int i = lane; i < n; i += 32) {
                const uint32_t p = chain[lineStart + i];
                const int index = ed_y(p) * W + ed_x(p);
                const double pd = atan2(-(double)F.dx[index], (double)F.dy[index]);
                const double dis = fabs((double)direction - pd);
                if (fabs(2 * ED_PI - dis) < 0.392699 || dis < 0.392699) k++;
            }
            k = ed_warp_sum_i(k);
            ok = cs_nfa_warp(F.lgam, n, k, 0.125, F.logNT, false) > 0;
        }
        if (ok) {
            const double a1 = lineEqu[1] * lineEqu[1], a2 = lineEqu[0] * lineEqu[0], a3 = lineEqu[0] * lineEqu[1];
            const double a4 = lineEqu[2] * lineEqu[0], a5 = lineEqu[2] * lineEqu[1];
            unsigned Px = ed_x(chain[lineStart]), Py = ed_y(chain[lineStart]);
            const float s1 = (float)(a1 * Px - a3 * Py - a4), s2 = (float)(a2 * Py - a3 * Px - a5);
            Px = ed_x(chain[S - 1]);
            Py = ed_y(chain[S - 1]);
            const float e1 = (float)(a1 * Px - a3 * Py - a4), e2 = (float)(a2 * Py - a3 * Px - a5);
            /* OctaveKeyLines: length and start / end ordering (:862-886,1069-1139) */
            float fdx = fabsf(s1 - e1), fdy = fabsf(s2 - e2);
            const float lineLength = sqrtf(fdx * fdx + fdy * fdy);
            fdx = e1 - s1;
            fdy = e2 - s2;
            bool sw = false;
            const double dr = (double)direction;
            if (dr >= -0.75 * ED_PI && dr < -0.25 * ED_PI && fdy > 0) sw = true;
            if (dr >= -0.25 * ED_PI && dr < 0.25 * ED_PI && fdx < 0) sw = true;
            if (dr >= 0.25 * ED_PI && dr < 0.75 * ED_PI && fdy < 0) sw = true;
            if (((dr >= 0.75 * ED_PI && dr < ED_PI) || (dr >= -ED_PI && dr < -0.75 * ED_PI)) && fdx > 0) sw = true;
            const bool kept = lineLength > line_length_thres;
            if (lane == 0) {
                float *o = seg + 5 * (size_t)n_raw;
                o[0] = sw ? e1 : s1;
                o[1] = sw ? e2 : s2;
                o[2] = sw ? s1 : e1;
                o[3] = sw ? s2 : e2;
                o[4] = __int_as_float(kept ? 1 : 0);
                if (segx) {
                    segx[2 * n_raw] = direction;
                    segx[2 * n_raw + 1] = __int_as_float(n);
                }
            }
            n_raw++;
            n_kept += kept ? 1 : 0;
        }
    }
}

__global__ void __launch_bounds__(128) k_ed_fit(int W, int H, const int16_t *__restrict__ dx_all, const int16_t *__restrict__ dy_all,
                                                const uint8_t *__restrict__ dir_all, const uint32_t *__restrict__ xy_all, size_t node_cap,
                                                uint32_t *__restrict__ scratch_all, size_t scratch_per_frame, double logNT, float line_length_thres,
                                                const int32_t *__restrict__ redo, const double *__restrict__ lgam, float *__restrict__ segx_all,
                                                size_t segx_per_frame)
{
    const int f = blockIdx.y, lane = threadIdx.x & 31;
    if (redo[f]) return;
    const size_t npx = (size_t)W * H;
    const unsigned P = (unsigned)(npx / 5), maxEdges = P / 20;
    EdScratch S = ed_scratch_of(scratch_all + (size_t)f * scratch_per_frame, P, maxEdges);
    const unsigned nE = (unsigned)S.hdr[0];
    EdFrame F;
    F.W = W;
    F.H = H;
    F.dx = dx_all + f * npx;
    F.dy = dy_all + f * npx;
    F.g = nullptr;
    F.dir = dir_all + f * npx;
    F.edge = nullptr;
    F.logNT = logNT;
    F.lgam = lgam;
    const uint32_t *xy = xy_all + (size_t)f * node_cap;
    const unsigned wpb = blockDim.x >> 5;
    for (unsigned e = blockIdx.x * wpb + (threadIdx.x >> 5); e < nE; e += gridDim.x * wpb) {
        /* chain assembly: first part reversed, then the second part without the anchor */
        const unsigned f0 = S.fS[e], f1 = S.fS[e + 1], s0 = S.sS[e], s1 = S.sS[e + 1], c0 = S.sId[e];
        const unsigned nf = f1 - f0, ns = s1 - s0 - 1;
        for (unsigned t = lane; t < nf; t += 32) S.chain[c0 + t] = xy[S.fP[f1 - 1 - t]];
        for (unsigned t = lane; t < ns; t += 32) S.chain[c0 + nf + t] = xy[S.sP[s0 + 1 + t]];
        __syncwarp();
        int n_raw, n_kept;
        ed_fit_chain(F, S.chain, c0, c0 + nf + ns, line_length_thres, S.seg + 5 * (size_t)(c0 / ED_MINLEN),
                     segx_all ? segx_all + (size_t)f * segx_per_frame + 2 * (size_t)(c0 / ED_MINLEN) : nullptr, n_raw, n_kept);
        if (lane == 0) S.segcnt[e] = (uint32_t)n_raw | ((uint32_t)n_kept << 16);
    }
}

/* segments of a frame in chain order */
__global__ void __launch_bounds__(256) k_ed_emit(int W, int H, uint32_t *__restrict__ scratch_all, size_t scratch_per_frame, float *__restrict__ raw_all,
                                                 int32_t *__restrict__ n_raw_all, float *__restrict__ out_all, int32_t *__restrict__ n_out_all, int cap,
                                                 const int32_t *__restrict__ redo, const float *__restrict__ segx_all, size_t segx_per_frame,
                                                 float *__restrict__ klx_all)
{
    __shared__ int s_w[8];
    __shared__ int s_base_raw, s_base_out;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const size_t npx = (size_t)W * H;
    const unsigned P = (unsigned)(npx / 5), maxEdges = P / 20;
    EdScratch S = ed_scratch_of(scratch_all + (size_t)f * scratch_per_frame, P, maxEdges);
    if (redo[f]) return; /* k_ed_route_fit writes this frame's segments */
    const int nE = S.hdr[0];
    float *raw = raw_all + (size_t)f * cap * 4;
    float *out = out_all + (size_t)f * cap * 4;
    if (tid == 0) {
        s_base_raw = 0;
        s_base_out = 0;
    }
    __syncthreads();
    for (int b = 0; b < nE; b += 256) {
        const int e = b + tid;
        const uint32_t c = e < nE ? S.segcnt[e] : 0u;
        const int nr = (int)(c & 0xffffu), nk = (int)(c >> 16);
        /* inclusive warp scans of both counts, packed */
        int inc = nr | (nk << 16);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        int pre = 0;
        for (int k = 0; k < wid; k++) pre += s_w[k];
        int off_r = s_base_raw + ((pre + inc) & 0xffff) - nr, off_o = s_base_out + ((pre + inc) >> 16) - nk;
        if (nr) {
            const float *seg = S.seg + 5 * (size_t)(S.sId[e] / ED_MINLEN);
            const float *segx = (segx_all && klx_all) ? segx_all + (size_t)f * segx_per_frame + 2 * (size_t)(S.sId[e] / ED_MINLEN) : nullptr;
            for (int k = 0; k < nr; k++) {
                const float *q = seg + 5 * k;
                if (off_r < cap)
                    for (int j = 0; j < 4; j++) raw[4 * off_r + j] = q[j];
                off_r++;
                if (__float_as_int(q[4])) {
                    if (off_o < cap) {
                        for (int j = 0; j < 4; j++) out[4 * off_o + j] = q[j];
                        if (segx) {
                            float *kx = klx_all + ((size_t)f * cap + off_o) * 2;
                            kx[0] = segx[2 * k];
                            kx[1] = segx[2 * k + 1];
                        }
                    }
                    off_o++;
                }
            }
        }
        __syncthreads();
        if (tid == 255) {
            s_base_raw += (pre + inc) & 0xffff;
            s_base_out += (pre + inc) >> 16;
        }
        __syncthreads();
    }
    if (tid == 0) {
        n_raw_all[f] = s_base_raw;
        n_out_all[f] = s_base_out;
    }
}

/* ---------------------------------------------------------------------------------------- host side */
struct Buf {
    void *p = nullptr;
    size_t cap = 0;
};
struct EdState {
    CsLineHead head; /* first: the error word (cs_internal.h) */
    Buf img, tmp, blur, dx, dy, g, dir, edge, anchors, nanch, scratch, raw, nraw, out, nout, err;
    Buf rowcnt, pid, xy, flags, next, anid, redo, abits, colcnt, lgam;
    Buf segx, klx; /* key-line extras for the descriptor (cs_edl_run_keylines): per temporary slot, per kept segment */
    bool lgam_filled = false;
    int last_frames = 0, last_w = 0, last_h = 0, cap = 0, anchor_cap = 0;
    size_t node_cap = 0;
    bool route_attr_set[64] = {};
};

int ed_ensure(cs_ctx *c, Buf &b, size_t bytes)
{
    if (bytes <= b.cap) return CS_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    const size_t want = bytes + bytes / 16 + 256;
    if (cudaMalloc(&b.p, want) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc(%zu) failed in the EDLines detector", want);
    b.cap = want;
    return CS_OK;
}
inline int ed_grid(int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, CS_SM_COUNT * 32); }
/* nodes of a frame's walk graph that k_ed_route keeps in shared memory (4 bytes + 1 bit each): 32,766 = the 15-bit id limit, one frame
 * per SM (H100, c3 EDLines with 12 batches in flight: 3.66 ms per step, 4.14 with 26,000 -- two frames per SM, where the densest frames
 * of a batch fall back to walking in HBM) */
#define ED_SM_NODES 32766

EdState *ed_state_of(cs_ctx *c)
{
    void **slot = cs_ctx_edl_slot(c);
    if (!*slot) *slot = new EdState();
    return (EdState *)*slot;
}

}  // namespace

void cs_edl_destroy(void *state)
{
    EdState *S = (EdState *)state;
    Buf *all[] = {&S->img, &S->tmp, &S->blur, &S->dx, &S->dy, &S->g, &S->dir, &S->edge, &S->anchors, &S->nanch, &S->scratch, &S->raw, &S->nraw, &S->out, &S->nout, &S->err,
                  &S->rowcnt, &S->pid, &S->xy, &S->flags, &S->next, &S->anid, &S->redo, &S->abits, &S->colcnt, &S->lgam, &S->segx, &S->klx};
    for (Buf *b : all)
        if (b->p) cudaFree(b->p);
    delete S;
}

/* frames in HBM (or host) -> filtered segments in HBM; want_keylines: also {direction, numOfPixels} of every kept segment (S.klx) */
static int ed_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
                  int cap, const float **d_lines, const int32_t **d_counts, bool want_keylines)
{
    EdState &S = *ed_state_of(c);
    cudaStream_t st = cs_ctx_stream(c);
    if (w < 8 || h < 8 || w > 65535 || h > 65535) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "image size unsupported by EDLines");
    const size_t px = (size_t)n_frames * w * h, npx = (size_t)w * h;
    const unsigned P = (unsigned)(npx / 5), maxEdges = P / 20;
    const size_t scratch_per_frame = std::max((size_t)P * 2 + (size_t)(maxEdges + 2) * 3 + (size_t)P * 4 + 64, ed_scratch_words(P, maxEdges));
    const size_t segx_per_frame = ((size_t)2 * P / ED_MINLEN + 2) * 2; /* one {direction, numOfPixels} pair per temporary segment slot */
    const int anchor_cap = (int)P + 1;
    const size_t node_cap = npx / 2; /* pixels with g > 0 (gradient magnitude above the threshold); denser frames take the pixel-map kernel */
    const int force_seq = cs_ctx_seq_lines(c);
    const int nw = (w - 2 + 1) / 2, nh = (h - 2 + 1) / 2, nhw = (nh + 31) / 32; /* anchor candidates: columns, rows, words of rows */
    int rc;
    const uint8_t *d_img = imgs;
    if (!imgs_on_device) {
        if ((rc = ed_ensure(c, S.img, (size_t)n_frames * h * stride))) return rc;
        if (cudaMemcpyAsync(S.img.p, imgs, (size_t)n_frames * h * stride, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames failed");
        d_img = (const uint8_t *)S.img.p;
    }
    if ((rc = ed_ensure(c, S.tmp, px * 2)) || (rc = ed_ensure(c, S.blur, px)) || (rc = ed_ensure(c, S.dx, px * 2)) || (rc = ed_ensure(c, S.dy, px * 2)) ||
        (rc = ed_ensure(c, S.g, px * 2)) || (rc = ed_ensure(c, S.dir, px)) || (rc = ed_ensure(c, S.edge, px)) ||
        (rc = ed_ensure(c, S.anchors, (size_t)n_frames * anchor_cap * 4)) || (rc = ed_ensure(c, S.nanch, (size_t)n_frames * 4)) ||
        (rc = ed_ensure(c, S.scratch, (size_t)n_frames * scratch_per_frame * 4)) || (rc = ed_ensure(c, S.raw, (size_t)n_frames * cap * 16)) ||
        (rc = ed_ensure(c, S.nraw, (size_t)n_frames * 4)) || (rc = ed_ensure(c, S.out, (size_t)n_frames * cap * 16)) ||
        (rc = ed_ensure(c, S.nout, (size_t)n_frames * 4)) || (rc = ed_ensure(c, S.err, 16)) ||
        (rc = ed_ensure(c, S.rowcnt, (size_t)n_frames * (h + 1) * 4)) || (rc = ed_ensure(c, S.pid, px * 4)) ||
        (rc = ed_ensure(c, S.xy, (size_t)n_frames * node_cap * 4)) || (rc = ed_ensure(c, S.flags, (size_t)n_frames * node_cap)) ||
        (rc = ed_ensure(c, S.next, (size_t)n_frames * node_cap * 8)) || (rc = ed_ensure(c, S.anid, (size_t)n_frames * anchor_cap * 4)) ||
        (rc = ed_ensure(c, S.redo, (size_t)n_frames * 4)) || (rc = ed_ensure(c, S.abits, (size_t)n_frames * nw * nhw * 4)) ||
        (rc = ed_ensure(c, S.colcnt, (size_t)n_frames * (nw + 1) * 4)) || (rc = ed_ensure(c, S.lgam, (size_t)CS_LGAMMA_TABLE * 8)))
        return rc;
    if (want_keylines && ((rc = ed_ensure(c, S.segx, (size_t)n_frames * segx_per_frame * 4)) || (rc = ed_ensure(c, S.klx, (size_t)n_frames * cap * 8)))) return rc;
    float *d_segx = want_keylines ? (float *)S.segx.p : nullptr, *d_klx = want_keylines ? (float *)S.klx.p : nullptr;
    if (!S.lgam_filled) { /* log_gamma of the integers 1 .. CS_LGAMMA_TABLE - 1, host libm like the reference */
        std::vector<double> t(CS_LGAMMA_TABLE, 0.0);
        for (int i = 1; i < CS_LGAMMA_TABLE; i++) t[i] = cs_lgamma_host((double)i);
        if (cudaMemcpyAsync(S.lgam.p, t.data(), t.size() * 8, cudaMemcpyHostToDevice, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the log_gamma table failed");
        S.lgam_filled = true;
    }
    const double logNT = 2.0 * (std::log10((double)w) + std::log10((double)h)); /* :2399, host libm like the reference */
    cudaMemsetAsync(S.edge.p, 0, px, st);
    S.head.d_err = (int32_t *)S.err.p;
    cudaMemsetAsync(S.err.p, 0, 16, st);
    if (force_seq) { /* A/B: the round-1 kernels */
        k_ed_hblur<<<ed_grid((int64_t)px), 256, 0, st>>>(d_img, n_frames, w, h, stride, channels, (uint16_t *)S.tmp.p);
        k_ed_vblur<<<ed_grid((int64_t)px), 256, 0, st>>>((const uint16_t *)S.tmp.p, n_frames, w, h, (uint8_t *)S.blur.p);
        k_ed_maps<<<ed_grid((int64_t)px), 256, 0, st>>>((const uint8_t *)S.blur.p, n_frames, w, h, (int16_t *)S.dx.p, (int16_t *)S.dy.p, (int16_t *)S.g.p,
                                                        (uint8_t *)S.dir.p);
        k_ed_anchors<<<n_frames, 256, 0, st>>>((const int16_t *)S.g.p, (const uint8_t *)S.dir.p, w, h, (int32_t *)S.anchors.p, (int32_t *)S.nanch.p, anchor_cap);
    } else {
        const dim3 g_tile((w + EDF_TW - 1) / EDF_TW, (h + EDF_TH - 1) / EDF_TH, n_frames);
        CUtensorMap tm;
        if (cs_ctx_use_tma(c) && channels == 3 && stride == 3 * w && cs_make_tmap_bytes(&tm, d_img, 3 * (int64_t)w, (int64_t)n_frames * h, stride, EDF_BOXW, EDF_TH + 6))
            k_ed_front<true><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, (uint8_t *)S.blur.p, (int16_t *)S.dx.p, (int16_t *)S.dy.p, (int16_t *)S.g.p,
                                                    (uint8_t *)S.dir.p, (int32_t *)S.err.p);
        else
            k_ed_front<false><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, (uint8_t *)S.blur.p, (int16_t *)S.dx.p, (int16_t *)S.dy.p, (int16_t *)S.g.p,
                                                     (uint8_t *)S.dir.p, (int32_t *)S.err.p);
        cudaMemsetAsync(S.colcnt.p, 0, (size_t)n_frames * (nw + 1) * 4, st);
        k_ed_anchor_flags<<<dim3((nw + 255) / 256, nhw, n_frames), 256, 0, st>>>((const int16_t *)S.g.p, (const uint8_t *)S.dir.p, w, h, nw, nh, nhw,
                                                                                 (uint32_t *)S.abits.p, (int32_t *)S.colcnt.p);
        k_ed_anchor_list<<<n_frames, 1024, 0, st>>>(w, nw, nhw, (const uint32_t *)S.abits.p, (int32_t *)S.colcnt.p, (int32_t *)S.anchors.p,
                                                    (int32_t *)S.nanch.p, anchor_cap);
    }
    /* the walk graph, routing on it, chains fitted in parallel, segments in order (see the comment above k_ed_rowcount) */
    const int dev = cs_ctx_device(c);
    const int sm_nodes = ED_SM_NODES;
    const size_t sm_bytes = (size_t)sm_nodes * 4 + (size_t)((sm_nodes + 31) / 32) * 4 + (size_t)ED_SM_ANCHORS * 2;
    if (dev >= 0 && dev < 64 && !S.route_attr_set[dev]) {
        cudaFuncSetAttribute(k_ed_route, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_bytes);
        S.route_attr_set[dev] = true;
    }
    const int warps = n_frames * h, row_blocks = (warps * 32 + 255) / 256;
    if (!force_seq) {
        k_ed_rowcount<<<row_blocks, 256, 0, st>>>((const int16_t *)S.g.p, w, h, n_frames, (int32_t *)S.rowcnt.p);
        k_ed_rowscan<<<n_frames, 1024, 0, st>>>(h, (int32_t *)S.rowcnt.p);
        k_ed_nodes<<<row_blocks, 256, 0, st>>>((const int16_t *)S.g.p, (const uint8_t *)S.dir.p, w, h, n_frames, (const int32_t *)S.rowcnt.p, (uint32_t *)S.pid.p,
                                              (uint32_t *)S.xy.p, (uint8_t *)S.flags.p, node_cap);
        k_ed_next<<<dim3(16, n_frames), 256, 0, st>>>((const int16_t *)S.g.p, w, h, n_frames, (const int32_t *)S.rowcnt.p, (const uint32_t *)S.pid.p,
                                                      (const uint32_t *)S.xy.p, (const uint8_t *)S.flags.p, node_cap, (uint2 *)S.next.p,
                                                      (const int32_t *)S.anchors.p, (const int32_t *)S.nanch.p, anchor_cap, (uint32_t *)S.anid.p);
        cs_ctx_count_launches(c, 4);
    } else
        cudaMemsetAsync(S.rowcnt.p, 0, (size_t)n_frames * (h + 1) * 4, st);
    k_ed_route<<<n_frames, 128, sm_bytes, st>>>(w, h, (const int32_t *)S.rowcnt.p, (const uint2 *)S.next.p, (uint8_t *)S.flags.p, node_cap,
                                                (const uint32_t *)S.anid.p, (const int32_t *)S.nanch.p, anchor_cap, (uint32_t *)S.scratch.p,
                                                scratch_per_frame, sm_nodes, (int32_t *)S.err.p, (int32_t *)S.redo.p, force_seq);
    if (!force_seq) {
        k_ed_fit<<<dim3(16, n_frames), 128, 0, st>>>(w, h, (const int16_t *)S.dx.p, (const int16_t *)S.dy.p, (const uint8_t *)S.dir.p, (const uint32_t *)S.xy.p,
                                                     node_cap, (uint32_t *)S.scratch.p, scratch_per_frame, logNT, line_length_thres, (const int32_t *)S.redo.p,
                                                     (const double *)S.lgam.p, d_segx, segx_per_frame);
        k_ed_emit<<<n_frames, 256, 0, st>>>(w, h, (uint32_t *)S.scratch.p, scratch_per_frame, (float *)S.raw.p, (int32_t *)S.nraw.p, (float *)S.out.p,
                                            (int32_t *)S.nout.p, cap, (const int32_t *)S.redo.p, d_segx, segx_per_frame, d_klx);
        cs_ctx_count_launches(c, 2);
    }
    /* frames flagged for redo (graph arrays too small; or the A/B switch): routing and fitting on the pixel maps, one thread per frame */
    k_ed_route_fit<<<n_frames, 32, 0, st>>>(w, h, (const int16_t *)S.dx.p, (const int16_t *)S.dy.p, (const int16_t *)S.g.p, (const uint8_t *)S.dir.p,
                                            (uint8_t *)S.edge.p, (const int32_t *)S.anchors.p, (const int32_t *)S.nanch.p, anchor_cap,
                                            (uint32_t *)S.scratch.p, scratch_per_frame, logNT, line_length_thres, (float *)S.raw.p, (int32_t *)S.nraw.p,
                                            (float *)S.out.p, (int32_t *)S.nout.p, cap, (int32_t *)S.err.p, (const int32_t *)S.redo.p, d_klx);
    cs_ctx_count_launches(c, 6);
    S.node_cap = node_cap;
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "EDLines kernel launch failed");
    S.last_frames = n_frames;
    S.last_w = w;
    S.last_h = h;
    S.cap = cap;
    S.anchor_cap = anchor_cap;
    if (d_lines) *d_lines = (const float *)S.out.p;
    if (d_counts) *d_counts = (const int32_t *)S.nout.p;
    return CS_OK;
}

uint8_t *cs_edl_frame_buffer(cs_ctx *c, size_t bytes)
{
    EdState &S = *ed_state_of(c);
    return ed_ensure(c, S.img, bytes) ? nullptr : (uint8_t *)S.img.p;
}

int cs_edl_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
               int cap, const float **d_lines, const int32_t **d_counts)
{
    return ed_run(c, imgs, imgs_on_device, n_frames, w, h, stride, channels, line_length_thres, cap, d_lines, d_counts, false);
}

/* the synchronous callers (the descriptor entry points, cs_lbd.cu): wait for the run and turn its error word into an error */
static int ed_check_run(cs_ctx *c, EdState &S)
{
    cudaStream_t st = cs_ctx_stream(c);
    int32_t err[4] = {0, 0, 0, 0};
    if (cudaMemcpyAsync(err, S.err.p, sizeof err, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "EDLines error word copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    return cs_edl_check_err(c, err);
}

int cs_edl_run_keylines(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels,
                        float line_length_thres, int cap, const float **d_lines, const int32_t **d_counts, const float **d_extra,
                        const int16_t **d_dx, const int16_t **d_dy)
{
    int rc = ed_run(c, imgs, imgs_on_device, n_frames, w, h, stride, channels, line_length_thres, cap, d_lines, d_counts, true);
    if (rc) return rc;
    EdState *S = ed_state_of(c);
    if ((rc = ed_check_run(c, *S))) return rc;
    *d_extra = (const float *)S->klx.p;
    *d_dx = (const int16_t *)S->dx.p;
    *d_dy = (const int16_t *)S->dy.p;
    return CS_OK;
}

/* The Sobel maps BinaryDescriptor::computeSobel builds for the descriptor (binary_descriptor.cpp:352-398, octave 0: GaussianBlur 5 x 5
 * sigma 1, then Sobel 3 x 3 into CV_16SC1) are the maps EDLineDetector::EdgeDrawing builds from OctaveKeyLines' blurred image (:811-814,
 * 1617-1622): the same front-end kernel produces them, into the EDLines workspace.  Any size from 1 x 1 works: the kernel reflects every
 * tap with ed_reflect101 and masks partial tiles, and computeSobel's BORDER_REFLECT_101 maps a 1-pixel side to its one pixel.  The
 * upper limit is the descriptor's: computeLBD clamps coordinates in a short (binary_descriptor.cpp:1184,1286-1288). */
int cs_edl_sobel_maps(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels,
                      const int16_t **d_dx, const int16_t **d_dy)
{
    EdState &S = *ed_state_of(c);
    cudaStream_t st = cs_ctx_stream(c);
    if (w < 1 || h < 1 || w > 32767 || h > 32767) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "image size unsupported by the line descriptor");
    const size_t px = (size_t)n_frames * w * h;
    int rc;
    const uint8_t *d_img = imgs;
    if (!imgs_on_device) {
        if ((rc = ed_ensure(c, S.img, (size_t)n_frames * h * stride))) return rc;
        if (cudaMemcpyAsync(S.img.p, imgs, (size_t)n_frames * h * stride, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames failed");
        d_img = (const uint8_t *)S.img.p;
    }
    if ((rc = ed_ensure(c, S.blur, px)) || (rc = ed_ensure(c, S.dx, px * 2)) || (rc = ed_ensure(c, S.dy, px * 2)) || (rc = ed_ensure(c, S.g, px * 2)) ||
        (rc = ed_ensure(c, S.dir, px)) || (rc = ed_ensure(c, S.err, 16)))
        return rc;
    S.head.d_err = (int32_t *)S.err.p;
    cudaMemsetAsync(S.err.p, 0, 16, st);
    const dim3 g_tile((w + EDF_TW - 1) / EDF_TW, (h + EDF_TH - 1) / EDF_TH, n_frames);
    CUtensorMap tm;
    if (cs_ctx_use_tma(c) && channels == 3 && stride == 3 * w && cs_make_tmap_bytes(&tm, d_img, 3 * (int64_t)w, (int64_t)n_frames * h, stride, EDF_BOXW, EDF_TH + 6))
        k_ed_front<true><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, (uint8_t *)S.blur.p, (int16_t *)S.dx.p, (int16_t *)S.dy.p, (int16_t *)S.g.p,
                                                (uint8_t *)S.dir.p, (int32_t *)S.err.p);
    else
        k_ed_front<false><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, (uint8_t *)S.blur.p, (int16_t *)S.dx.p, (int16_t *)S.dy.p, (int16_t *)S.g.p,
                                                 (uint8_t *)S.dir.p, (int32_t *)S.err.p);
    cs_ctx_count_launches(c, 1);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "Sobel-map kernel launch failed");
    S.last_frames = 0; /* the detector's debug views no longer describe these buffers */
    *d_dx = (const int16_t *)S.dx.p;
    *d_dy = (const int16_t *)S.dy.p;
    return ed_check_run(c, S);
}

extern "C" int cs_debug_edlines(cs_ctx *c, int frame, uint8_t *blur, int16_t *dx, int16_t *dy, int16_t *g, uint8_t *dir, int32_t *anchors,
                                int32_t *n_anchors, uint8_t *edge, float *raw_lines, int32_t *n_raw, int cap_raw)
{
    if (!c) return CS_ERR_INVALID_ARG;
    EdState *S = ed_state_of(c);
    if (frame < 0 || frame >= S->last_frames) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad frame index");
    cudaSetDevice(cs_ctx_device(c));
    cudaStreamSynchronize(cs_ctx_stream(c));
    const size_t npx = (size_t)S->last_w * S->last_h;
    if (blur) cudaMemcpy(blur, (uint8_t *)S->blur.p + frame * npx, npx, cudaMemcpyDeviceToHost);
    if (dx) cudaMemcpy(dx, (int16_t *)S->dx.p + frame * npx, npx * 2, cudaMemcpyDeviceToHost);
    if (dy) cudaMemcpy(dy, (int16_t *)S->dy.p + frame * npx, npx * 2, cudaMemcpyDeviceToHost);
    if (g) cudaMemcpy(g, (int16_t *)S->g.p + frame * npx, npx * 2, cudaMemcpyDeviceToHost);
    if (dir) cudaMemcpy(dir, (uint8_t *)S->dir.p + frame * npx, npx, cudaMemcpyDeviceToHost);
    if (edge) {
        int32_t redo = 1;
        if (S->redo.p) cudaMemcpy(&redo, (int32_t *)S->redo.p + frame, 4, cudaMemcpyDeviceToHost);
        if (!redo) { /* routed on the walk graph: the edge map is the set of nodes whose edge flag is set */
            int32_t n_nodes = 0;
            cudaMemcpy(&n_nodes, (int32_t *)S->rowcnt.p + (size_t)frame * (S->last_h + 1) + S->last_h, 4, cudaMemcpyDeviceToHost);
            cudaMemset((uint8_t *)S->edge.p + frame * npx, 0, npx);
            if (n_nodes > 0)
                k_ed_edge_map<<<(n_nodes + 255) / 256, 256>>>((const uint32_t *)S->xy.p + (size_t)frame * S->node_cap, (const uint8_t *)S->flags.p + (size_t)frame * S->node_cap,
                                                              n_nodes, S->last_w, (uint8_t *)S->edge.p + frame * npx);
            cudaDeviceSynchronize();
        }
        cudaMemcpy(edge, (uint8_t *)S->edge.p + frame * npx, npx, cudaMemcpyDeviceToHost);
    }
    int32_t na = 0, nr = 0;
    cudaMemcpy(&na, (int32_t *)S->nanch.p + frame, 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(&nr, (int32_t *)S->nraw.p + frame, 4, cudaMemcpyDeviceToHost);
    if (n_anchors) *n_anchors = na;
    if (n_raw) *n_raw = nr;
    if (anchors) cudaMemcpy(anchors, (int32_t *)S->anchors.p + (size_t)frame * S->anchor_cap, (size_t)std::min(na, S->anchor_cap) * 4, cudaMemcpyDeviceToHost);
    if (raw_lines) cudaMemcpy(raw_lines, (float *)S->raw.p + (size_t)frame * S->cap * 4, (size_t)std::min(nr, std::min(cap_raw, S->cap)) * 16, cudaMemcpyDeviceToHost);
    return cudaGetLastError() == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "debug copy failed");
}
