/*
 * cs_lsd.cu -- line_lbd_detect::detect_filter_lines, LSD flavour, for sm_90a (kernel group (i) of the north star).
 *
 * Replaces, for one octave (the only one filter_lines keeps, line_lbd/class/line_lbd_allclass.cpp:200-207):
 *   LSDDetector::detectImpl                line_lbd/libs/LSDDetector.cpp:153-256
 *   LineSegmentDetectorImpl::flsd & co.    line_lbd/libs/lsd.cpp:440-1154   (LSD_REFINE_ADV, default parameters)
 *   filter_lines + keylines_to_mat         line_lbd/class/line_lbd_allclass.cpp:26-36,200-221
 *
 * Front end (FP64, evaluation order of OpenCV's C paths, -fmad=false), one kernel on 32 x 32 tiles of the scaled frame:
 *   k_lsd_front   cvtColor + the 7 x 7 Gaussian (sigma 0.6/0.8), both passes             lsd.cpp:452-457
 *                 cv::resize(x0.8, INTER_LINEAR) on doubles                              lsd.cpp:459
 *                 2x2 gradient, modulus, fastAtan2 angle                                 lsd.cpp:562-586
 *                 interior tiles' BGR bytes come in by TMA; the blurred and scaled planes stay in shared memory
 *   (no ordering pass: ll_angle's 1024-bin pseudo-ordering, lsd.cpp:588-634, links the pixels by gradient bin, but flsd walks the node
 *   vector by index, lsd.cpp:478-480, i.e. in the raster order the nodes were allocated in -- established in round 2 by compiling the
 *   reference's own lsd.cpp, oracle/ref/; the counting-sort kernels of round 1 are gone)
 *
 * Seed loop (lsd.cpp:476-535).  The reference visits the ordered pixel list one seed at a time; a seed grows a region over the pixels no
 * earlier seed used, so the result is defined by the order -- but only through the `used` map.  It is cut in two:
 *   k_lsd_grow_seq   everything that reads or writes `used`: the raster scan for seeds, region_grow, region2rect, the density test, refine /
 *                    reduce_region_radius (lsd.cpp:478-519), one warp per frame (one 32-thread CTA, 8 KB of shared memory for the region
 *                    list, `used` as a bit per pixel in HBM read through L2).  Emits the candidate rectangles in seed order.  The scan
 *                    reads k_lsd_front's "angle defined" bit plane and the used map, both in row-padded words, 32 words (>= 1024 pixels)
 *                    per step: a word of seeds is defb & ~used.
 *   k_lsd_val_count / k_lsd_val_nfa (six rounds)   rect_improve and the NFA test (lsd.cpp:520-534, 873-1136) read the angle map only: one
 *                    warp per undecided candidate rectangle, all frames at once; a round's up-to-five rectangles counted in one scan of the
 *                    angle map, the binomial tails in a kernel of their own (as ONE kernel, its 6.6 k instructions would not fit the
 *                    instruction cache, and its warps would stall on instruction fetch).
 *   k_lsd_emit       accepted candidates in seed order + the key-line filter.
 * Why this shape: the one-warp loop is bound by instruction issue, not by memory latency; what stops more frames from sharing an SM is the instruction cache, so the sequential kernel is
 * kept small (grow -> rectangle -> density is ONE two-pass loop, 7.4 k instructions instead of 39 k) and everything order-free runs where
 * thousands of warps execute the same code.  An ordered-speculation kernel (many warps per frame claiming pixels by rank) was built and
 * removed: 74 % of the candidates it started were refused and redone (a property of the frames, not of the GPU), it needed ~25
 * barrier-separated rounds per frame, was not faster than one warp per frame where it was timed (not on H100), and emitted duplicate
 * segments on dense frames (git history: k_lsd_grow_par).
 *
 * Inside one candidate the warp parallelises what is order-free (the 3x3 neighbour tests of three region points per step from ONE 16-byte
 * record per pixel, the addends of the ordered sums, rectangle pixel counts over rows, min/max extents, the binomial tail's break tests) and
 * keeps every floating-point accumulation in the reference's order; neighbours whose angle difference is clear of the tolerance by more
 * than the region angle can drift within a round are accepted / rejected without re-deriving the angle per pixel (lsd_region_grow).
 */
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "cs_internal.h"
#include "cs_nfa.cuh"
#include "cs_tma.cuh"

#define LSD_PI 3.1415926535897932384626433832795
#define LSD_NOTDEF (-1024.0)
#define LSD_DEG2RAD (LSD_PI / 180)
#define LSD_3_2_PI ((3 * LSD_PI) / 2)
#define LSD_2PI (2 * LSD_PI)
#define LSD_LN10 2.30258509299404568402
#define LSD_NBINS 1024
#define LSD_CHUNK_ROWS 8
#define LSD_SCALE 0.8 /* lsd.cpp:459; k_lsd_front's tile spans assume it */

#define LSD_CAND_CAP 2048    /* candidate rectangles per frame handed from the seed loop to the validation kernels, until a frame needs more */
#define LSD_SEQ_SCAP 2048    /* region entries k_lsd_grow_seq keeps in shared memory (the rest spill to HBM; small, so that many frames share an SM) */
#define LSD_SEQ_SMEM (LSD_SEQ_SCAP * 4 + 96 * 8) /* its dynamic shared memory: region list + staging of the ordered sums (SCAP even: 8-byte aligned) */
#define LSD_HDR 8            /* ints of a candidate record header in the arena: n1, n2, has_line, x1 y1 x2 y2 (float bits), pad */

namespace {

/* One frame of a batch of frames of different sizes (kMixed instantiations): where its bytes are, its scaled size and flsd's constants for
 * it, and where its planes start.  The host builds the table as prefix sums (lsd_run_mixed); every kernel reads its frame's entry once. */
struct LsdGeom {
    int64_t img_off;                 /* bytes from the batch's base pointer to the frame's first row */
    int32_t w, h, stride, channels;  /* the frame */
    int32_t W, H;                    /* the scaled frame: lrint(w * LSD_SCALE) x lrint(h * LSD_SCALE) */
    int32_t min_reg_size, tile0;     /* flsd's min_reg_size; the frame's first tile in k_lsd_front's flattened tile list */
    double LOG_NT;
    int64_t px_off;                  /* first pixel of the frame in modgrad / angf / pix */
    int64_t bit_off;                 /* first word of the frame in defb / ubits (ceil(W / 32) * H words per frame) */
    int64_t arena_off;               /* first int of the frame in the region-list arena */
    int32_t tiles_x, pad_;           /* k_lsd_front tiles per row of the scaled frame */
};

/* cv2 4.x getGaussianKernel(7, 0.6 / 0.8, CV_64F): lsd.cpp:453 divides, sigma = 0.7499999999999999, not 0.75 */
__constant__ double c_gauss7[7] = {0x1.763496d347532p-13, 0x1.f1e23259cfdc1p-7, 0x1.bfd7fac1bd5a8p-3, 0x1.10562a79786afp-1,
                                   0x1.bfd7fac1bd5a8p-3, 0x1.f1e23259cfdc1p-7, 0x1.763496d347532p-13};

__device__ __forceinline__ int reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = (p < 0) ? -p : 2 * n - 2 - p;
    return p;
}

/* cv::fastAtan2 (degrees) */
__device__ __forceinline__ float fast_atan2(float y, float x)
{
    const float p1 = 0.9997878412794807f * (float)(180 / LSD_PI);
    const float p3 = -0.3258083974640975f * (float)(180 / LSD_PI);
    const float p5 = 0.1555786518463281f * (float)(180 / LSD_PI);
    const float p7 = -0.04432655554792128f * (float)(180 / LSD_PI);
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

/* ---------------------------------------------------------------------------------------- front end */
/* cv::resize(x0.8, INTER_LINEAR) on doubles, the source column / row of one output pixel and its float coefficient (OpenCV's HResize
 * tail: `single` = one tap at the right border).  Both mappings are monotone in the output coordinate. */
__device__ __forceinline__ void lsd_resize_col(int dx, int sw, double inv_scale, int &sx, float &fx, bool &single)
{
    fx = (float)((dx + 0.5) * inv_scale - 0.5);
    sx = (int)floorf(fx);
    fx -= sx;
    single = false;
    if (sx < 0) {
        fx = 0;
        sx = 0;
    }
    if (sx + 1 >= sw) {
        single = true;
        if (sx >= sw - 1) {
            fx = 0;
            sx = sw - 1;
        }
    }
}
__device__ __forceinline__ void lsd_resize_row(int dy, int sh, double inv_scale, int &y0, int &y1, float &fy)
{
    fy = (float)((dy + 0.5) * inv_scale - 0.5);
    const int sy = (int)floorf(fy);
    fy -= sy;
    y0 = (sy >= 0) ? (sy < sh ? sy : sh - 1) : 0;
    y1 = (sy + 1 >= 0) ? (sy + 1 < sh ? sy + 1 : sh - 1) : 0;
}

/* One CTA per 32 x 16 tile of the scaled frame, from the frame's bytes to the seed loop's inputs; nothing in between leaves shared memory:
 *   gray (cvtColor) of the source span the tile needs plus the blur's +-3 halo (reflect-101 at the frame border)     lsd.cpp:452-457
 *   the 7 x 7 Gaussian, horizontal then vertical pass (f64)
 *   the x0.8 bilinear resample of the 33 x 17 scaled pixels the tile's 2 x 2 gradients read                          lsd.cpp:459
 *   modulus, fastAtan2 angle and the 16-byte growth record per pixel                                                  lsd.cpp:562-586
 * Every operation and sum order is the one the separate blur / resize / gradient kernels used, so the planes are bit-identical to them.
 * At inverse scale 1.25, 33 consecutive output columns read exactly 41 + 1 source columns, 17 output rows 21 + 1 source rows: LSF_BW /
 * LSF_BH hold that.  20.5 KB of shared memory and 40 registers: a CTA fits on an SM beside the 21 one-warp CTAs of k_lsd_grow_seq the SM
 * holds when the seed loops of other batches fill the GPU (a 32 x 32 tile, 35.6 KB, does not: the front end then waits for seed loops to
 * finish: bench.py's c3 step, 12 batches in flight, took 10.0 ms instead of 8.8 on an H100 80GB HBM3 at 700 W).
 * kTma: an interior tile's BGR bytes are fetched by the copy engine (one cp.async.bulk.tensor.2d, completion on an mbarrier) instead of
 * three byte loads per pixel; border tiles keep the reflected loads.
 * Outputs: angf and pix for every pixel; modgrad only where the angle is defined (the only pixels the seed loop weights); defb, a bit per
 * pixel "angle defined" in row-padded words (bit x & 31 of word y * ceil(W / 32) + x / 32), which the seed loop scans for seeds.
 * kDebug (cs_debug_lsd, one frame): the scaled plane and the full modgrad plane instead. */
#define LSF_TW 32
#define LSF_TH 16
#define LSF_BW 44 /* blur columns a tile needs: 42 at inverse scale 1.25 */
#define LSF_BH 24 /* blur rows: 22 */
#define LSF_GW (LSF_BW + 6)                 /* gray columns: the blur's halo */
#define LSF_GH (LSF_BH + 6)
#define LSF_BOXW 176                        /* 3 * LSF_GW = 150 bytes of BGR + up to 15 of alignment slack (a TMA box starts at a multiple of 16 bytes) */
#define LSF_P_BYTES (LSF_GH * LSF_BW * 8)   /* the horizontal sums; before them the TMA box, after them the scaled pixels */
static_assert(LSF_GH * LSF_BOXW <= LSF_P_BYTES && (LSF_TH + 1) * (LSF_TW + 1) * 8 <= LSF_P_BYTES, "front-end shared-memory aliasing");
template <bool kTma, bool kDebug, bool kMixed>
__global__ void __launch_bounds__(256) k_lsd_front(const __grid_constant__ CUtensorMap tmap, const uint8_t *__restrict__ img, int w, int h, int stride,
                                                   int channels, int W, int H, double inv_scale, double threshold, double *__restrict__ modgrad,
                                                   float *__restrict__ angf, uint4 *__restrict__ pix, uint32_t *__restrict__ defb,
                                                   double *__restrict__ scaled, int32_t *__restrict__ err_flag, const LsdGeom *__restrict__ geom,
                                                   int n_geom)
{
    static_assert(!(kMixed && (kTma || kDebug)), "a mixed batch has no tensor map and no debug form");
    __shared__ __align__(128) unsigned char s_p[LSF_P_BYTES];
    __shared__ double s_b[LSF_BH][LSF_BW];
    __shared__ uint8_t s_g[LSF_GH][LSF_GW];
    __shared__ __align__(8) unsigned long long s_bar;
    double(*s_h)[LSF_BW] = reinterpret_cast<double(*)[LSF_BW]>(s_p);
    double(*s_sc)[LSF_TW + 1] = reinterpret_cast<double(*)[LSF_TW + 1]>(s_p);
    int f = blockIdx.z, X0 = blockIdx.x * LSF_TW, Y0 = blockIdx.y * LSF_TH;
    const int tid = threadIdx.x;
    const uint8_t *frame = img + (size_t)f * h * stride;
    if constexpr (kMixed) {
        /* blockIdx.x indexes the tiles of every frame, frame after frame: the frame is the last one whose first tile is <= it */
        const int t = blockIdx.x;
        int lo = 0, hi = n_geom - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (geom[mid].tile0 <= t)
                lo = mid;
            else
                hi = mid - 1;
        }
        const LsdGeom &G = geom[lo];
        f = lo;
        w = G.w;
        h = G.h;
        stride = G.stride;
        channels = G.channels;
        W = G.W;
        H = G.H;
        const int lt = t - G.tile0, ty = lt / G.tiles_x;
        X0 = (lt - ty * G.tiles_x) * LSF_TW;
        Y0 = ty * LSF_TH;
        frame = img + G.img_off;
        modgrad += G.px_off;
        angf += G.px_off;
        pix += G.px_off;
        defb += G.bit_off;
    }
    /* the scaled pixels [X0, xl] x [Y0, yl] and the blur span [bx0, bx0 + bw) x [by0, by0 + bh) they read */
    const int xl = min(X0 + LSF_TW, W - 1), yl = min(Y0 + LSF_TH, H - 1);
    int bx0, bx1, by0, by1, t0;
    {
        float ft;
        bool single;
        lsd_resize_col(X0, w, inv_scale, bx0, ft, single);
        lsd_resize_col(xl, w, inv_scale, bx1, ft, single);
        bx1 += single ? 0 : 1;
        lsd_resize_row(Y0, h, inv_scale, by0, t0, ft);
        lsd_resize_row(yl, h, inv_scale, t0, by1, ft);
    }
    const int bw = bx1 - bx0 + 1, bh = by1 - by0 + 1;
    const bool interior = kTma && bx0 - 3 >= 0 && bx1 + 3 <= w - 1 && by0 - 3 >= 0 && by1 + 3 <= h - 1;
    if (interior) {
        uint8_t *s_rgb = s_p;
        if (tid == 0) cs_mbar_init(&s_bar);
        __syncthreads();
        const int bxb = 3 * (bx0 - 3), boff = bxb & 15;
        if (tid == 0) cs_tma_load_2d(&tmap, s_rgb, &s_bar, bxb - boff, f * h + by0 - 3, LSF_GH * LSF_BOXW);
        if (!cs_mbar_wait(&s_bar, 0) && tid == 0) atomicOr(err_flag, 8);
        for (int i = tid; i < LSF_GH * LSF_GW; i += 256) {
            const int r = i / LSF_GW, c = i - r * LSF_GW;
            if (r >= bh + 6 || c >= bw + 6) continue;
            const uint8_t *q = &s_rgb[r * LSF_BOXW + boff + 3 * c];
            s_g[r][c] = (uint8_t)((q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15);
        }
    } else
        for (int i = tid; i < LSF_GH * LSF_GW; i += 256) {
            const int r = i / LSF_GW, c = i - r * LSF_GW;
            if (r >= bh + 6 || c >= bw + 6) continue;
            const int yy = reflect101(by0 - 3 + r, h), xx = reflect101(bx0 - 3 + c, w);
            const uint8_t *q = frame + (size_t)yy * stride;
            uint32_t g;
            if (channels == 3) {
                q += 3 * xx;
                g = (q[0] * 3735u + q[1] * 19235u + q[2] * 9798u + (1u << 14)) >> 15;
            } else
                g = q[xx];
            s_g[r][c] = (uint8_t)g;
        }
    __syncthreads();
    for (int i = tid; i < LSF_GH * LSF_BW; i += 256) {
        const int r = i / LSF_BW, c = i - r * LSF_BW;
        if (r >= bh + 6 || c >= bw) continue;
        double s = 0;
#pragma unroll
        for (int k = 0; k < 7; k++) {
            const double t = c_gauss7[k] * (double)(int)s_g[r][c + k];
            s = (k == 0) ? t : s + t;
        }
        s_h[r][c] = s;
    }
    __syncthreads();
    for (int i = tid; i < LSF_BH * LSF_BW; i += 256) {
        const int r = i / LSF_BW, c = i - r * LSF_BW;
        if (r >= bh || c >= bw) continue;
        double s = c_gauss7[3] * s_h[r + 3][c];
#pragma unroll
        for (int k = 1; k <= 3; k++) s += c_gauss7[3 + k] * (s_h[r + 3 + k][c] + s_h[r + 3 - k][c]);
        s_b[r][c] = s;
    }
    __syncthreads(); /* s_h is dead: s_sc takes its place */
    for (int i = tid; i < (LSF_TH + 1) * (LSF_TW + 1); i += 256) {
        const int r = i / (LSF_TW + 1), c = i - r * (LSF_TW + 1);
        if (Y0 + r > yl || X0 + c > xl) continue;
        int sx, y0, y1;
        float fx, fy;
        bool single;
        lsd_resize_col(X0 + c, w, inv_scale, sx, fx, single);
        lsd_resize_row(Y0 + r, h, inv_scale, y0, y1, fy);
        const double *S0 = s_b[y0 - by0], *S1 = s_b[y1 - by0];
        const int cx = sx - bx0;
        const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
        double r0, r1;
        if (!single) {
            r0 = S0[cx] * a0 + S0[cx + 1] * a1;
            r1 = S1[cx] * a0 + S1[cx + 1] * a1;
        } else {
            r0 = S0[cx] * 1.0;
            r1 = S1[cx] * 1.0;
        }
        s_sc[r][c] = r0 * b0 + r1 * b1;
    }
    __syncthreads();
    /* a warp covers one 32-pixel tile row (LSF_TW = 32, X0 a multiple of 32): one ballot makes the row's word of the defined-angle plane */
    const int WW = (W + 31) >> 5;
    for (int i = tid; i < LSF_TH * LSF_TW; i += 256) {
        const int r = i / LSF_TW, c = i - r * LSF_TW;
        const int x = X0 + c, y = Y0 + r;
        float deg = -1.f; /* pixels outside the frame vote 0 */
        if (x < W && y < H) {
            const size_t p = kMixed ? (size_t)y * W + x : ((size_t)f * H + y) * W + x;
            double norm = 0;
            if (x < W - 1 && y < H - 1) {
                const double DA = s_sc[r + 1][c + 1] - s_sc[r][c];
                const double BC = s_sc[r][c + 1] - s_sc[r + 1][c];
                const double gx = DA + BC, gy = DA - BC;
                norm = sqrt((gx * gx + gy * gy) / 4);
                if (!kDebug && !(norm <= threshold)) deg = fast_atan2((float)gx, (float)(-gy));
            }
            if (kDebug) {
                scaled[p] = s_sc[r][c];
                modgrad[p] = norm;
            } else {
                angf[p] = deg;
                uint4 rec = make_uint4(__float_as_uint(deg), 0u, 0u, 0u);
                if (deg >= 0.f) {
                    modgrad[p] = norm;
                    const double ang = (double)deg * LSD_DEG2RAD;
                    const double af = (double)(float)ang;
                    rec.y = __float_as_uint((float)cos(af));
                    rec.z = __float_as_uint((float)sin(af));
                }
                pix[p] = rec;
            }
        }
        if (!kDebug) {
            const uint32_t bits = __ballot_sync(0xffffffffu, deg >= 0.f);
            if (c == 0 && y < H) defb[(kMixed ? (size_t)y : (size_t)f * H + y) * WW + (X0 >> 5)] = bits;
        }
    }
}

/* ---------------------------------------------------------------------------------------- the seed loop */
/* cycle counters of the seed loop's phases (diagnostics, cs_debug_lsd_prof): grow, region2rect, refine, raster scan, used-map re-reads,
 * seeds grown, whole kernel, region pixels, region lists past the shared-memory part; then the per-seed hand-off (used-word re-read and
 * seed mask), the density decision and candidate store, reduce_region_radius (with its region2rect calls), seeds that reach region2rect,
 * refines, reduce iterations, and the sizes region2rect sees as three 21-bit counts (<= 32, <= 64, > 64 points) */
__device__ unsigned long long g_lsd_prof[16];
/* only in the instantiation for a profiling context (cs_set_profiling bit 0, kProf): a run that is not being measured pays neither the
 * clock reads nor the atomics of thousands of warps on the same sixteen words */
#define LSD_PROF_T0() const long long prof_t0__ = kProf ? clock64() : 0ll
#define LSD_PROF_ADD(slot)                                                                         \
    do {                                                                                           \
        if (kProf && (threadIdx.x & 31) == 0) atomicAdd(&g_lsd_prof[slot], (unsigned long long)(clock64() - prof_t0__)); \
    } while (0)
#define LSD_PROF_COUNT(slot, v)                                                    \
    do {                                                                           \
        if (kProf && (threadIdx.x & 31) == 0) atomicAdd(&g_lsd_prof[slot], (unsigned long long)(v)); \
    } while (0)
#define LSD_PROF_RECT_SIZE(n) LSD_PROF_COUNT(15, (n) <= 32 ? 1ull : (n) <= 64 ? 1ull << 21 : 1ull << 42)

/* k_lsd_grow_seq's dynamic shared memory (LSD_SEQ_SMEM): the first LSD_SEQ_SCAP entries of the region list (LsdReg), then 96 doubles
 * that stage the addends of the ordered sums.  Named here rather than handed around as a pointer in LsdReg / LsdFrame: those structs go
 * by reference to out-of-line functions, and a pointer that passes through them is a generic address, so every region-list read on the
 * growth chain was a generic load (LD) instead of a shared-memory load (LDS). */
extern __shared__ __align__(8) int s_seq[];
__device__ __forceinline__ double *lsd_stage() { return reinterpret_cast<double *>(s_seq + LSD_SEQ_SCAP); }

struct LsdFrame {
    int W, H;
    uint4 *pix;            /* {deg, cos, sin, 0}: one 16-byte record per neighbour test */
    const float *angf;     /* deg plane for the rectangle scans */
    const double *modgrad;
    double LOG_NT;
    /* the `used` map as a bit per pixel (HBM, read and written through L2 only, so that it costs no shared memory: the seed loop issues
     * is bound by instruction issue, and the more frames share an SM the better), in the row-padded words of the defined-angle plane:
     * bit x & 31 of word y * WW + x / 32, so that a word of seeds is defb & ~used */
    uint32_t *ubits;
    int WW; /* words per row: ceil(W / 32) */
    /* the word of pixel (y, x) and its bit: every access to the used map goes through here */
    __device__ __forceinline__ uint32_t *used_at(int y, int x, uint32_t &bit) const
    {
        bit = 1u << (x & 31);
        return ubits + y * WW + (x >> 5);
    }
    struct LsdSpan *span; /* k_lsd_val_count: room for five row-span records per warp (shared memory) */
    const double *lgam; /* log_gamma of small integers (cs_nfa.cuh) */
    unsigned long long wmagic; /* ceil(2^40 / W): row of a pixel address without an integer division (exact for addresses < 2^20 .. 2^30 / W) */
    __device__ __forceinline__ int row_of(int addr) const { return (int)(((unsigned long long)(unsigned)addr * wmagic) >> 40); }
};

/* the region list of the candidate a warp works on: the first LSD_SEQ_SCAP entries in shared memory (s_seq), the rest in HBM.  Only this
 * warp writes and reads its entries, so plain loads see the plain stores of put() once a __syncwarp() lies between them; an L2-only load
 * (__ldcg, a strong GPU-scope load in SASS) there, although it almost never executes, made region2rect and reduce_region_radius, which
 * read the list at every point, measurably slower (DESIGN.md section 8). */
struct LsdReg {
    int *g;
    int cap;
    __device__ __forceinline__ int get(int i) const { return i < LSD_SEQ_SCAP ? s_seq[i] : g[i]; }
    __device__ __forceinline__ void put(int i, int v) const
    {
        if (i < LSD_SEQ_SCAP)
            s_seq[i] = v;
        else
            g[i] = v;
    }
};

__device__ __forceinline__ void lsd_prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

struct LsdRect {
    double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p;
};

__device__ __forceinline__ double lsd_dist_sq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }
__device__ __forceinline__ double lsd_dist(double x1, double y1, double x2, double y2) { return sqrt(lsd_dist_sq(x1, y1, x2, y2)); }
__device__ __forceinline__ double lsd_angle_diff_signed(double a, double b)
{
    double diff = a - b;
    while (diff <= -LSD_PI) diff += LSD_2PI;
    while (diff > LSD_PI) diff -= LSD_2PI;
    return diff;
}
__device__ __forceinline__ bool lsd_double_equal(double a, double b)
{
    if (a == b) return true;
    const double abs_diff = fabs(a - b);
    const double aa = fabs(a), bb = fabs(b);
    double abs_max = (aa > bb) ? aa : bb;
    if (abs_max < DBL_MIN) abs_max = DBL_MIN;
    return (abs_diff / abs_max) <= (100.0 * DBL_EPSILON);
}
/* lsd.cpp:1138-1154 on the float level-line angle in degrees (negative = NOTDEF).  The decision is the reference's double comparison; a
 * float evaluation of the same difference (error < 1e-5 rad) settles every case that is not within 2e-4 rad of the tolerance, so the
 * double arithmetic (half-rate pipe, and this test runs for every pixel of every rectangle scan and every neighbour of every growth step)
 * is only executed on the rare borderline pixel. */
__device__ __forceinline__ bool lsd_aligned_deg(float deg, double theta, double prec)
{
    if (deg < 0.f) return false;
    {
        float nf = fabsf((float)theta - deg * 0.017453292f);
        if (nf > 4.712389f) nf = fabsf(nf - 6.2831855f);
        const float pf = (float)prec;
        if (nf < pf - 2e-4f) return true;
        if (nf > pf + 2e-4f) return false;
    }
    const double a = (double)deg * LSD_DEG2RAD;
    double n_theta = theta - a;
    if (n_theta < 0) n_theta = -n_theta;
    if (n_theta > LSD_3_2_PI) {
        n_theta -= LSD_2PI;
        if (n_theta < 0) n_theta = -n_theta;
    }
    return n_theta <= prec;
}

__device__ __noinline__ double lsd_log_gamma(double x)
{
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
    double b = 0;
    for (int n = 0; n < 7; ++n) {
        a -= log(x + (double)n);
        b += q[n] * pow(x, (double)n);
    }
    return a + log(b);
}

/* lsd.cpp:1100-1136; called with different (n, k, p) on different lanes */
__device__ __noinline__ double lsd_nfa(int n, int k, double p, double LOG_NT)
{
    if (n == 0 || k == 0) return -LOG_NT;
    if (n == k) return -LOG_NT - (double)n * log10(p);
    const double p_term = p / (1 - p);
    const double log1term = ((double)n + 1) - lsd_log_gamma((double)k + 1) - lsd_log_gamma((double)(n - k) + 1) + (double)k * log(p) + (double)(n - k) * log(1.0 - p);
    double term = exp(log1term);
    if (lsd_double_equal(term, 0)) {
        if (k > n * p) return -log1term / LSD_LN10 - LOG_NT;
        return -LOG_NT;
    }
    double bin_tail = term;
    const double tolerance = 0.1;
    for (int i = k + 1; i <= n; ++i) {
        const double bin_term = (double)(n - i + 1) / (double)i;
        const double mult_term = bin_term * p_term;
        term *= mult_term;
        bin_tail += term;
        if (bin_term < 1) {
            const double err = term * ((1 - pow(mult_term, (double)(n - i + 1))) / (1 - mult_term) - 1);
            if (err < tolerance * fabs(-log10(bin_tail) - LOG_NT) * bin_tail) break;
        }
    }
    return -log10(bin_tail) - LOG_NT;
}

/* lsd.cpp:637-688, one warp.  Three region points per round, their 3 x 3 neighbourhoods on lanes 0..26 in the reference's (point, yy, xx)
 * order, so "the first lane" is "the next pixel the reference would test".
 *
 * The reference updates the region angle after EVERY added pixel and tests the next neighbour against the new angle: a chain of
 * fastAtan2 -> compare -> add per pixel.  Most of those tests cannot come out differently, though.  Let S be the running sum of unit
 * vectors, L = |S|.  A pixel that passes the test lies within A = prec + D of the (computed) region direction, so adding it turns S by at
 * most sin(A + e) / L <= (A + e) / L and does not shorten it (e <= 1e-3 rad: error of the fastAtan2 polynomial, measured 1.7e-4).  With
 * at most m additions in this round, every angle the round will test against is within
 *     D = m (prec + 0.2 + e) / L + 2 e + float slack
 * of the angle at the start of the round (D <= 0.2 required).  A neighbour whose difference from the round-start angle is below prec - D
 * is accepted whenever its turn comes, one above prec + D is rejected whenever: neither needs the angle at its turn.  Only the pixels in
 * between are tested the reference's way, against fastAtan2 of the sums as they stand at their turn (the sums are always added in the
 * reference's order, in float, so they are the reference's bits).  prec + D stays below pi / 2, where the reference's wrapped difference
 * (lsd.cpp:1138-1154) equals the circular distance or exceeds pi / 2, so the argument holds across the 0 / 2 pi seam.
 */
__device__ void lsd_region_grow(const LsdFrame &F, const LsdReg &R, int base, int s_addr, int &reg_size, double &reg_angle, double prec)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    float reg_deg = F.angf[s_addr];
    reg_angle = (double)reg_deg * LSD_DEG2RAD;
    float sumdx = (float)cos(reg_angle);
    float sumdy = (float)sin(reg_angle);
    __syncwarp(); /* every lane is done reading the previous region's list before its slots are written again */
    if (lane == 0) {
        const int sy = F.row_of(s_addr);
        uint32_t bit;
        uint32_t *w = F.used_at(sy, s_addr - sy * F.W, bit);
        atomicOr(w, bit);
        R.put(base, s_addr);
    }
    reg_size = 1;
    __syncwarp();
    const int grp = lane / 9, kk = lane - grp * 9;
    const int ky = kk / 3 - 1, kx = kk - (kk / 3) * 3 - 1; /* (yy, xx) in the reference's loop order */
    const float precf = (float)prec;
    const unsigned lt_mask = (1u << lane) - 1u;
    for (int i = 0; i < reg_size;) {
        const int navail = min(3, reg_size - i);
        bool cand = false;
        int c_addr = -1;
        float deg = -1.f, csx = 0.f, csy = 0.f;
        if (grp < navail) {
            const int pa = R.get(base + i + grp);
            const int py = F.row_of(pa), px = pa - py * F.W;
            const int yy = py + ky, xx = px + kx;
            if (yy >= 0 && yy < F.H && xx >= 0 && xx < F.W) {
                c_addr = yy * F.W + xx;
                uint32_t ubit;
                const uint32_t *uw_p = F.used_at(yy, xx, ubit);
                const uint4 r = __ldg(F.pix + c_addr); /* {deg, cos, sin, -}: read-only */
                const uint32_t uw = __ldcg(uw_p);      /* issued together with the record: one round trip per round, not two */
                deg = __uint_as_float(r.x);
                if (deg >= 0.f && !(uw & ubit)) {
                    cand = true;
                    csx = __uint_as_float(r.y);
                    csy = __uint_as_float(r.z);
                }
            }
        }
        unsigned maybe = __ballot_sync(FULL, cand);
        if (maybe) {
            /* the float difference from the round-start angle (error < 1e-5 rad) and the drift bound D */
            float nf = fabsf(reg_deg * 0.017453292f - deg * 0.017453292f);
            if (nf > 4.712389f) nf = fabsf(nf - 6.2831855f);
            const float inv_l = rsqrtf(sumdx * sumdx + sumdy * sumdy) * 1.001f;
            const float per_add = (precf + 0.201f) * inv_l;
            unsigned sure = 0u;
            float D = (float)__popc(maybe) * per_add + 0.0022f;
            if (D <= 0.2f && precf + D < 1.5f) {
                const unsigned m1 = __ballot_sync(FULL, cand && nf < precf + D); /* everything else is rejected whatever the angle */
                D = (float)__popc(m1) * per_add + 0.0022f;                          /* at most popc(m1) additions this round */
                sure = __ballot_sync(FULL, cand && nf < precf - D);
                maybe = __ballot_sync(FULL, cand && nf < precf + D);
            }
            unsigned accepted = 0u;
            bool stale = false; /* sums changed since reg_deg was computed */
            while (maybe) {
                const int fl = __ffs(maybe) - 1;
                maybe &= ~(1u << fl);
                if (!((sure >> fl) & 1u)) {
                    /* the reference's own test, at this pixel's turn */
                    if (stale) {
                        reg_deg = fast_atan2(sumdy, sumdx);
                        stale = false;
                    }
                    const bool ok = lsd_aligned_deg(deg, (double)reg_deg * LSD_DEG2RAD, prec);
                    if (!((__ballot_sync(FULL, ok) >> fl) & 1u)) continue;
                }
                const int addrf = __shfl_sync(FULL, c_addr, fl);
                /* cos(float(angle)), sin(float(angle)): precomputed per pixel by k_lsd_front (pinned to the correctly rounded float) */
                sumdx += __shfl_sync(FULL, csx, fl);
                sumdy += __shfl_sync(FULL, csy, fl);
                stale = true;
                accepted |= 1u << fl;
                maybe &= ~__ballot_sync(FULL, c_addr == addrf); /* the same pixel seen from a later point of this round */
            }
            if (accepted) {
                if ((accepted >> lane) & 1u) {
                    R.put(base + reg_size + __popc(accepted & lt_mask), c_addr);
                    const int cy = F.row_of(c_addr); /* not kept from the gather: two registers fewer across the accept loop */
                    uint32_t ubit;
                    uint32_t *uw_p = F.used_at(cy, c_addr - cy * F.W, ubit);
                    atomicOr(uw_p, ubit);
                    /* this pixel is a region point now: its 3 x 3 neighbourhood will be gathered a few rounds from here.  Ask L2 for the three
                     * 48-byte runs of records (a DRAM miss is ~3x an L2 hit, and the gather is on the warp's critical path). */
                    const uint4 *q = F.pix + c_addr - 1;
                    if (c_addr >= F.W + 1) lsd_prefetch_l2(q - F.W);
                    lsd_prefetch_l2(q);
                    if (c_addr + F.W + 1 < F.W * F.H) lsd_prefetch_l2(q + F.W);
                }
                reg_size += __popc(accepted);
                if (stale) reg_deg = fast_atan2(sumdy, sumdx);
                __syncwarp();
            }
        }
        i += navail;
    }
    reg_angle = (double)reg_deg * LSD_DEG2RAD;
}

/* Sums over the region in the reference's order (the order decides the last bits of a double sum): 32 region points at a time, every lane
 * computes the addend(s) of ITS point -- the products round the same wherever they are computed -- and stages them in shared memory
 * (lsd_stage(), 96 doubles); then the additions run as one chain over the staged values, read as broadcasts. */
/* lsd.cpp:690-784 */
__device__ void lsd_region2rect(const LsdFrame &F, const LsdReg &R, int base, int reg_size, double reg_angle, double prec, double p, LsdRect &rec)
{
    const int lane = threadIdx.x & 31;
    double *st = lsd_stage();
    double x = 0, y = 0, sum = 0;
    for (int i0 = 0; i0 < reg_size; i0 += 32) {
        const int n = min(32, reg_size - i0);
        __syncwarp();
        if (lane < n) {
            const int addr = R.get(base + i0 + lane);
            const double weight = F.modgrad[addr];
            const int ry = F.row_of(addr), rx = addr - ry * F.W;
            st[lane] = (double)rx * weight;
            st[32 + lane] = (double)ry * weight;
            st[64 + lane] = weight;
        }
        __syncwarp();
        for (int j = 0; j < n; j++) {
            x += st[j];
            y += st[32 + j];
            sum += st[64 + j];
        }
    }
    x /= sum;
    y /= sum;
    /* get_theta */
    double Ixx = 0.0, Iyy = 0.0, Ixy = 0.0;
    for (int i0 = 0; i0 < reg_size; i0 += 32) {
        const int n = min(32, reg_size - i0);
        __syncwarp();
        if (lane < n) {
            const int addr = R.get(base + i0 + lane);
            const double weight = F.modgrad[addr];
            const int ry = F.row_of(addr), rx = addr - ry * F.W;
            const double ddx = (double)rx - x, ddy = (double)ry - y;
            st[lane] = ddy * ddy * weight;
            st[32 + lane] = ddx * ddx * weight;
            st[64 + lane] = ddx * ddy * weight;
        }
        __syncwarp();
        for (int j = 0; j < n; j++) {
            Ixx += st[j];
            Iyy += st[32 + j];
            Ixy -= st[64 + j];
        }
    }
    const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
    double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)fast_atan2((float)(lambda - Ixx), (float)Ixy) : (double)fast_atan2((float)Ixy, (float)(lambda - Iyy));
    theta *= LSD_DEG2RAD;
    if (fabs(lsd_angle_diff_signed(theta, reg_angle)) > prec) theta += LSD_PI;
    const double dx = cos(theta), dy = sin(theta);
    /* extents: min / max are order-free, so lanes split the region */
    double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
    for (int i = lane; i < reg_size; i += 32) {
        const int addr = R.get(base + i);
        const int ry = F.row_of(addr), rx = addr - ry * F.W;
        const double regdx = (double)rx - x, regdy = (double)ry - y;
        const double l = regdx * dx + regdy * dy;
        const double w = -regdx * dy + regdy * dx;
        l_max = fmax(l_max, l);
        l_min = fmin(l_min, l);
        w_max = fmax(w_max, w);
        w_min = fmin(w_min, w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        l_max = fmax(l_max, __shfl_xor_sync(0xffffffffu, l_max, o));
        l_min = fmin(l_min, __shfl_xor_sync(0xffffffffu, l_min, o));
        w_max = fmax(w_max, __shfl_xor_sync(0xffffffffu, w_max, o));
        w_min = fmin(w_min, __shfl_xor_sync(0xffffffffu, w_min, o));
    }
    rec.x1 = x + l_min * dx;
    rec.y1 = y + l_min * dy;
    rec.x2 = x + l_max * dx;
    rec.y2 = y + l_max * dy;
    rec.width = w_max - w_min;
    rec.x = x;
    rec.y = y;
    rec.theta = theta;
    rec.dx = dx;
    rec.dy = dy;
    rec.prec = prec;
    rec.p = p;
    if (rec.width < 1.0) rec.width = 1.0;
}

__device__ __noinline__ void lsd_region2rect_cold(const LsdFrame &F, const LsdReg &R, int base, int reg_size, double reg_angle, double prec, double p, LsdRect &rec);

/* lsd.cpp:834-871.  The reference removes the points outside the radius in place: a removed point at i takes the last point of the list
 * and i is tested again.  That fixes the order later sums run in, and it has a closed form: with K points kept, a kept point at i < K
 * stays at i, and the removed points below K ("holes", ascending) take the kept points at K and above, last one first.  The warp tests 32
 * points at a time and moves up to 32 points per step, pairing holes from the bottom with kept points from the top.
 * Returns 0 ok, 3 region rejected. */
template <bool kProf>
__device__ __noinline__ int lsd_reduce_region_radius(const LsdFrame &F, const LsdReg &R, int base, int &reg_size, double reg_angle, double prec, double p,
                                        LsdRect &rec, double density, double density_th)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u, gt_mask = ~((2u << lane) - 1u);
    int *st = reinterpret_cast<int *>(lsd_stage());
    const int a0 = R.get(base);
    const double xc = (double)(a0 - F.row_of(a0) * F.W), yc = (double)F.row_of(a0);
    const double radSq1 = lsd_dist_sq(xc, yc, rec.x1, rec.y1), radSq2 = lsd_dist_sq(xc, yc, rec.x2, rec.y2);
    double radSq = radSq1 > radSq2 ? radSq1 : radSq2;
    auto outside = [&](int addr) {
        const int ay = F.row_of(addr), ax = addr - ay * F.W;
        return lsd_dist_sq(xc, yc, (double)ax, (double)ay) > radSq;
    };
    while (density < density_th) {
        radSq *= 0.75 * 0.75;
        const int rs = reg_size;
        /* release the points outside the radius and count the ones kept */
        int K = 0;
        for (int i0 = 0; i0 < rs; i0 += 32) {
            bool out = false;
            if (i0 + lane < rs) {
                const int addr = R.get(base + i0 + lane);
                out = outside(addr);
                if (out) {
                    const int ay = F.row_of(addr);
                    uint32_t bit;
                    uint32_t *w = F.used_at(ay, addr - ay * F.W, bit);
                    atomicAnd(w, ~bit);
                }
            }
            K += __popc(__ballot_sync(FULL, i0 + lane < rs && !out));
        }
        /* fill the holes below K; hm: holes of chunk hc not filled yet, dm: kept points of chunk dc (>= K) not moved yet */
        int hc = -32, dc = (((rs - 1) >> 5) + 1) << 5, dval = 0;
        unsigned hm = 0u, dm = 0u;
        for (;;) {
            while (hm == 0u && hc + 32 < K) {
                hc += 32;
                hm = __ballot_sync(FULL, hc + lane < K && outside(R.get(base + hc + lane)));
            }
            if (hm == 0u) break;
            while (dm == 0u) { /* as many kept points at K and above as holes below it: one is left while a hole is */
                dc -= 32;
                const int i = dc + lane;
                dval = i < rs ? R.get(base + i) : 0;
                dm = __ballot_sync(FULL, i >= K && i < rs && !outside(dval));
            }
            const int t = min(__popc(hm), __popc(dm));
            const bool give = ((dm >> lane) & 1u) && __popc(dm & gt_mask) < t;
            const bool take = ((hm >> lane) & 1u) && __popc(hm & lt_mask) < t;
            __syncwarp();
            if (give) st[__popc(dm & gt_mask)] = dval;
            __syncwarp();
            if (take) R.put(base + hc + lane, st[__popc(hm & lt_mask)]);
            hm &= ~__ballot_sync(FULL, take);
            dm &= ~__ballot_sync(FULL, give);
        }
        reg_size = K;
        __syncwarp();
        LSD_PROF_COUNT(14, 1);
        if (reg_size < 2) return 3;
        LSD_PROF_RECT_SIZE(reg_size);
        lsd_region2rect_cold(F, R, base, reg_size, reg_angle, prec, p, rec);
        density = (double)reg_size / (lsd_dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
    }
    return 0;
}

/* lsd.cpp:977-1098 with the vendored slips kept: the (total, aligned) pixel counts of a rectangle.  The edge stepping of the
 * reference adds integer-valued steps (its slopes are int / int divisions) to integer starts, once per row INSIDE the image, so the
 * span of a row has a closed form (LsdSpan) and rows are scanned by separate lanes. */
struct LsdSpan {
    int mx, ly, ry, y0, y1; /* start column, the rows where the left / right edge changes slope, first and last row inside the image */
    int fl, sl, fr, sr;     /* the four integer steps */
};

__device__ void lsd_span_setup(const LsdFrame &F, const LsdRect &rec, LsdSpan &P)
{
    const double half_width = rec.width / 2.0;
    const double dyhw = rec.dy * half_width, dxhw = rec.dx * half_width;
    int ox[4], oy[4];
    ox[0] = (int)(rec.x1 - dyhw);
    oy[0] = (int)(rec.y1 + dxhw);
    ox[1] = (int)(rec.x2 - dyhw);
    oy[1] = (int)(rec.y2 + dxhw);
    ox[2] = (int)(rec.x2 + dyhw);
    oy[2] = (int)(rec.y2 - dxhw);
    ox[3] = (int)(rec.x1 + dyhw);
    oy[3] = (int)(rec.y1 - dxhw);
    /* sort by (x, y) */
#pragma unroll
    for (int i = 1; i < 4; i++) {
        const int vx = ox[i], vy = oy[i];
        int j = i - 1;
        while (j >= 0 && ((vx == ox[j]) ? (vy < oy[j]) : (vx < ox[j]))) {
            ox[j + 1] = ox[j];
            oy[j + 1] = oy[j];
            j--;
        }
        ox[j + 1] = vx;
        oy[j + 1] = vy;
    }
    int imin = 0, imax = 0;
    for (int i = 1; i < 4; ++i) {
        if (oy[imin] > oy[i]) imin = i;
        if (oy[imax] < oy[i]) imax = i;
    }
    unsigned taken = 1u << imin;
    int ileft = -1;
    for (int i = 0; i < 4; ++i)
        if (!((taken >> i) & 1u)) {
            if (ileft < 0)
                ileft = i;
            else if (ox[ileft] > ox[i])
                ileft = i;
        }
    taken |= 1u << ileft;
    int iright = -1;
    for (int i = 0; i < 4; ++i)
        if (!((taken >> i) & 1u)) {
            if (iright < 0)
                iright = i;
            else if (ox[iright] < ox[i])
                iright = i;
        }
    taken |= 1u << iright;
    int itail = -1;
    for (int i = 0; i < 4; ++i)
        if (!((taken >> i) & 1u)) {
            if (itail < 0)
                itail = i;
            else if (ox[itail] > ox[i])
                itail = i;
        }
    const int mx = ox[imin], my = oy[imin], lx = ox[ileft], ly = oy[ileft], rx = ox[iright], ry = oy[iright], tx = ox[itail];
    P.mx = mx;
    P.ly = ly;
    P.ry = ry;
    P.fl = (my != ly) ? (mx - lx) / (my - ly) : 0;
    P.sl = (ly != tx) ? (lx - tx) / (ly - tx) : 0;
    P.fr = (my != ry) ? (mx - rx) / (my - ry) : 0;
    P.sr = (ry != tx) ? (rx - tx) / (ry - tx) : 0;
    /* rows outside the image skip the edge stepping too (as the reference): only rows y0..y1 count */
    P.y0 = max(my, 0);
    P.y1 = min(oy[imax], F.H - 1);
}

/* the columns [lo, hi] of row y (y0 <= y <= y1); empty when hi < lo */
__device__ __forceinline__ void lsd_span_row(const LsdSpan &P, int y, int W, int &lo, int &hi)
{
    /* steps added before row y: one per earlier inside row y' in [y0, y); row y' adds the second slope iff y' >= ly (ry) */
    const long long n_l2 = (long long)max(0, y - max(P.ly, P.y0)), n_l1 = (long long)(y - P.y0) - n_l2;
    const long long n_r2 = (long long)max(0, y - max(P.ry, P.y0)), n_r1 = (long long)(y - P.y0) - n_r2;
    const long long left_x = (long long)P.mx + n_l1 * (long long)P.fl + n_l2 * (long long)P.sl;
    const long long right_x = (long long)P.mx + n_r1 * (long long)P.fr + n_r2 * (long long)P.sr;
    lo = (int)(left_x > 0 ? left_x : 0);
    hi = (int)(right_x < (long long)(W - 1) ? right_x : (long long)(W - 1));
}

__device__ void lsd_rect_count(const LsdFrame &F, const LsdRect &rec, int &total_pts, int &alg_pts)
{
    const int lane = threadIdx.x & 31;
    LsdSpan P;
    lsd_span_setup(F, rec, P);
    int tot = 0, alg = 0;
    /* lanes over rows AND over the pixels of a row: G lanes share a row, G the largest power of two with rows * G <= 32 (a nearly horizontal
     * segment has a handful of long rows, a nearly vertical one many short rows) */
    const int n_rows = P.y1 - P.y0 + 1;
    int G = 1;
    while (G < 32 && n_rows * G * 2 <= 32) G <<= 1;
    const int rows_per_step = 32 / G, sub = lane & (G - 1), rsel = lane / G;
    for (int yb = P.y0; yb <= P.y1; yb += rows_per_step) {
        const int y = yb + rsel;
        if (y > P.y1) continue;
        int lo, hi;
        lsd_span_row(P, y, F.W, lo, hi);
        if (hi >= lo) {
            if (sub == 0) tot += hi - lo + 1;
            const float *row = F.angf + (size_t)y * F.W;
            for (int x = lo + sub; x <= hi; x += G) alg += lsd_aligned_deg(row[x], rec.theta, rec.prec) ? 1 : 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tot += __shfl_xor_sync(0xffffffffu, tot, o);
        alg += __shfl_xor_sync(0xffffffffu, alg, o);
    }
    total_pts = tot;
    alg_pts = alg;
}

/* The (total, aligned) counts of the up to five rectangles of one rect_improve phase in ONE scan of the angle map.  Within a phase the
 * rectangles share the direction theta and differ either in the tolerance only (lsd.cpp:889-903, 957-972: p halved, same geometry) or in
 * the geometry only (lsd.cpp:905-955: width reduced / one side moved, same tolerance): the level-line angle of a pixel is loaded and
 * compared once, the per-rectangle part is a threshold or a column-range test.  The spans are built by lanes 0..n-1 in parallel and
 * shared through F.span (shared memory, 5 LsdSpan per warp). */
__device__ void lsd_rect_count_multi(const LsdFrame &F, const LsdRect *r, int n, bool same_geom, int *tot, int *alg)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    LsdSpan *sp = F.span;
    const int n_geom = same_geom ? 1 : n;
    __syncwarp();
    if (lane < n_geom) lsd_span_setup(F, r[lane], sp[lane]);
    __syncwarp();
    int y_min = sp[0].y0, y_max = sp[0].y1;
    for (int t = 1; t < n_geom; t++) {
        y_min = min(y_min, sp[t].y0);
        y_max = max(y_max, sp[t].y1);
    }
    const double theta = r[0].theta;
    const float thetaf = (float)theta;
    float pf[5];
#pragma unroll
    for (int t = 0; t < 5; t++) pf[t] = (float)r[t < n ? t : 0].prec;
    int c_tot[5] = {0, 0, 0, 0, 0}, c_alg[5] = {0, 0, 0, 0, 0};
    const int n_rows = y_max - y_min + 1;
    int G = 1;
    while (G < 32 && n_rows * G * 2 <= 32) G <<= 1;
    const int rows_per_step = 32 / G, sub = lane & (G - 1), rsel = lane / G;
    for (int yb = y_min; yb <= y_max; yb += rows_per_step) {
        const int y = yb + rsel;
        if (y > y_max) continue;
        int lo[5], hi[5];
        int x_lo = 0x7fffffff, x_hi = -1;
#pragma unroll
        for (int t = 0; t < 5; t++) {
            lo[t] = 1;
            hi[t] = 0;
            if (t < n_geom && y >= sp[t].y0 && y <= sp[t].y1) {
                lsd_span_row(sp[t], y, F.W, lo[t], hi[t]);
                if (hi[t] >= lo[t]) {
                    x_lo = min(x_lo, lo[t]);
                    x_hi = max(x_hi, hi[t]);
                    if (sub == 0) c_tot[t] += hi[t] - lo[t] + 1;
                }
            }
        }
        if (x_hi < 0) continue; /* no rectangle has pixels in this row */
        const float *row = F.angf + (size_t)y * F.W;
        for (int x = x_lo + sub; x <= x_hi; x += G) {
            const float deg = row[x];
            if (deg < 0.f) continue;
            float nf = fabsf(thetaf - deg * 0.017453292f);
            if (nf > 4.712389f) nf = fabsf(nf - 6.2831855f);
            if (same_geom) {
#pragma unroll
                for (int t = 0; t < 5; t++)
                    if (t < n) {
                        bool a = nf < pf[t] - 2e-4f;
                        if (!a && !(nf > pf[t] + 2e-4f)) a = lsd_aligned_deg(deg, theta, r[t].prec); /* borderline: the reference's doubles */
                        c_alg[t] += a ? 1 : 0;
                    }
            } else {
                bool a = nf < pf[0] - 2e-4f;
                if (!a && !(nf > pf[0] + 2e-4f)) a = lsd_aligned_deg(deg, theta, r[0].prec);
                if (a) {
#pragma unroll
                    for (int t = 0; t < 5; t++) c_alg[t] += (x >= lo[t] && x <= hi[t]) ? 1 : 0;
                }
            }
        }
    }
    if (same_geom) {
#pragma unroll
        for (int t = 1; t < 5; t++) c_tot[t] = c_tot[0];
    }
#pragma unroll
    for (int t = 0; t < 5; t++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            c_tot[t] += __shfl_xor_sync(FULL, c_tot[t], o);
            c_alg[t] += __shfl_xor_sync(FULL, c_alg[t], o);
        }
        if (t < n) {
            tot[t] = c_tot[t];
            alg[t] = c_alg[t];
        }
    }
}

/* The first half of one seed (lsd.cpp:478-519): grow, rectangle, density refinement.  has_rect = 1 when a rectangle comes out that
 * rect_improve / the NFA test still have to judge -- which they can do later, in any order and in parallel: they read the level-line
 * angles only and never touch the `used` map. */
__device__ __noinline__ void lsd_region2rect_cold(const LsdFrame &F, const LsdReg &R, int base, int reg_size, double reg_angle, double prec, double p, LsdRect &rec)
{
    lsd_region2rect(F, R, base, reg_size, reg_angle, prec, p, rec);
}

template <bool kProf>
__device__ void lsd_grow_candidate(const LsdFrame &F, const LsdReg &R, int s_addr, int min_reg_size, double prec, double p, int &n_all,
                                  int &has_rect, LsdRect &rec)
{
    /* region_grow -> region2rect -> density test, at most twice: the second round is refine()'s re-grow with the tolerance estimated from
     * the first region (lsd.cpp:786-832).  One loop, so that the two big inlined bodies exist once in the kernel (instruction cache). */
    const double DENSITY_TH = 0.7;
    const int lane = threadIdx.x & 31;
    int base = 0, reg_size = 0, seed = s_addr;
    double reg_angle = 0, tau = prec;
    has_rect = 0;
    n_all = 0;
    for (int pass = 0; pass < 2; pass++) {
        {
            LSD_PROF_T0();
            lsd_region_grow(F, R, base, seed, reg_size, reg_angle, tau);
            LSD_PROF_ADD(pass == 0 ? 0 : 2);
        }
        if (kProf && pass == 0 && lane == 0) {
            atomicAdd(&g_lsd_prof[5], 1ull);
            atomicAdd(&g_lsd_prof[7], (unsigned long long)reg_size);
        }
        n_all = base + reg_size;
        if (reg_size < (pass == 0 ? min_reg_size : 2)) return;
        if (pass == 0) LSD_PROF_COUNT(12, 1);
        LSD_PROF_RECT_SIZE(reg_size);
        {
            LSD_PROF_T0();
            lsd_region2rect(F, R, base, reg_size, reg_angle, prec, p, rec);
            LSD_PROF_ADD(1);
        }
        double density;
        {
            LSD_PROF_T0();
            density = (double)reg_size / (lsd_dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
            has_rect = density >= DENSITY_TH;
            LSD_PROF_ADD(10);
        }
        if (has_rect) return;
        if (pass == 1) { /* still too sparse after the re-grow: shrink it around the seed (lsd.cpp:834-871) */
            LSD_PROF_T0();
            if (lsd_reduce_region_radius<kProf>(F, R, base, reg_size, reg_angle, prec, p, rec, density, DENSITY_TH) == 0) has_rect = 1;
            LSD_PROF_ADD(11);
            return;
        }
        /* refine(): tolerance from the angle spread near the seed, give the region back, grow again from the same seed */
        LSD_PROF_COUNT(13, 1);
        LSD_PROF_T0();
        const int a0 = R.get(base);
        const double xc = (double)(a0 - F.row_of(a0) * F.W), yc = (double)F.row_of(a0);
        const double ang_c = (double)F.angf[a0] * LSD_DEG2RAD;
        double sum = 0, s_sum = 0;
        int n = 0;
        for (int i0 = 0; i0 < reg_size; i0 += 32) {
            const int m = min(32, reg_size - i0);
            bool near = false;
            __syncwarp();
            if (lane < m) {
                const int addr = R.get(base + i0 + lane);
                const int ry = F.row_of(addr), rx = addr - ry * F.W;
                if (lsd_dist(xc, yc, (double)rx, (double)ry) < rec.width) {
                    near = true;
                    const double ang_d = lsd_angle_diff_signed((double)F.angf[addr] * LSD_DEG2RAD, ang_c);
                    lsd_stage()[lane] = ang_d;
                    lsd_stage()[32 + lane] = ang_d * ang_d;
                }
            }
            __syncwarp();
            unsigned todo = __ballot_sync(0xffffffffu, near);
            n += __popc(todo);
            while (todo) {
                const int j = __ffs(todo) - 1;
                todo &= todo - 1;
                sum += lsd_stage()[j];
                s_sum += lsd_stage()[32 + j];
            }
        }
        for (int i = lane; i < reg_size; i += 32) {
            const int addr = R.get(base + i);
            const int ay = F.row_of(addr);
            uint32_t bit;
            uint32_t *w = F.used_at(ay, addr - ay * F.W, bit);
            atomicAnd(w, ~bit);
        }
        __syncwarp();
        const double mean_angle = sum / (double)n;
        tau = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)n + mean_angle * mean_angle);
        seed = a0;
        base += reg_size;
        LSD_PROF_ADD(2);
    }
}

/* checkLineExtremes + 10-px border rejection + length filter (LSDDetector.cpp:75-101,226-238; filter_lines): true = keep */
__device__ __forceinline__ bool lsd_keyline_filter(const float *raw, int img_w, int img_h, float line_length_thres, float *o)
{
    const float pre_boundary_thre = 10;
    float e[4] = {raw[0], raw[1], raw[2], raw[3]};
    if (e[0] < 0) e[0] = 0;
    if (e[0] >= img_w) e[0] = (float)img_w - 1.0f;
    if (e[2] < 0) e[2] = 0;
    if (e[2] >= img_w) e[2] = (float)img_w - 1.0f;
    if (e[1] < 0) e[1] = 0;
    if (e[1] >= img_h) e[1] = (float)img_h - 1.0f;
    if (e[3] < 0) e[3] = 0;
    if (e[3] >= img_h) e[3] = (float)img_h - 1.0f;
    const float sx = e[0], sy = e[1], ex = e[2], ey = e[3];
    if (((sx < pre_boundary_thre) && (ex < pre_boundary_thre)) || ((sx > img_w - pre_boundary_thre) && (ex > img_w - pre_boundary_thre)) ||
        ((sy < pre_boundary_thre) && (ey < pre_boundary_thre)) || ((sy > img_h - pre_boundary_thre) && (ey > img_h - pre_boundary_thre)))
        return false;
    const double ddx = (double)(e[0] - e[2]), ddy = (double)(e[1] - e[3]);
    const float line_length = (float)sqrt(ddx * ddx + ddy * ddy);
    if (!(line_length > line_length_thres)) return false;
    o[0] = sx;
    o[1] = sy;
    o[2] = ex;
    o[3] = ey;
    return true;
}

struct LsdGrowArgs {
    int W, H, img_w, img_h;
    uint4 *pix;
    const float *angf;
    const double *modgrad;
    int32_t *arena;
    int arena_cap;       /* ints per frame */
    double LOG_NT;
    int min_reg_size;
    double prec, p, scale;
    float line_length_thres;
    float *raw;
    int32_t *n_raw;
    float *out;
    int32_t *n_out;
    int cap;
    LsdRect *cand;       /* cand_cap rectangles per frame, seed order: k_lsd_grow_seq -> k_lsd_val_count / k_lsd_val_nfa */
    int32_t *n_cand;
    int cand_cap;
    int32_t *cand_line;  /* per candidate: {is a line, 4 floats} */
    struct LsdCandState *cand_state; /* per candidate: the state of the phase-split validation */
    int32_t *err;        /* [0]: 4 = more candidates in a frame than cand_cap, 8 = a TMA tile copy of k_lsd_front did not complete;
                          * [1]: the largest candidate count of a frame that overflowed, [2]: cand_cap */
    const double *lgam;  /* log_gamma table (cs_nfa.cuh) */
    uint32_t *ubits;     /* ceil(W / 32) * H words per frame: the used map of k_lsd_grow_seq (LsdFrame::used_at) */
    const uint32_t *defb; /* the same layout: "angle defined", from k_lsd_front */
    const LsdGeom *geom; /* kMixed: one entry per frame, and the fields above that describe a frame's size or place are not used */
};

/* The order-dependent half of the seed loop, one warp per frame (see the file header). */
template <bool kProf, bool kMixed>
__global__ void __launch_bounds__(32, 21) k_lsd_grow_seq(LsdGrowArgs A)
{
    const int f = blockIdx.x, lane = threadIdx.x;
    LsdGeom G = {};
    if constexpr (kMixed) G = A.geom[f];
    const int fW = kMixed ? G.W : A.W, fH = kMixed ? G.H : A.H;
    const size_t npx = (size_t)fW * fH;
    const size_t px0 = kMixed ? (size_t)G.px_off : f * npx;
    LsdFrame F;
    LSD_PROF_T0();
    F.W = fW;
    F.H = fH;
    F.pix = A.pix + px0;
    F.angf = A.angf + px0;
    F.modgrad = A.modgrad + px0;
    F.LOG_NT = kMixed ? G.LOG_NT : A.LOG_NT;
    const int WW = (fW + 31) >> 5, n_words = WW * fH;
    const size_t w0f = kMixed ? (size_t)G.bit_off : (size_t)f * n_words;
    F.ubits = A.ubits + w0f;
    F.WW = WW;
    F.span = nullptr;
    F.lgam = A.lgam;
    F.wmagic = ((1ull << 40) + (unsigned long long)fW - 1) / (unsigned long long)fW;
    for (int i = lane; i < n_words; i += 32) F.ubits[i] = 0u;
    __syncwarp();
    LsdReg R;
    R.g = A.arena /* region entries past the first LSD_SEQ_SCAP (shared memory): the (otherwise unused) record arena */ +
          (kMixed ? (size_t)G.arena_off : (size_t)f * A.arena_cap);
    R.cap = A.arena_cap;
    const int min_reg_size = kMixed ? G.min_reg_size : A.min_reg_size;
    int n_cand = 0;
    /* Seeds in RASTER order: flsd walks its coorlist vector by index (lsd.cpp:478-480), and ll_angle fills that vector in scan order; the
     * gradient-bin links it also builds (lsd.cpp:588-634) are never followed.  A step covers 32 words (1024 bit positions of the padded
     * layout), lane l holding word w0 + l: seeds are the bits of defb & ~used (pixels with a defined angle -- which excludes the last
     * row and column and the padding -- that no region holds), taken word by word, lowest bit first = raster order.  defb never changes:
     * the next step's words are loaded before this step's seeds grow.  The used map changes with every grow, and not only by setting bits:
     * refine and reduce_region_radius give pixels back, which may be later pixels of this very step.  So after each grow the used words of
     * this step and of the next are read again (one round trip) and the remaining seeds recomputed from them: a pixel is a seed iff it is
     * defined and unused at its turn, as in the reference, and the next step starts from words no grow has changed since. */
    const long long scan_t0 = kProf ? clock64() : 0ll;
    long long in_cand = 0, handoff_t0 = 0;
    const uint32_t *defb = A.defb + w0f;
    uint32_t d_next = lane < n_words ? __ldg(defb + lane) : 0u, u_next = 0u; /* the used map was just cleared */
    for (int w0 = 0; w0 < n_words; w0 += 32) {
        const int wi = w0 + lane;
        const uint32_t d = d_next;
        uint32_t u = u_next;
        d_next = wi + 32 < n_words ? __ldg(defb + wi + 32) : 0u;
        u_next = wi + 32 < n_words ? __ldcg(F.ubits + wi + 32) : 0u;
        const int wy = wi / WW, w_addr = wy * fW + ((wi - wy * WW) << 5); /* address of the word's bit 0 */
        uint32_t s = d & ~u;
        for (;;) {
            const unsigned nz = __ballot_sync(0xffffffffu, s != 0u);
            if (kProf && handoff_t0) {
                if (lane == 0) atomicAdd(&g_lsd_prof[9], (unsigned long long)(clock64() - handoff_t0));
                handoff_t0 = 0;
            }
            if (!nz) break;
            const int j = __ffs(nz) - 1;
            const int b = __ffs(__shfl_sync(0xffffffffu, s, j)) - 1;
            const int s_addr = __shfl_sync(0xffffffffu, w_addr, j) + b;
            int n_all = 0, has_rect = 0;
            LsdRect rec;
            const long long c0 = kProf ? clock64() : 0ll;
            lsd_grow_candidate<kProf>(F, R, s_addr, min_reg_size, A.prec, A.p, n_all, has_rect, rec); /* arena_cap >= 2 W H: both passes fit */
            if (kProf) {
                in_cand += clock64() - c0;
                if (lane == 0) {
                    atomicAdd(&g_lsd_prof[4], 1ull);
                    if (n_all > LSD_SEQ_SCAP) atomicAdd(&g_lsd_prof[8], 1ull);
                }
            }
            if (kProf) handoff_t0 = clock64(); /* counted up to the ballot over the new mask, which waits for the re-read */
            __syncwarp(); /* the grow's used-map atomics are visible to every lane */
            u = wi < n_words ? __ldcg(F.ubits + wi) : 0u;
            u_next = wi + 32 < n_words ? __ldcg(F.ubits + wi + 32) : 0u;
            /* what is left of the step after seed (j, b) */
            s = d & ~u & (lane > j ? 0xffffffffu : lane == j ? 0xfffffffeu << b : 0u);
            if (!has_rect) continue;
            /* the rectangle goes to the validation kernels (rect_improve + NFA never touch the used map): candidates in seed order */
            const long long st0 = kProf ? clock64() : 0ll;
            if (lane == 0 && n_cand < A.cand_cap) A.cand[(size_t)f * A.cand_cap + n_cand] = rec;
            n_cand++;
            if (kProf) {
                const long long dt = clock64() - st0;
                if (lane == 0) atomicAdd(&g_lsd_prof[10], (unsigned long long)dt);
                handoff_t0 += dt;
            }
        }
    }
    if (kProf && lane == 0) atomicAdd(&g_lsd_prof[3], (unsigned long long)(clock64() - scan_t0 - in_cand));
    if (lane == 0) {
        A.n_cand[f] = n_cand;
        if (n_cand > A.cand_cap) {
            atomicOr(A.err, 4);
            atomicMax(A.err + 1, n_cand);
            A.err[2] = A.cand_cap;
        }
    }
    LSD_PROF_ADD(6);
}

/* ---- rect_improve + NFA of every candidate rectangle (lsd.cpp:520-534), one warp each, split by phase into small kernels -----------
 * As one kernel this would be ~6.6 k instructions (the scans, the double-precision log / exp / pow of the binomial tail, the improvement
 * logic); the L1.5 instruction cache holds 2 k, and the warps would sit in different places of that code and stall on instruction fetch
 * (`no_instruction`).  rect_improve is six rounds of {count the pixels of up to five rectangles, turn the counts into NFA values, keep the
 * best} (lsd.cpp:873-975); run as twelve launches -- k_lsd_val_count(round), k_lsd_val_nfa(round) -- every warp of a launch is in the
 * same few hundred instructions.  State between launches: the candidate's current rectangle (A.cand, updated in place), its best
 * log_nfa and the counts of the round (A.cand_state). */
#define LSD_VAL_CTAS 64 /* CTAs of k_lsd_val_count / k_lsd_val_nfa per frame: 256 warps, a warp per candidate for all but the densest frames */

struct LsdCandState {
    double log_nfa;
    int32_t status; /* 0 = still being improved, 1 = decided (A.cand_line holds the verdict) */
    int32_t n;      /* rectangles counted in this round */
    int32_t tot[5], alg[5];
};

/* the rectangles round `round` evaluates, from the current one (lsd.cpp:873-975; round 0 = the rectangle itself) */
__device__ int lsd_improve_variants(const LsdRect &rec, int round, LsdRect *cand)
{
    const double delta = 0.5, delta_2 = delta / 2.0;
    LsdRect r = rec;
    if (round == 0) {
        cand[0] = r;
        return 1;
    }
    if (round == 1) {
        for (int n = 0; n < 5; ++n) {
            r.p /= 2;
            r.prec = r.p * LSD_PI;
            cand[n] = r;
        }
        return 5;
    }
    const int phase = round - 2;
    int m = 0;
    for (int n = 0; n < 5; ++n)
        if ((r.width - delta) >= 0.5) {
            if (phase == 0)
                r.width -= delta;
            else if (phase == 1) {
                r.x1 += -r.dy * delta_2;
                r.y1 += r.dx * delta_2;
                r.x2 += -r.dy * delta_2;
                r.y2 += r.dx * delta_2;
                r.width -= delta;
            } else if (phase == 2) {
                r.x1 -= -r.dy * delta_2;
                r.y1 -= r.dx * delta_2;
                r.x2 -= -r.dy * delta_2;
                r.y2 -= r.dx * delta_2;
                r.width -= delta;
            } else {
                r.p /= 2;
                r.prec = r.p * LSD_PI;
            }
            cand[m++] = r;
        }
    return m;
}

template <bool kMixed>
__global__ void __launch_bounds__(128, 5) k_lsd_val_count(LsdGrowArgs A, int round)
{
    /* kMixed: LSD_VAL_CTAS CTAs per frame along x (a frame count is not bounded by gridDim.y's 65535) */
    const int f = kMixed ? (int)(blockIdx.x / LSD_VAL_CTAS) : (int)blockIdx.y, lane = threadIdx.x & 31;
    const int bx = kMixed ? (int)(blockIdx.x % LSD_VAL_CTAS) : (int)blockIdx.x, gx = kMixed ? LSD_VAL_CTAS : (int)gridDim.x;
    LsdFrame F;
    if constexpr (kMixed) {
        const LsdGeom &G = A.geom[f];
        F.W = G.W;
        F.H = G.H;
        F.angf = A.angf + G.px_off;
        F.LOG_NT = G.LOG_NT;
    } else {
        const size_t npx = (size_t)A.W * A.H;
        F.W = A.W;
        F.H = A.H;
        F.angf = A.angf + f * npx;
        F.LOG_NT = A.LOG_NT;
    }
    F.pix = nullptr;
    F.modgrad = nullptr;
    F.ubits = nullptr;
    __shared__ LsdSpan s_span[4][5];
    F.span = s_span[threadIdx.x >> 5];
    F.lgam = A.lgam;
    F.wmagic = 0;
    const int n = min(A.n_cand[f], A.cand_cap);
    const int wpb = blockDim.x >> 5;
    for (int c = bx * wpb + (threadIdx.x >> 5); c < n; c += gx * wpb) {
        LsdCandState *S = A.cand_state + (size_t)f * A.cand_cap + c;
        if (round > 0 && S->status != 0) continue;
        const LsdRect rec = A.cand[(size_t)f * A.cand_cap + c];
        LsdRect cv[5];
        const int m = lsd_improve_variants(rec, round, cv);
        int tot[5] = {0, 0, 0, 0, 0}, alg[5] = {0, 0, 0, 0, 0};
        if (m == 1)
            lsd_rect_count(F, cv[0], tot[0], alg[0]);
        else if (m > 1)
            lsd_rect_count_multi(F, cv, m, round == 1 || round == 5, tot, alg);
        if (lane == 0) {
            S->n = m;
            for (int t = 0; t < 5; t++) {
                S->tot[t] = tot[t];
                S->alg[t] = alg[t];
            }
        }
    }
}

template <bool kMixed>
__global__ void __launch_bounds__(128, 5) k_lsd_val_nfa(LsdGrowArgs A, int round)
{
    /* kMixed: LSD_VAL_CTAS CTAs per frame along x (a frame count is not bounded by gridDim.y's 65535) */
    const int f = kMixed ? (int)(blockIdx.x / LSD_VAL_CTAS) : (int)blockIdx.y, lane = threadIdx.x & 31;
    const int bx = kMixed ? (int)(blockIdx.x % LSD_VAL_CTAS) : (int)blockIdx.x, gx = kMixed ? LSD_VAL_CTAS : (int)gridDim.x;
    const double LOG_NT = kMixed ? A.geom[f].LOG_NT : A.LOG_NT;
    const int n = min(A.n_cand[f], A.cand_cap);
    const int wpb = blockDim.x >> 5;
    for (int c = bx * wpb + (threadIdx.x >> 5); c < n; c += gx * wpb) {
        LsdCandState *S = A.cand_state + (size_t)f * A.cand_cap + c;
        if (round > 0 && S->status != 0) continue;
        LsdRect rec = A.cand[(size_t)f * A.cand_cap + c];
        LsdRect cv[5];
        const int m = lsd_improve_variants(rec, round, cv);
        double log_nfa = round == 0 ? 0.0 : S->log_nfa;
        bool changed = false;
        for (int t = 0; t < m; t++) {
            const double v = cs_nfa_warp(A.lgam, S->tot[t], S->alg[t], cv[t].p, LOG_NT, true); /* the whole warp on one binomial tail */
            if (round == 0 || v > log_nfa) {
                log_nfa = v;
                rec = cv[t];
                changed = round > 0;
            }
        }
        const bool done = round == 5 || log_nfa > 0.0; /* lsd.cpp:887,903,921,938,955: leave as soon as the rectangle is meaningful */
        __syncwarp();
        if (lane == 0) {
            if (done) {
                int32_t *o = A.cand_line + ((size_t)f * A.cand_cap + c) * 5;
                const bool ok = log_nfa > 0.0;
                o[0] = ok ? 1 : 0;
                /* lsd.cpp:524-534: the half-pixel offset, back to the scale of the input image */
                o[1] = __float_as_int((float)((rec.x1 + 0.5) / A.scale));
                o[2] = __float_as_int((float)((rec.y1 + 0.5) / A.scale));
                o[3] = __float_as_int((float)((rec.x2 + 0.5) / A.scale));
                o[4] = __float_as_int((float)((rec.y2 + 0.5) / A.scale));
                S->status = 1;
            } else {
                if (changed) A.cand[(size_t)f * A.cand_cap + c] = rec;
                S->log_nfa = log_nfa;
                S->status = 0;
            }
        }
    }
}

#define LSD_LAUNCHES_PER_RUN 15 /* kernels one LSD run launches: front end, seed loop, 12 validation phase kernels, emit */

/* the accepted candidates of a frame in seed order: raw segments, and those that pass the key-line filter */
template <bool kMixed>
__global__ void __launch_bounds__(256) k_lsd_emit(LsdGrowArgs A)
{
    __shared__ int s_warp_cnt[8], s_base_raw, s_base_out;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const unsigned FULL = 0xffffffffu;
    const int n = min(A.n_cand[f], A.cand_cap);
    float *raw = A.raw + (size_t)f * A.cap * 4;
    float *out = A.out + (size_t)f * A.cap * 4;
    if (tid == 0) {
        s_base_raw = 0;
        s_base_out = 0;
    }
    __syncthreads();
    for (int b = 0; b < n; b += 256) {
        const int i = b + tid;
        bool has = false, kept = false;
        float ln[4], fo[4];
        if (i < n) {
            const int32_t *o = A.cand_line + ((size_t)f * A.cand_cap + i) * 5;
            if (o[0]) {
                has = true;
                for (int k = 0; k < 4; k++) ln[k] = __int_as_float(o[1 + k]);
                kept = lsd_keyline_filter(ln, kMixed ? A.geom[f].w : A.img_w, kMixed ? A.geom[f].h : A.img_h, A.line_length_thres, fo);
            }
        }
        const unsigned mh = __ballot_sync(FULL, has), mk = __ballot_sync(FULL, kept);
        if (lane == 0) s_warp_cnt[wid] = __popc(mh) | (__popc(mk) << 16);
        __syncthreads();
        int pre_r = s_base_raw, pre_o = s_base_out;
        for (int k = 0; k < wid; k++) {
            pre_r += s_warp_cnt[k] & 0xffff;
            pre_o += s_warp_cnt[k] >> 16;
        }
        if (has) {
            const int slot = pre_r + __popc(mh & ((1u << lane) - 1u));
            if (slot < A.cap)
                for (int k = 0; k < 4; k++) raw[4 * slot + k] = ln[k];
        }
        if (kept) {
            const int slot = pre_o + __popc(mk & ((1u << lane) - 1u));
            if (slot < A.cap)
                for (int k = 0; k < 4; k++) out[4 * slot + k] = fo[k];
        }
        __syncthreads();
        if (tid == 0) {
            int tr = 0, to = 0;
            for (int k = 0; k < 8; k++) {
                tr += s_warp_cnt[k] & 0xffff;
                to += s_warp_cnt[k] >> 16;
            }
            s_base_raw += tr;
            s_base_out += to;
        }
        __syncthreads();
    }
    if (tid == 0) {
        /* more candidate rectangles than the hand-off buffer holds: report it the way a segment overflow is reported (count > capacity) */
        const bool overflow = A.n_cand[f] > A.cand_cap;
        A.n_raw[f] = overflow ? A.cap + 1 : s_base_raw;
        A.n_out[f] = overflow ? A.cap + 1 : s_base_out;
    }
}

/* ---------------------------------------------------------------------------------------- host side */
struct Buf {
    void *p = nullptr;
    size_t cap = 0;
};

struct LsdState {
    CsLineHead head; /* first: the error word (cs_internal.h) */
    Buf img, modgrad, angf, pix, defb, arena, raw, nraw, out, nout, lgam, ubits, cand, ncand, candline, candstate, err, geom;
    bool lgam_filled = false;
    bool last_mixed = false; /* the last run was a batch of frames of different sizes: its planes follow the geometry table */
    int last_frames = 0, last_W = 0, last_H = 0, cap = 0;
    /* the last run's frames (S.img, or the caller's device frames), from which cs_debug_lsd recomputes the scaled and modgrad planes */
    const uint8_t *last_img = nullptr;
    int last_w = 0, last_h = 0, last_stride = 0, last_channels = 0;
    int cand_cap = LSD_CAND_CAP; /* candidate rectangles per frame; grown when a frame had more (lsd_grow_candidates) */
};

int ensure(cs_ctx *c, Buf &b, size_t bytes)
{
    if (bytes <= b.cap) return CS_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    const size_t want = bytes + bytes / 16 + 256;
    if (cudaMalloc(&b.p, want) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc(%zu) failed in the line detector", want);
    b.cap = want;
    return CS_OK;
}

inline int grid_for(int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, CS_SM_COUNT * 32); }

/* k_lsd_front over n_frames frames (scaled == nullptr), or the debug instantiation over one frame: the scaled plane and the full modgrad plane */
void lsd_front(cs_ctx *c, const uint8_t *d_img, int n_frames, int w, int h, int stride, int channels, int W, int H, double rho, double *modgrad,
               float *angf, uint4 *pix, uint32_t *defb, double *scaled, int32_t *d_err)
{
    cudaStream_t st = cs_ctx_stream(c);
    const dim3 g_tile((W + LSF_TW - 1) / LSF_TW, (H + LSF_TH - 1) / LSF_TH, n_frames);
    const double inv_scale = 1. / LSD_SCALE;
    CUtensorMap tm;
    memset(&tm, 0, sizeof tm);
    if (scaled)
        k_lsd_front<false, true, false><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, W, H, inv_scale, rho, modgrad, angf, pix, defb, scaled,
                                                                d_err, nullptr, 0);
    /* BGR frames whose rows are a multiple of 16 bytes (640 and 1280 wide are) can be staged by the copy engine */
    else if (cs_ctx_use_tma(c) && channels == 3 && stride == 3 * w &&
             cs_make_tmap_bytes(&tm, d_img, 3 * (int64_t)w, (int64_t)n_frames * h, stride, LSF_BOXW, LSF_GH))
        k_lsd_front<true, false, false><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, W, H, inv_scale, rho, modgrad, angf, pix, defb, nullptr,
                                                                d_err, nullptr, 0);
    else
        k_lsd_front<false, false, false><<<g_tile, 256, 0, st>>>(tm, d_img, w, h, stride, channels, W, H, inv_scale, rho, modgrad, angf, pix, defb,
                                                                 nullptr, d_err, nullptr, 0);
}

/* host-side constants of flsd (lsd.cpp:445-447,468-469), evaluated with libm like the reference */
const double LSD_ANG_TH = 22.5, LSD_QUANT = 2.0;
inline double lsd_prec() { return LSD_PI * LSD_ANG_TH / 180; }
inline double lsd_p() { return LSD_ANG_TH / 180; }
inline double lsd_log_nt(int W, int H) { return 5 * (std::log10((double)W) + std::log10((double)H)) / 2 + std::log10(11.0); }
inline int lsd_min_reg_size(double LOG_NT) { return (int)(-LOG_NT / std::log10(lsd_p())); }
inline int lsd_arena_cap(int W, int H) { return (int)(((size_t)W * H * 2 + 64 + 3) & ~(size_t)3); } /* ints per frame */

/* every buffer of a run of n_frames frames with spx scaled pixels, bit_words words of each bit plane and arena_ints arena ints in all */
int lsd_buffers(cs_ctx *c, LsdState &S, int n_frames, size_t spx, size_t bit_words, size_t arena_ints, int cap)
{
    int rc;
    if ((rc = ensure(c, S.modgrad, spx * 8)) || (rc = ensure(c, S.angf, spx * 4)) || (rc = ensure(c, S.pix, spx * 16)) || (rc = ensure(c, S.defb, bit_words * 4)) ||
        (rc = ensure(c, S.arena, arena_ints * 4)) ||
        (rc = ensure(c, S.raw, (size_t)n_frames * cap * 16)) || (rc = ensure(c, S.nraw, (size_t)n_frames * 4)) ||
        (rc = ensure(c, S.out, (size_t)n_frames * cap * 16)) || (rc = ensure(c, S.nout, (size_t)n_frames * 4)) ||
        (rc = ensure(c, S.lgam, (size_t)CS_LGAMMA_TABLE * 8)) || (rc = ensure(c, S.ubits, bit_words * 4)) ||
        (rc = ensure(c, S.cand, (size_t)n_frames * S.cand_cap * sizeof(LsdRect))) || (rc = ensure(c, S.ncand, (size_t)n_frames * 4)) ||
        (rc = ensure(c, S.candline, (size_t)n_frames * S.cand_cap * 20)) || (rc = ensure(c, S.candstate, (size_t)n_frames * S.cand_cap * sizeof(LsdCandState))) || (rc = ensure(c, S.err, 16)))
        return rc;
    if (!S.lgam_filled) { /* log_gamma of the integers 1 .. CS_LGAMMA_TABLE - 1, host libm like the reference */
        std::vector<double> t(CS_LGAMMA_TABLE, 0.0);
        for (int i = 1; i < CS_LGAMMA_TABLE; i++) t[i] = cs_lgamma_host((double)i);
        if (cudaMemcpyAsync(S.lgam.p, t.data(), t.size() * 8, cudaMemcpyHostToDevice, cs_ctx_stream(c)) != cudaSuccess ||
            cudaStreamSynchronize(cs_ctx_stream(c)) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the log_gamma table failed");
        S.lgam_filled = true;
    }
    S.head.d_err = (int32_t *)S.err.p; /* the 16-byte error word (cs_internal.h) */
    cudaMemsetAsync(S.err.p, 0, 16, cs_ctx_stream(c));
    return CS_OK;
}

/* the seed-loop arguments every run shares; the frame geometry is the caller's */
LsdGrowArgs lsd_args(const LsdState &S, int cap, float line_length_thres)
{
    LsdGrowArgs A;
    memset(&A, 0, sizeof A);
    A.pix = (uint4 *)S.pix.p;
    A.angf = (const float *)S.angf.p;
    A.modgrad = (const double *)S.modgrad.p;
    A.arena = (int32_t *)S.arena.p;
    A.prec = lsd_prec();
    A.p = lsd_p();
    A.scale = LSD_SCALE;
    A.line_length_thres = line_length_thres;
    A.raw = (float *)S.raw.p;
    A.n_raw = (int32_t *)S.nraw.p;
    A.out = (float *)S.out.p;
    A.n_out = (int32_t *)S.nout.p;
    A.cap = cap;
    A.lgam = (const double *)S.lgam.p;
    A.ubits = (uint32_t *)S.ubits.p;
    A.defb = (const uint32_t *)S.defb.p;
    A.cand = (LsdRect *)S.cand.p;
    A.n_cand = (int32_t *)S.ncand.p;
    A.cand_cap = S.cand_cap;
    A.cand_line = (int32_t *)S.candline.p;
    A.cand_state = (LsdCandState *)S.candstate.p;
    A.err = (int32_t *)S.err.p;
    return A;
}

/* everything after the front end: the seed loop, the validation rounds and the emit */
template <bool kMixed>
int lsd_seed_loop(cs_ctx *c, const LsdGrowArgs &A, int n_frames)
{
    cudaStream_t st = cs_ctx_stream(c);
    const size_t smem = LSD_SEQ_SMEM;
    if (cs_ctx_profiling(c))
        k_lsd_grow_seq<true, kMixed><<<n_frames, 32, smem, st>>>(A);
    else
        k_lsd_grow_seq<false, kMixed><<<n_frames, 32, smem, st>>>(A);
    const dim3 g_val = kMixed ? dim3(LSD_VAL_CTAS * n_frames) : dim3(LSD_VAL_CTAS, n_frames);
    for (int round = 0; round < 6; round++) {
        k_lsd_val_count<kMixed><<<g_val, 128, 0, st>>>(A, round);
        k_lsd_val_nfa<kMixed><<<g_val, 128, 0, st>>>(A, round);
    }
    k_lsd_emit<kMixed><<<n_frames, 256, 0, st>>>(A);
    cs_ctx_count_launches(c, LSD_LAUNCHES_PER_RUN);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "LSD kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    return CS_OK;
}

int lsd_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
            int cap, LsdState &S)
{
    cudaStream_t st = cs_ctx_stream(c);
    const int W = (int)std::lrint(w * LSD_SCALE), H = (int)std::lrint(h * LSD_SCALE);
    if (W < 2 || H < 2) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "image too small for LSD");
    const size_t spx = (size_t)n_frames * W * H;
    const size_t bit_words = (size_t)n_frames * ((W + 31) / 32) * H; /* defb and the used map: row-padded bit planes */
    const int arena_cap = lsd_arena_cap(W, H);
    int rc;
    const uint8_t *d_img = imgs;
    if (!imgs_on_device) {
        if ((rc = ensure(c, S.img, (size_t)n_frames * h * stride))) return rc;
        if (cudaMemcpyAsync(S.img.p, imgs, (size_t)n_frames * h * stride, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames failed");
        d_img = (const uint8_t *)S.img.p;
    }
    if ((rc = lsd_buffers(c, S, n_frames, spx, bit_words, (size_t)n_frames * arena_cap, cap))) return rc;
    const double rho = LSD_QUANT / std::sin(lsd_prec());
    const double LOG_NT = lsd_log_nt(W, H);
    lsd_front(c, d_img, n_frames, w, h, stride, channels, W, H, rho, (double *)S.modgrad.p, (float *)S.angf.p, (uint4 *)S.pix.p, (uint32_t *)S.defb.p,
              nullptr, (int32_t *)S.err.p);
    LsdGrowArgs A = lsd_args(S, cap, line_length_thres);
    A.W = W;
    A.H = H;
    A.img_w = w;
    A.img_h = h;
    A.arena_cap = arena_cap;
    A.LOG_NT = LOG_NT;
    A.min_reg_size = lsd_min_reg_size(LOG_NT);
    if ((rc = lsd_seed_loop<false>(c, A, n_frames))) return rc;
    S.last_mixed = false;
    S.last_frames = n_frames;
    S.last_W = W;
    S.last_H = H;
    S.cap = cap;
    S.last_img = d_img;
    S.last_w = w;
    S.last_h = h;
    S.last_stride = stride;
    S.last_channels = channels;
    return CS_OK;
}

/* The same run over frames of different sizes already on the device: frame f at d_img + views[f].offset.  One geometry entry per frame, its
 * plane offsets the prefix sums of the frames before it; k_lsd_front walks one flattened list of every frame's tiles, and reads bytes with
 * plain loads (one tensor map cannot describe rows of different lengths). */
int lsd_run_mixed(cs_ctx *c, const uint8_t *d_img, const cs_frame_view *views, int n_frames, float line_length_thres, int cap, LsdState &S)
{
    cudaStream_t st = cs_ctx_stream(c);
    static_assert((int64_t)CS_LSD_MAX_MIXED_FRAMES * LSD_VAL_CTAS <= INT32_MAX, "the validation grid of a mixed run");
    if (n_frames > CS_LSD_MAX_MIXED_FRAMES)
        return cs_ctx_fail(c, CS_ERR_CAPACITY, "%d frames in one LSD batch: at most %d", n_frames, CS_LSD_MAX_MIXED_FRAMES);
    std::vector<LsdGeom> g((size_t)n_frames);
    size_t spx = 0, bit_words = 0, arena_ints = 0;
    int64_t tiles = 0;
    for (int f = 0; f < n_frames; f++) {
        const cs_frame_view &v = views[f];
        LsdGeom &G = g[(size_t)f];
        memset(&G, 0, sizeof G);
        G.W = (int)std::lrint(v.width * LSD_SCALE);
        G.H = (int)std::lrint(v.height * LSD_SCALE);
        if (G.W < 2 || G.H < 2) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: a %d x %d image is too small for LSD", f, v.width, v.height);
        G.img_off = v.offset;
        G.w = v.width;
        G.h = v.height;
        G.stride = v.stride;
        G.channels = v.channels;
        G.LOG_NT = lsd_log_nt(G.W, G.H);
        G.min_reg_size = lsd_min_reg_size(G.LOG_NT);
        G.tiles_x = (G.W + LSF_TW - 1) / LSF_TW;
        G.tile0 = (int)tiles;
        tiles += (int64_t)G.tiles_x * ((G.H + LSF_TH - 1) / LSF_TH);
        G.px_off = (int64_t)spx;
        spx += (size_t)G.W * G.H;
        G.bit_off = (int64_t)bit_words;
        bit_words += (size_t)((G.W + 31) / 32) * G.H;
        G.arena_off = (int64_t)arena_ints;
        arena_ints += (size_t)lsd_arena_cap(G.W, G.H);
    }
    if (tiles > INT32_MAX) return cs_ctx_fail(c, CS_ERR_CAPACITY, "%lld front-end tiles in one batch: more than a grid holds", (long long)tiles);
    int rc;
    if ((rc = ensure(c, S.geom, g.size() * sizeof(LsdGeom))) || (rc = lsd_buffers(c, S, n_frames, spx, bit_words, arena_ints, cap))) return rc;
    if (cudaMemcpyAsync(S.geom.p, g.data(), g.size() * sizeof(LsdGeom), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the LSD frame table failed");
    const LsdGeom *d_geom = (const LsdGeom *)S.geom.p;
    CUtensorMap tm;
    memset(&tm, 0, sizeof tm);
    k_lsd_front<false, false, true><<<(unsigned)tiles, 256, 0, st>>>(tm, d_img, 0, 0, 0, 0, 0, 0, 1. / LSD_SCALE, LSD_QUANT / std::sin(lsd_prec()),
                                                                     (double *)S.modgrad.p, (float *)S.angf.p, (uint4 *)S.pix.p, (uint32_t *)S.defb.p, nullptr,
                                                                     (int32_t *)S.err.p, d_geom, n_frames);
    LsdGrowArgs A = lsd_args(S, cap, line_length_thres);
    A.geom = d_geom;
    if ((rc = lsd_seed_loop<true>(c, A, n_frames))) return rc;
    S.last_mixed = true;
    S.last_frames = n_frames;
    S.cap = cap;
    return CS_OK;
}

LsdState *state_of(cs_ctx *c)
{
    void **slot = cs_ctx_lsd_slot(c);
    if (!*slot) *slot = new LsdState();
    return (LsdState *)*slot;
}

/* after a run whose error word (read back) says a frame had more candidate rectangles than the hand-off buffer held: grow the buffer to
 * the largest count, for the next run (false: nothing to grow) */
bool lsd_grow_candidates(LsdState &S, const int32_t err[4])
{
    if (!(err[0] & 4) || err[1] <= S.cand_cap) return false;
    S.cand_cap = (err[1] + 255) & ~255;
    return true;
}

}  // namespace

/* device-to-device entry used by the online batch path: frames already in HBM, results stay in HBM */
int cs_lsd_run_device(cs_ctx *c, const uint8_t *d_imgs, int n_frames, int w, int h, int stride, int channels, float line_length_thres, int cap,
                      const float **d_lines, const int32_t **d_counts)
{
    LsdState *S = state_of(c);
    const int rc = lsd_run(c, d_imgs, true, n_frames, w, h, stride, channels, line_length_thres, cap, *S);
    if (rc) return rc;
    *d_lines = (const float *)S->out.p;
    *d_counts = (const int32_t *)S->nout.p;
    return CS_OK;
}

/* host frames in, results stay in HBM (the synchronous descriptor path, cs_lbd.cu) */
int cs_lsd_run_host(cs_ctx *c, const uint8_t *imgs, int n_frames, int w, int h, int stride, int channels, float line_length_thres, int cap,
                    const float **d_lines, const int32_t **d_counts, const uint8_t **d_frames)
{
    return cs_lsd_run_sync(c, imgs, false, n_frames, w, h, stride, channels, line_length_thres, cap, d_lines, d_counts, d_frames);
}

namespace {
/* waits for the run `run` started and reads its error word back; a candidate overflow grows the buffer and runs once more, on the same
 * frames */
template <typename Run>
int lsd_sync(cs_ctx *c, LsdState &S, Run run)
{
    cudaStream_t st = cs_ctx_stream(c);
    for (int pass = 0;; pass++) {
        int rc = run();
        if (rc) return rc;
        int32_t err[4] = {0, 0, 0, 0};
        if (cudaMemcpyAsync(err, S.err.p, sizeof err, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "LSD error word copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        if (pass == 0 && lsd_grow_candidates(S, err)) continue;
        return cs_lsd_check_err(c, err);
    }
}
}  // namespace

/* host frames are copied in again on the rerun, device frames (the LSD frame buffer, cs_ingest.cu) are still where they were */
int cs_lsd_run_sync(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int w, int h, int stride, int channels, float line_length_thres,
                    int cap, const float **d_lines, const int32_t **d_counts, const uint8_t **d_frames)
{
    LsdState *S = state_of(c);
    const int rc = lsd_sync(c, *S, [&] { return lsd_run(c, imgs, imgs_on_device, n_frames, w, h, stride, channels, line_length_thres, cap, *S); });
    if (rc) return rc;
    *d_lines = (const float *)S->out.p;
    *d_counts = (const int32_t *)S->nout.p;
    *d_frames = imgs_on_device ? imgs : (const uint8_t *)S->img.p; /* the frames the run read (same stride), still in HBM */
    return CS_OK;
}

int cs_lsd_run_mixed_sync(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, float line_length_thres, int cap,
                          const float **d_lines, const int32_t **d_counts)
{
    LsdState *S = state_of(c);
    const int rc = lsd_sync(c, *S, [&] { return lsd_run_mixed(c, d_imgs, views, n_frames, line_length_thres, cap, *S); });
    if (rc) return rc;
    *d_lines = (const float *)S->out.p;
    *d_counts = (const int32_t *)S->nout.p;
    return CS_OK;
}

int cs_lsd_run_mixed_device(cs_ctx *c, const uint8_t *d_imgs, const cs_frame_view *views, int n_frames, float line_length_thres, int cap,
                            const float **d_lines, const int32_t **d_counts, const int32_t **d_err)
{
    LsdState *S = state_of(c);
    const int rc = lsd_run_mixed(c, d_imgs, views, n_frames, line_length_thres, cap, *S);
    if (rc) return rc;
    *d_lines = (const float *)S->out.p;
    *d_counts = (const int32_t *)S->nout.p;
    *d_err = (const int32_t *)S->err.p;
    return CS_OK;
}

int cs_check_frame_views(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames)
{
    if (!imgs || !views || n_frames <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    for (int f = 0; f < n_frames; f++) {
        const cs_frame_view &v = views[f];
        if (v.offset < 0 || v.width <= 0 || v.height <= 0)
            return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: offset %lld, %d x %d: the offset must not be negative and the size not empty", f,
                               (long long)v.offset, v.width, v.height);
        /* LSDDetector.cpp:163-164 throws on depth != 0 */
        if (v.channels != 1 && v.channels != 3) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: channels must be 1 or 3, got %d", f, v.channels);
        if ((int64_t)v.stride < (int64_t)v.width * v.channels)
            return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: stride %d smaller than a row of %d x %d bytes", f, v.stride, v.width, v.channels);
    }
    return CS_OK;
}

size_t cs_packed_frames_bytes(const cs_frame_view *views, int n_frames)
{
    size_t n = 0;
    for (int f = 0; f < n_frames; f++) n += (size_t)views[f].height * views[f].width * views[f].channels;
    return n;
}

/* Copies n_frames host frames (imgs + views[f].offset, rows of views[f].stride bytes) to d_dst, back to back with rows of width * channels
 * bytes, and gives their views there.  Frames that already lie back to back without row padding go in one copy. */
int cs_pack_host_frames(cs_ctx *c, uint8_t *d_dst, const uint8_t *imgs, const cs_frame_view *views, int n_frames, std::vector<cs_frame_view> &packed)
{
    cudaStream_t st = cs_ctx_stream(c);
    packed.assign(views, views + n_frames);
    size_t off = 0;
    for (int f = 0; f < n_frames;) {
        const cs_frame_view &v = views[f];
        const size_t row = (size_t)v.width * v.channels;
        if ((size_t)v.stride != row) {
            if (cudaMemcpy2DAsync(d_dst + off, row, imgs + v.offset, (size_t)v.stride, row, (size_t)v.height, cudaMemcpyHostToDevice, st) != cudaSuccess)
                return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frame %d failed", f);
            packed[f].offset = (int64_t)off;
            packed[f].stride = (int32_t)row;
            off += row * v.height;
            f++;
            continue;
        }
        /* a run of unpadded frames, each starting where the previous one ends */
        const int64_t src0 = v.offset;
        const size_t dst0 = off;
        int64_t src_end = v.offset;
        int g = f;
        for (; g < n_frames; g++) {
            const cs_frame_view &u = views[g];
            const size_t urow = (size_t)u.width * u.channels;
            if ((size_t)u.stride != urow || u.offset != src_end) break;
            packed[g].offset = (int64_t)off;
            off += urow * u.height;
            src_end += (int64_t)(urow * u.height);
        }
        if (cudaMemcpyAsync(d_dst + dst0, imgs + src0, off - dst0, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "H2D copy of frames %d .. %d failed", f, g - 1);
        f = g;
    }
    return CS_OK;
}

void cs_lsd_raw_segments(cs_ctx *c, const float **d_raw, const int32_t **d_nraw)
{
    LsdState *S = state_of(c);
    *d_raw = (const float *)S->raw.p;
    *d_nraw = (const int32_t *)S->nraw.p;
}

void cs_lsd_destroy(void *state)
{
    LsdState *S = (LsdState *)state;
    Buf *all[] = {&S->img, &S->modgrad, &S->angf, &S->pix, &S->defb, &S->arena, &S->raw, &S->nraw, &S->out, &S->nout, &S->lgam, &S->ubits, &S->cand, &S->ncand, &S->candline, &S->candstate, &S->err, &S->geom};
    for (Buf *b : all)
        if (b->p) cudaFree(b->p);
    delete S;
}

uint8_t *cs_lsd_frame_buffer(cs_ctx *c, size_t bytes)
{
    LsdState *S = state_of(c);
    return ensure(c, S->img, bytes) ? nullptr : (uint8_t *)S->img.p;
}

/* views: frames of different sizes on the device at imgs + views[f].offset (LSD only; width .. channels are then unused); frame_index: the
 * caller's number of each frame, for the capacity message (null: 0 .. n_frames - 1) */
int cs_detect_lines_run(cs_ctx *c, const uint8_t *imgs, bool imgs_on_device, int n_frames, int width, int height, int stride, int channels,
                        const cs_line_params *params, float *lines_xyxy, int32_t max_lines_per_frame, int32_t *n_lines, const cs_frame_view *views,
                        const int32_t *frame_index)
{
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    std::vector<int32_t> cnt(n_frames);
    for (int pass = 0;; pass++) {
        const float *d_out = nullptr;
        const int32_t *d_nout = nullptr, *d_err = nullptr;
        int rc;
        if (params->use_LSD) {
            LsdState *S = state_of(c);
            rc = views ? lsd_run_mixed(c, imgs, views, n_frames, params->line_length_thres, max_lines_per_frame, *S)
                       : lsd_run(c, imgs, imgs_on_device, n_frames, width, height, stride, channels, params->line_length_thres, max_lines_per_frame, *S);
            d_out = (const float *)S->out.p;
            d_nout = (const int32_t *)S->nout.p;
            d_err = (const int32_t *)S->err.p;
        } else {
            rc = cs_edl_run(c, imgs, imgs_on_device, n_frames, width, height, stride, channels, params->line_length_thres, max_lines_per_frame, &d_out,
                            &d_nout);
            d_err = cs_line_err_word(*cs_ctx_edl_slot(c));
        }
        if (rc) return rc;
        int32_t err[4] = {0, 0, 0, 0};
        if (cudaMemcpyAsync(cnt.data(), d_nout, (size_t)n_frames * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaMemcpyAsync(err, d_err, sizeof err, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaMemcpyAsync(lines_xyxy, d_out, (size_t)n_frames * max_lines_per_frame * 16, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "line result copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        /* a frame had more candidate rectangles than the hand-off buffer held: grow it to the batch's largest count and run once more */
        if (params->use_LSD && pass == 0 && lsd_grow_candidates(*state_of(c), err)) continue;
        if ((rc = params->use_LSD ? cs_lsd_check_err(c, err) : cs_edl_check_err(c, err))) return rc;
        break;
    }
    for (int f = 0; f < n_frames; f++) {
        if (cnt[f] > max_lines_per_frame)
            return cs_ctx_fail(c, CS_ERR_CAPACITY, "frame %d: %d segments exceed max_lines_per_frame", frame_index ? frame_index[f] : f, cnt[f]);
        n_lines[f] = cnt[f];
    }
    return CS_OK;
}

extern "C" {

int cs_detect_lines_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                          const cs_line_params *params, float *lines_xyxy, int32_t max_lines_per_frame, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!imgs || !params || !lines_xyxy || !n_lines || n_frames <= 0 || width <= 0 || height <= 0 || max_lines_per_frame <= 0)
        return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3"); /* LSDDetector.cpp:163-164 throws on depth != 0 */
    if (stride < width * channels) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    /* More octaves change nothing here: filter_lines keeps octave 0 only (line_lbd_allclass.cpp:200-207) and octave 0 is detected first and
     * independently of the others in both detectors, so the matrix is the one-octave one (checked against the compiled reference with 2 and
     * 3 octaves, tests/test_oracle_ref_octaves.py). */
    if (params->numoctaves < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1");
    return cs_detect_lines_run(c, imgs, false, n_frames, width, height, stride, channels, params, lines_xyxy, max_lines_per_frame, n_lines);
}

}

int cs_check_line_frames(cs_ctx *c, const cs_frame_view *views, int n_frames, const cs_line_params *params)
{
    if (params->use_LSD && n_frames > CS_LSD_MAX_MIXED_FRAMES)
        return cs_ctx_fail(c, CS_ERR_CAPACITY, "%d frames in one LSD batch: at most %d", n_frames, CS_LSD_MAX_MIXED_FRAMES);
    if (params->numoctaves < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1");
    for (int f = 0; f < n_frames; f++) {
        const int w = views[f].width, h = views[f].height;
        if (params->use_LSD && (std::lrint(w * LSD_SCALE) < 2 || std::lrint(h * LSD_SCALE) < 2))
            return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: a %d x %d image is too small for LSD", f, w, h);
        if (!params->use_LSD && (w < 8 || h < 8 || w > 65535 || h > 65535)) /* cs_edl_run's bounds, checked here before any group runs */
            return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "frame %d: a %d x %d image is outside EDLines' sizes (8 .. 65535 per side)", f, w, h);
    }
    return CS_OK;
}

extern "C" {

int cs_detect_lines_batch_mixed(cs_ctx *c, const uint8_t *imgs, const cs_frame_view *views, int n_frames, const cs_line_params *params,
                                float *lines_xyxy, int32_t max_lines_per_frame, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc;
    if ((rc = cs_check_frame_views(c, imgs, views, n_frames))) return rc;
    if (!params || !lines_xyxy || !n_lines || max_lines_per_frame <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if ((rc = cs_check_line_frames(c, views, n_frames, params))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const size_t slot = (size_t)max_lines_per_frame * 4;
    if (!params->use_LSD) {
        /* EDLines: one batch per (width, height, channels) group, its frames gathered on the host in call order */
        std::vector<int> done((size_t)n_frames, 0);
        std::vector<int32_t> idx, cnt;
        std::vector<uint8_t> pack;
        std::vector<float> out;
        for (int f0 = 0; f0 < n_frames; f0++) {
            if (done[f0]) continue;
            const cs_frame_view &v0 = views[f0];
            const size_t row = (size_t)v0.width * v0.channels, fb = row * v0.height;
            idx.clear();
            for (int f = f0; f < n_frames; f++)
                if (!done[f] && views[f].width == v0.width && views[f].height == v0.height && views[f].channels == v0.channels) {
                    idx.push_back(f);
                    done[f] = 1;
                }
            const int G = (int)idx.size();
            pack.resize(fb * G);
            for (int j = 0; j < G; j++)
                for (int y = 0; y < v0.height; y++)
                    memcpy(&pack[j * fb + y * row], imgs + views[idx[j]].offset + (size_t)y * views[idx[j]].stride, row);
            out.resize(slot * G);
            cnt.resize(G);
            if ((rc = cs_detect_lines_run(c, pack.data(), false, G, v0.width, v0.height, (int)row, v0.channels, params, out.data(), max_lines_per_frame,
                                          cnt.data(), nullptr, idx.data())))
                return rc;
            for (int j = 0; j < G; j++) {
                n_lines[idx[j]] = cnt[j];
                memcpy(lines_xyxy + idx[j] * slot, &out[j * slot], (size_t)cnt[j] * 16);
            }
        }
        return CS_OK;
    }
    uint8_t *buf = cs_lsd_frame_buffer(c, cs_packed_frames_bytes(views, n_frames));
    if (!buf) return CS_ERR_CUDA;
    std::vector<cs_frame_view> packed;
    if ((rc = cs_pack_host_frames(c, buf, imgs, views, n_frames, packed))) return rc;
    return cs_detect_lines_run(c, buf, true, n_frames, 0, 0, 0, 0, params, lines_xyxy, max_lines_per_frame, n_lines, packed.data(), nullptr);
}

int cs_detect_lines(cs_ctx *c, const uint8_t *img, int width, int height, int stride, int channels, const cs_line_params *params,
                    float *lines_xyxy, int32_t *n_inout)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!n_inout || *n_inout <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "n_inout must give the capacity of lines_xyxy");
    int32_t n = 0;
    const int rc = cs_detect_lines_batch(c, img, 1, width, height, stride, channels, params, lines_xyxy, *n_inout, &n);
    if (rc == CS_OK) *n_inout = n;
    return rc;
}

/* inspection of the last run's intermediate images of one frame (tests): any pointer may be NULL */
int cs_debug_lsd(cs_ctx *c, int frame, int32_t *scaled_wh, double *scaled, double *modgrad, double *angles, int32_t *list, int32_t *list_len,
                 float *raw_lines, int32_t *n_raw, int cap_raw)
{
    if (!c) return CS_ERR_INVALID_ARG;
    LsdState *S = state_of(c);
    if (S->last_mixed) return cs_ctx_fail(c, CS_ERR_UNSUPPORTED, "cs_debug_lsd reads one-size batches only: the last LSD run was a batch of mixed sizes");
    if (frame < 0 || frame >= S->last_frames) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad frame index");
    cudaSetDevice(cs_ctx_device(c));
    cudaStreamSynchronize(cs_ctx_stream(c));
    const size_t npx = (size_t)S->last_W * S->last_H;
    if (scaled_wh) {
        scaled_wh[0] = S->last_W;
        scaled_wh[1] = S->last_H;
    }
    if (scaled || modgrad) {
        /* the run keeps neither plane (modgrad only where the angle is defined): recompute both for this frame from its bytes */
        double *d_planes = nullptr;
        if (cudaMalloc(&d_planes, npx * 16) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc of the debug planes failed");
        lsd_front(c, S->last_img + (size_t)frame * S->last_h * S->last_stride, 1, S->last_w, S->last_h, S->last_stride, S->last_channels, S->last_W,
                  S->last_H, 0.0, d_planes + npx, nullptr, nullptr, nullptr, d_planes, nullptr);
        cudaStreamSynchronize(cs_ctx_stream(c));
        if (scaled) cudaMemcpy(scaled, d_planes, npx * 8, cudaMemcpyDeviceToHost);
        if (modgrad) cudaMemcpy(modgrad, d_planes + npx, npx * 8, cudaMemcpyDeviceToHost);
        cudaFree(d_planes);
    }
    if (angles) {
        /* the level-line angle map as the reference holds it: (double)fastAtan2 * DEG2RAD, NOTDEF = -1024 (the product is IEEE-exact on either side) */
        std::vector<float> deg(npx);
        cudaMemcpy(deg.data(), (float *)S->angf.p + frame * npx, npx * 4, cudaMemcpyDeviceToHost);
        for (size_t i = 0; i < npx; i++) angles[i] = deg[i] < 0.f ? LSD_NOTDEF : (double)deg[i] * LSD_DEG2RAD;
    }
    if (list || list_len) {
        /* the order seeds are visited in: raster order over the pixels with a defined angle (lsd.cpp:478-481) */
        std::vector<float> deg(npx);
        cudaMemcpy(deg.data(), (float *)S->angf.p + frame * npx, npx * 4, cudaMemcpyDeviceToHost);
        int32_t ll = 0;
        for (size_t i = 0; i < npx; i++)
            if (deg[i] >= 0.f) {
                if (list) list[ll] = (int32_t)i;
                ll++;
            }
        if (list_len) *list_len = ll;
    }
    int32_t nr = 0;
    cudaMemcpy(&nr, (int32_t *)S->nraw.p + frame, 4, cudaMemcpyDeviceToHost);
    if (n_raw) *n_raw = nr;
    if (raw_lines) cudaMemcpy(raw_lines, (float *)S->raw.p + (size_t)frame * S->cap * 4, (size_t)std::min(nr, std::min(cap_raw, S->cap)) * 16, cudaMemcpyDeviceToHost);
    return cudaGetLastError() == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "debug copy failed");
}

/* the last run's defined-angle bit plane of one frame (tests): *words_per_row = ceil(W / 32), bits = H * that many words (may be NULL) */
int cs_debug_lsd_defb(cs_ctx *c, int frame, uint32_t *bits, int32_t *words_per_row)
{
    if (!c) return CS_ERR_INVALID_ARG;
    LsdState *S = state_of(c);
    if (S->last_mixed)
        return cs_ctx_fail(c, CS_ERR_UNSUPPORTED, "cs_debug_lsd_defb reads one-size batches only: the last LSD run was a batch of mixed sizes");
    if (frame < 0 || frame >= S->last_frames) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad frame index");
    cudaSetDevice(cs_ctx_device(c));
    cudaStreamSynchronize(cs_ctx_stream(c));
    const size_t ww = ((size_t)S->last_W + 31) / 32, n = ww * S->last_H;
    if (words_per_row) *words_per_row = (int32_t)ww;
    if (bits) cudaMemcpy(bits, (const uint32_t *)S->defb.p + frame * n, n * 4, cudaMemcpyDeviceToHost);
    return cudaGetLastError() == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "debug copy failed");
}

/* cycle counters of the seed loop's phases summed over every warp since the last reset (diagnostics): {region_grow, region2rect, refine,
 * raster scan for seeds (everything outside lsd_grow_candidate), used-map re-reads after a grow, candidates grown, whole kernel (per CTA),
 * region pixels of the first grows, seeds whose region list outgrew its shared-memory part, per-seed hand-off, density decision and
 * candidate store, reduce_region_radius, seeds reaching region2rect, refines, reduce iterations, region2rect sizes (see g_lsd_prof)}. */
int cs_debug_lsd_prof(cs_ctx *c, uint64_t *out16, int reset)
{
    if (!c) return CS_ERR_INVALID_ARG;
    cudaSetDevice(cs_ctx_device(c));
    cudaStreamSynchronize(cs_ctx_stream(c));
    if (out16) cudaMemcpyFromSymbol(out16, g_lsd_prof, 128);
    if (reset) {
        const unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(g_lsd_prof, z, 128);
    }
    return cudaGetLastError() == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "debug copy failed");
}

/* resources and residency of the seed loop and the front end, as the device reports them (tools/lsd_occupancy.py) */
int cs_debug_lsd_occupancy(cs_ctx *c, int32_t *out14)
{
    if (!c || !out14) return CS_ERR_INVALID_ARG;
    cudaSetDevice(cs_ctx_device(c));
    struct {
        const void *fn;
        int threads, dyn_smem;
    } const k[2] = {{(const void *)k_lsd_grow_seq<false, false>, 32, LSD_SEQ_SMEM}, {(const void *)k_lsd_front<true, false, false>, 256, 0}};
    for (int i = 0; i < 2; i++) {
        cudaFuncAttributes a;
        int per_sm = 0;
        if (cudaFuncGetAttributes(&a, k[i].fn) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k[i].fn, k[i].threads, k[i].dyn_smem) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "LSD kernel attribute query failed: %s", cudaGetErrorString(cudaGetLastError()));
        int32_t *o = out14 + 7 * i;
        o[0] = a.numRegs;
        o[1] = (int32_t)a.localSizeBytes;
        o[2] = (int32_t)a.sharedSizeBytes;
        o[3] = k[i].dyn_smem;
        o[4] = k[i].threads;
        o[5] = per_sm;
        o[6] = a.preferredShmemCarveout;
    }
    return CS_OK;
}

/* kept for ABI stability (see the header): the seed loop runs one warp per frame with no speculative rounds, so stats4 reads zero and
 * redo[f] = 1 */
int cs_debug_lsd_stats(cs_ctx *c, int32_t *stats4, int32_t *redo, int n_frames)
{
    if (!c) return CS_ERR_INVALID_ARG;
    LsdState *S = state_of(c);
    if (n_frames > S->last_frames) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "more frames than the last run held");
    if (stats4) memset(stats4, 0, (size_t)n_frames * 16);
    if (redo)
        for (int f = 0; f < n_frames; f++) redo[f] = 1;
    return CS_OK;
}
}
