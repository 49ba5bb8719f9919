/*
 * cs_kernels_image.cu -- per-frame / per-ROI image stages of detect_cuboid for sm_90a.
 *
 *   k_bgr2gray      cv::cvtColor(BGR2GRAY)                      box_proposal_detail.cpp:62-66
 *   k_canny_nms     cv::Canny: Sobel 3x3 + L1 magnitude + NMS    box_proposal_detail.cpp:197
 *   k_canny_hyst    cv::Canny: hysteresis (order independent)    box_proposal_detail.cpp:197
 *   k_chamfer_dt    cv::distanceTransform(DIST_L2, 3)            box_proposal_detail.cpp:199
 *
 * All stages are integer / fixed-point and therefore reproduce OpenCV's results bit for bit (checked in tests/).
 *
 * Edge maps travel as BIT PLANES (1 bit per pixel): plane S = "edge" (strong, or weak reached by the
 * hysteresis), plane W = weak candidates.  A ROI of h rows x w columns is stored with a one-word / one-row
 * zero border: (h+2) rows of (bw+2) 32-bit words, bw = ceil(w/32).  That makes NMS output two ballots per
 * warp, hysteresis a word-parallel dilation in shared memory, and the distance transform's input 32x smaller.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "cs_internal.h"
#include "cs_kernels.h"

/* ------------------------------------------------------------------------------------------
 * BGR -> gray.  Pure stream: 3 B read + 1 B written per pixel, the one HBM-bound kernel of the
 * path.  Contiguous frames are treated as one flat pixel array so every thread moves 48 B in
 * (three 16-byte loads) and 16 B out, all naturally aligned.
 * ------------------------------------------------------------------------------------------ */
__device__ __forceinline__ uint32_t luma15(uint32_t b, uint32_t g, uint32_t r)
{
    return (b * 3735u + g * 19235u + r * 9798u + (1u << 14)) >> 15;
}

__global__ void __launch_bounds__(256) k_bgr2gray_flat(const uint4 *__restrict__ bgr, uint4 *__restrict__ gray,
                                                        int64_t n_groups /* of 16 pixels */)
{
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
        const uint4 a = __ldcs(bgr + 3 * g), b = __ldcs(bgr + 3 * g + 1), c = __ldcs(bgr + 3 * g + 2);
        const uint32_t w[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
        uint32_t out[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            /* 4 pixels = 12 bytes = words 3q .. 3q+2 */
            const uint32_t w0 = w[3 * q], w1 = w[3 * q + 1], w2 = w[3 * q + 2];
            const uint32_t p0 = luma15(w0 & 255u, (w0 >> 8) & 255u, (w0 >> 16) & 255u);
            const uint32_t p1 = luma15(w0 >> 24, w1 & 255u, (w1 >> 8) & 255u);
            const uint32_t p2 = luma15((w1 >> 16) & 255u, w1 >> 24, w2 & 255u);
            const uint32_t p3 = luma15((w2 >> 8) & 255u, (w2 >> 16) & 255u, w2 >> 24);
            out[q] = p0 | (p1 << 8) | (p2 << 16) | (p3 << 24);
        }
        gray[g] = make_uint4(out[0], out[1], out[2], out[3]);
    }
}

/* generic (strided / tail) variant: one pixel per thread */
__global__ void __launch_bounds__(256) k_bgr2gray_generic(const uint8_t *__restrict__ img, uint8_t *__restrict__ gray, int n_frames,
                                                           int w, int h, int stride, int channels, int64_t first_pixel)
{
    const int64_t total = (int64_t)n_frames * w * h;
    for (int64_t p = first_pixel + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = p / ((int64_t)w * h);
        const int64_t r = p - f * (int64_t)w * h;
        const int y = (int)(r / w), x = (int)(r - (int64_t)y * w);
        const uint8_t *s = img + ((size_t)f * h + y) * stride + (size_t)x * channels;
        gray[p] = (channels == 3) ? (uint8_t)luma15(s[0], s[1], s[2]) : s[0];
    }
}

/* ------------------------------------------------------------------------------------------
 * Canny part 1: Sobel + |dx|+|dy| + non-maximum suppression over 32x32 tiles of each ROI.
 * The gray tile (+2 halo, replicated at the ROI border: OpenCV filters an ROI in isolation) is staged
 * in shared memory; magnitudes of the +1 halo are held there too (zero outside the ROI).  A warp
 * owns 32 consecutive pixels of a row, so the strong / weak classification leaves as two ballots.
 * ------------------------------------------------------------------------------------------ */
#define CT 32  /* tile edge */
#define CTP 64 /* pitch of the staged gray tile in bytes (36 used) */

__global__ void __launch_bounds__(256) k_canny_nms(const uint8_t *__restrict__ gray, const CsJob *__restrict__ jobs,
                                                   const int32_t *__restrict__ tile_job, uint32_t *__restrict__ bits_arena, int low, int high)
{
    /* gray, +2 halo: 36 rows at a pitch of CTP bytes, in two buffers that alternate from tile to tile */
    __shared__ __align__(128) uint8_t s_gb_raw[2][((CT + 4) * CTP + 127) / 128 * 128];
    __shared__ int32_t s_d[CT + 2][CT + 2 + 1];   /* (dy << 16) | (dx & 0xffff), +1 halo */
    __shared__ uint16_t s_m[CT + 2][CT + 2 + 2];  /* |dx| + |dy|, zero outside the ROI */
    /* a block owns one ROW of tiles of one ROI and walks it left to right; the gray bytes of the next tile are fetched into
     * registers while the current tile is being processed, so only the first tile of a row pays the global-load latency */
    const int packed = tile_job[blockIdx.x];
    const CsJob &jb = jobs[packed >> 8];
    const int tile_y = packed & 255;
    const int w = jb.roi_w, h = jb.roi_h, tiles_x = jb.tiles_x;
    const int y0 = tile_y * CT;
    const uint8_t *src = gray + jb.gray_off; /* the ROI's top-left byte in its frame's gray plane (frames of a batch may differ in size) */
    const int pitch = jb.gray_pitch;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int tid = ty * 32 + tx;
    const int TG22 = 13573; /* (int)(0.4142135623730950488016887242097 * (1 << 15) + 0.5) */
    const int bwp = jb.bw + 2;
    uint32_t *planeS = bits_arena + jb.bit_off;
    uint32_t *planeW = planeS + (size_t)(h + 2) * bwp;
    const int MP = CT + 2 + 2; /* pitch of s_m in elements */
    const uint16_t *mflat = &s_m[0][0];
    constexpr int NPRE = ((CT + 4) * (CT + 4) + 255) / 256;
    uint8_t pre[NPRE];
    auto fetch = [&](int x0) { /* clamped byte loads into registers */
#pragma unroll
        for (int q = 0; q < NPRE; q++) {
            const int i = tid + q * 256;
            pre[q] = 0;
            if (i < (CT + 4) * (CT + 4)) {
                const int ly = i / (CT + 4), lx = i - ly * (CT + 4);
                const int gy = min(max(y0 + ly - 2, 0), h - 1);
                const int gx = min(max(x0 + lx - 2, 0), w - 1);
                pre[q] = __ldg(src + gy * pitch + gx);
            }
        }
    };
    fetch(0);
    for (int tile_x = 0; tile_x < tiles_x; tile_x++) {
        const int x0 = tile_x * CT;
        const int buf = tile_x & 1;
        uint8_t(*s_g)[CTP] = reinterpret_cast<uint8_t(*)[CTP]>(&s_gb_raw[buf][0]);
#pragma unroll
        for (int q = 0; q < NPRE; q++) {
            const int i = tid + q * 256;
            if (i < (CT + 4) * (CT + 4)) {
                const int ly = i / (CT + 4), lx = i - ly * (CT + 4);
                s_g[ly][lx] = pre[q];
            }
        }
        __syncthreads();
        if (tile_x + 1 < tiles_x) fetch(x0 + CT); /* the next tile, into registers */
        /* Sobel + magnitude for the (CT+2)^2 halo region: a thread owns one column and a strip of 5 rows, the three-row
         * window slides down in registers (21 shared loads for 5 results) */
        int loud = 0; /* does any pixel of the tile proper exceed the low threshold? (the +1 halo ring does not count) */
        if (tid < (CT + 2) * 7) {
            const int strip = tid / (CT + 2), lx = tid - strip * (CT + 2);
            const int r0 = strip * 5;
            int rs[7], rd[7];
#pragma unroll
            for (int r = 0; r < 7; r++) {
                const int row = min(r0 + r, CT + 3);
                const int a = s_g[row][lx], b = s_g[row][lx + 1], c = s_g[row][lx + 2];
                rs[r] = a + 2 * b + c;
                rd[r] = c - a;
            }
            const int gx = x0 + lx - 1;
            const bool col_in = (gx >= 0) && (gx < w);
#pragma unroll
            for (int j = 0; j < 5; j++) {
                const int ly = r0 + j;
                if (ly < CT + 2) {
                    const int gy = y0 + ly - 1;
                    const int dx = rd[j] + 2 * rd[j + 1] + rd[j + 2];
                    const int dy = rs[j + 2] - rs[j];
                    const bool in = col_in && (gy >= 0) && (gy < h);
                    const int m = in ? abs(dx) + abs(dy) : 0;
                    s_d[ly][lx] = (dy << 16) | (dx & 0xffff);
                    s_m[ly][lx] = (uint16_t)m;
                    loud |= (m > low) && (lx >= 1) && (lx <= CT) && (ly >= 1) && (ly <= CT);
                }
            }
        }
        /* a quiet tile has no edge pixel whatever its neighbours are: its words stay as the memset left them */
        if (!__syncthreads_or(loud)) continue;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int ly = ty + 8 * k, lx = tx;
            const int gy = y0 + ly, gx = x0 + lx;
            int code = 0;
            if (gy < h && gx < w) {
                const int mi = (ly + 1) * MP + lx + 1;
                const int m = mflat[mi];
                if (m > low) {
                    const int d = s_d[ly + 1][lx + 1];
                    const int xs = (int)(int16_t)(d & 0xffff), ys = d >> 16;
                    const int ax = abs(xs), ay = abs(ys) << 15;
                    const int tg22x = ax * TG22;
                    const int tg67x = tg22x + (ax << 16);
                    /* direction sector -> neighbour offset and comparison kind, without divergent branches */
                    const bool horiz = ay < tg22x;
                    const bool vert = !horiz && (ay > tg67x);
                    const int sgn = ((xs ^ ys) < 0) ? -1 : 1;
                    const int off = horiz ? 1 : (vert ? MP : MP + sgn);
                    const int ma = mflat[mi - off], mb = mflat[mi + off];
                    const bool is_max = (m > ma) && ((horiz || vert) ? (m >= mb) : (m > mb));
                    if (is_max) code = (m > high) ? 2 : 1;
                }
            }
            const unsigned strong = __ballot_sync(0xffffffffu, code == 2);
            const unsigned weak = __ballot_sync(0xffffffffu, code == 1);
            if (tx == 0 && gy < h) {
                const int wi = (gy + 1) * bwp + 1 + tile_x;
                planeS[wi] = strong;
                planeW[wi] = weak;
            }
        }
        __syncthreads();
    }
}

/* ------------------------------------------------------------------------------------------
 * Canny part 2: hysteresis on the bit planes.  One CTA per ROI; both planes sit in shared memory
 * (global memory for ROIs too large for it).  A thread owns one word column over a run of rows and
 * sweeps it down and up: new = dilate3x3(S) & W, closed horizontally inside the word, moved from W
 * to S.  Sweeps repeat until no thread changed anything.  The fixed point (every weak pixel
 * 8-connected to a strong one) is unique, hence identical to OpenCV's stack-based flood fill.
 * ------------------------------------------------------------------------------------------ */
#define HY_THREADS 256

template <class PT>
__device__ __forceinline__ bool hyst_word(PT S, PT W, int bwp, int r, int c)
{
    const size_t i = (size_t)r * bwp + c;
    uint32_t m = W[i];
    if (m == 0) return false;
    const uint32_t nC = S[i - bwp] | S[i] | S[i + bwp];
    const uint32_t nL = S[i - bwp - 1] | S[i - 1] | S[i + bwp - 1];
    const uint32_t nR = S[i - bwp + 1] | S[i + 1] | S[i + bwp + 1];
    const uint32_t d = nC | (nC << 1) | (nC >> 1) | (nL >> 31) | (nR << 31);
    uint32_t nw = d & m;
    if (nw == 0) return false;
    uint32_t s = S[i] | nw;
    m &= ~nw;
    /* close horizontally inside the word */
    while (true) {
        const uint32_t t = ((s << 1) | (s >> 1)) & m;
        if (t == 0) break;
        s |= t;
        m &= ~t;
    }
    S[i] = s;
    W[i] = m;
    return true;
}

extern __shared__ uint32_t hy_smem[];

__global__ void __launch_bounds__(HY_THREADS) k_canny_hyst(const CsJob *__restrict__ jobs, uint32_t *__restrict__ bits_arena, int smem_words)
{
    const CsJob &jb = jobs[blockIdx.x];
    const int h = jb.roi_h, bw = jb.bw, bwp = bw + 2;
    const int plane = (h + 2) * bwp;
    uint32_t *gS = bits_arena + jb.bit_off;
    const bool in_smem = (2 * plane <= smem_words);
    uint32_t *S = in_smem ? hy_smem : gS;
    uint32_t *W = S + plane;
    const int tid = threadIdx.x;
    if (in_smem) {
        for (int i = tid; i < 2 * plane; i += HY_THREADS) S[i] = gS[i];
        __syncthreads();
    }
    /* thread -> (word column, row run) */
    const int n_runs = max(HY_THREADS / bw, 1);
    const int rows_per = (h + n_runs - 1) / n_runs;
    const int c = 1 + tid % bw, run = tid / bw;
    const int r0 = 1 + run * rows_per, r1 = min(r0 + rows_per, h + 1);
    const bool active = (run < n_runs) && (tid < n_runs * bw);
    while (true) {
        bool changed = false;
        if (active) {
            if (in_smem) {
                for (int r = r0; r < r1; r++) changed |= hyst_word<uint32_t *>(S, W, bwp, r, c);
                for (int r = r1 - 2; r >= r0; r--) changed |= hyst_word<uint32_t *>(S, W, bwp, r, c);
            } else { /* oversized ROI: iterate in global memory (volatile: neighbours' updates must be re-read) */
                for (int r = r0; r < r1; r++) changed |= hyst_word<volatile uint32_t *>(S, W, bwp, r, c);
                for (int r = r1 - 2; r >= r0; r--) changed |= hyst_word<volatile uint32_t *>(S, W, bwp, r, c);
                __threadfence();
            }
        }
        if (!__syncthreads_or(changed ? 1 : 0)) break;
    }
    if (in_smem) {
        for (int i = tid; i < plane; i += HY_THREADS) gS[i] = S[i];
    }
}

/* ------------------------------------------------------------------------------------------
 * 3x3 chamfer distance transform, two raster passes in 16.16 fixed point (a = 62587, b = 89738).
 * One warp per ROI; a lane owns PPL consecutive columns of the current row in registers.  The
 * in-row recurrence tmp[j] = min(u[j], tmp[j-1] + a) is a min-plus prefix scan:
 *      tmp[j] = a*j + min_{k<=j} (u[k] - a*k)
 * evaluated as a local scan + a 5-step warp scan, all in exact integer arithmetic, so the result
 * equals the sequential OpenCV loop bit for bit.  "Infinity" is a sentinel BIG (> any reachable
 * distance) that is re-clamped every row; it is emitted as OpenCV's saturated DIST_MAX.
 * The edge bits of the next rows are prefetched into registers; the backward pass streams the forward
 * rows back through a cp.async ring in shared memory, so no row waits on an L2 round trip.
 * ------------------------------------------------------------------------------------------ */
#define DT_HV 62587
#define DT_DG 89738
#define DT_BIG (1 << 30)
#define DT_PF 4   /* prefetch depth (rows) */

/* raw bit-plane words covering columns [c0, c0+PPL) of one row (prefetched; shifted only when consumed so the
 * loads stay in flight across DT_PF rows) */
struct DtWords {
    uint32_t a, b, c;
};
template <int PPL>
__device__ __forceinline__ DtWords dt_row_words(const uint32_t *__restrict__ row_words /* word 0 = column 0 */, int c0, int bw)
{
    const int w0 = c0 >> 5;
    DtWords r;
    r.a = (w0 < bw) ? __ldg(row_words + w0) : 0u;
    r.b = (w0 + 1 < bw) ? __ldg(row_words + w0 + 1) : 0u;
    r.c = 0u;
    if (PPL > 32) r.c = (w0 + 2 < bw) ? __ldg(row_words + w0 + 2) : 0u;
    return r;
}
template <int PPL>
__device__ __forceinline__ uint64_t dt_bits_of(const DtWords &r, int c0)
{
    const int sh = c0 & 31;
    uint64_t bits = __funnelshift_r(r.a, r.b, sh);
    if (PPL > 32) bits |= (uint64_t)__funnelshift_r(r.b, r.c, sh) << 32;
    return bits;
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

template <int PPL>
__device__ __forceinline__ void dt_warp(const uint32_t *__restrict__ planeS, int bwp, uint32_t *__restrict__ tmp, int w, int h, int dpitch,
                                        uint32_t *ring /* DT_PF rows of dpitch words, shared */)
{
    const int lane = threadIdx.x & 31;
    const int c0 = lane * PPL;
    const unsigned FULL = 0xffffffffu;
    const int bw = bwp - 2;
    int up[PPL];
#pragma unroll
    for (int k = 0; k < PPL; k++) up[k] = DT_BIG;

    /* ---- forward pass ---- */
    DtWords pf[DT_PF];
#pragma unroll
    for (int d = 0; d < DT_PF; d++) pf[d] = dt_row_words<PPL>(planeS + (size_t)(min(d, h - 1) + 1) * bwp + 1, c0, bw);
    for (int i0 = 0; i0 < h; i0 += DT_PF) {
#pragma unroll
        for (int d = 0; d < DT_PF; d++) {
            const int i = i0 + d;
            if (i < h) {
                const uint64_t bits = dt_bits_of<PPL>(pf[d], c0);
                const int nxt = min(i + DT_PF, h - 1);
                pf[d] = dt_row_words<PPL>(planeS + (size_t)(nxt + 1) * bwp + 1, c0, bw);
                int upL = __shfl_up_sync(FULL, up[PPL - 1], 1);
                int upR = __shfl_down_sync(FULL, up[0], 1);
                if (lane == 0) upL = DT_BIG;
                if (lane == 31) upR = DT_BIG;
                int v[PPL];
#pragma unroll
                for (int k = 0; k < PPL; k++) {
                    const int col = c0 + k;
                    const int l = (k == 0) ? upL : up[k - 1];
                    const int r = (k == PPL - 1) ? upR : up[k + 1];
                    int u = min(min(l + DT_DG, up[k] + DT_HV), r + DT_DG);
                    if ((bits >> k) & 1ull) u = 0; /* bits beyond column w are zero (NMS writes none) */
                    if (col >= w) u = DT_BIG;
                    v[k] = u - DT_HV * col;
                }
#pragma unroll
                for (int k = 1; k < PPL; k++) v[k] = min(v[k], v[k - 1]);
                int incl = v[PPL - 1];
#pragma unroll
                for (int dd = 1; dd < 32; dd <<= 1) {
                    const int o = __shfl_up_sync(FULL, incl, dd);
                    if (lane >= dd) incl = min(incl, o);
                }
                int excl = __shfl_up_sync(FULL, incl, 1);
                if (lane == 0) excl = INT_MAX;
                uint32_t *trow = tmp + (size_t)i * dpitch;
#pragma unroll
                for (int k = 0; k < PPL; k++) {
                    const int col = c0 + k;
                    int t = min(v[k], excl) + DT_HV * col;
                    if (t >= DT_BIG || col >= w) t = DT_BIG;
                    up[k] = t;
                }
#pragma unroll
                for (int k = 0; k < PPL; k += 4)
                    if (c0 + k < dpitch) *reinterpret_cast<uint4 *>(trow + c0 + k) = make_uint4(up[k], up[k + 1], up[k + 2], up[k + 3]);
            }
        }
    }

    /* ---- backward pass: `up` now plays the role of the row below ---- */
#pragma unroll
    for (int k = 0; k < PPL; k++) up[k] = DT_BIG;
    const float scale = 1.f / 65536.f;
    const float dist_max = (float)(0xffffffffu - (uint32_t)DT_DG) * scale;
    const int chunks = dpitch >> 2; /* 16-byte chunks per row */
    __syncwarp();
    /* prime the ring with rows h-1 .. h-DT_PF */
#pragma unroll
    for (int d = 0; d < DT_PF; d++) {
        const int i = h - 1 - d;
        if (i >= 0)
            for (int q = lane; q < chunks; q += 32) cp_async16(ring + (size_t)d * dpitch + q * 4, tmp + (size_t)i * dpitch + q * 4);
        cp_async_commit();
    }
    int slot = 0;
    for (int i = h - 1; i >= 0; i--) {
        cp_async_wait<DT_PF - 1>();
        __syncwarp();
        const uint32_t *srow = ring + (size_t)slot * dpitch;
        int cur[PPL];
#pragma unroll
        for (int k = 0; k < PPL; k += 4) {
            uint4 q = make_uint4(DT_BIG, DT_BIG, DT_BIG, DT_BIG);
            if (c0 + k < dpitch) q = *reinterpret_cast<const uint4 *>(srow + c0 + k);
            cur[k] = (int)q.x;
            cur[k + 1] = (int)q.y;
            cur[k + 2] = (int)q.z;
            cur[k + 3] = (int)q.w;
        }
        __syncwarp();
        /* refill this slot with the row DT_PF above */
        {
            const int nxt = i - DT_PF;
            if (nxt >= 0)
                for (int q = lane; q < chunks; q += 32) cp_async16(ring + (size_t)slot * dpitch + q * 4, tmp + (size_t)nxt * dpitch + q * 4);
            cp_async_commit();
        }
        slot = (slot + 1 == DT_PF) ? 0 : slot + 1;
        int dnL = __shfl_up_sync(FULL, up[PPL - 1], 1);
        int dnR = __shfl_down_sync(FULL, up[0], 1);
        if (lane == 0) dnL = DT_BIG;
        if (lane == 31) dnR = DT_BIG;
        int v[PPL];
#pragma unroll
        for (int k = 0; k < PPL; k++) {
            const int col = c0 + k;
            const int l = (k == 0) ? dnL : up[k - 1];
            const int r = (k == PPL - 1) ? dnR : up[k + 1];
            int c = min(min(cur[k], r + DT_DG), min(up[k] + DT_HV, l + DT_DG));
            if (col >= w) c = DT_BIG;
            v[k] = c + DT_HV * col;
        }
#pragma unroll
        for (int k = PPL - 2; k >= 0; k--) v[k] = min(v[k], v[k + 1]);
        int incl = v[0];
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const int o = __shfl_down_sync(FULL, incl, dd);
            if (lane + dd < 32) incl = min(incl, o);
        }
        int excl = __shfl_down_sync(FULL, incl, 1);
        if (lane == 31) excl = INT_MAX;
        float *drow = reinterpret_cast<float *>(tmp + (size_t)i * dpitch);
        float outv[PPL];
#pragma unroll
        for (int k = 0; k < PPL; k++) {
            const int col = c0 + k;
            int t = min(v[k], excl) - DT_HV * col;
            if (t >= DT_BIG || col >= w) t = DT_BIG;
            up[k] = t;
            outv[k] = (t >= DT_BIG) ? dist_max : (float)(uint32_t)t * scale;
        }
#pragma unroll
        for (int k = 0; k < PPL; k += 4)
            if (c0 + k < dpitch) *reinterpret_cast<float4 *>(drow + c0 + k) = make_float4(outv[k], outv[k + 1], outv[k + 2], outv[k + 3]);
    }
    cp_async_wait<0>();
}

extern __shared__ uint32_t dt_smem[];

/* one warp per CTA; jobs are ordered by width class so neighbouring CTAs run the same instantiation */
__global__ void __launch_bounds__(32) k_chamfer_dt(const CsJob *__restrict__ jobs, const int32_t *__restrict__ job_ids,
                                                   const uint32_t *__restrict__ bits_arena, float *__restrict__ dist_arena)
{
    const CsJob &jb = jobs[job_ids[blockIdx.x]];
    const uint32_t *planeS = bits_arena + jb.bit_off;
    uint32_t *tmp = reinterpret_cast<uint32_t *>(dist_arena + jb.px_off);
    const int w = jb.roi_w, h = jb.roi_h, bwp = jb.bw + 2, dp = jb.dpitch;
    if (w <= 0 || h <= 0) return;
    if (w <= 32 * 4)
        dt_warp<4>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else if (w <= 32 * 8)
        dt_warp<8>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else if (w <= 32 * 12)
        dt_warp<12>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else if (w <= 32 * 16)
        dt_warp<16>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else if (w <= 32 * 24)
        dt_warp<24>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else if (w <= 32 * 40)
        dt_warp<40>(planeS, bwp, tmp, w, h, dp, dt_smem);
    else
        dt_warp<64>(planeS, bwp, tmp, w, h, dp, dt_smem);
}


/* ------------------------------------------------------------------------------------------
 * Distance transform, cone form (the default).  The two-pass 3x3 chamfer transform computes the exact path metric
 *      D(p) = min over edge pixels q of  a * max(|dx|,|dy|) + (b - a) * min(|dx|,|dy|)           (a = DT_HV < b = DT_DG < 2a),
 * so any evaluation order of that minimum gives the same integers.  Split the sources of p by octant pair:
 *   - q in the closed VERTICAL cone (|dx| <= |dy|) is reached by |dx| diagonal and |dy| - |dx| vertical moves:
 *        S(x,y) = min(edge ? 0 : inf, S(x,y-1) + a, S(x-1,y-1) + b, S(x+1,y-1) + b)      sources above:  top-down sweep
 *        N(x,y) = min(edge ? 0 : inf, N(x,y+1) + a, N(x-1,y+1) + b, N(x+1,y+1) + b)      sources below:  bottom-up sweep
 *        V = min(S, N)
 *     neither recurrence has a dependency inside a row (a row step is a handful of adds and mins per pixel), and the two sweeps are
 *     independent of each other;
 *   - q in the HORIZONTAL cone (|dy| <= |dx|) is reached by |dy| diagonal moves to a pixel p' of p's own row -- for which q lies on the rim of
 *     the vertical cone, so V(p') already holds that cost or less -- followed by horizontal moves:
 *        D(x,y) = min over x' of V(x',y) + a * |x - x'|                                   two 1-D min-plus scans per row
 *     rows are independent of each other: the scans are off the row-to-row dependency chain.
 * Every term is the cost of a real path (>= D) and the best path of either kind is among them (<= D), hence D exactly; values the
 * raster scan saturates at DIST_MAX (an edge-free ROI) come out >= DT_BIG and are written as DIST_MAX.  Columns between roi_w and the
 * padded pitch are treated as non-edge pixels of a wider image: a shortest path between two pixels of the ROI never leaves their
 * bounding box, so they change nothing inside the ROI.
 *
 * k_dt_bi<N>: one CTA of 8 warps per ROI.  Warp 0 sweeps down and warp 1 sweeps up AT THE SAME TIME, each from its end of the ROI.  Until
 * they meet in the middle they park their rows in the distance map itself (S in the top half, N in the bottom half).  Past the middle
 * each hands its rows through a shared-memory ring (named barriers, no polling) to three scan warps, which fetch the other sweep's row
 * from the map, take the minimum, run the two scans and write the final f32 row in place.  The dependency chain is H cheap row steps
 * (the raster scan: 2H steps with a 5-stage warp scan in each).
 * Layout: a lane owns 4 consecutive columns of every 128-column chunk, so a row moves as one coalesced 16-byte access per lane and chunk.
 * ------------------------------------------------------------------------------------------ */
#define DT_NC 3 /* scan warps behind each sweep warp, one ring slot each */

/* named barriers: the documented producer / consumer pairing of bar.arrive with bar.sync.  Ring r (0 down, 1 up), scan warp k:
 * barrier 1 + 6 r + k = "row ready", 4 + 6 r + k = "slot free"; every barrier has at most one arrival outstanding. */
__device__ __forceinline__ void dt_bar_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void dt_bar_arrive(int id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }

/* left / right neighbours of a lane's 4-column group in chunk c: the lane beside it, or the rim lane of the next chunk */
template <int NCH>
__device__ __forceinline__ void dt_rim(const int (&v)[NCH][4], int c, int lane, int &L, int &R)
{
    const unsigned FULL = 0xffffffffu;
    const int sendL = (c > 0 && lane == 31) ? v[c > 0 ? c - 1 : 0][3] : v[c][3];
    const int sendR = (c < NCH - 1 && lane == 0) ? v[c < NCH - 1 ? c + 1 : c][0] : v[c][0];
    L = __shfl_sync(FULL, sendL, (lane + 31) & 31);
    R = __shfl_sync(FULL, sendR, (lane + 1) & 31);
    if (c == 0 && lane == 0) L = DT_BIG;
    if (c == NCH - 1 && lane == 31) R = DT_BIG;
}

/* one sweep warp.  DIR = +1: rows 0 .. h-1, -1: rows h-1 .. 0.  The first n_park rows go to the map, the rest to the ring. */
template <int NCH, int DIR>
__device__ __forceinline__ void dt_sweep(const uint32_t *plane /* bordered strong plane, shared or global */, int bwp, uint32_t *__restrict__ tmp,
                                         int h, int dpitch, int n_park, uint32_t *ring, int bar_base)
{
    const int lane = threadIdx.x & 31;
    const int bw = bwp - 2;
    const int sh = (lane & 7) * 4;
    int v[NCH][4];
#pragma unroll
    for (int c = 0; c < NCH; c++)
#pragma unroll
        for (int j = 0; j < 4; j++) v[c][j] = DT_BIG;
    uint32_t nxt[NCH];
    auto fetch = [&](int y) {
        const uint32_t *rw = plane + (size_t)(y + 1) * bwp + 1;
#pragma unroll
        for (int c = 0; c < NCH; c++) {
            const int wi = 4 * c + (lane >> 3);
            nxt[c] = (wi < bw) ? rw[wi] : 0u; /* bits beyond roi_w are zero (NMS writes none) */
        }
    };
    fetch(DIR > 0 ? 0 : h - 1);
    if (n_park == 0) { /* nothing to park: the other sweep parks everything (h == 1) */
        __threadfence_block();
        __syncthreads();
    }
    for (int step = 0; step < h; step++) {
        const int y = DIR > 0 ? step : h - 1 - step;
        uint32_t nib[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) nib[c] = nxt[c] >> sh;
        if (step + 1 < h) fetch(y + DIR);
        int nv[NCH][4], Lr[NCH], Rr[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) dt_rim<NCH>(v, c, lane, Lr[c], Rr[c]); /* all shuffles of the row in flight together */
#pragma unroll
        for (int c = 0; c < NCH; c++) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int l = (j == 0) ? Lr[c] : v[c][j - 1];
                const int r = (j == 3) ? Rr[c] : v[c][j + 1];
                int u = min(min(min(l, r) + DT_DG, v[c][j] + DT_HV), DT_BIG);
                if ((nib[c] >> j) & 1u) u = 0;
                nv[c][j] = u;
            }
        }
#pragma unroll
        for (int c = 0; c < NCH; c++)
#pragma unroll
            for (int j = 0; j < 4; j++) v[c][j] = nv[c][j];
        if (step < n_park) {
            uint32_t *trow = tmp + (size_t)y * dpitch;
#pragma unroll
            for (int c = 0; c < NCH; c++) {
                const int col0 = c * 128 + lane * 4;
                if (col0 < dpitch) *reinterpret_cast<uint4 *>(trow + col0) = make_uint4(v[c][0], v[c][1], v[c][2], v[c][3]);
            }
            if (step == n_park - 1) { /* both sweeps are at the middle: parked rows become visible to the scan warps */
                __threadfence_block();
                __syncthreads();
            }
        } else {
            const int idx = step - n_park, k = idx % DT_NC;
            if (idx >= DT_NC) dt_bar_sync(bar_base + DT_NC + k); /* slot free? */
            uint32_t *vrow = ring + (size_t)k * dpitch;
#pragma unroll
            for (int c = 0; c < NCH; c++) {
                const int col0 = c * 128 + lane * 4;
                if (col0 < dpitch) *reinterpret_cast<uint4 *>(vrow + col0) = make_uint4(v[c][0], v[c][1], v[c][2], v[c][3]);
            }
            dt_bar_arrive(bar_base + k); /* row ready */
        }
    }
}

/* the two 1-D min-plus scans (slope a) of one row: V = min(ring row (shared), parked row (already in registers)) -> f32 row of the map.
 * A lane owns 4 consecutive columns of each 128-column chunk; the warp scans of all chunks advance together, stage by stage, so their
 * shuffles overlap (a warp issues in order: chunk after chunk would serialise the dependent shuffles) */
template <int NCH>
__device__ __forceinline__ void dt_row_scan(const uint32_t *vrow, const uint4 (&other)[NCH], float *__restrict__ drow, int dpitch, int lane)
{
    const unsigned FULL = 0xffffffffu;
    const float scale = 1.f / 65536.f;
    const float dist_max = (float)(0xffffffffu - (uint32_t)DT_DG) * scale;
    int t[NCH][4], incl[NCH], excl[NCH];
    /* ---- forward: F(x) = min over x' <= x of V(x') + a (x - x') ---- */
#pragma unroll
    for (int c = 0; c < NCH; c++) {
        const int col0 = c * 128 + lane * 4;
        uint4 q = make_uint4(DT_BIG, DT_BIG, DT_BIG, DT_BIG);
        if (col0 < dpitch) q = *reinterpret_cast<const uint4 *>(vrow + col0);
        t[c][0] = min((int)q.x, (int)other[c].x) - DT_HV * col0;
        t[c][1] = min(min((int)q.y, (int)other[c].y) - DT_HV * (col0 + 1), t[c][0]);
        t[c][2] = min(min((int)q.z, (int)other[c].z) - DT_HV * (col0 + 2), t[c][1]);
        t[c][3] = min(min((int)q.w, (int)other[c].w) - DT_HV * (col0 + 3), t[c][2]);
        incl[c] = t[c][3];
    }
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
        int o[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) o[c] = __shfl_up_sync(FULL, incl[c], dd);
        if (lane >= dd) {
#pragma unroll
            for (int c = 0; c < NCH; c++) incl[c] = min(incl[c], o[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < NCH; c++) excl[c] = __shfl_up_sync(FULL, incl[c], 1);
    {
        int tot[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) tot[c] = __shfl_sync(FULL, incl[c], 31);
        int carry = INT_MAX;
#pragma unroll
        for (int c = 0; c < NCH; c++) {
            if (lane == 0) excl[c] = INT_MAX;
            excl[c] = min(excl[c], carry);
            carry = min(carry, tot[c]);
        }
    }
    /* forward result, already shifted for the backward scan: F + a col = min(t, excl) + 2 a col; then the in-lane suffix minima */
#pragma unroll
    for (int c = 0; c < NCH; c++) {
        const int col0 = c * 128 + lane * 4;
        t[c][3] = min(t[c][3], excl[c]) + 2 * DT_HV * (col0 + 3);
        t[c][2] = min(min(t[c][2], excl[c]) + 2 * DT_HV * (col0 + 2), t[c][3]);
        t[c][1] = min(min(t[c][1], excl[c]) + 2 * DT_HV * (col0 + 1), t[c][2]);
        t[c][0] = min(min(t[c][0], excl[c]) + 2 * DT_HV * col0, t[c][1]);
        incl[c] = t[c][0];
    }
    /* ---- backward: D(x) = min over x' >= x of F(x') + a (x' - x) ---- */
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
        int o[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) o[c] = __shfl_down_sync(FULL, incl[c], dd);
        if (lane + dd < 32) {
#pragma unroll
            for (int c = 0; c < NCH; c++) incl[c] = min(incl[c], o[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < NCH; c++) excl[c] = __shfl_down_sync(FULL, incl[c], 1);
    {
        int tot[NCH];
#pragma unroll
        for (int c = 0; c < NCH; c++) tot[c] = __shfl_sync(FULL, incl[c], 0);
        int carry = INT_MAX;
#pragma unroll
        for (int c = NCH - 1; c >= 0; c--) {
            if (lane == 31) excl[c] = INT_MAX;
            excl[c] = min(excl[c], carry);
            carry = min(carry, tot[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < NCH; c++) {
        const int col0 = c * 128 + lane * 4;
        float o4[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int r = min(t[c][k], excl[c]) - DT_HV * (col0 + k);
            o4[k] = (r >= DT_BIG) ? dist_max : (float)(uint32_t)r * scale;
        }
        if (col0 < dpitch) *reinterpret_cast<float4 *>(drow + col0) = make_float4(o4[0], o4[1], o4[2], o4[3]);
    }
}

/* rows wider than 640 px: V = min(ring row, parked row) written back into the ring row, same scans, the forward result parked there too */
__device__ __noinline__ void dt_row_scan_wide(uint32_t *vrow, const uint32_t *__restrict__ orow, float *__restrict__ drow, int dpitch, int lane, int nch)
{
    const unsigned FULL = 0xffffffffu;
    const float scale = 1.f / 65536.f;
    const float dist_max = (float)(0xffffffffu - (uint32_t)DT_DG) * scale;
    int carry = INT_MAX;
    for (int c = 0; c < nch; c++) {
        const int col0 = c * 128 + lane * 4;
        uint4 q = make_uint4(DT_BIG, DT_BIG, DT_BIG, DT_BIG), o = q;
        if (col0 < dpitch) {
            q = *reinterpret_cast<const uint4 *>(vrow + col0);
            o = *reinterpret_cast<const uint4 *>(orow + col0);
        }
        int t[4] = {min((int)q.x, (int)o.x), min((int)q.y, (int)o.y), min((int)q.z, (int)o.z), min((int)q.w, (int)o.w)};
#pragma unroll
        for (int k = 0; k < 4; k++) t[k] -= DT_HV * (col0 + k);
        t[1] = min(t[1], t[0]);
        t[2] = min(t[2], t[1]);
        t[3] = min(t[3], t[2]);
        int incl = t[3];
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const int oo = __shfl_up_sync(FULL, incl, dd);
            if (lane >= dd) incl = min(incl, oo);
        }
        int excl = __shfl_up_sync(FULL, incl, 1);
        if (lane == 0) excl = INT_MAX;
        excl = min(excl, carry);
        carry = min(carry, __shfl_sync(FULL, incl, 31));
        if (col0 < dpitch)
            *reinterpret_cast<uint4 *>(vrow + col0) =
                make_uint4(min(t[0], excl) + 2 * DT_HV * col0, min(t[1], excl) + 2 * DT_HV * (col0 + 1), min(t[2], excl) + 2 * DT_HV * (col0 + 2),
                           min(t[3], excl) + 2 * DT_HV * (col0 + 3));
    }
    __syncwarp();
    carry = INT_MAX;
    for (int c = nch - 1; c >= 0; c--) {
        const int col0 = c * 128 + lane * 4;
        uint4 q = make_uint4(INT_MAX, INT_MAX, INT_MAX, INT_MAX);
        if (col0 < dpitch) q = *reinterpret_cast<const uint4 *>(vrow + col0);
        int t[4] = {(int)q.x, (int)q.y, (int)q.z, (int)q.w};
        t[2] = min(t[2], t[3]);
        t[1] = min(t[1], t[2]);
        t[0] = min(t[0], t[1]);
        int incl = t[0];
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) {
            const int oo = __shfl_down_sync(FULL, incl, dd);
            if (lane + dd < 32) incl = min(incl, oo);
        }
        int excl = __shfl_down_sync(FULL, incl, 1);
        if (lane == 31) excl = INT_MAX;
        excl = min(excl, carry);
        carry = min(carry, __shfl_sync(FULL, incl, 0));
        float o4[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int r = min(t[k], excl) - DT_HV * (col0 + k);
            o4[k] = (r >= DT_BIG) ? dist_max : (float)(uint32_t)r * scale;
        }
        if (col0 < dpitch) *reinterpret_cast<float4 *>(drow + col0) = make_float4(o4[0], o4[1], o4[2], o4[3]);
    }
}

/* scan warp k of ring r: rows first, first + stride, ... (n of them), row i of the list is ring slot k once "row ready" fires */
template <int NCH>
__device__ __forceinline__ void dt_scan_rows(uint32_t *__restrict__ tmp, int dpitch, int w, uint32_t *ring, int bar_base, int k, int first, int stride,
                                             int n_rows)
{
    const int lane = threadIdx.x & 31;
    uint32_t *vrow = ring + (size_t)k * dpitch;
    for (int i = 0; i < n_rows; i++) {
        const int y = first + i * stride;
        uint32_t *orow = tmp + (size_t)y * dpitch; /* the other sweep's row, parked before the middle barrier */
        if (NCH <= 5) {
            uint4 other[NCH <= 5 ? NCH : 1];
#pragma unroll
            for (int c = 0; c < (NCH <= 5 ? NCH : 1); c++) {
                const int col0 = c * 128 + lane * 4;
                other[c] = make_uint4(DT_BIG, DT_BIG, DT_BIG, DT_BIG);
                if (col0 < dpitch) other[c] = *reinterpret_cast<const uint4 *>(orow + col0); /* in flight while waiting for the ring */
            }
            dt_bar_sync(bar_base + k);
            dt_row_scan<(NCH <= 5 ? NCH : 1)>(vrow, other, reinterpret_cast<float *>(orow), dpitch, lane);
        } else {
            dt_bar_sync(bar_base + k);
            dt_row_scan_wide(vrow, orow, reinterpret_cast<float *>(orow), dpitch, lane, (w + 127) >> 7);
        }
        if (i + 1 < n_rows) dt_bar_arrive(bar_base + DT_NC + k); /* slot free (the sweep waits for it before the row after next) */
    }
}

template <int NCH>
__global__ void __launch_bounds__(32 * (2 + 2 * DT_NC), (NCH <= 3 ? 3 : (NCH <= 5 ? 2 : 1)))
    k_dt_bi(const CsJob *__restrict__ jobs, const int32_t *__restrict__ job_ids, const uint32_t *__restrict__ bits_arena,
            float *__restrict__ dist_arena, int plane_smem_words, int ring_pitch)
{
    const CsJob &jb = jobs[job_ids[blockIdx.x]];
    const uint32_t *planeS = bits_arena + jb.bit_off;
    uint32_t *tmp = reinterpret_cast<uint32_t *>(dist_arena + jb.px_off);
    const int w = jb.roi_w, h = jb.roi_h, bwp = jb.bw + 2, dp = jb.dpitch;
    if (w <= 0 || h <= 0) return;
    uint32_t *ringD = dt_smem, *ringU = dt_smem + (size_t)DT_NC * ring_pitch;
    uint32_t *plane_s = dt_smem + (size_t)2 * DT_NC * ring_pitch;
    /* the whole strong plane (1 bit per pixel) comes in with one burst of asynchronous copies; the sweeps then never wait on memory */
    const int n_words = (h + 2) * bwp;
    if (n_words <= plane_smem_words) {
        for (int q = threadIdx.x; q < n_words; q += blockDim.x) {
            const unsigned sa = (unsigned)__cvta_generic_to_shared(plane_s + q);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(sa), "l"(planeS + q));
        }
        cp_async_commit();
        cp_async_wait<0>();
        planeS = plane_s;
    }
    __syncthreads();
    const int mid = h >> 1; /* the down sweep parks rows [0, mid), the up sweep rows [mid, h) */
    const int wid = threadIdx.x >> 5;
    if (wid == 0)
        dt_sweep<NCH, 1>(planeS, bwp, tmp, h, dp, mid, ringD, 1);
    else if (wid == 1)
        dt_sweep<NCH, -1>(planeS, bwp, tmp, h, dp, h - mid, ringU, 1 + 2 * DT_NC);
    else {
        __syncthreads(); /* the middle barrier of the sweeps */
        const int r = (wid - 2) / DT_NC, k = (wid - 2) % DT_NC;
        if (r == 0) { /* rows mid .. h-1 from the down sweep; the parked row holds N */
            const int n = h - mid;
            dt_scan_rows<NCH>(tmp, dp, w, ringD, 1, k, mid + k, DT_NC, (n - k + DT_NC - 1) / DT_NC);
        } else { /* rows mid-1 .. 0 from the up sweep; the parked row holds S */
            const int n = mid;
            dt_scan_rows<NCH>(tmp, dp, w, ringU, 1 + 2 * DT_NC, k, mid - 1 - k, -DT_NC, (n - k + DT_NC - 1) / DT_NC);
        }
    }
}

/* ------------------------------------------------------------------------------------------ launchers */
/* ROI width classes of the distance transform: 1..5, 8 or 16 chunks of 128 columns (one kernel instantiation and one launch per class) */
const int cs_dt_class_width[CS_DT_CLASSES] = {128, 256, 384, 512, 640, 1024, 2048};

int cs_dt_class_of(int roi_w)
{
    for (int c = 0; c < CS_DT_CLASSES; c++)
        if (roi_w <= cs_dt_class_width[c]) return c;
    return -1;
}

void cs_launch_gray(const uint8_t *d_img, uint8_t *d_gray, int n_frames, int w, int h, int stride, int channels, cudaStream_t st,
                    int64_t *launches)
{
    const int64_t total = (int64_t)n_frames * w * h;
    int64_t done = 0;
    if (channels == 3 && stride == 3 * w && (((uintptr_t)d_img) & 15) == 0 && (((uintptr_t)d_gray) & 15) == 0) {
        const int64_t groups = total / 16;
        if (groups > 0) {
            const int blocks = (int)((groups + 255) / 256 < CS_SM_COUNT * 16 ? (groups + 255) / 256 : CS_SM_COUNT * 16);
            CS_APPLY_CARVEOUT(k_bgr2gray_flat);
            k_bgr2gray_flat<<<blocks, 256, 0, st>>>((const uint4 *)d_img, (uint4 *)d_gray, groups);
            (*launches)++;
        }
        done = groups * 16;
    }
    if (done < total) {
        const int64_t rest = total - done;
        const int blocks = (int)((rest + 255) / 256 < CS_SM_COUNT * 16 ? (rest + 255) / 256 : CS_SM_COUNT * 16);
        k_bgr2gray_generic<<<blocks, 256, 0, st>>>(d_img, d_gray, n_frames, w, h, stride, channels, done);
        (*launches)++;
    }
}

void cs_launch_canny(const uint8_t *d_base, int, int, const CsJob *d_jobs, int n_jobs, const int32_t *d_tile_job, int n_tiles, uint32_t *d_bits,
                     size_t bits_bytes, int low, int high, cudaStream_t st, int64_t *launches)
{
    if (n_jobs <= 0) return;
    cudaMemsetAsync(d_bits, 0, bits_bytes, st); /* zero borders (and stale bits) of every plane */
    if (n_tiles > 0) {
        CS_APPLY_CARVEOUT(k_canny_nms);
        k_canny_nms<<<n_tiles, dim3(32, 8), 0, st>>>(d_base, d_jobs, d_tile_job, d_bits, low, high);
        (*launches)++;
    }
}

void cs_launch_hyst(const CsJob *d_jobs, int n_jobs, uint32_t *d_bits, int max_plane_words, cudaStream_t st, int64_t *launches)
{
    if (n_jobs <= 0) return;
    int smem_words = 2 * max_plane_words;
    const int cap_words = (200 * 1024) / 4;
    if (smem_words > cap_words) smem_words = cap_words;
    const int bytes = smem_words * 4;
    CS_ONCE_PER_DEVICE(cs_allow_max_dynamic_smem(k_canny_hyst));
    CS_APPLY_CARVEOUT(k_canny_hyst);
    k_canny_hyst<<<n_jobs, HY_THREADS, bytes, st>>>(d_jobs, d_bits, smem_words);
    (*launches)++;
}

/* d_ids: job ids grouped by width class, tallest ROI first inside a class; class_off[c] .. class_off[c + 1] is the slice of class c;
 * class_plane_words[c]: words of the largest bordered bit plane of the class.
 * flags: bit 0 = the two-pass raster-scan kernel (A/B switch) instead of the cone form (k_dt_bi); bit 1 = cone form reading the edge bits
 * from global memory (the path of ROIs whose bit plane exceeds 96 KB, forced for the tests) */
template <int NCH>
static void dt_launch_class(const CsJob *d_jobs, const int32_t *d_ids, int count, int width, int plane_words, const uint32_t *d_bits, float *d_dist,
                            cudaStream_t st, int64_t *launches)
{
    int pw = plane_words;
    if (pw > (96 * 1024) / 4 || pw < 0) pw = 0; /* huge ROIs (or the debug switch): the sweeps read the bits from global memory */
    const int bytes = (2 * DT_NC * width + pw) * 4;
    CS_ONCE_PER_DEVICE(cs_allow_max_dynamic_smem(k_dt_bi<NCH>));
    CS_APPLY_CARVEOUT(k_dt_bi<NCH>);
    k_dt_bi<NCH><<<count, 32 * (2 + 2 * DT_NC), bytes, st>>>(d_jobs, d_ids, d_bits, d_dist, pw, width);
    (*launches)++;
}

void cs_launch_dt(const CsJob *d_jobs, const int32_t *d_ids, int n_jobs, int max_dpitch, const int *class_off, const int *class_plane_words,
                  const uint32_t *d_bits, float *d_dist, int raster_or_flags, cudaStream_t st, cudaStream_t st_side, cudaEvent_t ev_fork,
                  cudaEvent_t ev_join, int64_t *launches)
{
    if (n_jobs <= 0) return;
    if (raster_or_flags & 1) {
        const int bytes = DT_PF * max_dpitch * 4;
        CS_ONCE_PER_DEVICE(cs_allow_max_dynamic_smem(k_chamfer_dt));
        CS_APPLY_CARVEOUT(k_chamfer_dt);
        k_chamfer_dt<<<n_jobs, 32, bytes, st>>>(d_jobs, d_ids, d_bits, d_dist);
        (*launches)++;
        return;
    }
    /* the width classes are independent: the class with most work stays on `st`, the others run beside it on `st_side` */
    int main_cls = -1, n_cls = 0;
    int64_t best = -1;
    for (int c = 0; c < CS_DT_CLASSES; c++) {
        const int64_t work = (int64_t)(class_off[c + 1] - class_off[c]) * cs_dt_class_width[c];
        if (work > 0) n_cls++;
        if (work > best) {
            best = work;
            main_cls = c;
        }
    }
    const bool side = st_side != nullptr && n_cls > 1;
    if (side) {
        cudaEventRecord(ev_fork, st);
        cudaStreamWaitEvent(st_side, ev_fork, 0);
    }
    for (int c = CS_DT_CLASSES - 1; c >= 0; c--) {
        const int count = class_off[c + 1] - class_off[c];
        if (count <= 0) continue;
        const int32_t *ids = d_ids + class_off[c];
        const int width = cs_dt_class_width[c], pw = (raster_or_flags & 2) ? -1 : class_plane_words[c];
        cudaStream_t s = (side && c != main_cls) ? st_side : st;
        switch (c) {
        case 0: dt_launch_class<1>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        case 1: dt_launch_class<2>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        case 2: dt_launch_class<3>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        case 3: dt_launch_class<4>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        case 4: dt_launch_class<5>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        case 5: dt_launch_class<8>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        default: dt_launch_class<16>(d_jobs, ids, count, width, pw, d_bits, d_dist, s, launches); break;
        }
    }
    if (side) {
        cudaEventRecord(ev_join, st_side);
        cudaStreamWaitEvent(st, ev_join, 0);
    }
}
