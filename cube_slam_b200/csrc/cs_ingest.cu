/*
 * cs_ingest.cu -- frames that are already in GPU memory: the descriptor check, the layout kernel k_ingest_frames, and the entry points that
 * take a cs_device_frames (include/cube_slam_b200.h): the batch uploads, line detection, and the line descriptor's two calls.
 *
 * Every consumer of a batch's frames (k_bgr2gray_flat, k_lsd_front, k_ed_front) reads packed rows, BGR or gray, pitch width * channels.
 * A device view of any strides is brought into that layout once, on the context stream, so that everything downstream runs exactly the code
 * the host path runs.  The copy is HBM-bound: its algorithmic bytes are the view's bytes read plus the packed bytes written.
 */
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>

#include "cs_internal.h"

/* the context's two events that order a device-frame copy between the producer's stream and the context stream (cs_context.cu) */
void cs_ctx_ingest_events(cs_ctx *c, cudaEvent_t *in, cudaEvent_t *out);

#define ING_THREADS 256

/* the view as the kernel walks it: output byte k of a pixel reads the pixel's byte at ch_off[k] (BGR order: k * stride_channel; RGB: the
 * same bytes in reverse, a byte permutation and nothing else) */
struct CsIngest {
    int64_t total;        /* output bytes: n_frames * height * width * C */
    int64_t frame_bytes;  /* height * width * C */
    int32_t row_bytes;    /* width * C */
    int32_t width, height;
    int64_t stride_frame, stride_row, stride_col;
    int64_t ch_off0, ch_off1, ch_off2;
};

/* One thread per 16-byte chunk of the packed output: the chunk's first byte is located once (two divisions), then the source address walks
 * the view byte by byte with carries, and the 16 bytes leave as one 16-byte store (the buffer is cudaMalloc'ed, so chunks are aligned; the
 * last chunk of a batch may be partial and is stored byte by byte).  Lane i's chunk follows lane i - 1's, so a warp's loads of one
 * unrolled step cover one contiguous span of each source plane: the interleaved bytes of a row (NHWC, BGRA) or, for a planar view, a
 * contiguous span of each of the three planes, which the chunk interleaves in registers.  L1 merges the byte loads of a span. */
template <int C>
__global__ void k_ingest_frames(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, CsIngest g)
{
    const int64_t n_chunks = (g.total + 15) >> 4;
    for (int64_t chunk = (int64_t)blockIdx.x * ING_THREADS + threadIdx.x; chunk < n_chunks; chunk += (int64_t)gridDim.x * ING_THREADS) {
        const int64_t o0 = chunk << 4;
        const int64_t f = o0 / g.frame_bytes;
        const int64_t r = o0 - f * g.frame_bytes;
        int y = (int)(r / g.row_bytes);
        const int xk = (int)(r - (int64_t)y * g.row_bytes);
        int x = xk / C, k = xk - x * C;
        const uint8_t *pix = src + f * g.stride_frame + (int64_t)y * g.stride_row + (int64_t)x * g.stride_col;
        const int n = g.total - o0 < 16 ? (int)(g.total - o0) : 16;
        uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (i < n) {
                const int64_t off = C == 1 ? 0 : (k == 0 ? g.ch_off0 : (k == 1 ? g.ch_off1 : g.ch_off2));
                w[i >> 2] |= (uint32_t)__ldg(pix + off) << (8 * (i & 3));
                if (++k == C) { /* next pixel; past the row's end the next row, past the frame's end the next frame */
                    k = 0;
                    pix += g.stride_col;
                    if (++x == g.width) {
                        x = 0;
                        pix += g.stride_row - (int64_t)g.width * g.stride_col;
                        if (++y == g.height) {
                            y = 0;
                            pix += g.stride_frame - (int64_t)g.height * g.stride_row;
                        }
                    }
                }
            }
        }
        if (n == 16) {
            uint4 v;
            v.x = w[0];
            v.y = w[1];
            v.z = w[2];
            v.w = w[3];
            *reinterpret_cast<uint4 *>(dst + o0) = v;
        } else {
#pragma unroll
            for (int i = 0; i < 16; i++) /* unrolled: w stays in registers */
                if (i < n) dst[o0 + i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
        }
    }
}

/* Packed rows of the view into dst (n_frames * height * width * channels bytes) on `st`.  A view that already is packed BGR or gray with no
 * gaps is one device-to-device copy; any other goes through k_ingest_frames.  Returns the CUDA error of the enqueue; *launched tells which. */
cudaError_t cs_launch_ingest(const cs_device_frames *fr, uint8_t *dst, cudaStream_t st, bool *launched)
{
    const int C = fr->channels;
    const int64_t W = fr->width, H = fr->height, N = fr->n_frames;
    const int64_t total = N * H * W * C;
    /* a dimension of extent 1 has no stride that matters */
    const bool packed = (C == 1 || (fr->stride_channel == 1 && fr->channel_order == CS_ORDER_BGR)) && (W == 1 || fr->stride_col == C) &&
                        (H == 1 || fr->stride_row == W * C) && (N == 1 || fr->stride_frame == H * W * C);
    *launched = !packed;
    if (packed) return cudaMemcpyAsync(dst, fr->data, (size_t)total, cudaMemcpyDeviceToDevice, st);
    CsIngest g;
    g.total = total;
    g.frame_bytes = H * W * C;
    g.row_bytes = (int32_t)(W * C);
    g.width = (int32_t)W;
    g.height = (int32_t)H;
    g.stride_frame = fr->stride_frame;
    g.stride_row = fr->stride_row;
    g.stride_col = fr->stride_col;
    const bool rgb = C == 3 && fr->channel_order == CS_ORDER_RGB;
    g.ch_off0 = rgb ? 2 * fr->stride_channel : 0;
    g.ch_off1 = C == 3 ? fr->stride_channel : 0;
    g.ch_off2 = rgb ? 0 : 2 * fr->stride_channel;
    const int64_t n_chunks = (total + 15) / 16;
    const int64_t blocks = (n_chunks + ING_THREADS - 1) / ING_THREADS;
    const unsigned grid = (unsigned)(blocks < 16 * CS_SM_COUNT ? blocks : 16 * CS_SM_COUNT); /* grid-stride beyond 16 CTAs per SM */
    if (C == 1)
        k_ingest_frames<1><<<grid, ING_THREADS, 0, st>>>(fr->data, dst, g);
    else
        k_ingest_frames<3><<<grid, ING_THREADS, 0, st>>>(fr->data, dst, g);
    return cudaGetLastError();
}

namespace {

/* cuMemGetAddressRange through the runtime's driver entry point, as cs_tma.cuh reaches the driver: no link-time dependency on libcuda */
typedef CUresult (*AddressRangeFn)(CUdeviceptr *, size_t *, CUdeviceptr);
AddressRangeFn address_range_fn()
{
    static AddressRangeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (AddressRangeFn)p;
        cudaGetLastError();
    }
    return fn;
}

/* the descriptor check, host-only: nothing is read from the view and nothing is enqueued */
int check_frames(int device, const cs_device_frames *fr, char *msg, size_t cap)
{
    msg[0] = 0;
    if (!fr || !fr->data) return snprintf(msg, cap, "null frame descriptor or data pointer"), CS_ERR_INVALID_ARG;
    if (fr->n_frames <= 0 || fr->height <= 0 || fr->width <= 0)
        return snprintf(msg, cap, "empty frames (%d x %d x %d)", fr->n_frames, fr->height, fr->width), CS_ERR_INVALID_ARG;
    if (fr->channels != 1 && fr->channels != 3) return snprintf(msg, cap, "channels must be 1 or 3 (got %d)", fr->channels), CS_ERR_INVALID_ARG;
    if (fr->channels == 3 && fr->channel_order != CS_ORDER_BGR && fr->channel_order != CS_ORDER_RGB)
        return snprintf(msg, cap, "unknown channel order %d (CS_ORDER_BGR 0 or CS_ORDER_RGB 1)", fr->channel_order), CS_ERR_INVALID_ARG;
    if (fr->stride_frame < 0 || fr->stride_row < 0 || fr->stride_col < 0 || fr->stride_channel < 0)
        return snprintf(msg, cap, "negative stride"), CS_ERR_INVALID_ARG;
    if ((int64_t)fr->width * fr->channels > 0x7fffffff)
        return snprintf(msg, cap, "a row of %d x %d bytes is too long", fr->width, fr->channels), CS_ERR_INVALID_ARG;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, fr->data) != cudaSuccess) {
        cudaGetLastError();
        return snprintf(msg, cap, "cudaPointerGetAttributes failed on the frame pointer"), CS_ERR_INVALID_ARG;
    }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged)
        return snprintf(msg, cap, "the frame pointer is not device or managed memory"), CS_ERR_INVALID_ARG;
    if (at.device != device) return snprintf(msg, cap, "the frames are on device %d, the context on device %d", at.device, device), CS_ERR_INVALID_ARG;
    /* the last byte the view touches, in 128-bit arithmetic (extents below 2^31, strides below 2^63) */
    const __int128 last = (__int128)(fr->n_frames - 1) * fr->stride_frame + (__int128)(fr->height - 1) * fr->stride_row +
                          (__int128)(fr->width - 1) * fr->stride_col + (fr->channels == 3 ? (__int128)2 * fr->stride_channel : 0);
    AddressRangeFn range = address_range_fn();
    if (!range) return snprintf(msg, cap, "cuMemGetAddressRange is not available from the driver"), CS_ERR_CUDA;
    CUdeviceptr base = 0;
    size_t size = 0;
    if (range(&base, &size, (CUdeviceptr)(uintptr_t)fr->data) != CUDA_SUCCESS)
        return snprintf(msg, cap, "cuMemGetAddressRange failed on the frame pointer"), CS_ERR_INVALID_ARG;
    const __int128 room = (__int128)base + (__int128)size - (__int128)(uintptr_t)fr->data; /* bytes from data to the allocation's end */
    if (last >= room)
        return snprintf(msg, cap, "the view reaches byte %lld past its data pointer, the allocation ends %lld bytes after it", (long long)last,
                        (long long)room),
               CS_ERR_INVALID_ARG;
    return CS_OK;
}

int check_on_ctx(cs_ctx *c, const cs_device_frames *fr)
{
    char msg[256];
    const int rc = check_frames(cs_ctx_device(c), fr, msg, sizeof msg);
    return rc ? cs_ctx_fail(c, rc, "%s", msg) : CS_OK;
}

/* the view, packed, into dst on the context stream, ordered after the producer's work so far; the producer's later work is ordered after it */
int ingest(cs_ctx *c, const cs_device_frames *fr, uint8_t *dst)
{
    cudaStream_t st = cs_ctx_stream(c), producer = (cudaStream_t)fr->stream;
    cudaEvent_t ev_in, ev_out;
    cs_ctx_ingest_events(c, &ev_in, &ev_out);
    cudaError_t e;
    if ((e = cudaEventRecord(ev_in, producer)) != cudaSuccess || (e = cudaStreamWaitEvent(st, ev_in, 0)) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "ordering the frame copy after the producer stream: %s", cudaGetErrorString(e));
    bool launched = false;
    if ((e = cs_launch_ingest(fr, dst, st, &launched)) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "frame copy: %s", cudaGetErrorString(e));
    if ((e = cudaEventRecord(ev_out, st)) != cudaSuccess || (e = cudaStreamWaitEvent(producer, ev_out, 0)) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "ordering the producer stream after the frame copy: %s", cudaGetErrorString(e));
    return CS_OK;
}

int upload_device(cs_ctx *c, const cs_device_frames *fr, const double *T_wc, const double *boxes, const int32_t *box_offsets, const double *lines,
                  const int32_t *line_offsets, const cs_cuboid_params *params, const cs_line_params *online)
{
    int rc;
    if ((rc = check_on_ctx(c, fr))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    uint8_t *d_img = nullptr;
    /* the tables go first: their host-to-device copies must not queue behind the producer's work */
    if ((rc = cs_ctx_store_device_batch(c, fr->n_frames, fr->width, fr->height, fr->channels, T_wc, boxes, box_offsets, lines, line_offsets, params,
                                        online, &d_img)))
        return rc;
    if ((rc = ingest(c, fr, d_img))) return rc;
    cs_ctx_mark_prepared(c);
    return CS_OK;
}

}  // namespace

extern "C" {

int cs_check_device_frames(int device, const cs_device_frames *frames)
{
    char msg[256];
    const int rc = check_frames(device, frames, msg, sizeof msg);
    cs_set_frames_error(rc ? msg : "");
    return rc;
}

int cs_batch_upload_device(cs_ctx *c, const cs_device_frames *frames, const double *T_wc, const double *boxes, const int32_t *box_offsets,
                           const double *lines, const int32_t *line_offsets, const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    return upload_device(c, frames, T_wc, boxes, box_offsets, lines, line_offsets, params, nullptr);
}

int cs_batch_upload_online_device(cs_ctx *c, const cs_device_frames *frames, const double *T_wc, const double *boxes, const int32_t *box_offsets,
                                  const cs_line_params *line_params, const cs_cuboid_params *params)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!line_params) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null line params");
    return upload_device(c, frames, T_wc, boxes, box_offsets, nullptr, nullptr, params, line_params);
}

int cs_detect_lines_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_line_params *params, float *lines_xyxy,
                                 int32_t max_lines_per_frame, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!params || !lines_xyxy || !n_lines || max_lines_per_frame <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (params->numoctaves < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1"); /* as cs_detect_lines_batch */
    int rc;
    if ((rc = check_on_ctx(c, frames))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const int F = frames->n_frames, W = frames->width, H = frames->height, ch = frames->channels;
    const size_t bytes = (size_t)F * H * W * ch;
    /* the detector's own buffer: a batch uploaded to the context keeps its frames */
    uint8_t *buf = params->use_LSD ? cs_lsd_frame_buffer(c, bytes) : cs_edl_frame_buffer(c, bytes);
    if (!buf) return CS_ERR_CUDA; /* the allocation's failure is already the context's message */
    if ((rc = ingest(c, frames, buf))) return rc;
    return cs_detect_lines_run(c, buf, true, F, W, H, W * ch, ch, params, lines_xyxy, max_lines_per_frame, n_lines);
}

/* cs_detect_descrip_lines_batch on device frames: the detector runs on its own buffer, then the host form's body (cs_lbd.cu) */
int cs_detect_descrip_lines_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_line_params *params, cs_keyline *keylines,
                                         uint8_t *desc32, int32_t max_lines_per_frame, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!params || !keylines || !desc32 || !n_lines || max_lines_per_frame <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (params->numoctaves < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1"); /* as cs_detect_descrip_lines_batch */
    int rc;
    if ((rc = check_on_ctx(c, frames))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const int F = frames->n_frames, W = frames->width, H = frames->height, ch = frames->channels, cap = max_lines_per_frame;
    const size_t bytes = (size_t)F * H * W * ch;
    uint8_t *buf = params->use_LSD ? cs_lsd_frame_buffer(c, bytes) : cs_edl_frame_buffer(c, bytes);
    if (!buf) return CS_ERR_CUDA;
    if ((rc = ingest(c, frames, buf))) return rc;
    CsDetectedLines d;
    if (params->use_LSD) {
        if ((rc = cs_lsd_run_sync(c, buf, true, F, W, H, W * ch, ch, params->line_length_thres, cap, &d.lines, &d.counts, &d.lsd_frames))) return rc;
    } else if ((rc = cs_edl_run_keylines(c, buf, true, F, W, H, W * ch, ch, params->line_length_thres, cap, &d.lines, &d.counts, &d.extra, &d.dx, &d.dy)))
        return rc;
    return cs_lbd_describe_detected(c, d, params->use_LSD != 0, F, W, H, W * ch, ch, keylines, desc32, cap, n_lines);
}

/* cs_lbd_compute_batch on device frames: the frames go to the EDLines buffer, whose front end makes the descriptor's Sobel maps */
int cs_lbd_compute_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_keyline *keylines, const int32_t *keyline_offsets, uint8_t *desc32,
                                float *desc72)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc, n = 0;
    if ((rc = check_on_ctx(c, frames))) return rc;
    if ((rc = cs_lbd_check_given(c, frames->n_frames, keylines, keyline_offsets, desc32, &n)) || n == 0) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const int F = frames->n_frames, W = frames->width, H = frames->height, ch = frames->channels;
    uint8_t *buf = cs_edl_frame_buffer(c, (size_t)F * H * W * ch);
    if (!buf) return CS_ERR_CUDA;
    if ((rc = ingest(c, frames, buf))) return rc;
    return cs_lbd_compute_run(c, buf, true, F, W, H, W * ch, ch, keylines, keyline_offsets, desc32, desc72);
}

/* the octave calls on device frames: the frames go to the EDLines buffer (the LSD buffer takes the gray pyramid), then the host forms' body */
static int octaves_device(cs_ctx *c, const cs_device_frames *frames, const cs_line_params *params, bool describe, cs_keyline_octave *keylines,
                          uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc;
    if ((rc = check_on_ctx(c, frames))) return rc;
    if ((rc = cs_lsd_octaves_check(c, frames->width, frames->height, params, keylines, desc32, describe, max_lines_per_octave, n_lines))) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const int F = frames->n_frames, W = frames->width, H = frames->height, ch = frames->channels;
    uint8_t *buf = cs_edl_frame_buffer(c, (size_t)F * H * W * ch);
    if (!buf) return CS_ERR_CUDA;
    if ((rc = ingest(c, frames, buf))) return rc;
    return cs_lsd_octaves_run(c, buf, F, W, H, W * ch, ch, params, describe, keylines, desc32, max_lines_per_octave, n_lines);
}

int cs_detect_raw_lines_octaves_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_line_params *params, cs_keyline_octave *keylines,
                                             int32_t max_lines_per_octave, int32_t *n_lines)
{
    return octaves_device(c, frames, params, false, keylines, nullptr, max_lines_per_octave, n_lines);
}

int cs_detect_descrip_lines_octaves_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_line_params *params, cs_keyline_octave *keylines,
                                                 uint8_t *desc32, int32_t max_lines_per_octave, int32_t *n_lines)
{
    return octaves_device(c, frames, params, true, keylines, desc32, max_lines_per_octave, n_lines);
}

/* cs_lbd_compute_octaves_batch on device frames: the frames go to the EDLines buffer, then the host form's body (cs_lbd_octaves.cu) */
int cs_lbd_compute_octaves_batch_device(cs_ctx *c, const cs_device_frames *frames, const cs_keyline_octave *keylines, const int32_t *keyline_offsets,
                                        uint8_t *desc32, float *desc72)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc, n = 0;
    if ((rc = check_on_ctx(c, frames))) return rc;
    if ((rc = cs_lbd_octaves_check_given(c, frames->n_frames, frames->width, frames->height, keylines, keyline_offsets, desc32, &n)) || n == 0) return rc;
    cudaSetDevice(cs_ctx_device(c));
    const int F = frames->n_frames, W = frames->width, H = frames->height, ch = frames->channels;
    uint8_t *buf = cs_edl_frame_buffer(c, (size_t)F * H * W * ch);
    if (!buf) return CS_ERR_CUDA;
    if ((rc = ingest(c, frames, buf))) return rc;
    return cs_lbd_compute_octaves_run(c, buf, F, W, H, W * ch, ch, keylines, keyline_offsets, desc32, desc72);
}

} /* extern "C" */
