/* tests/host_core/lsd_octaves_standin.cpp -- a host stand-in for the part of libcubeslam_b200.so that shim/lsd_detector_b200.cpp calls:
 * cs_create, cs_destroy, cs_last_error, cs_default_line_params and cs_detect_raw_lines_octaves_batch.  The octave call answers from the CPU
 * oracle -- the gray frame (orc_bgr2gray), pyrDown per octave (lbd_oct_pyrdown), the LSD oracle's raw segments of each octave
 * (lsd_orc_detect) and the KeyLine fill (lbd_oct_keylines) -- with the C ABI's checks, slots and error statuses, so that the shim's host side
 * (grouping, packing, the mask rule, append semantics, messages, exceptions, the capacity retry) runs without a GPU
 * (tests/test_lsd_detector_shim_host.py).  It can also answer CS_ERR_CAPACITY on demand.  Test infrastructure, never shipped. */
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/cube_slam_b200.h"

extern "C" void orc_bgr2gray(const uint8_t *bgr, int w, int h, int stride, uint8_t *gray, int gstride, int fixed15);
extern "C" int lbd_oct_pyrdown(const uint8_t *src, int w, int h, uint8_t *dst, int dw, int dh);
extern "C" int lbd_oct_keylines(const float *raw, int n, int octave, int ow, int oh, int w, int h, void *out);
extern "C" int lsd_orc_detect(const uint8_t *img, int w, int h, int stride, int channels, float line_length_thres, float *lines_out, int cap,
                              float *raw_lines, int cap_raw, int *n_raw_out, double *scaled_out, double *modgrad_out, double *angles_out,
                              int32_t *list_out, int *list_len, int refine_mode);

struct cs_ctx {
    std::string err;
};

namespace {
int g_fail_below = 0; /* CS_ERR_CAPACITY whenever max_lines_per_octave is below this */
int g_calls = 0, g_last_cap = 0;

int fail(cs_ctx *c, int status, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    std::vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    c->err = buf;
    return status;
}
}  // namespace

extern "C" {
/* the knob and the record of the calls the shim made */
void standin_fail_below(int cap) { g_fail_below = cap; }
int standin_calls() { return g_calls; }
int standin_last_cap() { return g_last_cap; }
void standin_reset()
{
    g_fail_below = 0;
    g_calls = 0;
    g_last_cap = 0;
}

cs_ctx *cs_create(int, int, int, int, int, int) { return new cs_ctx; }
void cs_destroy(cs_ctx *c) { delete c; }
const char *cs_last_error(const cs_ctx *c) { return c ? c->err.c_str() : "no context"; }
void cs_default_line_params(cs_line_params *p)
{
    p->use_LSD = 0;
    p->numoctaves = 1;
    p->octaveratio = 1.0f;
    p->line_length_thres = 50.0f;
}

int cs_detect_raw_lines_octaves_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels,
                                      const cs_line_params *params, cs_keyline_octave *keylines, int32_t max_lines_per_octave, int32_t *n_lines)
{
    g_calls++;
    g_last_cap = max_lines_per_octave;
    if (!c) return CS_ERR_INVALID_ARG;
    if (!imgs || n_frames <= 0 || width <= 0 || height <= 0) return fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3");
    if (stride < width * channels) return fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    if (!params || !keylines || !n_lines || max_lines_per_octave <= 0) return fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (!params->use_LSD) return fail(c, CS_ERR_UNSUPPORTED, "the octave calls are provided for the LSD flavour (use_LSD = 1)");
    const int K = params->numoctaves;
    if (K < 1) return fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1");
    if (K > 1 && !(params->octaveratio >= 2.0f && params->octaveratio < 3.0f))
        return fail(c, CS_ERR_INVALID_ARG, "numoctaves > 1 needs (int)octaveratio == 2 (got %g)", (double)params->octaveratio);
    std::vector<int> ow((size_t)K, width), oh((size_t)K, height);
    for (int k = 1; k < K; k++) {
        ow[k] = ow[k - 1] / 2;
        oh[k] = oh[k - 1] / 2;
    }
    if (std::lrint(ow[K - 1] * 0.8) < 2 || std::lrint(oh[K - 1] * 0.8) < 2 || width > 32767 || height > 32767)
        return fail(c, CS_ERR_INVALID_ARG, "octave %d of a %d x %d frame is %d x %d: too small for LSD", K - 1, width, height, ow[K - 1], oh[K - 1]);
    const int cap = max_lines_per_octave;
    for (int f = 0; f < n_frames; f++) {
        const uint8_t *img = imgs + (size_t)f * height * stride;
        std::vector<std::vector<uint8_t>> pyr((size_t)K);
        pyr[0].resize((size_t)width * height);
        if (channels == 3)
            orc_bgr2gray(img, width, height, stride, pyr[0].data(), width, 1);
        else
            for (int y = 0; y < height; y++) std::memcpy(&pyr[0][(size_t)y * width], img + (size_t)y * stride, (size_t)width);
        for (int k = 1; k < K; k++) {
            pyr[k].resize((size_t)ow[k] * oh[k]);
            lbd_oct_pyrdown(pyr[k - 1].data(), ow[k - 1], oh[k - 1], pyr[k].data(), ow[k], oh[k]);
        }
        for (int k = 0; k < K; k++) {
            const int room = ow[k] * oh[k] + 16;
            std::vector<float> lines((size_t)room * 4), raw((size_t)room * 4);
            int n_raw = 0;
            lsd_orc_detect(pyr[k].data(), ow[k], oh[k], ow[k], 1, 15.0f, lines.data(), room, raw.data(), room, &n_raw, nullptr, nullptr, nullptr, nullptr, nullptr, 2);
            if (n_raw > cap || cap < g_fail_below)
                return fail(c, CS_ERR_CAPACITY, "frame %d, octave %d: %d LSD segments exceed max_lines_per_octave = %d", f, k, n_raw, cap);
            n_lines[(size_t)f * K + k] = lbd_oct_keylines(raw.data(), n_raw, k, ow[k], oh[k], width, height, keylines + ((size_t)f * K + k) * cap);
        }
    }
    return CS_OK;
}
}  // extern "C"
