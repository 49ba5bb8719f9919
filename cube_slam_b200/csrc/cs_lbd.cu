/* cs_lbd.cu -- LBD line descriptors and descriptor matching on the device: the descriptor / matcher half of class line_lbd_detect
 * (SURVEY.md section 8 row f4).
 *
 * Replaces   line_lbd/class/line_lbd_allclass.cpp:191-198,224-272,341-356   get_line_descriptors, detect_descrip_lines, match_line_descrip
 *            line_lbd/libs/binary_descriptor.cpp:352-416,587-790,1146-1509   computeSobel, binaryConversion, compute / computeImpl, computeLBD
 *            line_lbd/libs/LSDDetector.cpp:226-250                           the KeyLine fields of the LSD flavour (host)
 *            line_lbd/libs/binary_descriptor_matcher.cpp:196-262,598-756     BinaryDescriptorMatcher::match, Mihasher::batchquery / query
 *            line_lbd/libs/binary_descriptor_matcher.cpp:264-341,431-507     BinaryDescriptorMatcher::knnMatch, radiusMatch (pairwise forms)
 *
 *   k_lbd_describe   one 64-thread CTA per key line.  Thread hID walks row hID of the 63-row support region along the line (one int16
 *                    gather from each Sobel map per step, float sums in the reference's order); after a barrier 72 threads add the rows
 *                    into the 9 x 8 band sums, each in increasing row order; 9 threads turn them into mean / standard deviation; one thread
 *                    runs the two normalisations; 32 threads write the 32 comparison bytes.  The arithmetic lives in cs_lbd_core.h, which
 *                    the CPU test suite compiles for the host and checks against the oracle.
 *                    Algorithmic bytes per line: 63 x numOfPixels x 4 (two int16 gathers) + 32 out; the Sobel maps of a VGA frame are
 *                    1.2 MB, so the gathers of a batch are served from L2 after the first touch -- the kernel is bound by the dependent
 *                    float chain of each row (one add per step after a gather), thousands of rows in flight hide it.
 *   k_lbd_match      one 128-thread CTA per query descriptor: every thread takes train codes 128 apart, two 16-byte loads each, builds the
 *                    64-bit key (distance, radius, substring, pattern, train index) that reproduces the multi-index hash's visiting order
 *                    and the CTA reduces to the minimum.  32 bytes per (query, train) pair, all of it in L2 for a frame pair.
 *   k_lbd_knn2       knnMatch with k <= 2: k_lbd_match's shape keeping the two smallest keys per thread, merged by shuffles.
 *   k_lbd_match_sorted   knnMatch with k > 2 and radiusMatch: one 256-thread CTA per query counts the keys it keeps, stages them in shared
 *                    memory at a CTA-wide prefix and sorts them (bitonic); radius calls it twice (counts, then keys at host offsets).
 *   The Sobel maps come from the EDLines front-end kernel (cs_edlines.cu: k_ed_front), which is what computeSobel computes.
 *
 * Host side: cos / sin of the line direction, the mid point and the Gaussian weights are computed here with libm exactly as the reference
 * computes them (float overloads: see oracle/lbd_oracle.cpp's header for which ones and why); thresholding and compaction of the matches
 * run on the host over 8 bytes per query. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "cs_internal.h"
#include "cs_lbd_core.h"
#if defined(__CUDACC__)
#include "cs_kernels.h" /* CS_ONCE_PER_DEVICE */
#endif

namespace {

#include "cs_lbd_kernels.cuh"

struct Buf {
    void *p = nullptr;
    size_t cap = 0;
};
struct LbdState {
    Buf lines, desc, fdesc, coef, q, t, pairq, toff, keys;
    Buf mkeys, moff, mcnt; /* knn / radius matching: sorted keys, their per-query offsets and counts */
    bool coef_filled = false;
};

int ensure(cs_ctx *c, Buf &b, size_t bytes)
{
    if (bytes <= b.cap) return CS_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    const size_t want = bytes + bytes / 16 + 256;
    if (cudaMalloc(&b.p, want) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc(%zu) failed in the line descriptor", want);
    b.cap = want;
    return CS_OK;
}

LbdState *state_of(cs_ctx *c)
{
    void **slot = cs_ctx_lbd_slot(c);
    if (!*slot) *slot = new LbdState();
    return (LbdState *)*slot;
}

/* BinaryDescriptor::BinaryDescriptor (binary_descriptor.cpp:140-179): F_l over 3 x 7 rows, F_g over 63 rows; the integer divisions are the
 * reference's: u = (21 - 1) / 2 = 10, sigma = (14 + 1) / 2 = 7; then u = sigma = (63 - 1) / 2 = 31.  computeLBD narrows each weight to float
 * where it uses it (:1324,1340,1354,1368). */
void lbd_weights(float *g63, float *l21)
{
    const int wob = CS_LBD_BAND_WIDTH;
    double u = (wob * 3 - 1) / 2;
    double sigma = (wob * 2 + 1) / 2;
    double invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < wob * 3; i++) {
        const double dis = i - u;
        l21[i] = (float)exp(dis * dis * invsigma2);
    }
    u = (CS_LBD_BANDS * wob - 1) / 2;
    sigma = u;
    invsigma2 = -1 / (2 * sigma * sigma);
    for (int i = 0; i < CS_LBD_ROWS; i++) {
        const double dis = i - u;
        g63[i] = (float)exp(dis * dis * invsigma2);
    }
}

/* what computeLBD derives per line before its loops (:1233-1256) */
void lbd_prepare(const cs_keyline &k, int frame, CsLbdLine &o)
{
    o.mid_x = (float)(0.5 * (k.start_x + k.end_x));
    o.mid_y = (float)(0.5 * (k.start_y + k.end_y));
    o.dl_x = cosf(k.angle);
    o.dl_y = sinf(k.angle);
    o.length = (int32_t)(short)k.num_pixels;
    o.frame = frame;
}

/* number of pixels cv::LineIterator(img, Point2f, Point2f) reports for two points inside the image: Point2f -> Point rounds half to even
 * (cvRound), 8-connected: max(|dx|, |dy|) + 1.  LSDDetector clamps its extremes into the image first (checkLineExtremes, :75-101). */
int line_iterator_count(float x1, float y1, float x2, float y2, int w, int h)
{
    auto cl = [](long v, int n) { return (int)(v < 0 ? 0 : (v >= n ? n - 1 : v)); };
    const int ix1 = cl(lrintf(x1), w), iy1 = cl(lrintf(y1), h), ix2 = cl(lrintf(x2), w), iy2 = cl(lrintf(y2), h);
    return std::max(std::abs(ix2 - ix1), std::abs(iy2 - iy1)) + 1;
}

void keyline_from_lsd_row(const float *e, int w, int h, int class_id, cs_keyline &kl)
{
    kl.start_x = e[0];
    kl.start_y = e[1];
    kl.end_x = e[2];
    kl.end_y = e[3];
    const double lx = (double)(e[0] - e[2]), ly = (double)(e[1] - e[3]); /* sqrt(pow(float, 2) + pow(float, 2)): std::pow(float, int) is a double, */
    kl.line_length = (float)sqrt(lx * lx + ly * ly);                     /* and the square of a float is exact in double */
    kl.num_pixels = line_iterator_count(e[0], e[1], e[2], e[3], w, h);
    kl.angle = atan2f(kl.end_y - kl.start_y, kl.end_x - kl.start_x);
    kl.size = (kl.end_x - kl.start_x) * (kl.end_y - kl.start_y);
    kl.response = kl.line_length / std::max(w, h);
    kl.class_id = class_id;
}

/* BinaryDescriptor::detectImpl's KeyLine fill (binary_descriptor.cpp:526-545) for one EDLines segment: e = the ordered end points
 * (OctaveKeyLines :1083-1139), x = {lineDirection_, numOfPixels as an integer's bits} as the detector kernels leave them */
void keyline_from_edl_row(const float *e, const float *x, int w, int h, int class_id, cs_keyline &kl)
{
    int32_t npx;
    memcpy(&npx, x + 1, 4);
    kl.start_x = e[0];
    kl.start_y = e[1];
    kl.end_x = e[2];
    kl.end_y = e[3];
    kl.angle = x[0];
    const float ddx = fabsf(e[0] - e[2]), ddy = fabsf(e[1] - e[3]);
    kl.line_length = sqrtf(ddx * ddx + ddy * ddy); /* OctaveKeyLines :880-886, symmetric in the two ends */
    kl.num_pixels = npx;
    kl.size = (e[2] - e[0]) * (e[3] - e[1]);
    kl.response = kl.line_length / std::max(w, h);
    kl.class_id = class_id;
}

/* descriptors of `n` prepared lines over Sobel maps already in HBM; results to the host */
int describe(cs_ctx *c, LbdState &S, const std::vector<CsLbdLine> &lines, const int16_t *d_dx, const int16_t *d_dy, int w, int h, uint8_t *desc32, float *desc72)
{
    const size_t n = lines.size();
    if (!n) return CS_OK;
    cudaStream_t st = cs_ctx_stream(c);
    int rc;
    if ((rc = ensure(c, S.lines, n * sizeof(CsLbdLine))) || (rc = ensure(c, S.desc, n * CS_LBD_BYTES)) || (rc = ensure(c, S.coef, 84 * 4)) ||
        (desc72 && (rc = ensure(c, S.fdesc, n * CS_LBD_DESC * 4))))
        return rc;
    if (!S.coef_filled) {
        float coef[CS_LBD_ROWS + 3 * CS_LBD_BAND_WIDTH];
        lbd_weights(coef, coef + CS_LBD_ROWS);
        if (cudaMemcpyAsync(S.coef.p, coef, sizeof coef, cudaMemcpyHostToDevice, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the descriptor weights failed");
        S.coef_filled = true;
    }
    if (cudaMemcpyAsync(S.lines.p, lines.data(), n * sizeof(CsLbdLine), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the key lines failed");
    launch_lbd_describe((unsigned)n, st, (const CsLbdLine *)S.lines.p, (int)n, d_dx, d_dy, w, h, (const float *)S.coef.p, (uint8_t *)S.desc.p,
                        desc72 ? (float *)S.fdesc.p : nullptr);
    cs_ctx_count_launches(c, 1);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "descriptor kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (cudaMemcpyAsync(desc32, S.desc.p, n * CS_LBD_BYTES, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (desc72 && cudaMemcpyAsync(desc72, S.fdesc.p, n * CS_LBD_DESC * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "descriptor copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    return CS_OK;
}

int check_image_args(cs_ctx *c, const void *imgs, int n_frames, int width, int height, int stride, int channels)
{
    if (!imgs || n_frames <= 0 || width <= 0 || height <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (channels != 1 && channels != 3) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "channels must be 1 or 3"); /* computeImpl :617-618 throws on depth != 0 */
    if (stride < width * channels) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "stride smaller than a row");
    return CS_OK;
}

/* the pair CSRs of the knn / radius calls: start at 0, do not decrease, every train set within the shared-memory bound */
int check_pairs(cs_ctx *c, const int32_t *qo, const int32_t *to, int n_pairs)
{
    if (n_pairs <= 0 || !qo || !to) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (qo[0] != 0 || to[0] != 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "offsets must start at 0");
    for (int p = 0; p < n_pairs; p++) {
        if (qo[p + 1] < qo[p] || to[p + 1] < to[p]) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "offsets must not decrease");
        if (to[p + 1] - to[p] > CS_LBD_KNN_MAX_TRAIN)
            return cs_ctx_fail(c, CS_ERR_CAPACITY, "pair %d has %d train codes: knn / radius matching takes at most %d per pair", p, to[p + 1] - to[p],
                               CS_LBD_KNN_MAX_TRAIN);
    }
    return CS_OK;
}

/* codes of every pair to the device (S.q, S.t), with the pair of each query (S.pairq, and on the host in pair_of) and the train CSR (S.toff) */
int upload_pairs(cs_ctx *c, LbdState &S, const uint8_t *query32, const int32_t *qo, const uint8_t *train32, const int32_t *to, int n_pairs,
                 std::vector<int32_t> &pair_of)
{
    const int nq = qo[n_pairs], nt = to[n_pairs];
    cudaStream_t st = cs_ctx_stream(c);
    pair_of.assign((size_t)nq, 0);
    for (int p = 0; p < n_pairs; p++)
        for (int i = qo[p]; i < qo[p + 1]; i++) pair_of[i] = p;
    int rc;
    if ((rc = ensure(c, S.q, (size_t)nq * 32)) || (rc = ensure(c, S.t, (size_t)nt * 32)) || (rc = ensure(c, S.pairq, (size_t)nq * 4)) ||
        (rc = ensure(c, S.toff, (size_t)(n_pairs + 1) * 4)))
        return rc;
    if (cudaMemcpyAsync(S.q.p, query32, (size_t)nq * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.t.p, train32, (size_t)nt * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.pairq.p, pair_of.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.toff.p, to, (size_t)(n_pairs + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the descriptors failed");
    return CS_OK;
}

/* a sorted-match launch: room for out_off[nq] keys at S.mkeys, offsets uploaded to S.moff, counts at S.mcnt; with out_off == NULL the
 * counting launch (no keys, no shared memory) */
int launch_sorted(cs_ctx *c, LbdState &S, int nq, int max_dist, const std::vector<long long> *out_off, int max_m)
{
    cudaStream_t st = cs_ctx_stream(c);
    int rc;
    if ((rc = ensure(c, S.mcnt, (size_t)nq * 4))) return rc;
    unsigned sort_cap = 0;
    if (out_off) {
        sort_cap = 1;
        while ((int)sort_cap < max_m) sort_cap <<= 1;
        if ((rc = ensure(c, S.mkeys, (size_t)(*out_off)[nq] * 8)) || (rc = ensure(c, S.moff, (size_t)(nq + 1) * 8))) return rc;
        if (cudaMemcpyAsync(S.moff.p, out_off->data(), (size_t)(nq + 1) * 8, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the match offsets failed");
    }
    launch_lbd_match_sorted((unsigned)nq, st, sort_cap, (const uint4 *)S.q.p, (const uint4 *)S.t.p, (const int32_t *)S.pairq.p, (const int32_t *)S.toff.p, nq,
                            max_dist, out_off ? (const long long *)S.moff.p : nullptr, out_off ? (unsigned long long *)S.mkeys.p : nullptr, (int32_t *)S.mcnt.p);
    cs_ctx_count_launches(c, 1);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "matcher kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    return CS_OK;
}

/* cv::DMatch of a key, as match() builds it; beyond D = 128 the reference never writes results[], and the library reports train_idx -1 */
void key_to_dmatch(unsigned long long key, int query_idx, cs_dmatch &m)
{
    const int d = CS_LBD_KEY_DIST(key);
    m.query_idx = query_idx;
    m.train_idx = d <= 128 ? (int32_t)CS_LBD_KEY_TRAIN(key) : -1;
    m.img_idx = 0;
    m.distance = (float)d;
}

}  // namespace

void cs_lbd_destroy(void *state)
{
    LbdState *S = (LbdState *)state;
    Buf *all[] = {&S->lines, &S->desc, &S->fdesc, &S->coef, &S->q, &S->t, &S->pairq, &S->toff, &S->keys, &S->mkeys, &S->moff, &S->mcnt};
    for (Buf *b : all)
        if (b->p) cudaFree(b->p);
    delete S;
}

extern "C" {

int cs_keylines_from_lines(const float *lines_xyxy, int n, int width, int height, cs_keyline *out)
{
    if (n < 0 || width <= 0 || height <= 0 || (n > 0 && (!lines_xyxy || !out))) return CS_ERR_INVALID_ARG;
    for (int k = 0; k < n; k++) keyline_from_lsd_row(lines_xyxy + 4 * (size_t)k, width, height, k, out[k]);
    return CS_OK;
}

int cs_lbd_debug_keylines_edl(const float *lines_xyxy, const float *extra2, int n, int width, int height, cs_keyline *out)
{
    if (n < 0 || width <= 0 || height <= 0 || (n > 0 && (!lines_xyxy || !extra2 || !out))) return CS_ERR_INVALID_ARG;
    for (int k = 0; k < n; k++) keyline_from_edl_row(lines_xyxy + 4 * (size_t)k, extra2 + 2 * (size_t)k, width, height, k, out[k]);
    return CS_OK;
}

int cs_lbd_debug_prepare(const cs_keyline *keylines, int n, void *lines24, float *coef_g63, float *coef_l21)
{
    static_assert(sizeof(CsLbdLine) == 24, "CsLbdLine is 6 x 4 bytes");
    if (n < 0 || (n > 0 && (!keylines || !lines24))) return CS_ERR_INVALID_ARG;
    for (int i = 0; i < n; i++) lbd_prepare(keylines[i], 0, ((CsLbdLine *)lines24)[i]);
    if (coef_g63 && coef_l21) lbd_weights(coef_g63, coef_l21);
    return CS_OK;
}

int cs_lbd_compute_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const cs_keyline *keylines,
                         const int32_t *keyline_offsets, uint8_t *desc32, float *desc72)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc = check_image_args(c, imgs, n_frames, width, height, stride, channels);
    if (rc) return rc;
    if (!keyline_offsets || keyline_offsets[0] != 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "keyline_offsets must start at 0");
    for (int f = 0; f < n_frames; f++)
        if (keyline_offsets[f + 1] < keyline_offsets[f]) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "keyline_offsets must not decrease");
    const int n = keyline_offsets[n_frames];
    if (n == 0) return CS_OK; /* "Error: keypoint list is empty": descriptors left as they are (:622-626) */
    if (!keylines || !desc32) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null key lines or output");
    cudaSetDevice(cs_ctx_device(c));
    std::vector<CsLbdLine> lines((size_t)n);
    for (int f = 0; f < n_frames; f++)
        for (int i = keyline_offsets[f]; i < keyline_offsets[f + 1]; i++) lbd_prepare(keylines[i], f, lines[i]);
    const int16_t *d_dx = nullptr, *d_dy = nullptr;
    if ((rc = cs_edl_sobel_maps(c, imgs, false, n_frames, width, height, stride, channels, &d_dx, &d_dy))) return rc;
    return describe(c, *state_of(c), lines, d_dx, d_dy, width, height, desc32, desc72);
}

int cs_lbd_compute(cs_ctx *c, const uint8_t *img, int width, int height, int stride, int channels, const cs_keyline *keylines, int n, uint8_t *desc32,
                   float *desc72)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (n < 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "negative key line count");
    const int32_t off[2] = {0, n};
    return cs_lbd_compute_batch(c, img, 1, width, height, stride, channels, keylines, off, desc32, desc72);
}

int cs_detect_descrip_lines_batch(cs_ctx *c, const uint8_t *imgs, int n_frames, int width, int height, int stride, int channels, const cs_line_params *params,
                                  cs_keyline *keylines, uint8_t *desc32, int32_t max_lines_per_frame, int32_t *n_lines)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc = check_image_args(c, imgs, n_frames, width, height, stride, channels);
    if (rc) return rc;
    if (!params || !keylines || !desc32 || !n_lines || max_lines_per_frame <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    /* more octaves: both overloads of detect_descrip_lines keep octave 0 only (:239,266), whose lines and Sobel maps do not depend on the others */
    if (params->numoctaves < 1) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "numoctaves must be at least 1");
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    const int cap = max_lines_per_frame;
    const float *d_lines = nullptr, *d_extra = nullptr;
    const int32_t *d_counts = nullptr;
    const int16_t *d_dx = nullptr, *d_dy = nullptr;
    const uint8_t *d_lsd_frames = nullptr; /* LSD: the detector's copy of the frames, for the Sobel maps once the key lines are known */
    if (params->use_LSD) {
        if ((rc = cs_lsd_run_host(c, imgs, n_frames, width, height, stride, channels, params->line_length_thres, cap, &d_lines, &d_counts, &d_lsd_frames)))
            return rc;
    } else if ((rc = cs_edl_run_keylines(c, imgs, false, n_frames, width, height, stride, channels, params->line_length_thres, cap, &d_lines, &d_counts, &d_extra,
                                         &d_dx, &d_dy)))
        return rc;
    std::vector<int32_t> cnt((size_t)n_frames);
    std::vector<float> seg((size_t)n_frames * cap * 4), extra(d_extra ? (size_t)n_frames * cap * 2 : 0);
    if (cudaMemcpyAsync(cnt.data(), d_counts, (size_t)n_frames * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(seg.data(), d_lines, seg.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (d_extra && cudaMemcpyAsync(extra.data(), d_extra, extra.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "line result copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    /* the KeyLine fill of the two detectors (LSDDetector.cpp:226-250; binary_descriptor.cpp:526-545) for the kept lines */
    std::vector<CsLbdLine> lines;
    std::vector<int32_t> first((size_t)n_frames + 1, 0);
    for (int f = 0; f < n_frames; f++) {
        if (cnt[f] > cap) return cs_ctx_fail(c, CS_ERR_CAPACITY, "frame %d: %d segments exceed max_lines_per_frame", f, cnt[f]);
        n_lines[f] = cnt[f];
        first[f + 1] = first[f] + cnt[f];
        for (int k = 0; k < cnt[f]; k++) {
            const float *e = &seg[((size_t)f * cap + k) * 4];
            cs_keyline &kl = keylines[(size_t)f * cap + k];
            if (params->use_LSD)
                keyline_from_lsd_row(e, width, height, k, kl);
            else
                keyline_from_edl_row(e, &extra[((size_t)f * cap + k) * 2], width, height, k, kl);
            CsLbdLine L;
            lbd_prepare(kl, f, L);
            lines.push_back(L);
        }
    }
    /* computeImpl returns before computeSobel when there is no key line (binary_descriptor.cpp:617-622), and so does this */
    if (lines.empty()) return CS_OK;
    if (d_lsd_frames && (rc = cs_edl_sobel_maps(c, d_lsd_frames, true, n_frames, width, height, stride, channels, &d_dx, &d_dy))) return rc;
    /* descriptors come back line after line; hand each frame's rows to its slot */
    std::vector<uint8_t> packed(lines.size() * CS_LBD_BYTES);
    if ((rc = describe(c, *state_of(c), lines, d_dx, d_dy, width, height, packed.data(), nullptr))) return rc;
    for (int f = 0; f < n_frames; f++)
        if (cnt[f]) memcpy(desc32 + (size_t)f * cap * CS_LBD_BYTES, packed.data() + (size_t)first[f] * CS_LBD_BYTES, (size_t)cnt[f] * CS_LBD_BYTES);
    return CS_OK;
}

int cs_detect_descrip_lines(cs_ctx *c, const uint8_t *img, int width, int height, int stride, int channels, const cs_line_params *params, cs_keyline *keylines,
                            uint8_t *desc32, int32_t *n_inout)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (!n_inout || *n_inout <= 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "n_inout must give the capacity of keylines / desc32");
    int32_t n = 0;
    const int rc = cs_detect_descrip_lines_batch(c, img, 1, width, height, stride, channels, params, keylines, desc32, *n_inout, &n);
    if (rc == CS_OK) *n_inout = n;
    return rc;
}

int cs_match_line_descrip_batch(cs_ctx *c, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32, const int32_t *train_offsets,
                                int n_pairs, float thres, cs_dmatch *matches, int32_t *n_matches)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (n_pairs <= 0 || !query_offsets || !train_offsets || !n_matches) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null or empty argument");
    if (query_offsets[0] != 0 || train_offsets[0] != 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "offsets must start at 0");
    for (int p = 0; p < n_pairs; p++) {
        if (query_offsets[p + 1] < query_offsets[p] || train_offsets[p + 1] < train_offsets[p]) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "offsets must not decrease");
        n_matches[p] = 0;
    }
    const int nq = query_offsets[n_pairs], nt = train_offsets[n_pairs];
    if (nq == 0 || nt == 0) return CS_OK; /* "descriptors matrices cannot be void": no matches (:199-203) */
    if (!query32 || !train32 || !matches) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null descriptors or output");
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    LbdState &S = *state_of(c);
    std::vector<int32_t> pair_of_query((size_t)nq);
    for (int p = 0; p < n_pairs; p++)
        for (int i = query_offsets[p]; i < query_offsets[p + 1]; i++) pair_of_query[i] = p;
    int rc;
    if ((rc = ensure(c, S.q, (size_t)nq * 32)) || (rc = ensure(c, S.t, (size_t)nt * 32)) || (rc = ensure(c, S.pairq, (size_t)nq * 4)) ||
        (rc = ensure(c, S.toff, (size_t)(n_pairs + 1) * 4)) || (rc = ensure(c, S.keys, (size_t)nq * 8)))
        return rc;
    if (cudaMemcpyAsync(S.q.p, query32, (size_t)nq * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.t.p, train32, (size_t)nt * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.pairq.p, pair_of_query.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(S.toff.p, train_offsets, (size_t)(n_pairs + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "upload of the descriptors failed");
    launch_lbd_match((unsigned)nq, st, (const uint4 *)S.q.p, (const uint4 *)S.t.p, (const int32_t *)S.pairq.p, (const int32_t *)S.toff.p, nq,
                     (unsigned long long *)S.keys.p);
    cs_ctx_count_launches(c, 1);
    if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "matcher kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    std::vector<unsigned long long> keys((size_t)nq);
    if (cudaMemcpyAsync(keys.data(), S.keys.p, (size_t)nq * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "match copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    /* match_line_descrip's filter (:349-355), per pair, in query order */
    for (int p = 0; p < n_pairs; p++) {
        if (train_offsets[p + 1] == train_offsets[p]) continue; /* empty train set: the reference returns before matching */
        cs_dmatch *out = matches + query_offsets[p];
        int n = 0;
        for (int i = query_offsets[p]; i < query_offsets[p + 1]; i++) {
            const unsigned long long key = keys[i];
            if (key == ~0ull) continue; /* the hash visits no code for this query: no DMatch (:243-244) */
            const int d = CS_LBD_KEY_DIST(key);
            if (!((float)d < thres)) continue;
            out[n].query_idx = i - query_offsets[p];
            out[n].train_idx = d <= 128 ? (int32_t)CS_LBD_KEY_TRAIN(key) : -1; /* beyond D = 128 the reference never writes results[] */
            out[n].img_idx = 0;
            out[n].distance = (float)d;
            n++;
        }
        n_matches[p] = n;
    }
    return CS_OK;
}

int cs_match_line_descrip(cs_ctx *c, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, float thres, cs_dmatch *matches,
                          int32_t *n_matches)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (n_query < 0 || n_train < 0 || !n_matches) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad descriptor counts");
    const int32_t qo[2] = {0, n_query}, to[2] = {0, n_train};
    return cs_match_line_descrip_batch(c, query32, qo, train32, to, 1, thres, matches, n_matches);
}

int cs_knn_match_line_descrip_batch(cs_ctx *c, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32, const int32_t *train_offsets,
                                    int n_pairs, int k, const uint8_t *query_mask, cs_dmatch *matches, int32_t *n_per_query)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc = check_pairs(c, query_offsets, train_offsets, n_pairs);
    if (rc) return rc;
    if (k < 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "k must not be negative");
    const int nq = query_offsets[n_pairs], nt = train_offsets[n_pairs];
    if (nq > 0 && !n_per_query) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null n_per_query");
    for (int i = 0; i < nq; i++) n_per_query[i] = 0;
    if (nq == 0 || nt == 0 || k == 0) return CS_OK; /* "descriptors matrices cannot be void" (:270-274); k = 0: no entry per query */
    if (!query32 || !train32 || !matches) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null descriptors or output");
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    LbdState &S = *state_of(c);
    std::vector<int32_t> pair_of;
    if ((rc = upload_pairs(c, S, query32, query_offsets, train32, train_offsets, n_pairs, pair_of))) return rc;
    auto keep = [&](int i) { return !query_mask || query_mask[i]; };
    if (k <= 2) {
        if ((rc = ensure(c, S.mkeys, (size_t)nq * 16))) return rc;
        launch_lbd_knn2((unsigned)nq, st, (const uint4 *)S.q.p, (const uint4 *)S.t.p, (const int32_t *)S.pairq.p, (const int32_t *)S.toff.p, nq,
                        (unsigned long long *)S.mkeys.p);
        cs_ctx_count_launches(c, 1);
        if (cudaGetLastError() != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "matcher kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        std::vector<unsigned long long> keys((size_t)nq * 2);
        if (cudaMemcpyAsync(keys.data(), S.mkeys.p, keys.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return cs_ctx_fail(c, CS_ERR_CUDA, "match copy failed: %s", cudaGetErrorString(cudaGetLastError()));
        for (int i = 0; i < nq; i++) {
            if (!keep(i)) continue;
            int n = 0;
            while (n < k && keys[2 * (size_t)i + n] != ~0ull) {
                key_to_dmatch(keys[2 * (size_t)i + n], i - query_offsets[pair_of[i]], matches[(size_t)i * k + n]);
                n++;
            }
            n_per_query[i] = n;
        }
        return CS_OK;
    }
    /* k > 2: min(k, train set) slots per kept query, the first of its sorted met codes */
    std::vector<long long> off((size_t)nq + 1, 0);
    int max_nt = 0;
    for (int i = 0; i < nq; i++) {
        const int ntp = train_offsets[pair_of[i] + 1] - train_offsets[pair_of[i]];
        const int room = keep(i) ? std::min(k, ntp) : 0;
        off[i + 1] = off[i] + room;
        if (room) max_nt = std::max(max_nt, ntp);
    }
    if (off[nq] == 0) return CS_OK;
    if ((rc = launch_sorted(c, S, nq, 256 /* every met code */, &off, max_nt))) return rc;
    std::vector<unsigned long long> keys((size_t)off[nq]);
    std::vector<int32_t> cnt((size_t)nq);
    if (cudaMemcpyAsync(keys.data(), S.mkeys.p, keys.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(cnt.data(), S.mcnt.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "match copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    for (int i = 0; i < nq; i++) {
        for (int j = 0; j < cnt[i]; j++) key_to_dmatch(keys[(size_t)off[i] + j], i - query_offsets[pair_of[i]], matches[(size_t)i * k + j]);
        n_per_query[i] = cnt[i];
    }
    return CS_OK;
}

int cs_knn_match_line_descrip(cs_ctx *c, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, int k, const uint8_t *query_mask,
                              cs_dmatch *matches, int32_t *n_per_query)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (n_query < 0 || n_train < 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad descriptor counts");
    const int32_t qo[2] = {0, n_query}, to[2] = {0, n_train};
    return cs_knn_match_line_descrip_batch(c, query32, qo, train32, to, 1, k, query_mask, matches, n_per_query);
}

int cs_radius_match_line_descrip_batch(cs_ctx *c, const uint8_t *query32, const int32_t *query_offsets, const uint8_t *train32, const int32_t *train_offsets,
                                       int n_pairs, float max_distance, const uint8_t *query_mask, cs_dmatch *matches, int64_t max_matches,
                                       int64_t *match_offsets)
{
    if (!c) return CS_ERR_INVALID_ARG;
    int rc = check_pairs(c, query_offsets, train_offsets, n_pairs);
    if (rc) return rc;
    if (!match_offsets || max_matches < 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null match_offsets or negative max_matches");
    const int nq = query_offsets[n_pairs], nt = train_offsets[n_pairs];
    for (int i = 0; i <= nq; i++) match_offsets[i] = 0;
    /* k_distances[j] <= maxDistance (:484): an integer distance against a float; NaN and negative radii take nothing */
    const int max_dist = !(max_distance >= 0.0f) ? -1 : (max_distance >= 256.0f ? 256 : (int)floorf(max_distance));
    if (nq == 0 || nt == 0 || max_dist < 0) return CS_OK;
    if (!query32 || !train32) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null descriptors");
    cudaSetDevice(cs_ctx_device(c));
    cudaStream_t st = cs_ctx_stream(c);
    LbdState &S = *state_of(c);
    std::vector<int32_t> pair_of;
    if ((rc = upload_pairs(c, S, query32, query_offsets, train32, train_offsets, n_pairs, pair_of))) return rc;
    /* first launch: how many codes each query has within the radius */
    if ((rc = launch_sorted(c, S, nq, max_dist, nullptr, 0))) return rc;
    std::vector<int32_t> cnt((size_t)nq);
    if (cudaMemcpyAsync(cnt.data(), S.mcnt.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "match count copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    std::vector<long long> off((size_t)nq + 1, 0);
    int max_m = 0;
    for (int i = 0; i < nq; i++) {
        const int m = (!query_mask || query_mask[i]) ? cnt[i] : 0;
        off[i + 1] = off[i] + m;
        max_m = std::max(max_m, m);
    }
    for (int i = 0; i <= nq; i++) match_offsets[i] = off[i];
    if (off[nq] > max_matches)
        return cs_ctx_fail(c, CS_ERR_CAPACITY, "%lld matches within the radius exceed max_matches = %lld; match_offsets holds the layout they need",
                           (long long)off[nq], (long long)max_matches);
    if (off[nq] == 0) return CS_OK;
    if (!matches) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "null matches");
    /* second launch: the codes themselves, sorted, at their offsets */
    if ((rc = launch_sorted(c, S, nq, max_dist, &off, max_m))) return rc;
    std::vector<unsigned long long> keys((size_t)off[nq]);
    if (cudaMemcpyAsync(keys.data(), S.mkeys.p, keys.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return cs_ctx_fail(c, CS_ERR_CUDA, "match copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    for (int i = 0; i < nq; i++)
        for (long long j = off[i]; j < off[i + 1]; j++) key_to_dmatch(keys[(size_t)j], i - query_offsets[pair_of[i]], matches[j]);
    return CS_OK;
}

int cs_radius_match_line_descrip(cs_ctx *c, const uint8_t *query32, int n_query, const uint8_t *train32, int n_train, float max_distance,
                                 const uint8_t *query_mask, cs_dmatch *matches, int64_t max_matches, int64_t *match_offsets)
{
    if (!c) return CS_ERR_INVALID_ARG;
    if (n_query < 0 || n_train < 0) return cs_ctx_fail(c, CS_ERR_INVALID_ARG, "bad descriptor counts");
    const int32_t qo[2] = {0, n_query}, to[2] = {0, n_train};
    return cs_radius_match_line_descrip_batch(c, query32, qo, train32, to, 1, max_distance, query_mask, matches, max_matches, match_offsets);
}

}  // extern "C"
