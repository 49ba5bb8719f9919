/*
 * oracle/lbd_octaves_oracle.cpp -- CPU ORACLE for every octave of a multi-octave LSD line_lbd_detect.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates, without OpenCV, what the higher octaves add to the one-octave restatement of oracle/lbd_oracle.cpp:
 *   line_lbd/libs/LSDDetector.cpp:55-72                  computeGaussianPyramid: pyrDown to (cols / 2, rows / 2) per octave
 *   line_lbd/libs/LSDDetector.cpp:205-250                the KeyLine fill of octave k: extremes clamped to the octave, scaled by 2^k, the
 *                                                        10 px border test against the input frame, lineLength / numOfPixels / response on
 *                                                        the octave, angle and size of the scaled ends, class_id per octave
 *   line_lbd/libs/binary_descriptor.cpp:352-398          computeGaussianPyramid + computeSobel: the blurred frame, pyrDown per octave,
 *                                                        Sobel 3 x 3 to 16S on every octave
 *   line_lbd/libs/binary_descriptor.cpp:1146-1509        computeLBD over the Sobel maps of a key line's octave
 * oracle/pyoracle_octaves.py composes these with lsd_orc_detect's raw segments per octave (LSD of each octave is the one-octave LSD).
 *
 * computeLBD is oracle/lbd_oracle.cpp's own restatement: that file is compiled into this translation unit a second time, its C entry points
 * renamed so that liboracle.so does not define them twice; everything else it defines has internal linkage.
 *
 * PARITY: PINNED to the reference's own class built with (numoctaves, octaveratio) (tests/test_oracle_ref_lsd_octaves.py); pyrDown, the
 * blur and the Sobel maps also to cv2.
 */
#define lbd_orc_keylines_from_lsd lbd_oct_unused_keylines_from_lsd
#define lbd_orc_detect_keylines lbd_oct_unused_detect_keylines
#define lbd_orc_order_keylines lbd_oct_unused_order_keylines
#define lbd_orc_compute lbd_oct_unused_compute
#define lbd_orc_gauss_tables lbd_oct_unused_gauss_tables
#define lbd_orc_pattern_rank lbd_oct_unused_pattern_rank
#define lbd_orc_match lbd_oct_unused_match
#include "lbd_oracle.cpp"
#undef lbd_orc_keylines_from_lsd
#undef lbd_orc_detect_keylines
#undef lbd_orc_order_keylines
#undef lbd_orc_compute
#undef lbd_orc_gauss_tables
#undef lbd_orc_pattern_rank
#undef lbd_orc_match

/* a KeyLine of octave k: lbd_keyline's fields for the points in the input frame, then the in-octave points, the octave (64 bytes) */
struct lbd_keyline_octave {
    lbd_keyline kl;
    float s_oct_x, s_oct_y, e_oct_x, e_oct_y;
    int32_t octave, pad_;
};

/* cv::pyrDown(src, dst, Size(dw, dh)) on 8 bits: 1 4 6 4 1 in both directions at the even source positions, BORDER_REFLECT_101, one
 * rounding; -1 when |2 dw - w| or |2 dh - h| exceeds 2 (pyrDown's assertion) */
extern "C" int lbd_oct_pyrdown(const uint8_t *src, int w, int h, uint8_t *dst, int dw, int dh)
{
    if (dw <= 0 || dh <= 0 || std::abs(2 * dw - w) > 2 || std::abs(2 * dh - h) > 2) return -1;
    static const int k[5] = {1, 4, 6, 4, 1};
    for (int y = 0; y < dh; y++)
        for (int x = 0; x < dw; x++) {
            int a = 0;
            for (int j = 0; j < 5; j++) {
                int t = 0;
                for (int i = 0; i < 5; i++) t += k[i] * src[(size_t)reflect101(2 * y + j - 2, h) * w + reflect101(2 * x + i - 2, w)];
                a += k[j] * t;
            }
            dst[(size_t)y * dw + x] = (uint8_t)((a + 128) >> 8);
        }
    return 0;
}

/* cv::Sobel(img, dx / dy, CV_16S, 1, 0 / 0, 1, 3) of an 8-bit plane (computeSobel :389-390), no blur */
extern "C" void lbd_oct_sobel_u8(const uint8_t *b, int w, int h, int16_t *dx, int16_t *dy)
{
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            auto px = [&](int yy, int xx) -> int { return b[(size_t)reflect101(yy, h) * w + reflect101(xx, w)]; };
            dx[(size_t)y * w + x] = (int16_t)((px(y - 1, x + 1) + 2 * px(y, x + 1) + px(y + 1, x + 1)) - (px(y - 1, x - 1) + 2 * px(y, x - 1) + px(y + 1, x - 1)));
            dy[(size_t)y * w + x] = (int16_t)((px(y + 1, x - 1) + 2 * px(y + 1, x) + px(y + 1, x + 1)) - (px(y - 1, x - 1) + 2 * px(y - 1, x) + px(y - 1, x + 1)));
        }
}

/* computeLBD + binaryConversion of n key lines over given Sobel maps (the maps of their octave; sx .. ey are the in-octave ends) */
extern "C" void lbd_oct_compute_maps(const int16_t *dx, const int16_t *dy, int w, int h, const lbd_keyline *kl, int n, uint8_t *desc)
{
    double G[kRows], L[kBandWidth * 3];
    gauss_tables(G, L);
    for (int i = 0; i < n; i++) {
        float d[kDesc];
        lbd_one_line(dx, dy, w, h, kl[i], G, L, d);
        for (int comb = 0; comb < 32; comb++) { /* binaryConversion :405-416 */
            const float *f1 = &d[8 * kCombinations[comb][0]], *f2 = &d[8 * kCombinations[comb][1]];
            uint8_t r = 0;
            for (int b = 0; b < 8; b++)
                if (f1[b] > f2[b]) r += (uint8_t)(1 << b);
            desc[(size_t)i * 32 + comb] = r;
        }
    }
}

/* LSDDetector::detect's KeyLine fill (:205-250) for the n raw LSD segments of octave `octave` (ow x oh, octaveScale = pow((float)2, octave))
 * of a w x h frame, in order.  Returns the number kept. */
extern "C" int lbd_oct_keylines(const float *raw, int n, int octave, int ow, int oh, int w, int h, lbd_keyline_octave *out)
{
    const float octaveScale = (float)std::pow(2.0f, octave);
    const float pre_boundary_thre = 10;
    int m = 0;
    for (int k = 0; k < n; k++) {
        float e[4] = {raw[4 * k], raw[4 * k + 1], raw[4 * k + 2], raw[4 * k + 3]};
        if (e[0] < 0) e[0] = 0; /* checkLineExtremes against the octave's size (:75-101) */
        if (e[0] >= ow) e[0] = (float)ow - 1.0f;
        if (e[2] < 0) e[2] = 0;
        if (e[2] >= ow) e[2] = (float)ow - 1.0f;
        if (e[1] < 0) e[1] = 0;
        if (e[1] >= oh) e[1] = (float)oh - 1.0f;
        if (e[3] < 0) e[3] = 0;
        if (e[3] >= oh) e[3] = (float)oh - 1.0f;
        lbd_keyline_octave &o = out[m];
        o.kl.sx = e[0] * octaveScale;
        o.kl.sy = e[1] * octaveScale;
        o.kl.ex = e[2] * octaveScale;
        o.kl.ey = e[3] * octaveScale;
        if (((o.kl.sx < pre_boundary_thre) && (o.kl.ex < pre_boundary_thre)) || ((o.kl.sx > w - pre_boundary_thre) && (o.kl.ex > w - pre_boundary_thre)) ||
            ((o.kl.sy < pre_boundary_thre) && (o.kl.ey < pre_boundary_thre)) || ((o.kl.sy > h - pre_boundary_thre) && (o.kl.ey > h - pre_boundary_thre)))
            continue;
        o.s_oct_x = e[0];
        o.s_oct_y = e[1];
        o.e_oct_x = e[2];
        o.e_oct_y = e[3];
        o.kl.line_length = (float)std::sqrt(std::pow(e[0] - e[2], 2) + std::pow(e[1] - e[3], 2));
        o.kl.num_pixels = line_iterator_count(e[0], e[1], e[2], e[3], ow, oh);
        o.kl.angle = std::atan2(o.kl.ey - o.kl.sy, o.kl.ex - o.kl.sx); /* atan2f: see lbd_oracle.cpp's header */
        o.kl.class_id = m;
        o.octave = octave;
        o.pad_ = 0;
        o.kl.size = (o.kl.ex - o.kl.sx) * (o.kl.ey - o.kl.sy);
        o.kl.response = o.kl.line_length / std::max(ow, oh);
        m++;
    }
    return m;
}
