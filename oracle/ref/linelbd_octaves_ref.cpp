/*
 * oracle/ref/linelbd_octaves_ref.cpp -- CPU ORACLE, TEST INFRASTRUCTURE ONLY: the reference's own class line_lbd_detect built with more than
 * one octave, LSD flavour, every KeyLine field.
 *
 * The same translation unit as oracle/ref/linelbd_ref.cpp -- the reference's lsd.cpp, LSDDetector.cpp, binary_descriptor.cpp and
 * line_lbd_allclass.cpp and binary_descriptor_matcher.cpp (which the class links) included from where they lie under /root/reference, against oracle/ref/minicv.hpp in place of OpenCV -- with one
 * entry point of its own.  No reference source is copied.  Built on demand by oracle/pyoracle_octaves.py (build_ref) into
 * oracle/_ref/liblinelbd_octaves_ref.so where the reference checkout exists.
 */
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <vector>
#include <math.h> /* the float overloads of cos / sin / atan2, as in linelbd_ref.cpp */

#include "/root/reference/line_lbd/libs/lsd.cpp"
#include "/root/reference/line_lbd/libs/LSDDetector.cpp"
#include "/root/reference/line_lbd/libs/binary_descriptor.cpp"
#include "/root/reference/line_lbd/class/line_lbd_allclass.cpp"
#undef MAX_B
#include "/root/reference/line_lbd/libs/binary_descriptor_matcher.cpp"

namespace {
struct SilenceCout { /* the reference reports on std::cout on every call */
    SilenceCout() { std::cout.setstate(std::ios_base::failbit); }
} silence_cout;
}  // namespace

/* cs_keyline_octave's layout: the KeyLine fields of cs_keyline, the in-octave points, the octave */
struct ref_keyline_octave {
    float sx, sy, ex, ey, angle, line_length, response, size;
    int32_t num_pixels, class_id;
    float s_oct_x, s_oct_y, e_oct_x, e_oct_y;
    int32_t octave, pad_;
};

/* line_lbd_detect(numoctaves, octaveratio) with use_LSD: mode 0 detect_raw_lines(image, vector<vector<KeyLine>>&), mode 1
 * detect_raw_lines(image, vector<KeyLine>&) split by KeyLine::octave in list order, mode 2 detect_descrip_lines_octaves (desc_out: one
 * 32-byte row per key line).  Octave k's lines go to kl_out + k * cap, counts[k] of them.  Returns the number of octaves in the answer
 * (-1: exception, message on stderr; -6: a KeyLine::pt that is not the mid point of its ends; -7: more than cap lines in an octave). */
extern "C" int ref_lsd_octaves(const uint8_t *img, int w, int h, int channels, int numoctaves, float octaveratio, float line_length_thres, int mode,
                               ref_keyline_octave *kl_out, uint8_t *desc_out, int32_t *counts, int cap)
{
    try {
        line_lbd_detect det(numoctaves, octaveratio);
        det.use_LSD = true;
        det.line_length_thres = line_length_thres;
        cv::Mat image(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(image.data, img, (size_t)w * h * channels);
        std::vector<std::vector<KeyLine>> kls;
        std::vector<cv::Mat> descs;
        if (mode == 0)
            det.detect_raw_lines(image, kls);
        else if (mode == 1) {
            std::vector<KeyLine> flat;
            det.detect_raw_lines(image, flat);
            for (const KeyLine &k : flat) {
                if (k.octave >= (int)kls.size()) kls.resize(k.octave + 1);
                kls[k.octave].push_back(k);
            }
        } else
            det.detect_descrip_lines_octaves(image, kls, descs);
        for (size_t o = 0; o < kls.size(); o++) {
            const int n = (int)kls[o].size();
            if (n > cap) return -7;
            counts[o] = n;
            for (int i = 0; i < n; i++) {
                const KeyLine &k = kls[o][i];
                if (k.pt.x != (k.endPointX + k.startPointX) / 2 || k.pt.y != (k.endPointY + k.startPointY) / 2) return -6;
                kl_out[o * (size_t)cap + i] = ref_keyline_octave{k.startPointX, k.startPointY, k.endPointX, k.endPointY, k.angle, k.lineLength, k.response,
                                                                 k.size, k.numOfPixels, k.class_id, k.sPointInOctaveX, k.sPointInOctaveY,
                                                                 k.ePointInOctaveX, k.ePointInOctaveY, k.octave, 0};
                if (mode == 2) {
                    if (descs[o].rows != n || descs[o].cols != 32) return -2;
                    std::memcpy(desc_out + (o * (size_t)cap + i) * 32, descs[o].ptr(i), 32);
                }
            }
        }
        return (int)kls.size();
    } catch (const std::exception &e) {
        fprintf(stderr, "ref_lsd_octaves: %s\n", e.what());
        return -1;
    }
}
