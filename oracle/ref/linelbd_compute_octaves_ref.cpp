/*
 * oracle/ref/linelbd_compute_octaves_ref.cpp -- CPU ORACLE, TEST INFRASTRUCTURE ONLY: the reference's own BinaryDescriptor::compute on key
 * lines of any octave that the caller gives.
 *
 * The same translation unit as oracle/ref/linelbd_octaves_ref.cpp -- the reference's lsd.cpp, LSDDetector.cpp, binary_descriptor.cpp,
 * line_lbd_allclass.cpp and binary_descriptor_matcher.cpp included from where they lie under /root/reference, against oracle/ref/minicv.hpp in
 * place of OpenCV -- with one entry point of its own.  No reference source is copied.  Built on demand by oracle/pyoracle_compute_octaves.py
 * (build_ref) into oracle/_ref/liblinelbd_compute_octaves_ref.so where the reference checkout exists.
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

/* BinaryDescriptor::compute(image, keylines, descriptors, returnFloatDescr) (binary_descriptor.cpp:587-790) of the reference's own
 * BinaryDescriptor, built as line_lbd_detect builds it (default parameters: reductionRatio 2), on the caller's n key lines in their order:
 * desc32 n x 32 bytes, and desc72 n x 72 floats from a second call with returnFloatDescr when desc72 is not NULL.  The rows the reference does
 * not write (all but the first row of a repeated (class_id, octave) pair) hold whatever its output matrix held.  Returns 0, -2 for an output
 * matrix of an unexpected shape, or -1 with the exception's message in err (err_cap bytes). */
extern "C" int ref_lbd_compute_octaves(const uint8_t *img, int w, int h, int channels, const ref_keyline_octave *kl, int n, uint8_t *desc32,
                                       float *desc72, char *err, int err_cap)
{
    try {
        Ptr<BinaryDescriptor> lbd = BinaryDescriptor::createBinaryDescriptor();
        cv::Mat image(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(image.data, img, (size_t)w * h * channels);
        std::vector<KeyLine> kls((size_t)n);
        for (int i = 0; i < n; i++) {
            KeyLine &k = kls[i];
            const ref_keyline_octave &o = kl[i];
            k.startPointX = o.sx;
            k.startPointY = o.sy;
            k.endPointX = o.ex;
            k.endPointY = o.ey;
            k.pt = cv::Point2f((o.sx + o.ex) / 2, (o.sy + o.ey) / 2);
            k.angle = o.angle;
            k.lineLength = o.line_length;
            k.response = o.response;
            k.size = o.size;
            k.numOfPixels = o.num_pixels;
            k.class_id = o.class_id;
            k.sPointInOctaveX = o.s_oct_x;
            k.sPointInOctaveY = o.s_oct_y;
            k.ePointInOctaveX = o.e_oct_x;
            k.ePointInOctaveY = o.e_oct_y;
            k.octave = o.octave;
        }
        for (int want_float = 0; want_float < (desc72 ? 2 : 1); want_float++) {
            cv::Mat d;
            lbd->compute(image, kls, d, want_float != 0);
            if (n == 0) continue; /* "keypoint list is empty": the reference returns without touching d */
            if (d.rows != n || d.cols != (want_float ? 72 : 32)) return -2;
            if (want_float)
                std::memcpy(desc72, d.ptr<float>(0), (size_t)n * 72 * sizeof(float));
            else
                std::memcpy(desc32, d.ptr(0), (size_t)n * 32);
        }
        return 0;
    } catch (const std::exception &e) {
        if (err && err_cap > 0) snprintf(err, (size_t)err_cap, "%s", e.what());
        return -1;
    }
}
