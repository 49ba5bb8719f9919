/*
 * shim/test/lsd_detector_shim_driver.cpp -- TEST HARNESS for shim/lsd_detector_b200.cpp (not product code).
 *
 * Compiled twice by shim/test/Makefile, next to the reference's other line_lbd sources (lsd.cpp, binary_descriptor.cpp,
 * binary_descriptor_matcher.cpp, class/line_lbd_allclass.cpp) compiled as they are:
 *   oracle/_ref/libshim_lsd.so           with the shim in place of libs/LSDDetector.cpp (linked to libcubeslam_b200.so), LSDD_VIEWS defined;
 *   oracle/_ref/libref_lsd_detector.so   with the reference's own libs/LSDDetector.cpp: what the shim is compared with.
 * cv::Mat is oracle/ref/minicv.hpp (this image has no OpenCV C++ headers).  The entry points below construct a detector through
 * createLSDDetector, or the reference's line_lbd_detect, and call its members the way a user does; they flatten the KeyLine lists for ctypes.
 * minicv's Mat is always continuous: an ROI (a step wider than the row) is a strided view in the shim's build (LSDD_VIEWS), which reads
 * rows through Mat::step as it does on OpenCV, and a continuous copy of the same pixels in the reference's, which is what cv::Mat::clone of
 * an ROI gives the reference's detectImpl on OpenCV.
 */
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <iostream>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "line_lbd/line_lbd_allclass.h"

using cv::line_descriptor::KeyLine;
using cv::line_descriptor::LSDDetector;

/* one image or mask: rows x cols of `type`, row y at data + y * step (data NULL: an empty Mat) */
struct lsdd_mat {
    const uint8_t *data;
    int32_t rows, cols, type, step;
};

/* every KeyLine field, 17 x 4 bytes */
struct lsdd_rec {
    float sx, sy, ex, ey, angle, line_length, response, size;
    int32_t num_pixels, class_id;
    float s_oct_x, s_oct_y, e_oct_x, e_oct_y;
    int32_t octave;
    float pt_x, pt_y;
};

namespace {
cv::Mat mat_of(const lsdd_mat &d)
{
    if (!d.data) return cv::Mat();
    cv::Mat m(d.rows, d.cols, d.type);
    const size_t row = (size_t)d.cols * m.elemSize();
    if ((size_t)d.step != row) {
#ifdef LSDD_VIEWS
        cv::Mat parent(d.rows, (int)(d.step / m.elemSize()), d.type);
        for (int y = 0; y < d.rows; y++) std::memcpy(parent.data + (size_t)y * d.step, d.data + (size_t)y * d.step, row);
        cv::Mat view = parent;
        view.cols = d.cols;
        return view;
#endif
    }
    for (int y = 0; y < d.rows; y++) std::memcpy(m.data + y * row, d.data + (size_t)y * d.step, row);
    return m;
}

KeyLine keyline_of(const lsdd_rec &r)
{
    KeyLine kl;
    kl.startPointX = r.sx;
    kl.startPointY = r.sy;
    kl.endPointX = r.ex;
    kl.endPointY = r.ey;
    kl.angle = r.angle;
    kl.lineLength = r.line_length;
    kl.response = r.response;
    kl.size = r.size;
    kl.numOfPixels = r.num_pixels;
    kl.class_id = r.class_id;
    kl.sPointInOctaveX = r.s_oct_x;
    kl.sPointInOctaveY = r.s_oct_y;
    kl.ePointInOctaveX = r.e_oct_x;
    kl.ePointInOctaveY = r.e_oct_y;
    kl.octave = r.octave;
    kl.pt = cv::Point2f(r.pt_x, r.pt_y);
    return kl;
}

lsdd_rec rec_of(const KeyLine &k)
{
    return lsdd_rec{k.startPointX, k.startPointY, k.endPointX, k.endPointY, k.angle, k.lineLength, k.response, k.size, k.numOfPixels, k.class_id,
                    k.sPointInOctaveX, k.sPointInOctaveY, k.ePointInOctaveX, k.ePointInOctaveY, k.octave, k.pt.x, k.pt.y};
}

std::vector<std::vector<KeyLine>> lists_of(const int32_t *len, const lsdd_rec *recs, int n_lists)
{
    std::vector<std::vector<KeyLine>> out((size_t)(n_lists > 0 ? n_lists : 0));
    size_t at = 0;
    for (int l = 0; l < n_lists; l++)
        for (int i = 0; i < len[l]; i++) out[l].push_back(keyline_of(recs[at++]));
    return out;
}

/* lists -> list_len[l] records, l after l.  Returns the number of lists, -2 out of room. */
int flatten(const std::vector<std::vector<KeyLine>> &lists, int32_t *list_len, lsdd_rec *recs, int cap_lists, int64_t cap)
{
    if ((int64_t)lists.size() > cap_lists) return -2;
    int64_t n = 0;
    for (size_t l = 0; l < lists.size(); l++) {
        list_len[l] = (int32_t)lists[l].size();
        for (const KeyLine &k : lists[l]) {
            if (n >= cap) return -2;
            recs[n++] = rec_of(k);
        }
    }
    return (int)lists.size();
}

/* the exception the member threw: err_kind 1 std::runtime_error, 2 std::length_error, 3 another std::exception; its what() into err */
void report(const std::exception &e, int kind, int32_t *err_kind, char *err, int err_cap)
{
    *err_kind = kind;
    std::snprintf(err, (size_t)err_cap, "%s", e.what());
}
}  // namespace

/* the oracle's reference libraries switch std::cout off when they load; the messages the detector prints are checked with it on */
extern "C" void lsdd_cout_on() { std::cout.clear(); }

/* sizeof(lsdd_rec), for the test's dtype */
extern "C" int lsdd_rec_size() { return (int)sizeof(lsdd_rec); }

/* One call of a detector made by LSDDetector::createLSDDetector().  member 0: detect(image, vector<KeyLine>&, scale, numOctaves, opts,
 * mask), 1: detect(image, vector<vector<KeyLine>>&, ...), 2: detect(images, vector<vector<KeyLine>>&, ..., masks).  images[0] / masks[0]
 * are the single overloads' image and mask (n_masks 0: the default Mat()); the vector overload gets n_images images and n_masks masks.
 * The output vector starts as the n_pre lists of pre_len / pre (the flat overload: list 0) and is returned the same way, whether or not
 * the member threw.  *flag is opts.save_octave_line in and out.  Returns the number of lists (-2 out of room); *err_kind is 0 when the
 * member returned, else the kind of exception (report above). */
extern "C" int lsdd_detect(int member, const lsdd_mat *images, int n_images, const lsdd_mat *masks, int n_masks, int scale, int num_octaves, int32_t *flag,
                           const int32_t *pre_len, const lsdd_rec *pre, int n_pre, int32_t *list_len, lsdd_rec *recs, int cap_lists, int64_t cap,
                           int32_t *err_kind, char *err, int err_cap)
{
    *err_kind = 0;
    if (err_cap) err[0] = 0;
    cv::Ptr<LSDDetector> lsd = LSDDetector::createLSDDetector();
    LSDDetector::LSDOptions opts;
    opts.save_octave_line = *flag != 0;
    std::vector<cv::Mat> imgs, ms;
    for (int i = 0; i < n_images; i++) imgs.push_back(mat_of(images[i]));
    for (int i = 0; i < n_masks; i++) ms.push_back(mat_of(masks[i]));
    std::vector<std::vector<KeyLine>> lists = lists_of(pre_len, pre, n_pre);
    if (member == 0 && lists.empty()) lists.resize(1);
    try {
        if (member == 0)
            n_masks ? lsd->detect(imgs[0], lists[0], scale, num_octaves, opts, ms[0]) : lsd->detect(imgs[0], lists[0], scale, num_octaves, opts);
        else if (member == 1)
            n_masks ? lsd->detect(imgs[0], lists, scale, num_octaves, opts, ms[0]) : lsd->detect(imgs[0], lists, scale, num_octaves, opts);
        else
            n_masks ? lsd->detect(imgs, lists, scale, num_octaves, opts, ms) : lsd->detect(imgs, lists, scale, num_octaves, opts);
    } catch (const std::length_error &e) {
        report(e, 2, err_kind, err, err_cap);
    } catch (const std::runtime_error &e) {
        report(e, 1, err_kind, err, err_cap);
    } catch (const std::exception &e) {
        report(e, 3, err_kind, err, err_cap);
    }
    *flag = opts.save_octave_line ? 1 : 0;
    return flatten(lists, list_len, recs, cap_lists, cap);
}

/* n_threads host threads at once, thread t running the flat overload over images[t] (its own detector, numOctaves, scale 2) `repeat` times;
 * thread t's lines go to list t.  Returns the number of lists, -2 out of room, -1 when a thread threw (message on stderr). */
extern "C" int lsdd_threads(int n_threads, const lsdd_mat *images, int num_octaves, int repeat, int32_t *list_len, lsdd_rec *recs, int64_t cap)
{
    std::vector<std::vector<KeyLine>> lists((size_t)n_threads);
    std::vector<int> failed((size_t)n_threads, 0);
    std::vector<std::thread> ts;
    for (int t = 0; t < n_threads; t++)
        ts.emplace_back([&, t]() {
            try {
                const cv::Mat img = mat_of(images[t]);
                cv::Ptr<LSDDetector> lsd = LSDDetector::createLSDDetector();
                LSDDetector::LSDOptions opts;
                for (int r = 0; r < repeat; r++) {
                    std::vector<KeyLine> kl;
                    lsd->detect(img, kl, 2, num_octaves, opts);
                    if (r == 0)
                        lists[t] = kl;
                    else if (kl.size() != lists[t].size())
                        throw std::runtime_error("a repeated detection differs");
                }
            } catch (const std::exception &e) {
                std::fprintf(stderr, "lsdd_threads: %s\n", e.what());
                failed[t] = 1;
            }
        });
    for (std::thread &t : ts) t.join();
    for (int f : failed)
        if (f) return -1;
    return flatten(lists, list_len, recs, n_threads, cap);
}

/* The reference's own line_lbd_detect(num_octaves, 2.0) with use_LSD and line_length_thres, member 0 detect_raw_lines(gray, vector<KeyLine>&),
 * 1 detect_raw_lines(gray, vector<vector<KeyLine>>&), 2 detect_filter_lines(gray, vector<KeyLine>&), 3 detect_descrip_lines_octaves (desc:
 * 32 bytes per key line, in list order).  Returns the number of lists, -2 out of room, -1 exception (message on stderr). */
extern "C" int lsdd_line_lbd(int num_octaves, float line_length_thres, int member, const lsdd_mat *image, int32_t *list_len, lsdd_rec *recs, uint8_t *desc,
                             int cap_lists, int64_t cap)
{
    try {
        line_lbd_detect det(num_octaves, 2.0f);
        det.use_LSD = true;
        det.line_length_thres = line_length_thres;
        const cv::Mat img = mat_of(*image);
        std::vector<std::vector<KeyLine>> lists;
        std::vector<cv::Mat> descs;
        if (member == 0 || member == 2) {
            lists.resize(1);
            member == 0 ? det.detect_raw_lines(img, lists[0]) : det.detect_filter_lines(img, lists[0]);
        } else if (member == 1)
            det.detect_raw_lines(img, lists);
        else
            det.detect_descrip_lines_octaves(img, lists, descs);
        const int n = flatten(lists, list_len, recs, cap_lists, cap);
        if (n < 0 || member != 3) return n;
        size_t at = 0;
        for (size_t l = 0; l < lists.size(); l++) {
            if (descs[l].rows != (int)lists[l].size()) throw std::runtime_error("descriptor rows differ from the key lines");
            if (descs[l].rows) std::memcpy(desc + at * 32, descs[l].data, (size_t)descs[l].rows * 32);
            at += (size_t)descs[l].rows;
        }
        return n;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "lsdd_line_lbd: %s\n", e.what());
        return -1;
    }
}
