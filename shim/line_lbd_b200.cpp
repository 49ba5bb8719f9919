/*
 * shim/line_lbd_b200.cpp -- class line_lbd_detect (line_lbd/include/line_lbd/line_lbd_allclass.h:22-70;
 * line_lbd/class/line_lbd_allclass.cpp:110-356) on libcubeslam_b200.so: the detection members (detect_raw_lines, detect_filter_lines) and
 * the descriptor / matcher members (get_line_descriptors, detect_descrip_lines x 2, detect_descrip_lines_octaves, match_line_descrip).  In the
 * reference's line_lbd package, compile this file and drop the definitions of the same member functions from line_lbd_allclass.cpp (the
 * constructor, filter_lines, keylines_to_mat / mat_to_keylines stay).  Callers: object_slam/src/main_obj.cpp:363-366,428 and
 * line_lbd/src/detect_lines.cpp:60-69, unchanged.
 *
 * Guarded like detect_3d_cuboid_b200.cpp: an empty translation unit where OpenCV's C++ headers are absent.
 */
#if defined(__has_include)
#if __has_include(<opencv2/core/core.hpp>) && __has_include("line_lbd/line_lbd_allclass.h")
#define CS_SHIM_ENABLED 1
#endif
#endif

#ifdef CS_SHIM_ENABLED
#include <cmath>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "cube_slam_b200.h"
#include "line_lbd/line_lbd_allclass.h"

namespace {
struct CtxTable { /* one context per detector object, see detect_3d_cuboid_b200.cpp */
    std::mutex mu;
    std::unordered_map<const line_lbd_detect *, cs_ctx *> map;
    cs_ctx *get(const line_lbd_detect *self)
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = map.find(self);
        if (it != map.end()) return it->second;
        cs_ctx *c = cs_create(0, 2048, 2048, 1, 64, 8192);
        if (!c) throw std::runtime_error("cube_slam_b200: cs_create failed (no CUDA device?)");
        map.emplace(self, c);
        return c;
    }
};
CtxTable &table()
{
    static CtxTable t;
    return t;
}

/* n x 4 float [x1 y1 x2 y2], with or without the length filter (line_length_thres = 0 keeps every octave-0 segment) */
void run(line_lbd_detect *self, const cv::Mat &gray_img, float length_thres, std::vector<float> &seg, int32_t &n)
{
    cs_ctx *ctx = table().get(self);
    cs_line_params lp;
    cs_default_line_params(&lp);
    lp.use_LSD = self->use_LSD ? 1 : 0;
    lp.line_length_thres = length_thres;
    lp.numoctaves = self->numoctaves_;
    lp.octaveratio = self->octaveratio_;
    const cv::Mat img = gray_img.isContinuous() ? gray_img : gray_img.clone();
    seg.resize(4 * 8192);
    n = 8192;
    const int rc = cs_detect_lines(ctx, img.data, img.cols, img.rows, (int)img.step, img.channels(), &lp, seg.data(), &n);
    if (rc != CS_OK) throw std::runtime_error(cs_last_error(ctx)); /* LSDDetector throws on bad input too (LSDDetector.cpp:112-113,163-164) */
}

/* what the reference's KeyLine carries for a detected segment (LSDDetector.cpp:205-256): enough for filter_lines / keylines_to_mat */
void to_keylines(const std::vector<float> &seg, int n, std::vector<cv::line_descriptor::KeyLine> &out)
{
    out.clear();
    for (int i = 0; i < n; i++) {
        cv::line_descriptor::KeyLine kl;
        kl.startPointX = kl.sPointInOctaveX = seg[4 * i + 0];
        kl.startPointY = kl.sPointInOctaveY = seg[4 * i + 1];
        kl.endPointX = kl.ePointInOctaveX = seg[4 * i + 2];
        kl.endPointY = kl.ePointInOctaveY = seg[4 * i + 3];
        kl.lineLength = std::sqrt((seg[4 * i] - seg[4 * i + 2]) * (seg[4 * i] - seg[4 * i + 2]) + (seg[4 * i + 1] - seg[4 * i + 3]) * (seg[4 * i + 1] - seg[4 * i + 3]));
        kl.angle = std::atan2(kl.endPointY - kl.startPointY, kl.endPointX - kl.startPointX);
        kl.class_id = i;
        kl.octave = 0;
        kl.size = (kl.endPointX - kl.startPointX) * (kl.endPointY - kl.startPointY);
        kl.response = 0;
        kl.pt = cv::Point2f((kl.endPointX + kl.startPointX) / 2, (kl.endPointY + kl.startPointY) / 2);
        out.push_back(kl);
    }
}
}  // namespace

/* weak: the shim still loads against a build of the library without the octave calls (a host-only build of the descriptor); the
 * multi-octave members then throw */
#pragma weak cs_detect_raw_lines_octaves_batch
#pragma weak cs_detect_descrip_lines_octaves_batch

namespace {
void octaves(line_lbd_detect *self, const cv::Mat &gray_img, std::vector<std::vector<cv::line_descriptor::KeyLine>> &out, std::vector<cv::Mat> *descrips);
}

/* line_lbd_allclass.cpp:125-135.  More octaves (LSD flavour): the key lines of every octave, octave after octave */
void line_lbd_detect::detect_raw_lines(const cv::Mat &gray_img, std::vector<cv::line_descriptor::KeyLine> &keylines_out)
{
    if (numoctaves_ > 1) {
        if (!use_LSD) throw std::runtime_error("cube_slam_b200: detect_raw_lines with more than one octave is provided for the LSD flavour");
        std::vector<std::vector<cv::line_descriptor::KeyLine>> per;
        octaves(this, gray_img, per, nullptr);
        keylines_out.clear();
        for (const auto &o : per) keylines_out.insert(keylines_out.end(), o.begin(), o.end());
        return;
    }
    std::vector<float> seg;
    int32_t n = 0;
    run(this, gray_img, -1.f, seg, n); /* lineLength > -1: every segment */
    to_keylines(seg, n, keylines_out);
}

/* line_lbd_allclass.cpp:150-172: one list per octave.  (The third overload, :174-189 -- detect_raw_lines(gray, lines_mat, downsample_img)
 * -- is written in terms of the first one and stays the reference's source.) */
void line_lbd_detect::detect_raw_lines(const cv::Mat &gray_img, std::vector<std::vector<cv::line_descriptor::KeyLine>> &keyline_octaves)
{
    if (numoctaves_ > 1) {
        if (!use_LSD) throw std::runtime_error("cube_slam_b200: detect_raw_lines with more than one octave is provided for the LSD flavour");
        octaves(this, gray_img, keyline_octaves, nullptr);
        return;
    }
    keyline_octaves.assign(1, std::vector<cv::line_descriptor::KeyLine>());
    detect_raw_lines(gray_img, keyline_octaves[0]);
}

/* line_lbd_allclass.cpp:216-221 */
void line_lbd_detect::detect_filter_lines(const cv::Mat &gray_img, cv::Mat &linesmat_out)
{
    std::vector<float> seg;
    int32_t n = 0;
    run(this, gray_img, line_length_thres, seg, n);
    linesmat_out.create(n, 4, CV_32FC1);
    if (n) std::memcpy(linesmat_out.data, seg.data(), sizeof(float) * 4 * (size_t)n);
}

void line_lbd_detect::detect_filter_lines(const cv::Mat &gray_img, std::vector<cv::line_descriptor::KeyLine> &keylines_out)
{
    std::vector<float> seg;
    int32_t n = 0;
    run(this, gray_img, line_length_thres, seg, n);
    to_keylines(seg, n, keylines_out);
}

/* ---- descriptors and matching (line_lbd_allclass.cpp:191-198,224-356) ---- */
namespace {
cs_line_params line_params(const line_lbd_detect *self, float length_thres)
{
    cs_line_params lp;
    cs_default_line_params(&lp);
    lp.use_LSD = self->use_LSD ? 1 : 0;
    lp.line_length_thres = length_thres;
    lp.numoctaves = self->numoctaves_;
    lp.octaveratio = self->octaveratio_;
    return lp;
}

void to_keyline(const cs_keyline &k, cv::line_descriptor::KeyLine &kl)
{
    kl.startPointX = kl.sPointInOctaveX = k.start_x;
    kl.startPointY = kl.sPointInOctaveY = k.start_y;
    kl.endPointX = kl.ePointInOctaveX = k.end_x;
    kl.endPointY = kl.ePointInOctaveY = k.end_y;
    kl.angle = k.angle;
    kl.lineLength = k.line_length;
    kl.response = k.response;
    kl.size = k.size;
    kl.numOfPixels = k.num_pixels;
    kl.class_id = k.class_id;
    kl.octave = 0;
    kl.pt = cv::Point2f((k.end_x + k.start_x) / 2, (k.end_y + k.start_y) / 2);
}

/* detect + describe + length filter on the device: key lines and the n x 32 CV_8UC1 descriptor matrix */
void detect_descrip(line_lbd_detect *self, const cv::Mat &gray_img, float length_thres, std::vector<cs_keyline> &kls, cv::Mat &descrips)
{
    cs_ctx *ctx = table().get(self);
    const cs_line_params lp = line_params(self, length_thres);
    const cv::Mat img = gray_img.isContinuous() ? gray_img : gray_img.clone();
    int32_t n = 8192;
    kls.resize((size_t)n);
    std::vector<uint8_t> desc((size_t)n * 32);
    const int rc = cs_detect_descrip_lines(ctx, img.data, img.cols, img.rows, (int)img.step, img.channels(), &lp, kls.data(), desc.data(), &n);
    if (rc != CS_OK) throw std::runtime_error(cs_last_error(ctx));
    kls.resize((size_t)n);
    descrips = cv::Mat();
    if (n) {
        descrips.create(n, 32, CV_8UC1);
        std::memcpy(descrips.data, desc.data(), (size_t)n * 32);
    }
}

/* every octave of a multi-octave LSD detector (cs_detect_raw_lines_octaves_batch / cs_detect_descrip_lines_octaves_batch, one frame):
 * one list per octave with every KeyLine field, and with `descrips` one descriptor matrix per octave.  A ratio pyrDown refuses throws, as
 * the reference's pyrDown does. */
void octaves(line_lbd_detect *self, const cv::Mat &gray_img, std::vector<std::vector<cv::line_descriptor::KeyLine>> &out, std::vector<cv::Mat> *descrips)
{
    if (!cs_detect_raw_lines_octaves_batch || !cs_detect_descrip_lines_octaves_batch)
        throw std::runtime_error("cube_slam_b200: the loaded library has no octave calls");
    cs_ctx *ctx = table().get(self);
    const cs_line_params lp = line_params(self, self->line_length_thres);
    const cv::Mat img = gray_img.isContinuous() ? gray_img : gray_img.clone();
    const int K = self->numoctaves_, cap = 8192;
    std::vector<cs_keyline_octave> kls((size_t)K * cap);
    std::vector<uint8_t> desc(descrips ? (size_t)K * cap * 32 : 0);
    std::vector<int32_t> n((size_t)K);
    const int rc = descrips ? cs_detect_descrip_lines_octaves_batch(ctx, img.data, 1, img.cols, img.rows, (int)img.step, img.channels(), &lp, kls.data(),
                                                                    desc.data(), cap, n.data())
                            : cs_detect_raw_lines_octaves_batch(ctx, img.data, 1, img.cols, img.rows, (int)img.step, img.channels(), &lp, kls.data(), cap,
                                                                n.data());
    if (rc != CS_OK) throw std::runtime_error(cs_last_error(ctx));
    out.assign((size_t)K, std::vector<cv::line_descriptor::KeyLine>());
    if (descrips) descrips->assign((size_t)K, cv::Mat());
    for (int k = 0; k < K; k++) {
        out[k].resize((size_t)n[k]);
        for (int i = 0; i < n[k]; i++) {
            const cs_keyline_octave &o = kls[(size_t)k * cap + i];
            cv::line_descriptor::KeyLine &kl = out[k][i];
            to_keyline(o.kl, kl);
            kl.sPointInOctaveX = o.s_oct_x;
            kl.sPointInOctaveY = o.s_oct_y;
            kl.ePointInOctaveX = o.e_oct_x;
            kl.ePointInOctaveY = o.e_oct_y;
            kl.octave = o.octave;
        }
        if (descrips && n[k]) {
            (*descrips)[k].create(n[k], 32, CV_8UC1);
            std::memcpy((*descrips)[k].data, &desc[(size_t)k * cap * 32], (size_t)n[k] * 32);
        }
    }
}
}  // namespace

/* :191-198.  The reference goes through mat_to_keylines (:68-108), which reads KeyLine fields before setting them and returns key lines
 * without class_id / octave: undefined there.  Here the key lines of the given rows are filled as LSDDetector fills them. */
void line_lbd_detect::get_line_descriptors(const cv::Mat &gray_img, const cv::Mat &linesmat_src, cv::Mat &line_descrips)
{
    cs_ctx *ctx = table().get(this);
    const cv::Mat img = gray_img.isContinuous() ? gray_img : gray_img.clone();
    const cv::Mat rows = linesmat_src.isContinuous() ? linesmat_src : linesmat_src.clone();
    const int n = rows.rows;
    if (n == 0) return; /* "Error: keypoint list is empty" (binary_descriptor.cpp:622-626) */
    std::vector<cs_keyline> kls((size_t)n);
    if (cs_keylines_from_lines((const float *)rows.data, n, img.cols, img.rows, kls.data()) != CS_OK) throw std::runtime_error("cs_keylines_from_lines failed");
    line_descrips.create(n, 32, CV_8UC1);
    const int rc = cs_lbd_compute(ctx, img.data, img.cols, img.rows, (int)img.step, img.channels(), kls.data(), n, line_descrips.data, nullptr);
    if (rc != CS_OK) throw std::runtime_error(cs_last_error(ctx));
}

/* :224-250: every octave-0 line, no length filter */
void line_lbd_detect::detect_descrip_lines(const cv::Mat &gray_img, cv::Mat &lines_mat, cv::Mat &line_descrips)
{
    std::vector<cs_keyline> kls;
    detect_descrip(this, gray_img, -1.f, kls, line_descrips);
    lines_mat.create((int)kls.size(), 4, CV_32FC1);
    for (size_t i = 0; i < kls.size(); i++) {
        float *r = (float *)lines_mat.data + 4 * i;
        r[0] = kls[i].start_x;
        r[1] = kls[i].start_y;
        r[2] = kls[i].end_x;
        r[3] = kls[i].end_y;
    }
}

/* :253-272 */
void line_lbd_detect::detect_descrip_lines(const cv::Mat &gray_img, std::vector<cv::line_descriptor::KeyLine> &keylines_out, cv::Mat &line_descrips)
{
    std::vector<cs_keyline> kls;
    detect_descrip(this, gray_img, line_length_thres, kls, line_descrips);
    keylines_out.resize(kls.size());
    for (size_t i = 0; i < kls.size(); i++) to_keyline(kls[i], keylines_out[i]);
}

/* :285-339.  One octave: lineLength * 1 > line_length_thres, start x <= end x (ends swapped, the angle folded by normalize_to_PI,
 * :272-281), class_id = position.  More octaves (LSD flavour): every octave from cs_detect_descrip_lines_octaves_batch */
void line_lbd_detect::detect_descrip_lines_octaves(const cv::Mat &gray_img, std::vector<std::vector<cv::line_descriptor::KeyLine>> &keylines_out,
                                                   std::vector<cv::Mat> &line_descrips)
{
    if (numoctaves_ > 1) {
        if (!use_LSD) throw std::runtime_error("cube_slam_b200: detect_descrip_lines_octaves with more than one octave is provided for the LSD flavour");
        octaves(this, gray_img, keylines_out, &line_descrips);
        return;
    }
    keylines_out.assign((size_t)numoctaves_, std::vector<cv::line_descriptor::KeyLine>());
    line_descrips.assign((size_t)numoctaves_, cv::Mat());
    if (numoctaves_ < 1) return;
    std::vector<cs_keyline> kls;
    detect_descrip(this, gray_img, line_length_thres, kls, line_descrips[0]);
    keylines_out[0].resize(kls.size());
    const double PI_ = 3.14159265; /* line_lbd_allclass.cpp:19 */
    for (size_t i = 0; i < kls.size(); i++) {
        cv::line_descriptor::KeyLine &kl = keylines_out[0][i];
        to_keyline(kls[i], kl);
        if (kl.startPointX > kl.endPointX) {
            std::swap(kl.startPointX, kl.endPointX);
            std::swap(kl.startPointY, kl.endPointY);
            std::swap(kl.sPointInOctaveX, kl.ePointInOctaveX);
            std::swap(kl.sPointInOctaveY, kl.ePointInOctaveY);
            if (kl.angle > PI_ / 2)
                kl.angle = (float)(kl.angle - PI_);
            else if (kl.angle < -PI_ / 2)
                kl.angle = (float)(kl.angle + PI_);
        }
        kl.class_id = (int)i;
    }
}

/* :341-356 */
void line_lbd_detect::match_line_descrip(const cv::Mat &descrips_query, const cv::Mat &descrips_train, std::vector<cv::DMatch> &good_matches,
                                         float matching_dist_thres)
{
    good_matches.clear();
    if (descrips_query.rows == 0 || descrips_train.rows == 0) return; /* "descriptors matrices cannot be void" */
    cs_ctx *ctx = table().get(this);
    const cv::Mat q = descrips_query.isContinuous() ? descrips_query : descrips_query.clone();
    const cv::Mat t = descrips_train.isContinuous() ? descrips_train : descrips_train.clone();
    std::vector<cs_dmatch> m((size_t)q.rows);
    int32_t n = 0;
    const int rc = cs_match_line_descrip(ctx, q.data, q.rows, t.data, t.rows, matching_dist_thres, m.data(), &n);
    if (rc != CS_OK) throw std::runtime_error(cs_last_error(ctx));
    for (int i = 0; i < n; i++) good_matches.push_back(cv::DMatch(m[i].query_idx, m[i].train_idx, m[i].img_idx, m[i].distance));
}
#endif /* CS_SHIM_ENABLED */
