/*
 * shim/lsd_detector_b200.cpp -- class cv::line_descriptor::LSDDetector (line_lbd/include/line_lbd/line_descriptor/descriptor.hpp:1004-1067;
 * line_lbd/libs/LSDDetector.cpp:49-287) on libcubeslam_b200.so.  In the reference's line_lbd package, compile this file in place of
 * libs/LSDDetector.cpp.  line_lbd_detect's constructor (line_lbd_allclass.cpp:119) then creates this detector as its lsd, so det.lsd->detect
 * and line_lbd_detect's LSD members (detect_raw_lines, detect_filter_lines, detect_descrip_lines_octaves) run LSD on the GPU with the caller's
 * code unchanged.
 *
 * Members: createLSDDetector, the three detect overloads, computeGaussianPyramid and detectImpl.  Every detection goes through
 * cs_detect_raw_lines_octaves_batch, for any numOctaves >= 1 (1 included), so every KeyLine field is filled as LSDDetector.cpp:214-249 fills
 * it: both pairs of end points, lineLength, numOfPixels (cv::LineIterator's count on the octave image), angle, class_id, octave, size,
 * response and pt.  The vector overload groups the images by (cols, rows, channels) and makes one call per group; the pyramid, LSD of every
 * octave and the KeyLine fill run on the device.  gaussianPyrs stays empty (it is private and nothing outside the class reads it);
 * computeGaussianPyramid is defined for the class's sake: it only clears gaussianPyrs, and nothing here calls it.
 *
 * Semantics are the reference's:
 *   - opts.save_octave_line: the flat overload prints "LSD line detector reset save octave lines to False  to match output !!!" on std::cout
 *     when it is true and sets it to false; the per-octave overload prints the "to True" message when it is false and sets it to true; the
 *     vector overload sets it to false, silently, once it reaches its first image.  The other LSDOptions fields are ignored (LSD_REFINE_ADV
 *     and LSD's default parameters, as the reference hard-codes them).
 *   - a mask with data whose size differs from the image's, or whose type is not CV_8UC1, throws std::runtime_error with the reference's
 *     message ("Masks error ..." in the vector overload); an image whose depth is not 8 bits throws "Error, depth image!= 0"; 3-channel
 *     images are BGR and converted to gray as cvtColor does.
 *   - the flat overload APPENDS to `keylines` and never clears it; the per-octave overload replaces the caller's lists by numOctaves new
 *     ones; the vector overload appends image i's lines to keylines[i].
 *   - lines come octave after octave, in LSD's order; class_id counts the kept lines of an octave from 0 before the mask test, so masked
 *     lines leave gaps.
 *   - the mask rule (LSDDetector.cpp:258-286), on the host after detection: a key line is erased when the mask is 0 at both
 *     ((int)startPointY, (int)startPointX) and ((int)endPointY, (int)endPointX).  In the flat and the vector overload the rule runs over the
 *     whole vector it appends to, entries the caller put there included.
 *   - vector overload: the reference checks image i's mask just before it detects image i, so a bad mask (or a bad image) at position i
 *     leaves the lines of images 0 .. i-1 appended and then throws; so does this one (the images before it are detected, appended, then it
 *     throws).
 *   - numOctaves == 1: scale is unused (the reference never calls pyrDown).  numOctaves > 1 with scale != 2 throws std::runtime_error (the
 *     reference's pyrDown asserts |2 * dst - src| <= 2).  numOctaves == 0 detects nothing: the flat overload still runs the mask rule over the
 *     entries already there, the per-octave overload returns no list.  numOctaves < 0 throws std::length_error, the reference's
 *     vector::resize.  These are checked after the mask, channel and depth checks of the same image, in the reference's order.
 * Where the reference's answer is undefined, or where this drop-in's answer differs from it, this one is defined as follows:
 *   - vector overload with keylines.size() < images.size(): keylines is resized up to images.size() first (never shrunk);
 *   - vector overload with masks shorter than images (the default empty vector included): the images without a mask entry are unmasked;
 *   - a key line already in the caller's vector whose truncated end point lies outside the mask: that end point does not count as 0, so
 *     the line is kept unless the other end is inside the mask and 0;
 *   - per-octave overload given a non-empty vector shorter than numOctaves: every list is cleared (the reference indexes past the end);
 *   - images with 4 channels are BGRA and converted as cvtColor's BGR2GRAY converts them (the alpha is ignored); any other channel count
 *     but 1, 3 and 4 throws std::runtime_error (cvtColor throws cv::Exception there);
 *   - a smallest octave with a side of one pixel or less (LSD's 0.8 scaling rounds it below 2 pixels) is refused by the C ABI: this drop-in
 *     throws std::runtime_error with the ABI's message, where the reference returns no line for that octave and the lines of the others.
 * There is no visible cap: a call whose octave holds more LSD segments than the buffer (CS_ERR_CAPACITY) is repeated with a buffer twice as
 * large, so any line count is answered.  Any other failure of the C ABI throws std::runtime_error(cs_last_error).
 *
 * State.  Each host thread gets one small cs_ctx on device 0 (the device shim/line_lbd_b200.cpp uses), created at its first detection and
 * destroyed when the thread ends, following the C ABI's one-context-per-thread rule; every detector used in that thread shares it.
 *
 * Guarded like the other shims: an empty translation unit where OpenCV's C++ headers or the reference's header are absent.
 */
#if defined(__has_include)
#if __has_include(<opencv2/core/core.hpp>) && __has_include("line_lbd/line_descriptor/descriptor.hpp")
#define CS_SHIM_ENABLED 1
#endif
#endif

#ifdef CS_SHIM_ENABLED
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <exception>
#include <iostream>
#include <map>
#include <stdexcept>
#include <tuple>
#include <vector>

#include "cube_slam_b200.h"
#include "line_lbd/line_descriptor/descriptor.hpp"

namespace cv {
namespace line_descriptor {

namespace {
const int kFirstCap = 2048; /* LSD segments per octave the first call has room for; doubled while the ABI answers CS_ERR_CAPACITY */

struct ThreadCtx {
    cs_ctx *ctx = nullptr;
    ~ThreadCtx()
    {
        if (ctx) cs_destroy(ctx);
    }
};
thread_local ThreadCtx thread_ctx_slot;

cs_ctx *thread_ctx()
{
    if (!thread_ctx_slot.ctx) {
        thread_ctx_slot.ctx = cs_create(0, 64, 64, 1, 1, 64); /* the octave calls size their own device buffers: the capacities are not used */
        if (!thread_ctx_slot.ctx) throw std::runtime_error("cube_slam_b200: cs_create failed (no CUDA device?)");
    }
    return thread_ctx_slot.ctx;
}

/* the checks detectImpl and its callers make of one image before LSD runs, in the reference's order: mask, channels, depth, pyrDown's size
 * rule, vector::resize(numOctaves) */
void check_image(const Mat &image, const Mat &mask, int scale, int numOctaves, const char *mask_message)
{
    if (mask.data != NULL && (mask.size() != image.size() || mask.type() != CV_8UC1)) throw std::runtime_error(mask_message);
    const int ch = image.channels();
    if (ch != 1 && ch != 3 && ch != 4)
        throw std::runtime_error("cube_slam_b200: LSDDetector takes gray, BGR or BGRA images (cvtColor BGR2GRAY refuses other channel counts)");
    if (image.depth() != CV_8U) throw std::runtime_error("Error, depth image!= 0");
    if (numOctaves > 1 && scale != 2)
        throw std::runtime_error("cube_slam_b200: LSDDetector with more than one octave needs scale 2 (cv::pyrDown makes an octave of (cols / scale, "
                                 "rows / scale) only when |2 * dst - src| <= 2)");
    if (numOctaves < 0) std::vector<KeyLine>().resize((size_t)numOctaves); /* throws std::length_error, as the reference's resize does */
}

void fill_keyline(const cs_keyline_octave &o, KeyLine &kl)
{
    kl.startPointX = o.kl.start_x;
    kl.startPointY = o.kl.start_y;
    kl.endPointX = o.kl.end_x;
    kl.endPointY = o.kl.end_y;
    kl.sPointInOctaveX = o.s_oct_x;
    kl.sPointInOctaveY = o.s_oct_y;
    kl.ePointInOctaveX = o.e_oct_x;
    kl.ePointInOctaveY = o.e_oct_y;
    kl.lineLength = o.kl.line_length;
    kl.numOfPixels = o.kl.num_pixels;
    kl.angle = o.kl.angle;
    kl.class_id = o.kl.class_id;
    kl.octave = o.octave;
    kl.size = o.kl.size;
    kl.response = o.kl.response;
    kl.pt = Point2f((kl.endPointX + kl.startPointX) / 2, (kl.endPointY + kl.startPointY) / 2);
}

/* mask value at a truncated point; a point outside the mask does not count as 0 */
bool masked_out(const Mat &mask, float x, float y)
{
    if (!(x > -1.f && y > -1.f && x < (float)mask.cols && y < (float)mask.rows)) return false;
    return mask.data[(size_t)(int)y * (size_t)mask.step + (size_t)(int)x] == 0;
}

void apply_mask(const Mat &mask, std::vector<KeyLine> &kls)
{
    if (mask.empty()) return;
    size_t n = 0;
    for (size_t i = 0; i < kls.size(); i++) {
        const KeyLine &kl = kls[i];
        if (masked_out(mask, kl.startPointX, kl.startPointY) && masked_out(mask, kl.endPointX, kl.endPointY)) continue;
        if (n != i) kls[n] = kls[i];
        n++;
    }
    kls.resize(n);
}

/* every octave of n images of one size and channel count: out[i][k] the key lines of image i, octave k (numOctaves >= 1, scale checked) */
void detect_group(const std::vector<const Mat *> &images, int numOctaves, std::vector<std::vector<std::vector<KeyLine>>> &out)
{
    const int n = (int)images.size(), K = numOctaves;
    const Mat &first = *images[0];
    const int w = first.cols, h = first.rows, ch = first.channels() == 1 ? 1 : 3;
    const size_t row = (size_t)w * ch;
    const uint8_t *frames;
    int stride;
    std::vector<uint8_t> packed;
    if (n == 1 && first.channels() == ch) { /* one gray or BGR image: its rows as they lie, whatever the step */
        frames = first.data;
        stride = (int)(size_t)first.step;
    } else {
        packed.resize((size_t)n * h * row);
        for (int i = 0; i < n; i++) {
            const Mat &m = *images[i];
            for (int y = 0; y < h; y++) {
                const uint8_t *src = m.data + (size_t)y * (size_t)m.step;
                uint8_t *dst = &packed[((size_t)i * h + y) * row];
                if (m.channels() == ch)
                    std::memcpy(dst, src, row);
                else /* BGRA: its first three channels */
                    for (int x = 0; x < w; x++) std::memcpy(dst + 3 * x, src + 4 * x, 3);
            }
        }
        frames = packed.data();
        stride = (int)row;
    }
    cs_ctx *ctx = thread_ctx();
    cs_line_params lp;
    cs_default_line_params(&lp);
    lp.use_LSD = 1;
    lp.numoctaves = K;
    lp.octaveratio = K > 1 ? 2.0f : 1.0f;
    std::vector<cs_keyline_octave> kls;
    std::vector<int32_t> cnt((size_t)n * K);
    int64_t cap = kFirstCap;
    for (;;) {
        kls.resize((size_t)n * K * cap);
        const int rc = cs_detect_raw_lines_octaves_batch(ctx, frames, n, w, h, stride, ch, &lp, kls.data(), (int32_t)cap, cnt.data());
        if (rc == CS_OK) break;
        /* LSD finds fewer segments in an octave than it has pixels: past that the error is not a matter of room */
        if (rc == CS_ERR_CAPACITY && cap < (int64_t)w * h && 2 * cap <= INT32_MAX) {
            cap *= 2;
            continue;
        }
        throw std::runtime_error(cs_last_error(ctx));
    }
    out.assign((size_t)n, std::vector<std::vector<KeyLine>>((size_t)K));
    for (int i = 0; i < n; i++)
        for (int k = 0; k < K; k++) {
            const size_t s = (size_t)i * K + k;
            std::vector<KeyLine> &dst = out[i][k];
            dst.resize((size_t)cnt[s]);
            for (int j = 0; j < cnt[s]; j++) fill_keyline(kls[s * cap + j], dst[j]);
        }
}

/* detect every image of `images` (numOctaves >= 0, each image checked), one call per (cols, rows, channels) group: out[i][k] */
void detect_all(const std::vector<const Mat *> &images, int numOctaves, std::vector<std::vector<std::vector<KeyLine>>> &out)
{
    out.assign(images.size(), std::vector<std::vector<KeyLine>>((size_t)std::max(numOctaves, 0)));
    if (numOctaves < 1) return;
    std::map<std::tuple<int, int, int>, std::vector<size_t>> groups; /* (cols, rows, channels) -> image positions, in order */
    for (size_t i = 0; i < images.size(); i++) groups[std::make_tuple(images[i]->cols, images[i]->rows, images[i]->channels())].push_back(i);
    for (const auto &g : groups) {
        std::vector<const Mat *> members;
        for (size_t i : g.second) members.push_back(images[i]);
        std::vector<std::vector<std::vector<KeyLine>>> got;
        detect_group(members, numOctaves, got);
        for (size_t j = 0; j < g.second.size(); j++) out[g.second[j]].swap(got[j]);
    }
}

void append_octaves(std::vector<std::vector<KeyLine>> &octaves, std::vector<KeyLine> &keylines)
{
    for (const std::vector<KeyLine> &o : octaves) keylines.insert(keylines.end(), o.begin(), o.end());
}

const char kMaskMessage[] = "Mask error while detecting lines: please check its dimensions and that data type is CV_8UC1";
const char kMasksMessage[] = "Masks error while detecting lines: please check their dimensions and that data types are CV_8UC1";
}  // namespace

Ptr<LSDDetector> LSDDetector::createLSDDetector() { return Ptr<LSDDetector>(new LSDDetector()); }

/* defined for the class's sake: the detection builds its pyramid on the device and leaves gaussianPyrs empty */
void LSDDetector::computeGaussianPyramid(const Mat &image, int numOctaves, int scale)
{
    (void)image;
    (void)numOctaves;
    (void)scale;
    gaussianPyrs.clear();
}

void LSDDetector::detect(const Mat &image, CV_OUT std::vector<KeyLine> &keylines, int scale, int numOctaves, LSDOptions &opts, const Mat &mask)
{
    if (opts.save_octave_line == true) {
        std::cout << "LSD line detector reset save octave lines to False  to match output !!!" << std::endl;
        opts.save_octave_line = false;
    }
    if (mask.data != NULL && (mask.size() != image.size() || mask.type() != CV_8UC1)) throw std::runtime_error(kMaskMessage);
    std::vector<std::vector<KeyLine>> keyline_octaves;
    detectImpl(image, keylines, keyline_octaves, numOctaves, scale, opts, mask);
}

void LSDDetector::detect(const Mat &image, CV_OUT std::vector<std::vector<KeyLine>> &keyline_octaves, int scale, int numOctaves, LSDOptions &opts,
                         const Mat &mask)
{
    if (opts.save_octave_line == false) {
        std::cout << "LSD line detector reset save octave lines to True to match output !!!" << std::endl;
        opts.save_octave_line = true;
    }
    if (mask.data != NULL && (mask.size() != image.size() || mask.type() != CV_8UC1)) throw std::runtime_error(kMaskMessage);
    std::vector<KeyLine> keylines;
    detectImpl(image, keylines, keyline_octaves, numOctaves, scale, opts, mask);
}

void LSDDetector::detect(const std::vector<Mat> &images, std::vector<std::vector<KeyLine>> &keylines, int scale, int numOctaves, LSDOptions &opts,
                         const std::vector<Mat> &masks)
{
    if (images.empty()) return;
    opts.save_octave_line = false;
    if (keylines.size() < images.size()) keylines.resize(images.size());
    const Mat no_mask;
    auto mask_of = [&](size_t i) -> const Mat & { return i < masks.size() ? masks[i] : no_mask; };
    /* the images the reference detects before it throws: those before the first that fails its checks */
    std::exception_ptr failure;
    size_t n_ok = images.size();
    for (size_t i = 0; i < images.size() && !failure; i++) {
        try {
            check_image(images[i], mask_of(i), scale, numOctaves, kMasksMessage);
        } catch (...) {
            failure = std::current_exception();
            n_ok = i;
        }
    }
    std::vector<const Mat *> ok;
    for (size_t i = 0; i < n_ok; i++) ok.push_back(&images[i]);
    std::vector<std::vector<std::vector<KeyLine>>> found;
    detect_all(ok, numOctaves, found);
    for (size_t i = 0; i < n_ok; i++) {
        append_octaves(found[i], keylines[i]);
        apply_mask(mask_of(i), keylines[i]);
    }
    if (failure) std::rethrow_exception(failure);
}

/* LSDDetector.cpp:153-287 for one image: the flat list (opts.save_octave_line false: appended to keylines) or one list per octave */
void LSDDetector::detectImpl(const Mat &imageSrc, std::vector<KeyLine> &keylines, std::vector<std::vector<KeyLine>> &keyline_octaves, int numOctaves,
                             int scale, const LSDOptions &opts, const Mat &mask) const
{
    check_image(imageSrc, Mat(), scale, numOctaves, kMaskMessage); /* the mask was checked by the caller */
    std::vector<std::vector<std::vector<KeyLine>>> found;
    detect_all(std::vector<const Mat *>(1, &imageSrc), numOctaves, found);
    if (opts.save_octave_line) {
        keyline_octaves.swap(found[0]);
        for (std::vector<KeyLine> &o : keyline_octaves) apply_mask(mask, o);
    } else {
        append_octaves(found[0], keylines);
        apply_mask(mask, keylines);
    }
}

}  // namespace line_descriptor
}  // namespace cv
#endif /* CS_SHIM_ENABLED */
