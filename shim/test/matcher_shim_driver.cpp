/*
 * shim/test/matcher_shim_driver.cpp -- TEST HARNESS for shim/binary_descriptor_matcher_b200.cpp (not product code).
 *
 * Linked with the shim in place of the reference's libs/binary_descriptor_matcher.cpp, next to the reference's other line_lbd sources
 * (lsd.cpp, LSDDetector.cpp, binary_descriptor.cpp, class/line_lbd_allclass.cpp) compiled as they are: the reference's line_lbd library with
 * the one file swapped, as a maintainer builds it.  cv::Mat is oracle/ref/minicv.hpp (this image has no OpenCV C++ headers).  The entry
 * points below build matchers and call their members the way a user does -- by hand, or as line_lbd_detect's bdm -- and flatten the
 * DMatch lists for ctypes.  Built by shim/test/Makefile into oracle/_ref/libshim_matcher.so; tests/test_gpu_matcher_shim.py loads it.
 */
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <iostream>
#include <new>
#include <stdexcept>
#include <thread>
#include <vector>

#include "line_lbd/line_lbd_allclass.h"

using cv::line_descriptor::BinaryDescriptorMatcher;

namespace {
cv::Mat codes_mat(const uint8_t *codes, int n)
{
    cv::Mat m(n, 32, CV_8UC1);
    if (n) std::memcpy(m.data, codes, (size_t)n * 32);
    return m;
}

/* mask i: shapes[2i] x shapes[2i+1] bytes, the masks back to back in `bytes` */
std::vector<cv::Mat> masks_of(const uint8_t *bytes, const int32_t *shapes, int n_masks)
{
    std::vector<cv::Mat> out;
    size_t at = 0;
    for (int i = 0; i < n_masks; i++) {
        cv::Mat m(shapes[2 * i], shapes[2 * i + 1], CV_8UC1);
        const size_t n = (size_t)shapes[2 * i] * shapes[2 * i + 1];
        if (n) std::memcpy(m.data, bytes + at, n);
        at += n;
        out.push_back(m);
    }
    return out;
}

const cv::DMatch kSentinel(-7, -7, -7, -7.f);

bool is_sentinel(const cv::DMatch &m)
{
    return m.queryIdx == kSentinel.queryIdx && m.trainIdx == kSentinel.trainIdx && m.imgIdx == kSentinel.imgIdx && m.distance == kSentinel.distance;
}

/* lists -> list_len[l] entries of (query_idx, train_idx, img_idx, distance), l after l.  Returns the number of lists, -2 out of room. */
int flatten(const std::vector<std::vector<cv::DMatch>> &lists, size_t first, int32_t *list_len, int32_t *qi, int32_t *ti, int32_t *ii, float *d, int cap_lists,
            int64_t cap)
{
    int64_t n = 0;
    for (size_t l = first; l < lists.size(); l++) {
        if ((int)(l - first) >= cap_lists) return -2;
        list_len[l - first] = (int32_t)lists[l].size();
        for (const cv::DMatch &m : lists[l]) {
            if (n >= cap) return -2;
            qi[n] = m.queryIdx;
            ti[n] = m.trainIdx;
            ii[n] = m.imgIdx;
            d[n++] = m.distance;
        }
    }
    return (int)(lists.size() - first);
}

/* One query of matcher m.  kind 0 match, 1 knnMatch(k), 2 radiusMatch(max_distance); with train (n_train rows) the pairwise form and mask
 * 0 if n_masks, else the collection form with the n_masks masks.  `matches` holds one entry (match) or one list (knn / radius) before the
 * call, so that the call is seen to append to it.  match returns each DMatch as a list of one. */
int query(BinaryDescriptorMatcher *m, int kind, const uint8_t *q, int nq, const uint8_t *train, int n_train, int k, float max_distance, const uint8_t *mask_bytes,
          const int32_t *mask_shapes, int n_masks, int compact, int32_t *list_len, int32_t *qi, int32_t *ti, int32_t *ii, float *d, int cap_lists, int64_t cap)
{
    const cv::Mat mq = codes_mat(q, nq);
    const std::vector<cv::Mat> masks = masks_of(mask_bytes, mask_shapes, n_masks);
    std::vector<std::vector<cv::DMatch>> lists;
    if (kind == 0) {
        std::vector<cv::DMatch> ms(1, kSentinel);
        if (train)
            m->match(mq, codes_mat(train, n_train), ms, n_masks ? masks[0] : cv::Mat());
        else
            m->match(mq, ms, masks);
        if (ms.empty() || !is_sentinel(ms[0])) return -4;
        lists.push_back({});
        for (size_t i = 1; i < ms.size(); i++) lists.push_back({ms[i]});
    } else {
        lists.assign(1, std::vector<cv::DMatch>(1, kSentinel));
        if (kind == 1 && train)
            m->knnMatch(mq, codes_mat(train, n_train), lists, k, n_masks ? masks[0] : cv::Mat(), compact != 0);
        else if (kind == 1)
            m->knnMatch(mq, lists, k, masks, compact != 0);
        else if (train)
            m->radiusMatch(mq, codes_mat(train, n_train), lists, max_distance, n_masks ? masks[0] : cv::Mat(), compact != 0);
        else
            m->radiusMatch(mq, lists, max_distance, masks, compact != 0);
        if (lists.empty() || lists[0].size() != 1 || !is_sentinel(lists[0][0])) return -4;
    }
    return flatten(lists, 1, list_len, qi, ti, ii, d, cap_lists, cap);
}

std::vector<cv::Mat> images_of(const uint8_t *codes, const int32_t *image_offsets, int n_images)
{
    std::vector<cv::Mat> imgs;
    for (int i = 0; i < n_images; i++) imgs.push_back(codes_mat(codes + (size_t)image_offsets[i] * 32, image_offsets[i + 1] - image_offsets[i]));
    return imgs;
}
}  // namespace

#define GUARD(name, body)                                   \
    try {                                                   \
        body                                                \
    } catch (const std::exception &e) {                     \
        fprintf(stderr, "%s: %s\n", name, e.what());        \
        return -1;                                          \
    }

/* the oracle's reference libraries switch std::cout off when they load (oracle/ref/linelbd_ref.cpp); the messages the matcher prints where the
 * reference does are checked with it on */
extern "C" void shim_cout_on() { std::cout.clear(); }

/* a matcher of the user's own */
extern "C" void *shim_bdm_new() { return new BinaryDescriptorMatcher(); }
extern "C" void shim_bdm_free(void *m) { delete (BinaryDescriptorMatcher *)m; }

/* the matcher at m destroyed and a new one constructed at the same address */
extern "C" void shim_bdm_recreate(void *m)
{
    ((BinaryDescriptorMatcher *)m)->~BinaryDescriptorMatcher();
    new (m) BinaryDescriptorMatcher();
}

/* a line_lbd_detect made by the reference's constructor (line_lbd_allclass.cpp:110-123), and its bdm */
extern "C" void *shim_detector_new() { return new line_lbd_detect(1, 2.0f); }
extern "C" void shim_detector_free(void *det) { delete (line_lbd_detect *)det; }
extern "C" void *shim_detector_bdm(void *det) { return ((line_lbd_detect *)det)->bdm.get(); }

/* the reference's line_lbd_detect::match_line_descrip (:341-356) over the shim's pairwise match */
extern "C" int shim_detector_match_line_descrip(void *det, const uint8_t *q, int nq, const uint8_t *t, int nt, float thres, int32_t *qi, int32_t *ti, int32_t *ii,
                                                float *d)
{
    GUARD("shim_detector_match_line_descrip", {
        std::vector<cv::DMatch> good;
        ((line_lbd_detect *)det)->match_line_descrip(codes_mat(q, nq), codes_mat(t, nt), good, thres);
        for (size_t i = 0; i < good.size(); i++) {
            qi[i] = good[i].queryIdx;
            ti[i] = good[i].trainIdx;
            ii[i] = good[i].imgIdx;
            d[i] = good[i].distance;
        }
        return (int)good.size();
    })
}

/* add(images): codes / image_offsets (n_images + 1) hold the images' rows back to back */
extern "C" int shim_bdm_add(void *m, const uint8_t *codes, const int32_t *image_offsets, int n_images)
{
    GUARD("shim_bdm_add", {
        ((BinaryDescriptorMatcher *)m)->add(images_of(codes, image_offsets, n_images));
        return 0;
    })
}

extern "C" int shim_bdm_train(void *m) { GUARD("shim_bdm_train", { ((BinaryDescriptorMatcher *)m)->train(); return 0; }) }
extern "C" int shim_bdm_clear(void *m) { GUARD("shim_bdm_clear", { ((BinaryDescriptorMatcher *)m)->clear(); return 0; }) }

/* one query (see query() above); -1 exception (message on stderr), -2 out of room, -4 the call did not append */
extern "C" int shim_bdm_query(void *m, int kind, const uint8_t *q, int nq, const uint8_t *train, int n_train, int k, float max_distance, const uint8_t *mask_bytes,
                              const int32_t *mask_shapes, int n_masks, int compact, int32_t *list_len, int32_t *qi, int32_t *ti, int32_t *ii, float *d, int cap_lists,
                              int64_t cap)
{
    GUARD("shim_bdm_query", {
        return query((BinaryDescriptorMatcher *)m, kind, q, nq, train, n_train, k, max_distance, mask_bytes, mask_shapes, n_masks, compact, list_len, qi, ti, ii, d,
                     cap_lists, cap);
    })
}

/* a descriptor matrix that is not n x 32 bytes: which 0 add() of a 4 x 16 image, 1 pairwise knnMatch against a 4 x 16 train matrix, 2 a
 * collection knnMatch of a 4 x 64 query.  Returns 1 when the member threw std::invalid_argument, 0 when it did not throw, -1 otherwise. */
extern "C" int shim_bdm_wrong_shape(void *p, int which)
{
    BinaryDescriptorMatcher *m = (BinaryDescriptorMatcher *)p;
    const cv::Mat q(4, 32, CV_8UC1), narrow(4, 16, CV_8UC1), wide(4, 64, CV_8UC1);
    std::vector<std::vector<cv::DMatch>> lists;
    try {
        if (which == 0) m->add({narrow});
        if (which == 1) m->knnMatch(q, narrow, lists, 1);
        if (which == 2) m->knnMatch(wide, lists, 1);
        return 0;
    } catch (const std::invalid_argument &) {
        return 1;
    } catch (const std::exception &) {
        return -1;
    }
}

/* n_threads host threads at once, each with a matcher of its own: add(images), knnMatch(q, k) against the collection and knnMatch(q, train =
 * all codes, k) pairwise, then (clear_after) clear().  Thread t writes its two answers at list slots 2t, 2t + 1 of cap_lists each and entry
 * slots of cap each; n_lists[2t + j] is the number of lists or a negative code. */
extern "C" int shim_bdm_threads(int n_threads, const uint8_t *codes, const int32_t *image_offsets, int n_images, const uint8_t *q, int nq, int k, int clear_after,
                                int32_t *n_lists, int32_t *list_len, int32_t *qi, int32_t *ti, int32_t *ii, float *d, int cap_lists, int64_t cap)
{
    std::vector<std::thread> ts;
    for (int t = 0; t < n_threads; t++)
        ts.emplace_back([=]() {
            try {
                BinaryDescriptorMatcher m;
                m.add(images_of(codes, image_offsets, n_images));
                for (int j = 0; j < 2; j++) {
                    const size_t s = 2 * (size_t)t + j;
                    n_lists[s] = query(&m, 1, q, nq, j ? codes : nullptr, j ? image_offsets[n_images] : 0, k, 0.f, nullptr, nullptr, 0, 0, list_len + s * cap_lists,
                                       qi + s * cap, ti + s * cap, ii + s * cap, d + s * cap, cap_lists, cap);
                }
                if (clear_after) m.clear();
            } catch (const std::exception &e) {
                fprintf(stderr, "shim_bdm_threads: %s\n", e.what());
                n_lists[2 * t] = n_lists[2 * t + 1] = -1;
            }
        });
    for (std::thread &t : ts) t.join();
    return 0;
}
