/*
 * shim/binary_descriptor_matcher_b200.cpp -- class cv::line_descriptor::BinaryDescriptorMatcher (line_lbd/include/line_lbd/line_descriptor/
 * descriptor.hpp:1094-1218; line_lbd/libs/binary_descriptor_matcher.cpp:54-595) on libcubeslam_b200.so.  In the reference's line_lbd package,
 * compile this file in place of libs/binary_descriptor_matcher.cpp.  line_lbd_detect's constructor (line_lbd_allclass.cpp:117) then creates
 * this matcher as its bdm, so det.bdm->knnMatch / radiusMatch / add / train / match and line_lbd_detect::match_line_descrip run on the GPU
 * with the caller's code unchanged.
 *
 * Members: the constructor, createBinaryDescriptorMatcher, add, train, clear, both forms of match, knnMatch and radiusMatch.  Nothing else of
 * the class is reachable from a caller; Mihasher, SparseHashtable, BucketGroup and checkKDistances are not defined, and `dataset` stays null.
 *
 * Semantics are the reference's:
 *   - results are APPENDED to `matches`, which is never cleared, as in the reference;
 *   - an empty query (or, pairwise, train) matrix prints the reference's message on std::cout and returns; so does a pairwise mask the
 *     reference refuses (match / radiusMatch: rows != query rows AND cols != 1; knnMatch: rows != query rows OR cols != 1) and a collection
 *     query given a number of masks other than the number of images added;
 *   - a mask value is mask.at<uchar>(i); compactResult leaves out the lists that end up empty (pairwise knnMatch: the masked queries' lists);
 *   - add() keeps the codes on the host and records each image's first row as the reference does (an empty image owns the rows of the images
 *     that start where it does, and its mask is the one consulted for them); train() uploads what add() kept to the matcher's device
 *     collection; every collection query calls train() first, as the reference does, so it searches every image added since construction or
 *     clear(); clear() forgets the images and frees the collection's device memory;
 *   - collection forms: trainIdx is the row over all images added, imgIdx the image as add() recorded it.  A per-image mask of the wrong shape
 *     makes match skip that image's matches silently, and knnMatch / radiusMatch print the reference's message and return with the lists
 *     completed before the first entry of that image.
 * Where the reference's result is undefined, the C ABI's documented answer is returned (include/cube_slam_b200.h, above
 * cs_knn_match_line_descrip and cs_lbd_collection_create):
 *   - only codes the multi-index hash meets count (a code none of whose 32 bytes is within 4 bits of the query's is never met): a query gets
 *     fewer than k entries, or no match at all, where the reference returns uninitialised entries or reads past a vector;
 *   - an entry further than 128 bits away has trainIdx -1 (collection forms: imgIdx -1 too, and it is dropped when masks are given);
 *   - k = 0 gives empty lists; k < 0 throws std::invalid_argument (the reference's new[] of a negative size throws too);
 *   - a collection query with no code added gives no entries;
 *   - a pairwise mask that passes the reference's check but holds fewer bytes than there are queries is refused like one that fails it.
 * Descriptor matrices must be n x 32 CV_8UC1 (the binary LBD codes); any other non-empty matrix throws std::invalid_argument.
 * The pairwise C ABI calls take at most 16384 train codes (CS_LBD_KNN_MAX_TRAIN); a larger pairwise knnMatch / radiusMatch goes through a
 * temporary device collection, which has no cap, and gives the same answer.
 *
 * State.  Each host thread gets one small cs_ctx on device 0 (the device shim/line_lbd_b200.cpp uses), shared by every matcher used in that
 * thread, following the C ABI's one-context-per-thread rule.  Each matcher gets one cs_lbd_collection, created by its first add() on the
 * context of the thread that calls it; the class cannot grow a member, so it lives in a side table keyed by the matcher's address.  The
 * header's destructor is inline and empty (descriptor.hpp:1216-1218), so nothing is freed when a matcher is destroyed -- the reference
 * leaks its `dataset` there too: a destroyed matcher's codes stay on the device until clear() is called on it, a new matcher is constructed
 * at the same address (the constructor drops what a former one left there), or the process exits.  A thread's context outlives the thread
 * while a collection on it still holds codes.
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
#include <cmath>
#include <cstring>
#include <iostream>
#include <mutex>
#include <sstream>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "cube_slam_b200.h"
#include "line_lbd/line_descriptor/descriptor.hpp"

namespace cv {
namespace line_descriptor {

namespace {
const int kMaxPairTrain = 16384; /* CS_LBD_KNN_MAX_TRAIN: the most train codes a pairwise knn / radius call takes */

std::mutex &table_mutex()
{
    static std::mutex m;
    return m;
}

/* the context of one host thread, and how many collections live on it: it is destroyed once its thread has ended and none is left */
struct ThreadCtx {
    cs_ctx *ctx = nullptr;
    int collections = 0;
    bool thread_ended = false;
};

void release_if_unused(ThreadCtx *t) /* under table_mutex */
{
    if (t->thread_ended && t->collections == 0) {
        cs_destroy(t->ctx);
        delete t;
    }
}

struct ThreadSlot {
    ThreadCtx *t = nullptr;
    ~ThreadSlot()
    {
        if (!t) return;
        std::lock_guard<std::mutex> g(table_mutex());
        t->thread_ended = true;
        release_if_unused(t);
    }
};
thread_local ThreadSlot thread_slot;

ThreadCtx *thread_ctx()
{
    if (!thread_slot.t) {
        cs_ctx *c = cs_create(0, 64, 64, 1, 1, 64); /* matching allocates its own device buffers on demand: the capacities are not used */
        if (!c) throw std::runtime_error("cube_slam_b200: cs_create failed (no CUDA device?)");
        thread_slot.t = new ThreadCtx;
        thread_slot.t->ctx = c;
    }
    return thread_slot.t;
}

/* what a matcher holds besides the class's own members */
struct State {
    std::vector<uint8_t> pending;          /* codes add() kept and train() has not uploaded yet (the reference's descriptorsMat) */
    std::vector<int32_t> pending_off{0};   /* their images, as offsets into `pending` */
    cs_lbd_collection *coll = nullptr;
    ThreadCtx *owner = nullptr;            /* the context coll was created on */
};

std::unordered_map<const BinaryDescriptorMatcher *, State> &table()
{
    static std::unordered_map<const BinaryDescriptorMatcher *, State> t;
    return t;
}

State &state_of(const BinaryDescriptorMatcher *m) /* entries are nodes: the reference stays valid while others are added or erased */
{
    std::lock_guard<std::mutex> g(table_mutex());
    return table()[m];
}

void forget(const BinaryDescriptorMatcher *m)
{
    std::lock_guard<std::mutex> g(table_mutex());
    auto it = table().find(m);
    if (it == table().end()) return;
    State &s = it->second;
    if (s.coll) {
        cs_lbd_collection_destroy(s.coll);
        s.owner->collections--;
        release_if_unused(s.owner);
    }
    table().erase(it);
}

void check(cs_ctx *c, int rc)
{
    if (rc != CS_OK) throw std::runtime_error(std::string("cube_slam_b200: ") + cs_last_error(c));
}

/* an n x 32 CV_8UC1 matrix as the C ABI takes it, rows back to back */
Mat codes_of(const Mat &d, const char *what)
{
    if (d.type() != CV_8UC1 || d.cols != 32) {
        std::ostringstream ss;
        ss << "BinaryDescriptorMatcher: " << what << " must be n x 32 CV_8UC1 binary descriptors, got " << d.rows << " x " << d.cols << " of type "
           << d.type();
        throw std::invalid_argument(ss.str());
    }
    return d.isContinuous() ? d : d.clone();
}

void check_k(int k)
{
    if (k < 0) throw std::invalid_argument("BinaryDescriptorMatcher: k must not be negative");
}

/* mask.at<uchar>(i) != 0 for the n queries; false when the mask holds fewer than n bytes */
bool mask_values(const Mat &mask, int n, std::vector<uint8_t> &out)
{
    const Mat m = mask.isContinuous() ? mask : mask.clone();
    if (m.total() * m.elemSize() < (size_t)n) return false;
    out.resize((size_t)n);
    for (int i = 0; i < n; i++) out[i] = m.data[i] != 0;
    return true;
}

bool wrong_shape(const Mat &mask, int n) { return mask.rows != n || mask.cols != 1; }

DMatch to_dmatch(const cs_dmatch &m, int img_idx) { return DMatch(m.query_idx, m.train_idx, img_idx, m.distance); }

/* the radius protocol of the C ABI: call with room for 8 entries per query, again with the size it reports when they do not fit */
template <typename Call>
void radius_call(cs_ctx *c, int nq, Call call, std::vector<cs_dmatch> &out, std::vector<int64_t> &off)
{
    int64_t cap = 8 * (int64_t)nq;
    off.assign((size_t)nq + 1, 0);
    for (int attempt = 0;; attempt++) {
        out.resize((size_t)std::max<int64_t>(cap, 1));
        const int rc = call(out.data(), cap, off.data());
        if (rc == CS_ERR_CAPACITY && attempt == 0 && off[nq] > cap) {
            cap = off[nq];
            continue;
        }
        check(c, rc);
        return;
    }
}

/* A pair whose train set exceeds the pairwise calls' cap: one image in a temporary collection.  Its entries are the pairwise answer with
 * imgIdx 0; the query mask is applied here (a masked query has no entries), as the pairwise calls apply it. */
struct TempCollection {
    cs_ctx *ctx;
    cs_lbd_collection *coll;
    TempCollection(cs_ctx *c, const Mat &t) : ctx(c), coll(cs_lbd_collection_create(c))
    {
        if (!coll) throw std::runtime_error("cube_slam_b200: cs_lbd_collection_create failed");
        const int32_t off[2] = {0, t.rows};
        const int rc = cs_lbd_collection_add(coll, t.data, off, 1);
        if (rc != CS_OK) {
            cs_lbd_collection_destroy(coll);
            check(c, rc);
        }
    }
    ~TempCollection() { cs_lbd_collection_destroy(coll); }
};

/* pairwise knn: per query its entries in the hash's order */
std::vector<std::vector<DMatch>> pair_knn(const Mat &q, const Mat &t, int k, const std::vector<uint8_t> &keep)
{
    cs_ctx *c = thread_ctx()->ctx;
    const int nq = q.rows, kk = std::min(k, t.rows); /* no query gets more entries than the train set has codes */
    std::vector<cs_dmatch> out(std::max<size_t>((size_t)nq * kk, 1));
    std::vector<int32_t> n((size_t)nq);
    if (t.rows <= kMaxPairTrain) {
        check(c, cs_knn_match_line_descrip(c, q.data, nq, t.data, t.rows, kk, keep.empty() ? nullptr : keep.data(), out.data(), n.data()));
    } else {
        TempCollection tc(c, t);
        check(c, cs_lbd_collection_knn_match(tc.coll, q.data, nq, kk, nullptr, 0, out.data(), n.data()));
    }
    std::vector<std::vector<DMatch>> lists((size_t)nq);
    for (int i = 0; i < nq; i++)
        if (keep.empty() || keep[i])
            for (int j = 0; j < n[i]; j++) lists[i].push_back(to_dmatch(out[(size_t)i * kk + j], 0));
    return lists;
}

std::vector<std::vector<DMatch>> pair_radius(const Mat &q, const Mat &t, float max_distance, const std::vector<uint8_t> &keep)
{
    cs_ctx *c = thread_ctx()->ctx;
    const int nq = q.rows;
    std::vector<cs_dmatch> out;
    std::vector<int64_t> off;
    if (t.rows <= kMaxPairTrain) {
        radius_call(c, nq, [&](cs_dmatch *m, int64_t cap, int64_t *o) {
            return cs_radius_match_line_descrip(c, q.data, nq, t.data, t.rows, max_distance, keep.empty() ? nullptr : keep.data(), m, cap, o);
        }, out, off);
    } else {
        TempCollection tc(c, t);
        radius_call(c, nq, [&](cs_dmatch *m, int64_t cap, int64_t *o) {
            return cs_lbd_collection_radius_match(tc.coll, q.data, nq, max_distance, nullptr, 0, m, cap, o);
        }, out, off);
    }
    std::vector<std::vector<DMatch>> lists((size_t)nq);
    for (int i = 0; i < nq; i++)
        if (keep.empty() || keep[i])
            for (int64_t j = off[i]; j < off[i + 1]; j++) lists[i].push_back(to_dmatch(out[j], 0));
    return lists;
}

/* The masks of a collection query as the C ABI takes them (n_masks rows of nq bytes), with bad[i] for mask i of the wrong shape: its row
 * keeps every query, and the caller treats that image's entries as the reference does. */
int collection_masks(const std::vector<Mat> &masks, int nq, std::vector<uint8_t> &rows, std::vector<char> &bad)
{
    rows.assign(masks.size() * (size_t)nq, 1);
    bad.assign(masks.size(), 0);
    std::vector<uint8_t> v;
    for (size_t i = 0; i < masks.size(); i++) {
        if (wrong_shape(masks[i], nq)) {
            bad[i] = 1;
            continue;
        }
        mask_values(masks[i], nq, v);
        std::copy(v.begin(), v.end(), rows.begin() + i * (size_t)nq);
    }
    return (int)masks.size();
}

void print_mask_error(int img, const char *fn, int nq)
{
    std::cout << "Error: mask " << img << " in " << fn << " function " << "should have " << nq << " and " << "1 column. Program will be terminated"
              << std::endl;
}
}  // namespace

/* binary_descriptor_matcher.cpp:55-61.  `dataset` stays null: no hash is built on the host. */
BinaryDescriptorMatcher::BinaryDescriptorMatcher()
{
    dataset = 0;
    nextAddedIndex = 0;
    numImages = 0;
    descrInDS = 0;
    forget(this); /* a matcher destroyed at this address left its collection behind: the header's destructor cannot free it */
}

/* :64-67 */
Ptr<BinaryDescriptorMatcher> BinaryDescriptorMatcher::createBinaryDescriptorMatcher()
{
    return Ptr<BinaryDescriptorMatcher>(new BinaryDescriptorMatcher());
}

/* :70-80: the codes stay on the host until train() */
void BinaryDescriptorMatcher::add(const std::vector<Mat> &descriptors)
{
    std::vector<Mat> codes;
    for (const Mat &d : descriptors) codes.push_back(d.rows > 0 ? codes_of(d, "added descriptors") : Mat());
    State &s = state_of(this);
    for (const Mat &c : codes) {
        s.pending.insert(s.pending.end(), c.data, c.data + (size_t)c.rows * 32);
        s.pending_off.push_back(s.pending_off.back() + c.rows);
        indexesMap.insert(std::pair<int, int>(nextAddedIndex, numImages));
        nextAddedIndex += c.rows;
        numImages++;
    }
    if (!s.coll) {
        ThreadCtx *t = thread_ctx();
        s.coll = cs_lbd_collection_create(t->ctx);
        if (!s.coll) throw std::runtime_error("cube_slam_b200: cs_lbd_collection_create failed");
        std::lock_guard<std::mutex> g(table_mutex());
        s.owner = t;
        t->collections++;
    }
}

/* :83-93: what add() kept goes to the device collection */
void BinaryDescriptorMatcher::train()
{
    State &s = state_of(this);
    const int n_images = (int)s.pending_off.size() - 1;
    if (!s.coll || n_images == 0) return;
    check(s.owner->ctx, cs_lbd_collection_add(s.coll, s.pending.empty() ? nullptr : s.pending.data(), s.pending_off.data(), n_images));
    s.pending.clear();
    s.pending_off.assign(1, 0);
    descrInDS = nextAddedIndex;
}

/* :96-104, and the collection's device memory is freed */
void BinaryDescriptorMatcher::clear()
{
    descriptorsMat.release();
    indexesMap.clear();
    dataset = 0;
    nextAddedIndex = 0;
    numImages = 0;
    descrInDS = 0;
    forget(this);
}

/* :126-193 */
void BinaryDescriptorMatcher::match(const Mat &queryDescriptors, std::vector<DMatch> &matches, const std::vector<Mat> &masks)
{
    if (queryDescriptors.rows == 0) {
        std::cout << "Error: query descriptors'matrix is empty" << std::endl;
        return;
    }
    if (masks.size() != 0 && (int)masks.size() != numImages) {
        std::cout << "Error: the number of images in dataset is " << numImages << " but match function received " << masks.size()
                  << " masks. Program will be terminated" << std::endl;
        return;
    }
    const Mat q = codes_of(queryDescriptors, "query descriptors");
    train();
    State &s = state_of(this);
    if (!s.coll) return;
    const int nq = q.rows;
    std::vector<uint8_t> rows;
    std::vector<char> bad;
    const int n_masks = collection_masks(masks, nq, rows, bad);
    std::vector<cs_dmatch> out((size_t)nq);
    int32_t n = 0;
    check(s.owner->ctx, cs_lbd_collection_match(s.coll, q.data, nq, n_masks ? rows.data() : nullptr, n_masks, out.data(), &n));
    for (int i = 0; i < n; i++)
        if (!n_masks || out[i].img_idx < 0 || !bad[out[i].img_idx]) /* a mask of the wrong shape: the match is left out (:165-171) */
            matches.push_back(to_dmatch(out[i], out[i].img_idx));
}

/* :196-261 */
void BinaryDescriptorMatcher::match(const Mat &queryDescriptors, const Mat &trainDescriptors, std::vector<DMatch> &matches, const Mat &mask) const
{
    if (queryDescriptors.rows == 0 || trainDescriptors.rows == 0) {
        std::cout << "Error: descriptors matrices cannot be void" << std::endl;
        return;
    }
    std::vector<uint8_t> keep;
    if (!mask.empty() && ((mask.rows != queryDescriptors.rows && mask.cols != 1) || !mask_values(mask, queryDescriptors.rows, keep))) {
        std::cout << "Error: input mask should have " << queryDescriptors.rows << " rows and 1 column. " << "Program will be terminated" << std::endl;
        return;
    }
    const Mat q = codes_of(queryDescriptors, "query descriptors"), t = codes_of(trainDescriptors, "train descriptors");
    cs_ctx *c = thread_ctx()->ctx;
    std::vector<cs_dmatch> out((size_t)q.rows);
    int32_t n = 0;
    check(c, cs_match_line_descrip(c, q.data, q.rows, t.data, t.rows, INFINITY, out.data(), &n));
    for (int i = 0; i < n; i++)
        if (keep.empty() || keep[out[i].query_idx]) matches.push_back(to_dmatch(out[i], 0));
}

/* :264-341 */
void BinaryDescriptorMatcher::knnMatch(const Mat &queryDescriptors, const Mat &trainDescriptors, std::vector<std::vector<DMatch>> &matches, int k,
                                       const Mat &mask, bool compactResult) const
{
    if (queryDescriptors.rows == 0 || trainDescriptors.rows == 0) {
        std::cout << "Error: descriptors matrices cannot be void" << std::endl;
        return;
    }
    if (!mask.empty() && wrong_shape(mask, queryDescriptors.rows)) {
        std::cout << "Error: input mask should have " << queryDescriptors.rows << " rows and 1 column. " << "Program will be terminated" << std::endl;
        return;
    }
    check_k(k);
    std::vector<uint8_t> keep;
    if (!mask.empty()) mask_values(mask, queryDescriptors.rows, keep);
    const Mat q = codes_of(queryDescriptors, "query descriptors"), t = codes_of(trainDescriptors, "train descriptors");
    std::vector<std::vector<DMatch>> lists = pair_knn(q, t, k, keep);
    for (int i = 0; i < q.rows; i++)
        if (keep.empty() || keep[i] || !compactResult) matches.push_back(lists[i]); /* an unmasked query's list is kept even when empty */
}

/* :344-428 */
void BinaryDescriptorMatcher::knnMatch(const Mat &queryDescriptors, std::vector<std::vector<DMatch>> &matches, int k, const std::vector<Mat> &masks,
                                       bool compactResult)
{
    if (queryDescriptors.rows == 0) {
        std::cout << "Error: descriptors matrix cannot be void" << std::endl;
        return;
    }
    if (masks.size() != 0 && (int)masks.size() != numImages) {
        std::cout << "Error: the number of images in dataset is " << numImages << " but knnMatch function received " << masks.size()
                  << " masks. Program will be terminated" << std::endl;
        return;
    }
    check_k(k);
    const Mat q = codes_of(queryDescriptors, "query descriptors");
    train();
    State &s = state_of(this);
    const int nq = q.rows;
    std::vector<cs_dmatch> out;
    std::vector<int32_t> n((size_t)nq, 0);
    std::vector<uint8_t> rows;
    std::vector<char> bad;
    const int n_masks = collection_masks(masks, nq, rows, bad);
    int kk = 0;
    if (s.coll) {
        int64_t n_codes = 0;
        check(s.owner->ctx, cs_lbd_collection_size(s.coll, nullptr, &n_codes));
        kk = (int)std::min<int64_t>(k, n_codes); /* no query gets more entries than the collection has codes */
        out.resize(std::max<size_t>((size_t)nq * kk, 1));
        check(s.owner->ctx, cs_lbd_collection_knn_match(s.coll, q.data, nq, kk, n_masks ? rows.data() : nullptr, n_masks, out.data(), n.data()));
    }
    for (int i = 0; i < nq; i++) {
        std::vector<DMatch> list;
        for (int j = 0; j < n[i]; j++) {
            const cs_dmatch &m = out[(size_t)i * kk + j];
            if (n_masks && m.img_idx >= 0 && bad[m.img_idx]) {
                print_mask_error(m.img_idx, "knnMatch", nq);
                return;
            }
            list.push_back(to_dmatch(m, m.img_idx));
        }
        if (!list.empty() || !compactResult) matches.push_back(list);
    }
}

/* :431-507 */
void BinaryDescriptorMatcher::radiusMatch(const Mat &queryDescriptors, const Mat &trainDescriptors, std::vector<std::vector<DMatch>> &matches,
                                          float maxDistance, const Mat &mask, bool compactResult) const
{
    if (queryDescriptors.rows == 0 || trainDescriptors.rows == 0) {
        std::cout << "Error: descriptors matrices cannot be void" << std::endl;
        return;
    }
    std::vector<uint8_t> keep;
    if (!mask.empty() && ((mask.rows != queryDescriptors.rows && mask.cols != 1) || !mask_values(mask, queryDescriptors.rows, keep))) {
        std::cout << "Error: input mask should have " << queryDescriptors.rows << " rows and 1 column. " << "Program will be terminated" << std::endl;
        return;
    }
    const Mat q = codes_of(queryDescriptors, "query descriptors"), t = codes_of(trainDescriptors, "train descriptors");
    std::vector<std::vector<DMatch>> lists = pair_radius(q, t, maxDistance, keep);
    for (int i = 0; i < q.rows; i++)
        if (!lists[i].empty() || !compactResult) matches.push_back(lists[i]);
}

/* :510-595 */
void BinaryDescriptorMatcher::radiusMatch(const Mat &queryDescriptors, std::vector<std::vector<DMatch>> &matches, float maxDistance,
                                          const std::vector<Mat> &masks, bool compactResult)
{
    if (queryDescriptors.rows == 0) {
        std::cout << "Error: descriptors matrices cannot be void" << std::endl;
        return;
    }
    if (masks.size() != 0 && (int)masks.size() != numImages) {
        std::cout << "Error: the number of images in dataset is " << numImages << " but radiusMatch function received " << masks.size()
                  << " masks. Program will be terminated" << std::endl;
        return;
    }
    const Mat q = codes_of(queryDescriptors, "query descriptors");
    train();
    State &s = state_of(this);
    const int nq = q.rows;
    std::vector<cs_dmatch> out;
    std::vector<int64_t> off((size_t)nq + 1, 0);
    std::vector<uint8_t> rows;
    std::vector<char> bad;
    const int n_masks = collection_masks(masks, nq, rows, bad);
    if (s.coll)
        radius_call(s.owner->ctx, nq, [&](cs_dmatch *m, int64_t cap, int64_t *o) {
            return cs_lbd_collection_radius_match(s.coll, q.data, nq, maxDistance, n_masks ? rows.data() : nullptr, n_masks, m, cap, o);
        }, out, off);
    for (int i = 0; i < nq; i++) {
        std::vector<DMatch> list;
        for (int64_t j = off[i]; j < off[i + 1]; j++) {
            if (n_masks && out[j].img_idx >= 0 && bad[out[j].img_idx]) {
                print_mask_error(out[j].img_idx, "radiusMatch", nq);
                return;
            }
            list.push_back(to_dmatch(out[j], out[j].img_idx));
        }
        if (!list.empty() || !compactResult) matches.push_back(list);
    }
}

}  // namespace line_descriptor
}  // namespace cv
#endif /* CS_SHIM_ENABLED */
