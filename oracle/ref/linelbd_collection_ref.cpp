/*
 * oracle/ref/linelbd_collection_ref.cpp -- CPU ORACLE, TEST INFRASTRUCTURE ONLY: the reference's own collection forms of
 * BinaryDescriptorMatcher -- add (line_lbd/libs/binary_descriptor_matcher.cpp:70-80), then one of match (:126-193), knnMatch (:344-428) or
 * radiusMatch (:510-595) without a train matrix, which call train() (:83-93) themselves.
 *
 * The translation unit of oracle/ref/linelbd_ref.cpp (the reference's detection, descriptor and matcher sources, included from where they
 * lie, against the OpenCV stand-in) plus the entry point below; nothing of the reference is copied.  Built into
 * oracle/_ref/liblinelbd_collection_ref.so by oracle/pyoracle_collection.py with the flags oracle/Makefile uses for liblinelbd_ref.so, where
 * the reference checkout exists.  Every call uses a fresh matcher: add() of the images, one query call.
 */
#include <algorithm>

#include "linelbd_ref.cpp"

namespace {
/* distances of the codes Mihasher::query meets for one query over all rows, ascending (a code is met when one of its 32 bytes is within 4
 * bits of the query's).  Past the first min(K, met) positions the reference reads results[] that query() never wrote and k_distances past
 * its end: the part of its answer that is not defined.  A met code further than D = 128 has no written trainIdx either. */
std::vector<int> met_distances(const uint8_t *qrow, const uint8_t *t, int nt)
{
    std::vector<int> out;
    for (int j = 0; j < nt; j++) {
        int d = 0, smin = 9;
        for (int k = 0; k < 32; k++) {
            const int s = __builtin_popcount(qrow[k] ^ t[(size_t)j * 32 + k]);
            d += s;
            smin = s < smin ? s : smin;
        }
        if (smin <= 4) out.push_back(d);
    }
    std::sort(out.begin(), out.end());
    return out;
}
}  // namespace

/* kind 0 match, 1 knnMatch(k), 2 radiusMatch(max_distance) of a fresh BinaryDescriptorMatcher after add(images): codes / image_offsets
 * (n_images + 1) hold the images' rows back to back, masks (NULL, or n_images x nq bytes) become one nq x 1 Mat per image.  Output, defined
 * part only: list l is query list_query[l] with list_len[l] entries, flattened into query_idx / train_idx / img_idx / dist (match: one list
 * per DMatch).  train_idx and img_idx are -1 beyond D = 128.  Returns the number of lists; -1 exception, -2 out of room, -3 unexpected list
 * shape, -5 k <= 0 (setK(0) makes query() write every code into a result buffer of 0 entries: not run), -7 no codes at all (train()
 * leaves the hash unpopulated and the query reads its empty tables: not run), -8 a query that meets no code (the reference then reads
 * element 0 of an empty k_distances: not run), -6 masks given where some entry the
 * reference would look a mask up for is undefined (its image index is then garbage and the mask lookup may read out of bounds: not run).
 * cap < 0: the call alone, nothing written (timing). */
extern "C" int ref_collection_query(int kind, const uint8_t *codes, const int32_t *image_offsets, int n_images, const uint8_t *q, int nq, int k,
                                    float max_distance, const uint8_t *masks, int compact, int32_t *list_query, int32_t *list_len, int32_t *query_idx,
                                    int32_t *train_idx, int32_t *img_idx, float *dist, int cap)
{
    if (kind == 1 && k <= 0) return -5;
    const int nt = n_images > 0 ? image_offsets[n_images] : 0;
    if (nt == 0) return -7;
    std::vector<std::vector<int>> met((size_t)nq);
    for (int i = 0; i < nq; i++) {
        met[i] = met_distances(q + (size_t)i * 32, codes, nt);
        if (met[i].empty()) return -8;
    }
    if (masks)
        for (int i = 0; i < nq; i++) {
            const std::vector<int> &m = met[i];
            if (kind == 0 && (m.empty() || m[0] > 128)) return -6;
            if (kind == 1 && ((int)m.size() < k || m[k - 1] > 128)) return -6;
            if (kind == 2) {
                if ((int)m.size() < nt) return -6;
                for (int d : m)
                    if (d <= max_distance && d > 128) return -6;
            }
        }
    try {
        cv::line_descriptor::BinaryDescriptorMatcher bdm;
        std::vector<cv::Mat> imgs, mm;
        for (int i = 0; i < n_images; i++) {
            const int n = image_offsets[i + 1] - image_offsets[i];
            cv::Mat m(n, 32, CV_8UC1);
            if (n) std::memcpy(m.data, codes + (size_t)image_offsets[i] * 32, (size_t)n * 32);
            imgs.push_back(m);
            if (masks) {
                cv::Mat mk(nq, 1, CV_8UC1);
                std::memcpy(mk.data, masks + (size_t)i * nq, (size_t)nq);
                mm.push_back(mk);
            }
        }
        cv::Mat mq(nq, 32, CV_8UC1);
        if (nq) std::memcpy(mq.data, q, (size_t)nq * 32);
        bdm.add(imgs);
        std::vector<std::vector<cv::DMatch>> lists;
        if (kind == 0) {
            std::vector<cv::DMatch> ms;
            bdm.match(mq, ms, mm);
            for (const cv::DMatch &m : ms) lists.push_back({m});
        } else if (kind == 1) {
            bdm.knnMatch(mq, lists, k, mm, compact != 0);
        } else {
            bdm.radiusMatch(mq, lists, max_distance, mm, compact != 0);
        }
        if (cap < 0) return (int)lists.size();
        /* the defined entries of each query: with masks every entry (the guard above); else the first min(k, met) (knn), the met codes
         * within the radius (radius), the nearest met code (match) -- they come first in its list */
        std::vector<int> defined_of((size_t)nq, 0);
        for (int i = 0; i < nq; i++) {
            const std::vector<int> &m = met[i];
            if (kind == 0) defined_of[i] = !m.empty();
            if (kind == 1) defined_of[i] = std::min<int>(k, (int)m.size());
            if (kind == 2)
                for (int d : m) defined_of[i] += d <= max_distance;
        }
        int n = 0, n_lists = 0;
        for (size_t l = 0; l < lists.size(); l++) {
            int i;
            if (kind == 0 || compact) {
                if (lists[l].empty()) return -3;
                i = lists[l][0].queryIdx;
            } else {
                i = (int)l;
            }
            if (i < 0 || i >= nq) return -3;
            const int len = masks ? (int)lists[l].size() : std::min<int>(defined_of[i], (int)lists[l].size());
            if (!masks && (int)lists[l].size() < defined_of[i]) return -3;
            if (len == 0 && (kind == 0 || compact)) continue; /* a list of undefined entries only: the library has none, and drops it */
            list_query[n_lists] = i;
            list_len[n_lists] = len;
            n_lists++;
            for (int j = 0; j < len; j++, n++) {
                if (n >= cap) return -2;
                const cv::DMatch &m = lists[l][j];
                query_idx[n] = m.queryIdx;
                train_idx[n] = m.distance > 128 ? -1 : m.trainIdx;
                img_idx[n] = m.distance > 128 ? -1 : m.imgIdx;
                dist[n] = m.distance;
            }
        }
        if (kind != 0 && !compact && (int)lists.size() != nq) return -3;
        return n_lists;
    } catch (const std::exception &e) {
        fprintf(stderr, "ref_collection_query: %s\n", e.what());
        return -1;
    }
}
