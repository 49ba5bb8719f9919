/*
 * oracle/ref/linelbd_knn_ref.cpp -- CPU ORACLE, TEST INFRASTRUCTURE ONLY: the reference's own pairwise BinaryDescriptorMatcher::knnMatch and
 * radiusMatch (line_lbd/libs/binary_descriptor_matcher.cpp:264-341, 431-507), called on the matcher line_lbd_detect creates (bdm).
 *
 * The translation unit of oracle/ref/linelbd_ref.cpp (the reference's detection, descriptor and matcher sources, included from where they
 * lie, against the OpenCV stand-in) plus the two entry points below; nothing of the reference is copied.  Built into
 * oracle/_ref/liblinelbd_knn_ref.so by oracle/pyoracle_knn.py with the flags oracle/Makefile uses for liblinelbd_ref.so, where the reference
 * checkout exists; the library travels with the tree like the others.
 */
#include <algorithm>

#include "linelbd_ref.cpp"


/* The distances of the codes Mihasher::query meets for one query, ascending: a code is met when one of its 32 bytes is within d = 4 bits
 * of the query's (the 32 hash tables are looked up at radius 0 .. 4 per byte); query() stops early only once K codes are counted.  So
 * checkKDistances' k_distances has min(K, met codes) entries -- these -- and past them knnMatch reads results[] that query() never wrote
 * and radiusMatch reads k_distances past its end: the part of the reference's answer that is not defined. */
static std::vector<int> ref_met_distances(const uint8_t *qrow, const uint8_t *t, int nt)
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

/* The lists of a pairwise knnMatch / radiusMatch, defined part only: list l is query list_query[l] with list_len[l] entries, flattened into
 * query_idx / train_idx / dist (train_idx -1 beyond D = 128, where the reference never writes it).  Returns the number of lists (-1:
 * exception, -2: out of room).  With cap < 0 the entry points below return after the reference's call, writing nothing (for timing it). */
static int ref_lists_out(const std::vector<std::vector<cv::DMatch>> &lists, const std::vector<int> &list_query, const std::vector<int> &defined,
                         int32_t *lq, int32_t *ll, int32_t *query_idx, int32_t *train_idx, float *dist, int cap)
{
    int n = 0;
    for (size_t l = 0; l < lists.size(); l++) {
        lq[l] = list_query[l];
        ll[l] = defined[l];
        for (int j = 0; j < defined[l]; j++, n++) {
            if (n >= cap) return -2;
            const cv::DMatch &m = lists[l][j];
            query_idx[n] = m.queryIdx;
            train_idx[n] = m.distance > 128 ? -1 : m.trainIdx;
            dist[n] = m.distance;
        }
    }
    return (int)lists.size();
}

/* bdm->knnMatch(query, train, matches, k, mask, compactResult), the pairwise form (binary_descriptor_matcher.cpp:264-341) */
extern "C" int ref_knn_match(const uint8_t *q, int nq, const uint8_t *t, int nt, int k, const uint8_t *mask, int compact, int32_t *list_query, int32_t *list_len,
                             int32_t *query_idx, int32_t *train_idx, float *dist, int cap)
{
    /* k = 0: setK(0) makes query() search for every code, and it stores them into res[] of K * (D + 1) = 0 entries -- not run */
    if (k <= 0) return -5;
    try {
        line_lbd_detect &det = ref_detector(1, 0);
        cv::Mat mq(nq, 32, CV_8UC1), mt(nt, 32, CV_8UC1), mm;
        if (nq) std::memcpy(mq.data, q, (size_t)nq * 32);
        if (nt) std::memcpy(mt.data, t, (size_t)nt * 32);
        if (mask) {
            mm = cv::Mat(nq, 1, CV_8UC1);
            std::memcpy(mm.data, mask, (size_t)nq);
        }
        std::vector<std::vector<cv::DMatch>> lists;
        det.bdm->knnMatch(mq, mt, lists, k, mm, compact != 0);
        if (lists.empty() || cap < 0) return (int)lists.size(); /* cap < 0: the call alone (timing) */
        std::vector<int> lq, defined;
        for (int i = 0; i < nq; i++) {
            const bool skip = mask && !mask[i];
            if (skip && compact) continue;
            lq.push_back(i);
            defined.push_back(skip ? 0 : std::min<int>(k, (int)ref_met_distances(q + (size_t)i * 32, t, nt).size()));
        }
        if (lq.size() != lists.size()) return -3;
        return ref_lists_out(lists, lq, defined, list_query, list_len, query_idx, train_idx, dist, cap);
    } catch (const std::exception &e) {
        fprintf(stderr, "ref_knn_match: %s\n", e.what());
        return -1;
    }
}

/* bdm->radiusMatch(query, train, matches, maxDistance, mask, compactResult), the pairwise form (:431-507).  The defined entries of a query
 * are those of the first k_distances.size() positions; they come first in its list. */
extern "C" int ref_radius_match(const uint8_t *q, int nq, const uint8_t *t, int nt, float max_distance, const uint8_t *mask, int compact, int32_t *list_query,
                                int32_t *list_len, int32_t *query_idx, int32_t *train_idx, float *dist, int cap)
{
    try {
        line_lbd_detect &det = ref_detector(1, 0);
        cv::Mat mq(nq, 32, CV_8UC1), mt(nt, 32, CV_8UC1), mm;
        if (nq) std::memcpy(mq.data, q, (size_t)nq * 32);
        if (nt) std::memcpy(mt.data, t, (size_t)nt * 32);
        if (mask) {
            mm = cv::Mat(nq, 1, CV_8UC1);
            std::memcpy(mm.data, mask, (size_t)nq);
        }
        std::vector<std::vector<cv::DMatch>> lists;
        det.bdm->radiusMatch(mq, mt, lists, max_distance, mm, compact != 0);
        if (lists.empty() || cap < 0) return (int)lists.size(); /* cap < 0: the call alone (timing) */
        std::vector<int> defined_of((size_t)nq, 0);
        for (int i = 0; i < nq; i++)
            if (!mask || mask[i])
                for (int d : ref_met_distances(q + (size_t)i * 32, t, nt)) defined_of[i] += d <= max_distance;
        /* which query each list belongs to: every query in order, or (compactResult) the non-empty ones, named by their entries; a list
         * whose entries are all undefined is left out there, as the library leaves out an empty one */
        std::vector<std::vector<cv::DMatch>> kept;
        std::vector<int> lq, defined;
        for (size_t l = 0; l < lists.size(); l++) {
            const int i = compact ? lists[l][0].queryIdx : (int)l;
            if (i < 0 || i >= nq) return -3;
            if (compact && defined_of[i] == 0) continue;
            if ((int)lists[l].size() < defined_of[i]) return -4;
            kept.push_back(lists[l]);
            lq.push_back(i);
            defined.push_back(defined_of[i]);
        }
        if (!compact && (int)lists.size() != nq) return -3;
        return ref_lists_out(kept, lq, defined, list_query, list_len, query_idx, train_idx, dist, cap);
    } catch (const std::exception &e) {
        fprintf(stderr, "ref_radius_match: %s\n", e.what());
        return -1;
    }
}
