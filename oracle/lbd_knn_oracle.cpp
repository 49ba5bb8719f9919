/*
 * oracle/lbd_knn_oracle.cpp -- CPU ORACLE for k-nearest-neighbour and radius matching of line descriptors.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates, without OpenCV, the pairwise forms of
 *   line_lbd/libs/binary_descriptor_matcher.cpp:264-341     BinaryDescriptorMatcher::knnMatch(query, train, matches, k, mask)
 *   line_lbd/libs/binary_descriptor_matcher.cpp:431-507     BinaryDescriptorMatcher::radiusMatch(query, train, matches, maxDistance, mask)
 *   line_lbd/libs/binary_descriptor_matcher.cpp:637-755     Mihasher::query
 * on the key lbd_orc_match orders codes by (oracle/lbd_oracle.cpp: distance, search radius, substring, rank of the xor pattern in
 * query()'s enumeration -- lbd_orc_pattern_rank -- and train index).  The knnMatch / radiusMatch views with masks and compactResult are in
 * oracle/pyoracle_knn.py.
 *
 * PARITY: PINNED to the reference.  oracle/ref/linelbd_knn_ref.cpp calls the reference's own knnMatch / radiusMatch and returns the part of
 * their answer that is defined; tests/test_oracle_ref_lbd_knn.py requires equal lists.
 */
#include <algorithm>
#include <cstdint>
#include <vector>

extern "C" void lbd_orc_pattern_rank(int32_t *rank256);

/* The met codes of one query in ascending key order -- the order lbd_orc_match takes the first of.  BinaryDescriptorMatcher::knnMatch and
 * radiusMatch over Mihasher::query (:264-341, 431-507, 637-755) return a prefix of it: query() stops once n >= K codes are counted, and by
 * the pigeonhole argument of multi-index hashing every code at distance <= s * 32 + k has been met by then, so the stop drops no nearer
 * code; knnMatch takes the first k, radiusMatch those with distance <= maxDistance. */
static void mih_sorted_keys(const uint8_t *qrow, const uint8_t *t, int nt, const int32_t rank[256], std::vector<uint64_t> &keys)
{
    keys.clear();
    for (int j = 0; j < nt; j++) {
        int d = 0, smin = 9, kmin = 0;
        for (int k = 0; k < 32; k++) {
            const int s = __builtin_popcount(qrow[k] ^ t[(size_t)j * 32 + k]);
            d += s;
            if (s < smin) {
                smin = s;
                kmin = k;
            }
        }
        if (smin > 4) continue;
        const int x = qrow[kmin] ^ t[(size_t)j * 32 + kmin];
        keys.push_back(((uint64_t)d << 47) | ((uint64_t)smin << 44) | ((uint64_t)kmin << 39) | ((uint64_t)rank[x] << 32) | (uint64_t)j);
    }
    std::sort(keys.begin(), keys.end());
}

static void mih_key_out(uint64_t key, int32_t *train_idx, float *dist)
{
    const int d = (int)(key >> 47);
    *train_idx = d <= 128 ? (int32_t)(key & 0xffffffffu) : -1; /* beyond D = 128 results[] is never written: -1, as lbd_orc_match */
    *dist = (float)d;
}

/* knnMatch(query, train, matches, k, mask) for one pair: row i (k slots at query_idx / train_idx / dist + i * k) holds n_per_query[i] entries,
 * the first k met codes; a query masked out (mask[i] == 0) and every query of an empty query or train set gets none.  -1 for k < 0. */
extern "C" int lbd_orc_knn_match(const uint8_t *q, int nq, const uint8_t *t, int nt, int k, const uint8_t *mask, int32_t *n_per_query, int32_t *query_idx,
                                 int32_t *train_idx, float *dist)
{
    if (k < 0) return -1;
    for (int i = 0; i < nq; i++) n_per_query[i] = 0;
    if (nq <= 0 || nt <= 0) return 0;
    int32_t rank[256];
    lbd_orc_pattern_rank(rank);
    std::vector<uint64_t> keys;
    for (int i = 0; i < nq; i++) {
        if (mask && !mask[i]) continue;
        mih_sorted_keys(q + (size_t)i * 32, t, nt, rank, keys);
        const int n = std::min<int>(k, (int)keys.size());
        for (int j = 0; j < n; j++) {
            query_idx[(size_t)i * k + j] = i;
            mih_key_out(keys[j], &train_idx[(size_t)i * k + j], &dist[(size_t)i * k + j]);
        }
        n_per_query[i] = n;
    }
    return 0;
}

/* radiusMatch(query, train, matches, maxDistance, mask) for one pair: query i's entries at [offsets[i], offsets[i + 1]) -- every met code
 * with distance <= max_distance, in key order.  Writes at most cap entries; returns the total (offsets always complete). */
extern "C" int64_t lbd_orc_radius_match(const uint8_t *q, int nq, const uint8_t *t, int nt, float max_distance, const uint8_t *mask, int64_t *offsets,
                                        int32_t *query_idx, int32_t *train_idx, float *dist, int64_t cap)
{
    offsets[0] = 0;
    int32_t rank[256];
    lbd_orc_pattern_rank(rank);
    std::vector<uint64_t> keys;
    int64_t n = 0;
    for (int i = 0; i < nq; i++) {
        if (nt > 0 && (!mask || mask[i])) {
            mih_sorted_keys(q + (size_t)i * 32, t, nt, rank, keys);
            for (uint64_t key : keys) {
                if (!((float)(int)(key >> 47) <= max_distance)) break;
                if (n < cap) {
                    query_idx[n] = i;
                    mih_key_out(key, &train_idx[n], &dist[n]);
                }
                n++;
            }
        }
        offsets[i + 1] = n;
    }
    return n;
}
