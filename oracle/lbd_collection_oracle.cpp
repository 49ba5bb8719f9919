/*
 * oracle/lbd_collection_oracle.cpp -- CPU ORACLE for matching line descriptors against a collection of images.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates, without OpenCV, the collection forms of BinaryDescriptorMatcher ("from one image to a set"):
 *   line_lbd/libs/binary_descriptor_matcher.cpp:70-93      add (the image map: std::map::insert of each image's first row) and train
 *   line_lbd/libs/binary_descriptor_matcher.cpp:126-193    match(query, matches, masks)
 *   line_lbd/libs/binary_descriptor_matcher.cpp:344-428    knnMatch(query, matches, k, masks, compactResult)
 *   line_lbd/libs/binary_descriptor_matcher.cpp:510-595    radiusMatch(query, matches, maxDistance, masks, compactResult)
 * as the pairwise restatement (oracle/lbd_knn_oracle.cpp) over the concatenation of the images -- train() populates one hash over all rows,
 * so the order and the global train index are the pairwise ones -- followed by the image of each row and the mask post-filter: an entry
 * stays when masks[imgIdx][queryIdx] != 0.  match is knnMatch with k = 1 and no fall-back.  Entries beyond D = 128 (train_idx -1) have no
 * image: img_idx -1, and with masks they are dropped.  The list views (compactResult) are in oracle/pyoracle_collection.py.
 *
 * PARITY: PINNED to the reference.  oracle/ref/linelbd_collection_ref.cpp calls the reference's own collection forms and returns the part of
 * their answer that is defined; tests/test_oracle_ref_lbd_collection.py requires equal lists.
 */
#include <cstdint>
#include <map>
#include <vector>

extern "C" int lbd_orc_knn_match(const uint8_t *q, int nq, const uint8_t *t, int nt, int k, const uint8_t *mask, int32_t *n_per_query, int32_t *query_idx,
                                 int32_t *train_idx, float *dist);
extern "C" int64_t lbd_orc_radius_match(const uint8_t *q, int nq, const uint8_t *t, int nt, float max_distance, const uint8_t *mask, int64_t *offsets,
                                        int32_t *query_idx, int32_t *train_idx, float *dist, int64_t cap);

namespace {
/* add()'s indexesMap: image i's first row -> i, inserted in order, never overwritten */
std::map<int, int> image_map(const int32_t *image_offsets, int n_images)
{
    std::map<int, int> m;
    for (int i = 0; i < n_images; i++) m.insert({image_offsets[i], i});
    return m;
}

/* image of an entry and whether the masks keep it (masks: n_images x nq bytes, or NULL) */
bool keep_entry(const std::map<int, int> &m, int32_t train_idx, int query, int nq, const uint8_t *masks, int32_t *img)
{
    if (train_idx < 0) {
        *img = -1;
        return masks == nullptr;
    }
    auto it = m.upper_bound(train_idx);
    --it;
    *img = it->second;
    return !masks || masks[(size_t)it->second * nq + query] != 0;
}
}  // namespace

/* knnMatch(query, matches, k, masks) over the images' concatenated codes (image_offsets: n_images + 1): row i (k slots at i * k) holds
 * n_per_query[i] entries.  -1 for k < 0. */
extern "C" int lbd_orc_collection_knn(const uint8_t *codes, const int32_t *image_offsets, int n_images, const uint8_t *q, int nq, int k, const uint8_t *masks,
                                      int32_t *n_per_query, int32_t *query_idx, int32_t *train_idx, int32_t *img_idx, float *dist)
{
    if (k < 0) return -1;
    const int nt = n_images > 0 ? image_offsets[n_images] : 0;
    const int rc = lbd_orc_knn_match(q, nq, codes, nt, k, nullptr, n_per_query, query_idx, train_idx, dist);
    if (rc) return rc;
    const std::map<int, int> m = image_map(image_offsets, n_images);
    for (int i = 0; i < nq; i++) {
        int n = 0;
        for (int j = 0; j < n_per_query[i]; j++) {
            const size_t s = (size_t)i * k + j, o = (size_t)i * k + n;
            int32_t img;
            if (!keep_entry(m, train_idx[s], i, nq, masks, &img)) continue;
            query_idx[o] = query_idx[s];
            train_idx[o] = train_idx[s];
            dist[o] = dist[s];
            img_idx[o] = img;
            n++;
        }
        n_per_query[i] = n;
    }
    return 0;
}

/* radiusMatch(query, matches, maxDistance, masks) over the concatenated codes: query i's entries at [offsets[i], offsets[i + 1]).  Writes at
 * most cap entries; returns the total (offsets always complete). */
extern "C" int64_t lbd_orc_collection_radius(const uint8_t *codes, const int32_t *image_offsets, int n_images, const uint8_t *q, int nq, float max_distance,
                                             const uint8_t *masks, int64_t *offsets, int32_t *query_idx, int32_t *train_idx, int32_t *img_idx, float *dist,
                                             int64_t cap)
{
    const int nt = n_images > 0 ? image_offsets[n_images] : 0;
    std::vector<int64_t> off((size_t)nq + 1);
    const int64_t all = lbd_orc_radius_match(q, nq, codes, nt, max_distance, nullptr, off.data(), nullptr, nullptr, nullptr, 0);
    std::vector<int32_t> qi((size_t)all + 1), ti((size_t)all + 1);
    std::vector<float> di((size_t)all + 1);
    lbd_orc_radius_match(q, nq, codes, nt, max_distance, nullptr, off.data(), qi.data(), ti.data(), di.data(), all);
    const std::map<int, int> m = image_map(image_offsets, n_images);
    int64_t n = 0;
    offsets[0] = 0;
    for (int i = 0; i < nq; i++) {
        for (int64_t j = off[i]; j < off[i + 1]; j++) {
            int32_t img;
            if (!keep_entry(m, ti[j], i, nq, masks, &img)) continue;
            if (n < cap) {
                query_idx[n] = qi[j];
                train_idx[n] = ti[j];
                img_idx[n] = img;
                dist[n] = di[j];
            }
            n++;
        }
        offsets[i + 1] = n;
    }
    return n;
}
