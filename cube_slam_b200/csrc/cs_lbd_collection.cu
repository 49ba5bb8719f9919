/* cs_lbd_collection.cu -- matching line descriptors against a device-resident collection of many images' codes: the "from one image to a
 * set" forms of BinaryDescriptorMatcher (relocalisation and loop closure: this frame's lines against every keyframe's).
 *
 * Replaces   line_lbd/libs/binary_descriptor_matcher.cpp:70-104    BinaryDescriptorMatcher::add, train, clear
 *            line_lbd/libs/binary_descriptor_matcher.cpp:126-193   match(query, matches, masks)
 *            line_lbd/libs/binary_descriptor_matcher.cpp:344-428   knnMatch(query, matches, k, masks, compactResult)
 *            line_lbd/libs/binary_descriptor_matcher.cpp:510-595   radiusMatch(query, matches, maxDistance, masks, compactResult)
 *
 * The answers are the pairwise answers over the concatenation of every image added (cs_lbd.cu), ordered by the same key -- cs_lbd_match_key
 * (cs_lbd_core.h) called with the global row -- so ties break as the reference's one multi-index hash over all rows breaks them.  The
 * image of a row and the masks are applied on the host to the few keys that come back.
 *
 *   k_coll_scan<MODE>  one CTA of 64 threads holds a tile of 64 queries, one per thread, in registers, and streams a contiguous split of the
 *                      collection through shared memory in tiles of 128 codes (4 KB), double-buffered: one thread starts the bulk copy
 *                      (cp.async.bulk + mbarrier) of tile t + 2 as soon as the CTA is done with tile t.  Every thread reads each staged
 *                      code by broadcast.  The grid is query tiles x train splits, so a frame's few hundred queries fill the GPU against a
 *                      large collection.  Per (query, code) the full Hamming distance comes first (8 x XOR + POPC); the key is built only
 *                      when the distance can matter.  A code at distance <= 159 is always met by the hash (some byte then differs in <= 4
 *                      bits, pigeonhole), so the "met" test (cs_lbd_match_key != ~0) is needed only at distances >= 160.
 *     KNN2             k <= 2 (match, the ratio test): the two smallest keys per (query, split) in registers -> k_coll_merge2.
 *     HIST             knn with k > 2: a per-thread histogram of met distances in shared memory (257 x 16-bit bins per query: a split holds
 *                      at most 65408 codes), added into a per-query histogram in HBM.  The host finds the distance of the k-th met code.
 *     COUNT            radius: the number of met codes within the radius per query.
 *     GATHER           the keys of met codes at distance <= the query's threshold into its segment (offsets from a scan of the counts).
 *   Then a segmented sort of the 64-bit keys (CUB's DeviceSegmentedSort) and, for knn, k_coll_emit copies the first k of each segment.
 */
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/device/device_segmented_sort.cuh>

#include "cs_internal.h"
#include "cs_lbd_core.h"
#include "cs_tma.cuh"

#define CS_COLL_QT 64                        /* queries per CTA, one per thread */
#define CS_COLL_TT 128                       /* codes per staged tile: 4 KB */
#define CS_COLL_BINS 257                     /* distances 0 .. 256 */
#define CS_COLL_MAX_SPLIT (511 * CS_COLL_TT) /* codes per split, so that a 16-bit histogram bin cannot overflow */
#define CS_COLL_TARGET_CTAS (CS_SM_COUNT * 8)

namespace {

enum { COLL_KNN2 = 0, COLL_HIST = 1, COLL_COUNT = 2, COLL_GATHER = 3 };

struct CollArgs {
    const uint4 *q;               /* nq x 32 bytes */
    const uint4 *t;               /* nt x 32 bytes, the collection */
    int nq, nt, chunk;            /* chunk: codes per split (a multiple of CS_COLL_TT) */
    int max_dist;                 /* COUNT */
    unsigned long long *part2;    /* KNN2: [split][nq][2] */
    uint32_t *hist;               /* HIST: [nq][257] */
    int32_t *cnt;                 /* COUNT: [nq] */
    const int32_t *thr;           /* GATHER: per query, -1 = nothing */
    const int32_t *off;           /* GATHER: segment starts */
    int32_t *cursor;              /* GATHER: [nq], zeroed */
    unsigned long long *seg;      /* GATHER */
    int32_t *err;                 /* bit 0: a tile copy did not complete; bit 1: a segment would overflow */
};

#ifdef __CUDACC__
/* one thread: expect `bytes` on the barrier and start a 1-D bulk copy of them (16-byte aligned, a multiple of 16) into shared memory */
__device__ __forceinline__ void coll_bulk_load(void *dst, const void *src, uint32_t bytes, unsigned long long *bar)
{
    const uint32_t b = cs_smem_u32(bar);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(cs_smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(b)
                 : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(CS_COLL_QT) k_coll_scan(CollArgs a)
{
    __shared__ __align__(128) uint4 s_t[2][CS_COLL_TT * 2];
    __shared__ __align__(8) unsigned long long s_bar[2];
    __shared__ uint16_t s_hist[MODE == COLL_HIST ? CS_COLL_BINS * CS_COLL_QT : 2];
    const int tid = threadIdx.x, qi = blockIdx.x * CS_COLL_QT + tid;
    const int j0 = (int)blockIdx.y * a.chunk; /* < nt for every split the grid has */
    const int j1 = (int)min((long long)a.nt, (long long)j0 + a.chunk); /* 64-bit: j0 + chunk may pass 2^31 - 1 in the last split */
    if (j0 >= a.nt) return; /* the whole CTA */
    const bool live = qi < a.nq;
    uint32_t q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (live) {
        const uint4 qa = a.q[2 * (size_t)qi], qb = a.q[2 * (size_t)qi + 1];
        q[0] = qa.x, q[1] = qa.y, q[2] = qa.z, q[3] = qa.w, q[4] = qb.x, q[5] = qb.y, q[6] = qb.z, q[7] = qb.w;
    }
    const int thr = MODE == COLL_GATHER ? (live ? a.thr[qi] : -1) : a.max_dist;
    if (MODE == COLL_HIST)
        for (int b = 0; b < CS_COLL_BINS; b++) s_hist[b * CS_COLL_QT + tid] = 0;
    const int n_tiles = (j1 - j0 + CS_COLL_TT - 1) / CS_COLL_TT;
    if (tid == 0) {
        cs_mbar_init(&s_bar[0]);
        cs_mbar_init(&s_bar[1]);
    }
    __syncthreads();
    auto issue = [&](int tl) {
        const int base = j0 + tl * CS_COLL_TT, n = min(CS_COLL_TT, j1 - base);
        coll_bulk_load(s_t[tl & 1], a.t + 2 * (size_t)base, (uint32_t)n * 32u, &s_bar[tl & 1]);
    };
    if (tid == 0) {
        issue(0);
        if (n_tiles > 1) issue(1);
    }
    unsigned long long b0 = ~0ull, b1 = ~0ull;
    unsigned c_in = 0;
    const bool active = live && (MODE != COLL_GATHER || thr >= 0);
    for (int tl = 0; tl < n_tiles; tl++) {
        const int buf = tl & 1;
        if (!cs_mbar_wait(&s_bar[buf], (uint32_t)((tl >> 1) & 1)) && tid == 0) atomicOr(a.err, 1);
        const int base = j0 + tl * CS_COLL_TT, n = min(CS_COLL_TT, j1 - base);
        if (active)
            for (int c = 0; c < n; c++) {
                const uint4 ta = s_t[buf][2 * c], tb = s_t[buf][2 * c + 1];
                const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
                int d = 0;
#pragma unroll
                for (int w = 0; w < 8; w++) d += __popc(q[w] ^ t[w]);
                if (MODE == COLL_KNN2) {
                    if (d <= (int)(b1 >> 48)) { /* a farther code cannot enter the best two: the distance is the key's top field */
                        const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)(base + c));
                        if (key < b0) {
                            b1 = b0;
                            b0 = key;
                        } else if (key < b1) {
                            b1 = key;
                        }
                    }
                } else if (MODE == COLL_HIST) {
                    if (d < 160 || cs_lbd_match_key(q, t, 0) != ~0ull) s_hist[d * CS_COLL_QT + tid]++;
                } else if (MODE == COLL_COUNT) {
                    if (d <= thr && (d < 160 || cs_lbd_match_key(q, t, 0) != ~0ull)) c_in++;
                } else if (d <= thr) {
                    const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)(base + c));
                    if (key != ~0ull) {
                        const int pos = a.off[qi] + atomicAdd(&a.cursor[qi], 1);
                        if (pos < a.off[qi + 1])
                            a.seg[pos] = key;
                        else
                            atomicOr(a.err, 2); /* more keys than the counting pass found: reported, never written past the segment */
                    }
                }
            }
        __syncthreads(); /* every thread is done with this buffer */
        if (tid == 0 && tl + 2 < n_tiles) issue(tl + 2);
    }
    if (!live) return;
    if (MODE == COLL_KNN2) {
        unsigned long long *p = a.part2 + 2 * ((size_t)blockIdx.y * a.nq + qi);
        p[0] = b0;
        p[1] = b1;
    } else if (MODE == COLL_HIST) {
        for (int b = 0; b < CS_COLL_BINS; b++) {
            const unsigned v = s_hist[b * CS_COLL_QT + tid];
            if (v) atomicAdd(&a.hist[(size_t)qi * CS_COLL_BINS + b], v);
        }
    } else if (MODE == COLL_COUNT) {
        if (c_in) atomicAdd(&a.cnt[qi], (int)c_in);
    }
}

/* the best two keys of every query over the splits: two ascending pairs (a0, a1), (c0, c1) merge into (min(a0, c0), min(max(a0, c0), a1, c1)) */
__global__ void __launch_bounds__(128) k_coll_merge2(const unsigned long long *__restrict__ part2, int n_split, int nq, unsigned long long *__restrict__ keys2)
{
    const int qi = blockIdx.x * 128 + threadIdx.x;
    if (qi >= nq) return;
    unsigned long long b0 = ~0ull, b1 = ~0ull;
    for (int s = 0; s < n_split; s++) {
        const unsigned long long c0 = part2[2 * ((size_t)s * nq + qi)], c1 = part2[2 * ((size_t)s * nq + qi) + 1];
        const unsigned long long hi = b0 < c0 ? c0 : b0, lo1 = b1 < c1 ? b1 : c1;
        b0 = b0 < c0 ? b0 : c0;
        b1 = hi < lo1 ? hi : lo1;
    }
    keys2[2 * (size_t)qi] = b0;
    keys2[2 * (size_t)qi + 1] = b1;
}

/* knn: the first n_out[q] sorted keys of query q's segment to out[q * k ..] */
__global__ void __launch_bounds__(64) k_coll_emit(const unsigned long long *__restrict__ sorted, const int32_t *__restrict__ off,
                                                  const int32_t *__restrict__ n_out, int k, unsigned long long *__restrict__ out)
{
    const int qi = blockIdx.x;
    for (int i = threadIdx.x; i < n_out[qi]; i += 64) out[(size_t)qi * k + i] = sorted[(size_t)off[qi] + i];
}
#endif

struct DBuf {
    void *p = nullptr;
    size_t cap = 0;
};

}  // namespace

struct cs_lbd_collection {
    cs_ctx *ctx = nullptr;
    void *codes = nullptr;            /* n_codes x 32 bytes on the device */
    size_t codes_cap = 0;             /* codes of room */
    int64_t n_codes = 0;
    int32_t n_images = 0;
    std::vector<int64_t> starts;      /* add()'s indexesMap, flattened: distinct first rows, ascending, */
    std::vector<int32_t> owner;       /* and the first image added at each (std::map::insert keeps the first) */
    DBuf q, part2, keys2, hist, cnt, thr, off, cursor, seg, sorted, out, temp, err;
};

namespace {

int grow(cs_lbd_collection *L, DBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return CS_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    const size_t want = bytes + bytes / 8 + 256;
    if (cudaMalloc(&b.p, want) != cudaSuccess) {
        cudaGetLastError();
        return cs_ctx_fail(L->ctx, CS_ERR_CUDA, "cudaMalloc(%zu) failed in the descriptor collection", want);
    }
    b.cap = want;
    return CS_OK;
}

int cuda_fail(cs_lbd_collection *L, const char *what)
{
    const cudaError_t e = cudaGetLastError();
    return cs_ctx_fail(L->ctx, CS_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
}

/* splits of the collection: about CS_COLL_TARGET_CTAS CTAs over the query tiles, each split a whole number of tiles and at most
 * CS_COLL_MAX_SPLIT codes */
void plan_splits(int nq, int nt, int *chunk, int *n_split)
{
    /* 64-bit: nt + CS_COLL_TT - 1 and nt + chunk - 1 pass 2^31 - 1 for collections near the bound */
    const int64_t qtiles = ((int64_t)nq + CS_COLL_QT - 1) / CS_COLL_QT;
    const int64_t tiles = ((int64_t)nt + CS_COLL_TT - 1) / CS_COLL_TT;
    const int64_t s = std::max<int64_t>(1, std::min<int64_t>(tiles, (CS_COLL_TARGET_CTAS + qtiles - 1) / qtiles));
    const int64_t per = std::min<int64_t>((tiles + s - 1) / s, CS_COLL_MAX_SPLIT / CS_COLL_TT);
    *chunk = (int)(per * CS_COLL_TT);
    *n_split = (int)(((int64_t)nt + *chunk - 1) / *chunk);
}

int launch_scan(cs_lbd_collection *L, int mode, CollArgs a, int n_split)
{
    const dim3 grid((unsigned)((a.nq + CS_COLL_QT - 1) / CS_COLL_QT), (unsigned)n_split);
    cudaStream_t st = cs_ctx_stream(L->ctx);
    switch (mode) {
    case COLL_KNN2: k_coll_scan<COLL_KNN2><<<grid, CS_COLL_QT, 0, st>>>(a); break;
    case COLL_HIST: k_coll_scan<COLL_HIST><<<grid, CS_COLL_QT, 0, st>>>(a); break;
    case COLL_COUNT: k_coll_scan<COLL_COUNT><<<grid, CS_COLL_QT, 0, st>>>(a); break;
    default: k_coll_scan<COLL_GATHER><<<grid, CS_COLL_QT, 0, st>>>(a); break;
    }
    cs_ctx_count_launches(L->ctx, 1);
    if (cudaGetLastError() != cudaSuccess) return cuda_fail(L, "collection matcher kernel launch");
    return CS_OK;
}

/* common entry: checks, queries to the device, the scan arguments.  Returns CS_OK with *go = false when there is nothing to search. */
int begin_query(cs_lbd_collection *L, const uint8_t *query32, int n_query, const uint8_t *masks, int n_masks, bool *go, CollArgs &a, int *n_split)
{
    *go = false;
    if (n_query < 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "negative query count");
    if (masks && n_masks != L->n_images)
        return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "%d masks for a collection of %d images: one mask per image", n_masks, L->n_images);
    if (!masks && n_masks != 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "n_masks = %d without masks", n_masks);
    if (n_query == 0 || L->n_codes == 0) return CS_OK;
    if (!query32) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null query descriptors");
    cudaSetDevice(cs_ctx_device(L->ctx));
    cudaStream_t st = cs_ctx_stream(L->ctx);
    int rc;
    if ((rc = grow(L, L->q, (size_t)n_query * 32)) || (rc = grow(L, L->err, 4))) return rc;
    if (cudaMemcpyAsync(L->q.p, query32, (size_t)n_query * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(L->err.p, 0, 4, st) != cudaSuccess)
        return cuda_fail(L, "upload of the query descriptors");
    memset(&a, 0, sizeof a);
    a.q = (const uint4 *)L->q.p;
    a.t = (const uint4 *)L->codes;
    a.nq = n_query;
    a.nt = (int)L->n_codes;
    plan_splits(n_query, a.nt, &a.chunk, n_split);
    a.err = (int32_t *)L->err.p;
    *go = true;
    return CS_OK;
}

int check_err(cs_lbd_collection *L)
{
    int32_t e = 0;
    if (cudaMemcpyAsync(&e, L->err.p, 4, cudaMemcpyDeviceToHost, cs_ctx_stream(L->ctx)) != cudaSuccess ||
        cudaStreamSynchronize(cs_ctx_stream(L->ctx)) != cudaSuccess)
        return cuda_fail(L, "collection matcher");
    if (e & 1) return cs_ctx_fail(L->ctx, CS_ERR_CUDA, "a bulk copy of collection codes into shared memory did not complete");
    if (e & 2) return cs_ctx_fail(L->ctx, CS_ERR_CUDA, "the gather pass met more keys than the counting pass (internal error)");
    return CS_OK;
}

/* the image a global row belongs to, as the reference's indexesMap.upper_bound(row) - 1 finds it */
int32_t image_of_row(const cs_lbd_collection *L, int64_t row)
{
    return L->owner[std::upper_bound(L->starts.begin(), L->starts.end(), row) - L->starts.begin() - 1];
}

/* a key as a DMatch of the collection; false when the masks drop it */
bool key_entry(const cs_lbd_collection *L, unsigned long long key, int query_idx, int n_query, const uint8_t *masks, cs_dmatch &m)
{
    const int d = CS_LBD_KEY_DIST(key);
    m.query_idx = query_idx;
    m.distance = (float)d;
    if (d > 128) { /* the reference never writes this entry's trainIdx, so there is no image (and no mask) to consult */
        m.train_idx = -1;
        m.img_idx = -1;
        return masks == nullptr;
    }
    m.train_idx = (int32_t)CS_LBD_KEY_TRAIN(key);
    m.img_idx = image_of_row(L, m.train_idx);
    return !masks || masks[(size_t)m.img_idx * n_query + query_idx] != 0;
}

/* the best two keys of every query (k <= 2) to the host */
int best_two(cs_lbd_collection *L, CollArgs a, int n_split, std::vector<unsigned long long> &keys2)
{
    const int nq = a.nq;
    cudaStream_t st = cs_ctx_stream(L->ctx);
    int rc;
    if ((rc = grow(L, L->part2, (size_t)n_split * nq * 16)) || (rc = grow(L, L->keys2, (size_t)nq * 16))) return rc;
    a.part2 = (unsigned long long *)L->part2.p;
    if ((rc = launch_scan(L, COLL_KNN2, a, n_split))) return rc;
    k_coll_merge2<<<(nq + 127) / 128, 128, 0, st>>>((const unsigned long long *)L->part2.p, n_split, nq, (unsigned long long *)L->keys2.p);
    cs_ctx_count_launches(L->ctx, 1);
    if (cudaGetLastError() != cudaSuccess) return cuda_fail(L, "collection merge kernel launch");
    keys2.resize((size_t)nq * 2);
    if (cudaMemcpyAsync(keys2.data(), L->keys2.p, (size_t)nq * 16, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_fail(L, "match copy");
    return check_err(L);
}

/* the keys of every met code at distance <= thr[q] of each query, sorted, in segments at off[q] (thr[q] < 0: none).  Leaves them at
 * L->sorted. */
int gather_sorted(cs_lbd_collection *L, CollArgs a, int n_split, const std::vector<int32_t> &thr, const std::vector<int32_t> &off)
{
    const int nq = a.nq;
    const int total = off[nq];
    cudaStream_t st = cs_ctx_stream(L->ctx);
    int rc;
    if ((rc = grow(L, L->thr, (size_t)nq * 4)) || (rc = grow(L, L->off, (size_t)(nq + 1) * 4)) || (rc = grow(L, L->cursor, (size_t)nq * 4)) ||
        (rc = grow(L, L->seg, (size_t)total * 8)) || (rc = grow(L, L->sorted, (size_t)total * 8)))
        return rc;
    if (cudaMemcpyAsync(L->thr.p, thr.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(L->off.p, off.data(), (size_t)(nq + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(L->cursor.p, 0, (size_t)nq * 4, st) != cudaSuccess)
        return cuda_fail(L, "upload of the match thresholds");
    a.thr = (const int32_t *)L->thr.p;
    a.off = (const int32_t *)L->off.p;
    a.cursor = (int32_t *)L->cursor.p;
    a.seg = (unsigned long long *)L->seg.p;
    if ((rc = launch_scan(L, COLL_GATHER, a, n_split))) return rc;
    const int *b = (const int *)L->off.p;
    size_t temp = 0;
    if (cub::DeviceSegmentedSort::SortKeys(nullptr, temp, (const unsigned long long *)L->seg.p, (unsigned long long *)L->sorted.p, total, nq, b, b + 1, st) !=
        cudaSuccess)
        return cuda_fail(L, "segmented sort sizing");
    if ((rc = grow(L, L->temp, temp))) return rc;
    if (cub::DeviceSegmentedSort::SortKeys(L->temp.p, temp, (const unsigned long long *)L->seg.p, (unsigned long long *)L->sorted.p, total, nq, b, b + 1, st) !=
        cudaSuccess)
        return cuda_fail(L, "segmented sort");
    cs_ctx_count_launches(L->ctx, 1);
    return CS_OK;
}

/* every device buffer of the collection back to the device, after the work queued on the context stream */
void release_device(cs_lbd_collection *L)
{
    cudaSetDevice(cs_ctx_device(L->ctx));
    cudaStreamSynchronize(cs_ctx_stream(L->ctx));
    if (L->codes) cudaFree(L->codes);
    L->codes = nullptr;
    L->codes_cap = 0;
    DBuf *all[] = {&L->q, &L->part2, &L->keys2, &L->hist, &L->cnt, &L->thr, &L->off, &L->cursor, &L->seg, &L->sorted, &L->out, &L->temp, &L->err};
    for (DBuf *b : all) {
        if (b->p) cudaFree(b->p);
        b->p = nullptr;
        b->cap = 0;
    }
}

/* exclusive scan of the counts; CS_ERR_CAPACITY when the keys would not be addressable with 32-bit offsets */
int scan_counts(cs_lbd_collection *L, const std::vector<int64_t> &cnt, std::vector<int32_t> &off)
{
    const size_t nq = cnt.size();
    off.assign(nq + 1, 0);
    int64_t s = 0;
    for (size_t i = 0; i < nq; i++) {
        s += cnt[i];
        if (s > INT32_MAX) return cs_ctx_fail(L->ctx, CS_ERR_CAPACITY, "more than 2^31 - 1 keys to sort in one call: query fewer descriptors at once");
        off[i + 1] = (int32_t)s;
    }
    return CS_OK;
}

}  // namespace

extern "C" {

cs_lbd_collection *cs_lbd_collection_create(cs_ctx *ctx)
{
    if (!ctx) return nullptr;
    cs_lbd_collection *L = new cs_lbd_collection();
    L->ctx = ctx;
    return L;
}

void cs_lbd_collection_destroy(cs_lbd_collection *L)
{
    if (!L) return;
    release_device(L);
    delete L;
}

int cs_lbd_collection_add(cs_lbd_collection *L, const uint8_t *codes32, const int32_t *image_offsets, int n_images)
{
    if (!L) return CS_ERR_INVALID_ARG;
    if (n_images < 0 || (n_images > 0 && !image_offsets)) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null image_offsets or negative image count");
    if (n_images == 0) return CS_OK;
    if (image_offsets[0] != 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "image_offsets must start at 0");
    for (int i = 0; i < n_images; i++)
        if (image_offsets[i + 1] < image_offsets[i]) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "image_offsets must not decrease");
    const int64_t n = image_offsets[n_images];
    if (n > 0 && !codes32) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null codes");
    if (L->n_codes + n > INT32_MAX)
        return cs_ctx_fail(L->ctx, CS_ERR_CAPACITY, "a collection holds fewer than 2^31 codes (%lld + %lld)", (long long)L->n_codes, (long long)n);
    if ((int64_t)L->n_images + n_images > INT32_MAX) return cs_ctx_fail(L->ctx, CS_ERR_CAPACITY, "too many images");
    cudaSetDevice(cs_ctx_device(L->ctx));
    cudaStream_t st = cs_ctx_stream(L->ctx);
    if (n > 0 && (size_t)(L->n_codes + n) > L->codes_cap) { /* grow by half again, keeping what is there */
        const size_t cap = std::max((size_t)(L->n_codes + n), L->codes_cap + L->codes_cap / 2);
        void *p = nullptr;
        if (cudaMalloc(&p, cap * 32) != cudaSuccess) {
            cudaGetLastError();
            return cs_ctx_fail(L->ctx, CS_ERR_CUDA, "cudaMalloc(%zu) failed for the descriptor collection", cap * 32);
        }
        if (L->n_codes && cudaMemcpyAsync(p, L->codes, (size_t)L->n_codes * 32, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
            cudaFree(p);
            return cuda_fail(L, "collection growth copy");
        }
        cudaStreamSynchronize(st);
        if (L->codes) cudaFree(L->codes);
        L->codes = p;
        L->codes_cap = cap;
    }
    if (n > 0 && (cudaMemcpyAsync((uint8_t *)L->codes + (size_t)L->n_codes * 32, codes32, (size_t)n * 32, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                  cudaStreamSynchronize(st) != cudaSuccess))
        return cuda_fail(L, "upload of the collection codes");
    for (int i = 0; i < n_images; i++) /* starts only grow; an image starting where the last one did leaves it its owner */
        if (L->starts.empty() || L->starts.back() != L->n_codes + image_offsets[i]) {
            L->starts.push_back(L->n_codes + image_offsets[i]);
            L->owner.push_back(L->n_images + i);
        }
    L->n_codes += n;
    L->n_images += n_images;
    return CS_OK;
}

int cs_lbd_collection_clear(cs_lbd_collection *L)
{
    if (!L) return CS_ERR_INVALID_ARG;
    L->n_codes = 0;
    L->n_images = 0;
    L->starts.clear();
    L->owner.clear();
    release_device(L); /* clear() returns the device memory: the codes and every scratch buffer */
    return CS_OK;
}

int cs_lbd_collection_size(const cs_lbd_collection *L, int32_t *n_images, int64_t *n_codes)
{
    if (!L) return CS_ERR_INVALID_ARG;
    if (n_images) *n_images = L->n_images;
    if (n_codes) *n_codes = L->n_codes;
    return CS_OK;
}

int cs_lbd_collection_knn_match(cs_lbd_collection *L, const uint8_t *query32, int n_query, int k, const uint8_t *masks, int n_masks, cs_dmatch *matches,
                                int32_t *n_per_query)
{
    if (!L) return CS_ERR_INVALID_ARG;
    if (k < 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "k must not be negative");
    if (n_query > 0 && !n_per_query) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null n_per_query");
    for (int i = 0; i < n_query; i++) n_per_query[i] = 0;
    if (k == 0) return CS_OK;
    bool go;
    CollArgs a;
    int n_split, rc;
    if ((rc = begin_query(L, query32, n_query, masks, n_masks, &go, a, &n_split)) || !go) return rc;
    if (!matches) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null matches");
    cudaStream_t st = cs_ctx_stream(L->ctx);
    const int nq = n_query;
    auto put = [&](int i, const unsigned long long *keys, int n) {
        int m = 0;
        for (int j = 0; j < n; j++)
            if (key_entry(L, keys[j], i, nq, masks, matches[(size_t)i * k + m])) m++;
        n_per_query[i] = m;
    };
    if (k <= 2) {
        std::vector<unsigned long long> keys2;
        if ((rc = best_two(L, a, n_split, keys2))) return rc;
        for (int i = 0; i < nq; i++) {
            int n = 0;
            while (n < k && keys2[2 * (size_t)i + n] != ~0ull) n++;
            put(i, &keys2[2 * (size_t)i], n);
        }
        return CS_OK;
    }
    /* k > 2: histogram of met distances -> the distance of the k-th met code -> gather, sort, first k */
    if ((rc = grow(L, L->hist, (size_t)nq * CS_COLL_BINS * 4))) return rc;
    if (cudaMemsetAsync(L->hist.p, 0, (size_t)nq * CS_COLL_BINS * 4, st) != cudaSuccess) return cuda_fail(L, "histogram clear");
    a.hist = (uint32_t *)L->hist.p;
    if ((rc = launch_scan(L, COLL_HIST, a, n_split))) return rc;
    std::vector<uint32_t> hist((size_t)nq * CS_COLL_BINS);
    if (cudaMemcpyAsync(hist.data(), L->hist.p, hist.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_fail(L, "histogram copy");
    if ((rc = check_err(L))) return rc;
    std::vector<int32_t> thr((size_t)nq, -1), n_out((size_t)nq, 0), off;
    std::vector<int64_t> cnt((size_t)nq, 0);
    for (int i = 0; i < nq; i++) {
        int64_t s = 0;
        for (int d = 0; d < CS_COLL_BINS && s < k; d++)
            if (hist[(size_t)i * CS_COLL_BINS + d]) {
                s += hist[(size_t)i * CS_COLL_BINS + d];
                thr[i] = d;
            }
        cnt[i] = s;
        n_out[i] = (int32_t)std::min<int64_t>(k, s);
    }
    if ((rc = scan_counts(L, cnt, off))) return rc;
    if (off[nq] == 0) return CS_OK;
    if ((rc = gather_sorted(L, a, n_split, thr, off))) return rc;
    const int kk = (int)std::min<int64_t>(k, L->n_codes); /* no query has more entries than the collection has codes */
    if ((rc = grow(L, L->out, (size_t)nq * kk * 8)) || (rc = grow(L, L->cnt, (size_t)nq * 4))) return rc;
    if (cudaMemcpyAsync(L->cnt.p, n_out.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_fail(L, "upload of the counts");
    k_coll_emit<<<nq, 64, 0, st>>>((const unsigned long long *)L->sorted.p, (const int32_t *)L->off.p, (const int32_t *)L->cnt.p, kk, (unsigned long long *)L->out.p);
    cs_ctx_count_launches(L->ctx, 1);
    if (cudaGetLastError() != cudaSuccess) return cuda_fail(L, "collection emit kernel launch");
    std::vector<unsigned long long> keys((size_t)nq * kk);
    if (cudaMemcpyAsync(keys.data(), L->out.p, keys.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_fail(L, "match copy");
    if ((rc = check_err(L))) return rc;
    for (int i = 0; i < nq; i++) put(i, &keys[(size_t)i * kk], n_out[i]);
    return CS_OK;
}

int cs_lbd_collection_match(cs_lbd_collection *L, const uint8_t *query32, int n_query, const uint8_t *masks, int n_masks, cs_dmatch *matches, int32_t *n_matches)
{
    if (!L) return CS_ERR_INVALID_ARG;
    if (!n_matches) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null n_matches");
    *n_matches = 0;
    if (n_query < 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "negative query count");
    std::vector<int32_t> n1((size_t)std::max(n_query, 1));
    if (!matches && n_query > 0 && L->n_codes > 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null matches");
    const int rc = cs_lbd_collection_knn_match(L, query32, n_query, 1, masks, n_masks, matches, n1.data());
    if (rc) return rc;
    int n = 0; /* the nearest code of each query, kept unless its image masks the query; compacted in query order */
    for (int i = 0; i < n_query; i++)
        if (n1[i]) matches[n++] = matches[i];
    *n_matches = n;
    return CS_OK;
}

int cs_lbd_collection_radius_match(cs_lbd_collection *L, const uint8_t *query32, int n_query, float max_distance, const uint8_t *masks, int n_masks,
                                   cs_dmatch *matches, int64_t max_matches, int64_t *match_offsets)
{
    if (!L) return CS_ERR_INVALID_ARG;
    if (!match_offsets || max_matches < 0) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null match_offsets or negative max_matches");
    for (int i = 0; i <= std::max(n_query, 0); i++) match_offsets[i] = 0;
    /* k_distances[j] <= maxDistance (:565): an integer distance against a float; NaN and negative radii take nothing */
    const int max_dist = !(max_distance >= 0.0f) ? -1 : (max_distance >= 256.0f ? 256 : (int)floorf(max_distance));
    bool go;
    CollArgs a;
    int n_split, rc;
    if ((rc = begin_query(L, query32, n_query, masks, n_masks, &go, a, &n_split)) || !go || max_dist < 0) return rc;
    cudaStream_t st = cs_ctx_stream(L->ctx);
    const int nq = n_query;
    if ((rc = grow(L, L->cnt, (size_t)nq * 4))) return rc;
    if (cudaMemsetAsync(L->cnt.p, 0, (size_t)nq * 4, st) != cudaSuccess) return cuda_fail(L, "count clear");
    a.cnt = (int32_t *)L->cnt.p;
    a.max_dist = max_dist;
    if ((rc = launch_scan(L, COLL_COUNT, a, n_split))) return rc;
    std::vector<int32_t> c32((size_t)nq), thr((size_t)nq), off;
    if (cudaMemcpyAsync(c32.data(), L->cnt.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_fail(L, "count copy");
    if ((rc = check_err(L))) return rc;
    std::vector<int64_t> cnt((size_t)nq);
    for (int i = 0; i < nq; i++) {
        cnt[i] = c32[i];
        thr[i] = c32[i] ? max_dist : -1;
    }
    if ((rc = scan_counts(L, cnt, off))) return rc;
    if (off[nq] == 0) return CS_OK;
    if ((rc = gather_sorted(L, a, n_split, thr, off))) return rc;
    std::vector<unsigned long long> keys((size_t)off[nq]);
    if (cudaMemcpyAsync(keys.data(), L->sorted.p, keys.size() * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_fail(L, "match copy");
    if ((rc = check_err(L))) return rc;
    /* the entries the masks keep, query after query: their layout, then (when they fit) the entries */
    std::vector<cs_dmatch> kept(keys.size());
    int64_t total = 0;
    for (int i = 0; i < nq; i++) {
        for (int j = off[i]; j < off[i + 1]; j++) total += key_entry(L, keys[j], i, nq, masks, kept[total]);
        match_offsets[i + 1] = total;
    }
    if (total > max_matches)
        return cs_ctx_fail(L->ctx, CS_ERR_CAPACITY, "%lld matches within the radius exceed max_matches = %lld; match_offsets holds the layout they need",
                           (long long)total, (long long)max_matches);
    if (total && !matches) return cs_ctx_fail(L->ctx, CS_ERR_INVALID_ARG, "null matches");
    if (total) memcpy(matches, kept.data(), (size_t)total * sizeof(cs_dmatch));
    return CS_OK;
}

}  // extern "C"
