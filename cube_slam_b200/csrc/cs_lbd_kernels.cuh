/* cs_lbd_kernels.cuh -- the kernels of cs_lbd.cu (included there, inside its unnamed namespace): k_lbd_describe, k_lbd_match, and the
 * knn / radius matchers k_lbd_knn2 and k_lbd_match_sorted (tests/host_core/lbd_knn_emu.cpp runs those two under the same emulation).
 * They live in a file of their own so that the CPU test suite can compile this very source against a small emulation of the CUDA
 * execution model (tests/host_core/lbd_kernels_emu.cpp: one std::thread per CUDA thread, a std::barrier for __syncthreads, function-local
 * statics for __shared__) and run whole launches against the oracle -- index arithmetic, phase split and barrier placement included -- on
 * machines without a GPU.  The arithmetic itself is cs_lbd_core.h; see cs_lbd.cu's header for what each kernel does. */
__global__ void __launch_bounds__(64) k_lbd_describe(const CsLbdLine *__restrict__ lines, int n_lines, const int16_t *__restrict__ dx_all,
                                                     const int16_t *__restrict__ dy_all, int w, int h, const float *__restrict__ coef /* F_g 63, F_l 21 */,
                                                     uint8_t *__restrict__ desc, float *__restrict__ fdesc)
{
    __shared__ float s_rows[CS_LBD_ROWS * 4];
    __shared__ float s_sums[CS_LBD_DESC];
    __shared__ float s_des[CS_LBD_DESC];
    __shared__ float s_coefL[3 * CS_LBD_BAND_WIDTH];
    const int li = blockIdx.x, tid = threadIdx.x;
    if (li >= n_lines) return; /* the whole CTA leaves together */
    const CsLbdLine L = lines[li];
    if (tid < 3 * CS_LBD_BAND_WIDTH) s_coefL[tid] = coef[CS_LBD_ROWS + tid];
    if (tid < CS_LBD_ROWS) {
        const size_t off = (size_t)L.frame * w * h;
        float r[4];
        cs_lbd_row(L, tid, dx_all + off, dy_all + off, w, h, coef[tid], r);
        s_rows[tid * 4 + 0] = r[0];
        s_rows[tid * 4 + 1] = r[1];
        s_rows[tid * 4 + 2] = r[2];
        s_rows[tid * 4 + 3] = r[3];
    }
    __syncthreads();
    for (int t = tid; t < CS_LBD_DESC; t += 64) s_sums[t] = cs_lbd_band_sum(t, s_rows, s_coefL);
    __syncthreads();
    if (tid < CS_LBD_BANDS) cs_lbd_band_stats(tid, s_sums, s_des);
    __syncthreads();
    if (tid == 0) cs_lbd_finish(s_des);
    __syncthreads();
    if (tid < CS_LBD_BYTES) desc[(size_t)li * CS_LBD_BYTES + tid] = cs_lbd_byte(tid, s_des);
    if (fdesc)
        for (int t = tid; t < CS_LBD_DESC; t += 64) fdesc[(size_t)li * CS_LBD_DESC + t] = s_des[t];
}

__global__ void __launch_bounds__(128) k_lbd_match(const uint4 *__restrict__ q_all, const uint4 *__restrict__ t_all, const int32_t *__restrict__ pair_of_query,
                                                   const int32_t *__restrict__ t_off, int n_queries, unsigned long long *__restrict__ keys)
{
    __shared__ unsigned long long s_best[4];
    const int qi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (qi >= n_queries) return;
    const uint4 qa = q_all[2 * (size_t)qi], qb = q_all[2 * (size_t)qi + 1];
    const uint32_t q[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    const int p = pair_of_query[qi], t0 = t_off[p], t1 = t_off[p + 1];
    unsigned long long best = ~0ull;
    for (int j = t0 + tid; j < t1; j += 128) {
        const uint4 ta = t_all[2 * (size_t)j], tb = t_all[2 * (size_t)j + 1];
        const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
        const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)(j - t0));
        best = key < best ? key : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other < best ? other : best;
    }
    if (lane == 0) s_best[wid] = best;
    __syncthreads();
    if (tid == 0) {
        unsigned long long b = s_best[0];
        for (int k = 1; k < 4; k++) b = s_best[k] < b ? s_best[k] : b;
        keys[qi] = b;
    }
}

/* ---- k nearest neighbours and radius matching (BinaryDescriptorMatcher::knnMatch / radiusMatch over pairs).  Both answers are a prefix
 * of the query's met train codes in ascending key order (cs_lbd_match_key): the first k, or every code at distance <= r -- the distance is
 * the key's top field, so those come first. */
#define CS_LBD_KNN_MAX_TRAIN 16384 /* train codes per pair: k_lbd_match_sorted stages up to this many keys, 128 KB of shared memory */
#define CS_LBD_SORT_THREADS 256

/* k <= 2, the ratio test's case: the two smallest keys of each query in registers, merged by shuffles, no shared-memory staging.
 * keys2[2 qi], keys2[2 qi + 1]: ascending, ~0 where fewer codes are met. */
__global__ void __launch_bounds__(128) k_lbd_knn2(const uint4 *__restrict__ q_all, const uint4 *__restrict__ t_all, const int32_t *__restrict__ pair_of_query,
                                                  const int32_t *__restrict__ t_off, int n_queries, unsigned long long *__restrict__ keys2)
{
    __shared__ unsigned long long s_best[4][2];
    const int qi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (qi >= n_queries) return;
    const uint4 qa = q_all[2 * (size_t)qi], qb = q_all[2 * (size_t)qi + 1];
    const uint32_t q[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    const int p = pair_of_query[qi], t0 = t_off[p], t1 = t_off[p + 1];
    unsigned long long b0 = ~0ull, b1 = ~0ull;
    for (int j = t0 + tid; j < t1; j += 128) {
        const uint4 ta = t_all[2 * (size_t)j], tb = t_all[2 * (size_t)j + 1];
        const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
        const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)(j - t0));
        if (key < b0) {
            b1 = b0;
            b0 = key;
        } else if (key < b1) {
            b1 = key;
        }
    }
    /* two ascending pairs (a0, a1), (c0, c1) merge into (min(a0, c0), min(max(a0, c0), a1, c1)); keys are distinct but for ~0 */
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long c0 = __shfl_xor_sync(0xffffffffu, b0, o), c1 = __shfl_xor_sync(0xffffffffu, b1, o);
        const unsigned long long hi = b0 < c0 ? c0 : b0, lo1 = b1 < c1 ? b1 : c1;
        b0 = b0 < c0 ? b0 : c0;
        b1 = hi < lo1 ? hi : lo1;
    }
    if (lane == 0) {
        s_best[wid][0] = b0;
        s_best[wid][1] = b1;
    }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < 4; w++) {
            const unsigned long long c0 = s_best[w][0], c1 = s_best[w][1];
            const unsigned long long hi = b0 < c0 ? c0 : b0, lo1 = b1 < c1 ? b1 : c1;
            b0 = b0 < c0 ? b0 : c0;
            b1 = hi < lo1 ? hi : lo1;
        }
        keys2[2 * (size_t)qi] = b0;
        keys2[2 * (size_t)qi + 1] = b1;
    }
}

/* Any k, and radius matching: one 256-thread CTA per query.  Pass 1 counts the met keys at distance <= max_dist (m); keys == NULL stops
 * there and writes counts[qi] = m (the radius call's first launch, no shared memory).  Otherwise each thread stages its keys at its
 * exclusive prefix of the counts, the CTA sorts the m keys (bitonic, padded with ~0 to a power of two <= sort_cap, the dynamic shared
 * memory in keys) and writes the first min(m, room) at keys + out_off[qi], room = out_off[qi + 1] - out_off[qi]; counts[qi] = that number.
 * The keys are computed twice (pass 1, staging): two reads of the pair's train codes, which L1 / L2 serve, instead of a stage of every key. */
__global__ void __launch_bounds__(CS_LBD_SORT_THREADS) k_lbd_match_sorted(const uint4 *__restrict__ q_all, const uint4 *__restrict__ t_all,
                                                                          const int32_t *__restrict__ pair_of_query, const int32_t *__restrict__ t_off,
                                                                          int n_queries, int max_dist, const long long *__restrict__ out_off,
                                                                          unsigned long long *__restrict__ keys, int32_t *__restrict__ counts)
{
#if defined(__CUDACC__)
    extern __shared__ unsigned long long s_keys[];
#else
    static unsigned long long s_keys[CS_LBD_KNN_MAX_TRAIN]; /* host emulation: one block at a time */
#endif
    __shared__ unsigned s_warp[CS_LBD_SORT_THREADS / 32];
    const int qi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (qi >= n_queries) return;
    if (keys && out_off[qi + 1] == out_off[qi]) { /* no room: a masked query (the whole CTA leaves together) */
        if (tid == 0) counts[qi] = 0;
        return;
    }
    const uint4 qa = q_all[2 * (size_t)qi], qb = q_all[2 * (size_t)qi + 1];
    const uint32_t q[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    const int p = pair_of_query[qi], t0 = t_off[p], nt = t_off[p + 1] - t0;
    unsigned c = 0;
    for (int j = tid; j < nt; j += CS_LBD_SORT_THREADS) {
        const uint4 ta = t_all[2 * (size_t)(t0 + j)], tb = t_all[2 * (size_t)(t0 + j) + 1];
        const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
        const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)j);
        c += key != ~0ull && CS_LBD_KEY_DIST(key) <= max_dist;
    }
    /* exclusive prefix of c over the CTA: a butterfly inside the warp (pre: lanes below in the group of 2 o), then the warps' totals */
    unsigned sum = c, pre = 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned other = (unsigned)__shfl_xor_sync(0xffffffffu, sum, o);
        if (lane & o) pre += other;
        sum += other;
    }
    if (lane == 0) s_warp[wid] = sum;
    __syncthreads();
    unsigned m = 0;
    for (int w = 0; w < CS_LBD_SORT_THREADS / 32; w++) {
        if (w < wid) pre += s_warp[w];
        m += s_warp[w];
    }
    if (!keys) {
        if (tid == 0) counts[qi] = (int32_t)m;
        return;
    }
    for (int j = tid; j < nt && c; j += CS_LBD_SORT_THREADS) {
        const uint4 ta = t_all[2 * (size_t)(t0 + j)], tb = t_all[2 * (size_t)(t0 + j) + 1];
        const uint32_t t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
        const unsigned long long key = cs_lbd_match_key(q, t, (uint32_t)j);
        if (key != ~0ull && CS_LBD_KEY_DIST(key) <= max_dist) {
            s_keys[pre++] = key;
            c--;
        }
    }
    unsigned P = 1;
    while (P < m) P <<= 1;
    for (unsigned i = m + tid; i < P; i += CS_LBD_SORT_THREADS) s_keys[i] = ~0ull;
    __syncthreads();
    for (unsigned size = 2; size <= P; size <<= 1)
        for (unsigned stride = size >> 1; stride > 0; stride >>= 1) {
            for (unsigned i = tid; i < P / 2; i += CS_LBD_SORT_THREADS) {
                const unsigned lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const unsigned long long a = s_keys[lo], b = s_keys[hi];
                if ((a > b) == ((lo & size) == 0)) {
                    s_keys[lo] = b;
                    s_keys[hi] = a;
                }
            }
            __syncthreads();
        }
    const long long o0 = out_off[qi], room = out_off[qi + 1] - o0;
    const int n_out = (long long)m < room ? (int)m : (int)room;
    for (int i = tid; i < n_out; i += CS_LBD_SORT_THREADS) keys[o0 + i] = s_keys[i];
    if (tid == 0) counts[qi] = n_out;
}

/* the launches: a CTA of 64 threads per key line, a CTA of 128 (k_lbd_match, k_lbd_knn2) or 256 (k_lbd_match_sorted) threads per query.
 * Under the CPU emulation of the test suite (CS_LBD_EMU_LAUNCH defined by tests/host_core/*.cpp) the same grids run as threads of the host. */
#if defined(__CUDACC__)
inline void launch_lbd_describe(unsigned grid, cudaStream_t st, const CsLbdLine *lines, int n_lines, const int16_t *dx_all, const int16_t *dy_all, int w, int h,
                                const float *coef, uint8_t *desc, float *fdesc)
{
    k_lbd_describe<<<grid, 64, 0, st>>>(lines, n_lines, dx_all, dy_all, w, h, coef, desc, fdesc);
}
inline void launch_lbd_match(unsigned grid, cudaStream_t st, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries,
                             unsigned long long *keys)
{
    k_lbd_match<<<grid, 128, 0, st>>>(q_all, t_all, pair_of_query, t_off, n_queries, keys);
}
inline void launch_lbd_knn2(unsigned grid, cudaStream_t st, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries,
                            unsigned long long *keys2)
{
    k_lbd_knn2<<<grid, 128, 0, st>>>(q_all, t_all, pair_of_query, t_off, n_queries, keys2);
}
/* sort_cap: keys of shared memory to reserve (a power of two, at most CS_LBD_KNN_MAX_TRAIN; 0 with keys == NULL).  The kernel's dynamic
 * shared-memory limit is raised once per device to the most any launch asks for (CS_LBD_KNN_MAX_TRAIN keys, 128 KB), not to this launch's
 * own size: the attribute belongs to the function on the device, shared by every context and host thread, so a limit lowered by one call
 * could land between another thread's raise and its launch.  The limit is only a cap: occupancy still follows each launch's size. */
inline void launch_lbd_match_sorted(unsigned grid, cudaStream_t st, unsigned sort_cap, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query,
                                    const int32_t *t_off, int n_queries, int max_dist, const long long *out_off, unsigned long long *keys, int32_t *counts)
{
    const int smem = (int)(sort_cap * sizeof(unsigned long long));
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(k_lbd_match_sorted, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)(CS_LBD_KNN_MAX_TRAIN * sizeof(unsigned long long))));
    k_lbd_match_sorted<<<grid, CS_LBD_SORT_THREADS, smem, st>>>(q_all, t_all, pair_of_query, t_off, n_queries, max_dist, out_off, keys, counts);
}
#elif defined(CS_LBD_EMU_LAUNCH)
inline void launch_lbd_describe(unsigned grid, cudaStream_t, const CsLbdLine *lines, int n_lines, const int16_t *dx_all, const int16_t *dy_all, int w, int h,
                                const float *coef, uint8_t *desc, float *fdesc)
{
    CS_LBD_EMU_LAUNCH(grid, 64, [&] { k_lbd_describe(lines, n_lines, dx_all, dy_all, w, h, coef, desc, fdesc); });
}
inline void launch_lbd_match(unsigned grid, cudaStream_t, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries,
                             unsigned long long *keys)
{
    CS_LBD_EMU_LAUNCH(grid, 128, [&] { k_lbd_match(q_all, t_all, pair_of_query, t_off, n_queries, keys); });
}
inline void launch_lbd_knn2(unsigned grid, cudaStream_t, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries,
                            unsigned long long *keys2)
{
    CS_LBD_EMU_LAUNCH(grid, 128, [&] { k_lbd_knn2(q_all, t_all, pair_of_query, t_off, n_queries, keys2); });
}
inline void launch_lbd_match_sorted(unsigned grid, cudaStream_t, unsigned, const uint4 *q_all, const uint4 *t_all, const int32_t *pair_of_query, const int32_t *t_off,
                                    int n_queries, int max_dist, const long long *out_off, unsigned long long *keys, int32_t *counts)
{
    CS_LBD_EMU_LAUNCH(grid, CS_LBD_SORT_THREADS, [&] { k_lbd_match_sorted(q_all, t_all, pair_of_query, t_off, n_queries, max_dist, out_off, keys, counts); });
}
#endif
