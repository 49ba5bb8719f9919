/*
 * cs_kernels_sweep.cu -- the proposal sweep, scoring and selection kernels (sm_90a).
 *
 *   k_sweep_score : getVanishingPoints + VP_support_edge_infos + the yaw x top-corner x configuration
 *                   corner chain + box_edge_sum_dists + box_edge_alignment_angle_error
 *                   (box_proposal_detail.cpp:229-465; object_3d_util.cpp:380-492,602-607)
 *   k_fuse_rank   : fuse_normalize_scores_v2 + change_2d_corner_to_3d_object + skew-penalised ranking
 *                   (box_proposal_detail.cpp:472-536; object_3d_util.cpp:495-648)
 *
 * FP64 throughout (compiled -fmad=false); the only float32 arithmetic is the dist-map running sum,
 * which the reference also does in float32 and in the same order.
 */
#include "cs_pmath.h"
#include <cuda_runtime.h>
#include <stdint.h>

#include "cs_geom.cuh"
#include "cs_internal.h"
#include "cs_kernels.h"

#define SW_THREADS 256
#define SW_WARPS (SW_THREADS / 32)
#define SW_MAX_YC 16
#define SW_LPL (CS_MAXL_OUT / 32) /* lines per lane */

struct SweepShared {
    double ang[CS_MAXL_OUT], midx[CS_MAXL_OUT], midy[CS_MAXL_OUT];
    D2 vps[SW_MAX_YC][3];
    double vp_angles[SW_MAX_YC][6];
    D2 corners[SW_THREADS][8];
    int32_t slot_cand[SW_THREADS];
    int warp_cnt[SW_WARPS];
};

/* (value, index) comparators with first-occurrence semantics of Eigen's maxCoeff / minCoeff */
__device__ __forceinline__ void arg_better_max(double &v, int &i, double ov, int oi)
{
    if (oi >= 0 && (i < 0 || ov > v || (ov == v && oi < i))) {
        v = ov;
        i = oi;
    }
}
__device__ __forceinline__ void arg_better_min(double &v, int &i, double ov, int oi)
{
    if (oi >= 0 && (i < 0 || ov < v || (ov == v && oi < i))) {
        v = ov;
        i = oi;
    }
}

/* VP_support_edge_infos for one (yaw, vp) by one warp (object_3d_util.cpp:380-425) */
__device__ __forceinline__ void vp_support_warp(const SweepShared &S, int n_lines, D2 vp, double thre, int vp_id, double *out2)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    double raw[SW_LPL];
    bool inl[SW_LPL];
    int first = INT_MAX;
#pragma unroll
    for (int k = 0; k < SW_LPL; k++) {
        const int e = lane + 32 * k;
        inl[k] = false;
        raw[k] = 0;
        if (e < n_lines) {
            raw[k] = cs_pm_atan2(S.midy[e] - vp.y, S.midx[e] - vp.x);
            const double nrm = g_normalize_to_pi(raw[k]);
            double d = fabs(S.ang[e] - nrm);
            d = g_min(d, CS_PI - d);
            inl[k] = d < thre;
            if (inl[k] && e < first) first = e;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(FULL, first, o));
    if (first == INT_MAX) { /* no inlier: NaN (object_3d_util.cpp:383) */
        if (lane == 0) {
            out2[0] = nan("");
            out2[1] = nan("");
        }
        return;
    }
    /* smooth_jump_angles (object_3d_util.cpp:175-189): base = first inlier's raw angle */
    const int owner = first & 31, slot = first >> 5;
    double base = 0;
#pragma unroll
    for (int k = 0; k < SW_LPL; k++)
        if (k == slot) base = raw[k];
    base = __shfl_sync(FULL, base, owner);
    double vmax = 0, vmin = 0;
    int imax = -1, imin = -1;
#pragma unroll
    for (int k = 0; k < SW_LPL; k++) {
        if (inl[k]) {
            const int e = lane + 32 * k;
            double v = raw[k];
            if ((raw[k] - base) < -CS_PI)
                v = raw[k] + 2 * CS_PI;
            else if ((raw[k] - base) > CS_PI)
                v = raw[k] - 2 * CS_PI;
            arg_better_max(vmax, imax, v, e);
            arg_better_min(vmin, imin, v, e);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(FULL, vmax, o);
        const int oi = __shfl_xor_sync(FULL, imax, o);
        arg_better_max(vmax, imax, ov, oi);
        const double pv = __shfl_xor_sync(FULL, vmin, o);
        const int pi = __shfl_xor_sync(FULL, imin, o);
        arg_better_min(vmin, imin, pv, pi);
    }
    if (lane == 0) {
        int low = imax, top = imin;
        if (vp_id > 0) {
            const int t = low;
            low = top;
            top = t;
        }
        out2[0] = S.ang[low];
        out2[1] = S.ang[top];
    }
}

extern __shared__ unsigned char sw_smem_raw[];

__global__ void __launch_bounds__(SW_THREADS) k_sweep_score(const CsJob *__restrict__ jobs, const CsFrame *__restrict__ frames,
                                                            const CsPose *__restrict__ poses, const double *__restrict__ yaw_table,
                                                            const int2 *__restrict__ blocks /* (job, pose) */,
                                                            const double *__restrict__ merged_lines, const int32_t *__restrict__ line_counts,
                                                            const float *__restrict__ dist_arena, uint8_t *__restrict__ c_valid,
                                                            double *__restrict__ c_dist, double *__restrict__ c_angle, cs_cuboid_params prm)
{
    SweepShared &S = *reinterpret_cast<SweepShared *>(sw_smem_raw);
    const int2 bp = blocks[blockIdx.x];
    const CsJob jb = jobs[bp.x];
    const CsFrame fr = frames[jb.frame];
    const CsPose &pose = poses[fr.pose_off + bp.y];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int n_lines = line_counts[bp.x * 2 + 1];
    const int n_yaw = fr.n_yaw, n_top = jb.n_top;
    const double *yaws = yaw_table + 3 * (size_t)fr.yaw_off; /* {yaw, cos, sin} per entry */

    /* the ROI's merged line set -> shared memory */
    {
        const double *ml = merged_lines + (size_t)bp.x * CS_MAXL_OUT * 7;
        for (int i = tid; i < n_lines; i += SW_THREADS) {
            S.ang[i] = ml[4 * CS_MAXL_OUT + i];
            S.midx[i] = ml[5 * CS_MAXL_OUT + i];
            S.midy[i] = ml[6 * CS_MAXL_OUT + i];
        }
    }
    if (n_top <= 0 || n_yaw <= 0) return;
    int YC = SW_THREADS / (2 * n_top);
    YC = max(1, min(YC, SW_MAX_YC));
    const float *dist = dist_arena + jb.px_off;
    const int64_t cbase = jb.cand_off + (int64_t)bp.y * n_yaw * n_top * 2;
    const bool cfg1 = prm.consider_config_1 != 0, cfg2 = prm.consider_config_2 != 0;

    for (int y0 = 0; y0 < n_yaw; y0 += YC) {
        const int yc = min(YC, n_yaw - y0);
        __syncthreads();
        if (tid < yc) g_vanishing_points(pose.KinvR, yaws + 3 * (y0 + tid), S.vps[tid]);
        __syncthreads();
        for (int t = wid; t < yc * 3; t += SW_WARPS) {
            const int yi = t / 3, vp_id = t - yi * 3;
            const double thre = ((vp_id != 2) ? prm.vp12_edge_angle_thre : prm.vp3_edge_angle_thre) / 180.0 * CS_PI;
            if (n_lines > 0)
                vp_support_warp(S, n_lines, S.vps[yi][vp_id], thre, vp_id, &S.vp_angles[yi][vp_id * 2]);
            else if (lane == 0) {
                S.vp_angles[yi][vp_id * 2] = nan("");
                S.vp_angles[yi][vp_id * 2 + 1] = nan("");
            }
        }
        __syncthreads();

        const int n_group = yc * n_top * 2;
        for (int g0 = 0; g0 < n_group; g0 += SW_THREADS) {
            const int gi = g0 + tid;
            bool valid = false;
            D2 c[8];
            int yi = 0, config_id = 1;
            if (gi < n_group) {
                yi = gi / (n_top * 2);
                const int r = gi - yi * (n_top * 2);
                const int ti = r >> 1;
                config_id = (r & 1) + 1;
                int vp1pos;
                if ((config_id == 1) ? cfg1 : cfg2) valid = g_build_corners(jb, S.vps[yi], g_top_x(jb, ti), config_id, prm.shorted_edge_thre, c, vp1pos);
                c_valid[cbase + (int64_t)y0 * n_top * 2 + gi] = valid ? 1 : 0;
            }
            /* ordered compaction of the valid candidates of this stride */
            const unsigned m = __ballot_sync(0xffffffffu, valid);
            if (lane == 0) S.warp_cnt[wid] = __popc(m);
            __syncthreads();
            int off = 0, total = 0;
            for (int k = 0; k < SW_WARPS; k++) {
                if (k < wid) off += S.warp_cnt[k];
                total += S.warp_cnt[k];
            }
            if (valid) {
                const int slot = off + __popc(m & ((1u << lane) - 1u));
#pragma unroll
                for (int k = 0; k < 8; k++) S.corners[slot][k] = c[k];
                S.slot_cand[slot] = gi;
            }
            __syncthreads();
            /* scoring: one thread per valid proposal, no idle lanes in the low warps */
            if (tid < total) {
                const int sg = S.slot_cand[tid];
                const int syi = sg / (n_top * 2);
                const int scfg = ((sg - syi * (n_top * 2)) & 1) + 1;
                const double sum_dist = g_edge_sum_dists(dist, jb.dpitch, jb.roi_w, jb.roi_h, S.corners[tid], (double)jb.roi_l, (double)jb.roi_t, scfg,
                                                         prm.reweight_edge_distance != 0);
                const double ang_err = g_angle_error(S.vp_angles[syi], scfg, S.corners[tid]);
                const int64_t ci = cbase + (int64_t)y0 * n_top * 2 + sg;
                c_dist[ci] = sum_dist / jb.diag;
                c_angle[ci] = ang_err;
            }
            __syncthreads();
        }
    }
}

/* ------------------------------------------------------------------------------------------ selection */
#define FU_THREADS 256
#define FU_SMEM_SORT 4096

__device__ __forceinline__ uint64_t sort_key(double v)
{
    if (isnan(v)) return ~0ull;
    if (v == 0.0) v = 0.0; /* -0 -> +0 */
    const uint64_t b = (uint64_t)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

/* bitonic sort of (key, idx) ascending, ties by idx.  P is a power of two; any address space. */
__device__ void bitonic_sort(uint64_t *key, uint32_t *idx, int P)
{
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int i = threadIdx.x; i < P; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const uint64_t ki = key[i], kl = key[l];
                    const uint32_t ii = idx[i], il = idx[l];
                    const bool gt = (ki > kl) || (ki == kl && ii > il);
                    const bool up = ((i & k) == 0);
                    if (gt == up) {
                        key[i] = kl;
                        key[l] = ki;
                        idx[i] = il;
                        idx[l] = ii;
                    }
                }
            }
        }
    __syncthreads();
}

__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int &total)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    __syncthreads();
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int off = 0;
    total = 0;
    for (int k = 0; k < FU_THREADS / 32; k++) {
        if (k < wid) off += s_warp[k];
        total += s_warp[k];
    }
    return off + incl - v;
}

/* rebuild the 8 corners of valid proposal `cand` (index inside its job) -- same code path as the sweep */
__device__ __forceinline__ bool rebuild_corners(const CsJob &jb, const CsFrame &fr, const CsPose *poses, const double *yaw_table,
                                                const cs_cuboid_params &prm, int cand, D2 *c, int &vp1pos, int &config_id, const double *&ycs,
                                                int &pose_id, int &top_id)
{
    const int per_pose = fr.n_yaw * jb.n_top * 2;
    pose_id = cand / per_pose;
    int r = cand - pose_id * per_pose;
    const int yi = r / (jb.n_top * 2);
    r -= yi * (jb.n_top * 2);
    top_id = r >> 1;
    config_id = (r & 1) + 1;
    ycs = yaw_table + 3 * (size_t)(fr.yaw_off + yi);
    D2 vps[3];
    g_vanishing_points(poses[fr.pose_off + pose_id].KinvR, ycs, vps);
    return g_build_corners(jb, vps, g_top_x(jb, top_id), config_id, prm.shorted_edge_thre, c, vp1pos);
}

/* combined_score of an emitted record: the ranking key, except where the key stands in for a NaN score with +inf (NaN ranks last but is
 * still a cuboid).  There the record reports the reference's own sum, normalized_error + skew penalty of its skew_ratio
 * (box_proposal_detail.cpp:517-536), which is NaN when either term is. */
__device__ __forceinline__ double g_record_score(double key, const cs_cuboid_rec &o, const cs_cuboid_params &prm)
{
    if (!isinf(key)) return key;
    double skew_error = prm.weight_skew_error * g_max(o.skew_ratio - prm.nominal_skew_ratio, 0.0);
    if (o.skew_ratio > prm.max_cut_skew) skew_error = 100;
    return o.normalized_error + prm.weight_skew_error * skew_error;
}

extern __shared__ unsigned char fu_smem_raw[];

__global__ void __launch_bounds__(FU_THREADS) k_fuse_rank(const CsObj *__restrict__ objs, const CsJob *__restrict__ jobs,
                                                          const CsFrame *__restrict__ frames, const CsPose *__restrict__ poses,
                                                          const double *__restrict__ yaw_table, const uint8_t *__restrict__ c_valid,
                                                          const double *__restrict__ c_dist, const double *__restrict__ c_angle,
                                                          int32_t *__restrict__ w_vlist, uint64_t *__restrict__ w_key, uint32_t *__restrict__ w_idx,
                                                          uint8_t *__restrict__ w_flag, int32_t *__restrict__ w_keep, double *__restrict__ w_norm,
                                                          double *__restrict__ w_score, int32_t *__restrict__ job_counts /* n_jobs x 2: valid, kept */,
                                                          cs_cuboid_rec *__restrict__ out, int32_t *__restrict__ out_counts, int topk,
                                                          cs_cuboid_params prm)
{
    __shared__ int s_warp[FU_THREADS / 32];
    __shared__ int s_i[4];
    __shared__ double s_red[4][FU_THREADS / 32];
    __shared__ double s_best_v[FU_THREADS / 32];
    __shared__ long long s_best_p[FU_THREADS / 32];
    __shared__ long long s_chosen[CS_MAX_TOPK];
    uint64_t *sm_key = reinterpret_cast<uint64_t *>(fu_smem_raw);
    uint32_t *sm_idx = reinterpret_cast<uint32_t *>(fu_smem_raw + sizeof(uint64_t) * FU_SMEM_SORT);

    const CsObj ob = objs[blockIdx.x];
    const CsFrame fr = frames[ob.frame];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    for (int jj = 0; jj < ob.n_jobs; jj++) {
        const int job = ob.job_off + jj;
        const CsJob jb = jobs[job];
        const int64_t co = jb.cand_off;
        int32_t *vlist = w_vlist + co;
        /* 1. valid proposals in enumeration order == the reference's row order */
        int n = 0;
        for (int base = 0; base < jb.n_cand; base += FU_THREADS) {
            const int i = base + tid;
            const int v = (i < jb.n_cand) ? (int)c_valid[co + i] : 0;
            int tot;
            const int pos = block_excl_scan(v, s_warp, tot);
            if (v) vlist[n + pos] = i;
            n += tot;
        }
        __syncthreads();
        int32_t *keep = w_keep + co;
        double *normv = w_norm + co;
        int n_keep = 0;
        /* 2. fuse_normalize_scores_v2 (object_3d_util.cpp:495-565) */
        if (n > 4) {
            const int bn = (int)round((double)((float)n) / 3.0 * 2.0);
            int P = 1;
            while (P < n) P <<= 1;
            uint64_t *key = (P <= FU_SMEM_SORT) ? sm_key : (w_key + 2 * co);
            uint32_t *idx = (P <= FU_SMEM_SORT) ? sm_idx : (w_idx + 2 * co);
            uint8_t *flag = w_flag + co;
            /* distance ranking */
            for (int i = tid; i < P; i += FU_THREADS) {
                key[i] = (i < n) ? sort_key(c_dist[co + vlist[i]]) : ~0ull;
                idx[i] = (i < n) ? (uint32_t)i : 0xffffffffu;
            }
            bitonic_sort(key, idx, P);
            for (int i = tid; i < n; i += FU_THREADS) flag[i] = 0;
            __syncthreads();
            for (int i = tid; i < bn - 1; i += FU_THREADS) {
                flag[idx[i]] = 1;
                keep[i] = (int32_t)idx[i]; /* distance order; used when the angle set is skipped */
            }
            __syncthreads();
            /* angle ranking */
            for (int i = tid; i < P; i += FU_THREADS) {
                key[i] = (i < n) ? sort_key(c_angle[co + vlist[i]]) : ~0ull;
                idx[i] = (i < n) ? (uint32_t)i : 0xffffffffu;
            }
            bitonic_sort(key, idx, P);
            if (tid == 0) {
                const double a1 = c_angle[co + vlist[idx[bn - 1]]], a2 = c_angle[co + vlist[idx[bn - 2]]];
                s_i[0] = (a1 > a2) ? 1 : 0;
            }
            __syncthreads();
            if (s_i[0]) {
                for (int i = tid; i < bn - 1; i += FU_THREADS) flag[idx[i]] |= 2;
                __syncthreads();
                /* set_intersection of the two index-sorted sets == ascending index order */
                int cnt = 0;
                for (int base = 0; base < n; base += FU_THREADS) {
                    const int i = base + tid;
                    const int v = (i < n && flag[i] == 3) ? 1 : 0;
                    int tot;
                    const int pos = block_excl_scan(v, s_warp, tot);
                    if (v) keep[cnt + pos] = i;
                    cnt += tot;
                }
                n_keep = cnt;
            } else
                n_keep = bn - 1;
            __syncthreads();
        } else {
            for (int i = tid; i < n; i += FU_THREADS) keep[i] = i;
            n_keep = n;
            __syncthreads();
        }
        /* min / max of the kept errors */
        double mn_d = 1e6, mx_d = -1, mn_a = 1e6, mx_a = -1;
        for (int i = tid; i < n_keep; i += FU_THREADS) {
            const double td = c_dist[co + vlist[keep[i]]], ta = c_angle[co + vlist[keep[i]]];
            mn_d = g_min(mn_d, td);
            mx_d = g_max(mx_d, td);
            mn_a = g_min(mn_a, ta);
            mx_a = g_max(mx_a, ta);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn_d = g_min(mn_d, __shfl_xor_sync(0xffffffffu, mn_d, o));
            mx_d = g_max(mx_d, __shfl_xor_sync(0xffffffffu, mx_d, o));
            mn_a = g_min(mn_a, __shfl_xor_sync(0xffffffffu, mn_a, o));
            mx_a = g_max(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, o));
        }
        __syncthreads();
        if (lane == 0) {
            s_red[0][wid] = mn_d;
            s_red[1][wid] = mx_d;
            s_red[2][wid] = mn_a;
            s_red[3][wid] = mx_a;
        }
        __syncthreads();
        mn_d = 1e6;
        mx_d = -1;
        mn_a = 1e6;
        mx_a = -1;
        for (int k = 0; k < FU_THREADS / 32; k++) {
            mn_d = g_min(mn_d, s_red[0][k]);
            mx_d = g_max(mx_d, s_red[1][k]);
            mn_a = g_min(mn_a, s_red[2][k]);
            mx_a = g_max(mx_a, s_red[3][k]);
        }
        /* 3. normalised score, 3D lift, skew penalty (box_proposal_detail.cpp:477-528) */
        double *score = w_score + co;
        for (int i = tid; i < n_keep; i += FU_THREADS) {
            const int raw = keep[i];
            const double dk = c_dist[co + vlist[raw]];
            double ak = c_angle[co + vlist[raw]];
            double comb;
            if (prm.whether_normalize_two_errors && n_keep > 1) {
                comb = (dk - mn_d) / (mx_d - mn_d);
                if ((mx_a - mn_a) > 0) ak = (ak - mn_a) / (mx_a - mn_a);
                comb = (comb + prm.weight_vp_angle * ak) / (1 + prm.weight_vp_angle);
            } else
                comb = (dk + prm.weight_vp_angle * ak) / (1 + prm.weight_vp_angle);
            normv[i] = comb;
            D2 c[8];
            int vp1pos, config_id, pose_id, top_id;
            const double *yaw;
            rebuild_corners(jb, fr, poses, yaw_table, prm, vlist[raw], c, vp1pos, config_id, yaw, pose_id, top_id);
            cs_cuboid_rec o;
            const CsPose &ps = poses[fr.pose_off + pose_id];
            g_lift_to_3d(c, (double)config_id, (double)vp1pos, yaw, ps.ground, ps.T, fr.invK, o);
            double sc;
            if (o.scale[0] < 0 || o.scale[1] < 0 || o.scale[2] < 0)
                sc = nan(""); /* dropped: scale should be positive (:493) */
            else {
                const double skew_ratio = g_max(o.scale[0], o.scale[1]) / g_min(o.scale[0], o.scale[1]);
                double skew_error = prm.weight_skew_error * g_max(skew_ratio - prm.nominal_skew_ratio, 0.0);
                if (skew_ratio > prm.max_cut_skew) skew_error = 100;
                sc = comb + prm.weight_skew_error * skew_error;
                if (isnan(sc)) sc = __longlong_as_double(0x7ff0000000000000ll); /* NaN ranks with +inf, still a cuboid */
            }
            score[i] = sc;
        }
        if (tid == 0) {
            job_counts[job * 2 + 0] = n;
            job_counts[job * 2 + 1] = n_keep;
        }
        __syncthreads();
    }

    /* 4. final ranking over all height samples: K rounds of arg-min by (score, position) (:517-536) */
    const int K = min(topk, CS_MAX_TOPK);
    int n_out = 0;
    for (int round = 0; round < K; round++) {
        double bv = 0;
        long long bp = -1; /* position = (job index in object << 32) | kept index */
        for (int jj = 0; jj < ob.n_jobs; jj++) {
            const int job = ob.job_off + jj;
            const int64_t co = jobs[job].cand_off;
            const int nk = job_counts[job * 2 + 1];
            for (int i = tid; i < nk; i += FU_THREADS) {
                const double sc = w_score[co + i];
                if (isnan(sc)) continue;
                const long long p = ((long long)jj << 32) | (long long)i;
                bool taken = false;
                for (int r = 0; r < round; r++) taken |= (s_chosen[r] == p);
                if (taken) continue;
                if (bp < 0 || sc < bv || (sc == bv && p < bp)) {
                    bv = sc;
                    bp = p;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const long long op = __shfl_xor_sync(0xffffffffu, bp, o);
            if (op >= 0 && (bp < 0 || ov < bv || (ov == bv && op < bp))) {
                bv = ov;
                bp = op;
            }
        }
        __syncthreads();
        if (lane == 0) {
            s_best_v[wid] = bv;
            s_best_p[wid] = bp;
        }
        __syncthreads();
        if (tid == 0) {
            double v = 0;
            long long p = -1;
            for (int k = 0; k < FU_THREADS / 32; k++) {
                const double ov = s_best_v[k];
                const long long op = s_best_p[k];
                if (op >= 0 && (p < 0 || ov < v || (ov == v && op < p))) {
                    v = ov;
                    p = op;
                }
            }
            s_chosen[round] = p;
        }
        __syncthreads();
        const long long p = s_chosen[round];
        if (p < 0) break;
        n_out++;
        if (tid == 0) {
            const int jj = (int)(p >> 32), i = (int)(p & 0xffffffffll);
            const int job = ob.job_off + jj;
            const CsJob jb = jobs[job];
            const int64_t co = jb.cand_off;
            const int raw = w_keep[co + i];
            const int cand = w_vlist[co + raw];
            D2 c[8];
            int vp1pos, config_id, pose_id, top_id;
            const double *yaw;
            rebuild_corners(jb, fr, poses, yaw_table, prm, cand, c, vp1pos, config_id, yaw, pose_id, top_id);
            cs_cuboid_rec o;
            const CsPose &ps = poses[fr.pose_off + pose_id];
            g_lift_to_3d(c, (double)config_id, (double)vp1pos, yaw, ps.ground, ps.T, fr.invK, o);
            o.rect_detect_2d[0] = ob.left;
            o.rect_detect_2d[1] = ob.top;
            o.rect_detect_2d[2] = ob.width_raw;
            o.rect_detect_2d[3] = ob.height_raw;
            o.edge_distance_error = c_dist[co + cand];
            o.edge_angle_error = c_angle[co + cand];
            o.normalized_error = w_norm[co + i];
            o.skew_ratio = g_max(o.scale[0], o.scale[1]) / g_min(o.scale[0], o.scale[1]);
            o.down_expand_height = (double)jb.down_expand;
            if (prm.whether_sample_cam_roll_pitch) {
                o.camera_roll_delta = ps.roll - fr.euler_raw[0];
                o.camera_pitch_delta = ps.pitch - fr.euler_raw[1];
            } else {
                o.camera_roll_delta = 0;
                o.camera_pitch_delta = 0;
            }
            o.combined_score = g_record_score(w_score[co + i], o, prm);
            o.proposal_index = raw;
            o.height_sample_id = jb.hs;
            o.valid = 1;
            o.pad_ = 0;
            out[(size_t)blockIdx.x * topk + round] = o;
        }
    }
    if (tid == 0) out_counts[blockIdx.x] = n_out;
}


/* ==========================================================================================
 * Warp-centric variants (the default when they apply).  The batch holds only ~10^5 candidates, so the CTA-wide
 * kernels above spend most of their time at __syncthreads; here one warp owns an independent unit of work and only
 * __syncwarp is used.
 * ========================================================================================== */
#define SWW_WARPS 4
#define SWW_YAWS 4   /* yaws handled by one warp, one after the other */
#define SWW_SLOTS 64

struct SweepWarpShared {
    double ang[CS_MAXL_OUT], midx[CS_MAXL_OUT], midy[CS_MAXL_OUT];
    double vp_angles[SWW_WARPS * SWW_YAWS][6];
    D2 vps[SWW_WARPS * SWW_YAWS][3];
    D2 corners[SWW_WARPS][SWW_SLOTS][8];
    int32_t slot_cand[SWW_WARPS][SWW_SLOTS]; /* candidate index inside the (job, pose) block */
    int8_t slot_yaw[SWW_WARPS][SWW_SLOTS];
    int8_t slot_cfg[SWW_WARPS][SWW_SLOTS];
};

/* scale (half sizes) of a lifted proposal only: what the ranking needs (object_3d_util.cpp:615-625) */
__device__ __forceinline__ void g_lift_scale(const D2 *c, const double *ground, const double *T, const double *invK, double *scale)
{
    double g[4][3];
    for (int i = 0; i < 4; i++) g_plane_hit(T, invK, ground, c[4 + i], g[i]);
    double dx = g[0][0] - g[3][0], dy = g[0][1] - g[3][1], dz = g[0][2] - g[3][2];
    scale[0] = sqrt((dx * dx + dy * dy) + dz * dz) / 2;
    dx = g[0][0] - g[1][0];
    dy = g[0][1] - g[1][1];
    dz = g[0][2] - g[1][2];
    scale[1] = sqrt((dx * dx + dy * dy) + dz * dz) / 2;
    double nrm[3] = {dy * 1.0 - dz * 0.0, dz * 0.0 - dx * 1.0, dx * 0.0 - dy * 0.0};
    const double nn = sqrt((nrm[0] * nrm[0] + nrm[1] * nrm[1]) + nrm[2] * nrm[2]);
    for (int i = 0; i < 3; i++) nrm[i] /= nn;
    const double dist = -((nrm[0] * g[0][0] + nrm[1] * g[0][1]) + nrm[2] * g[0][2]);
    double pw[4] = {nrm[0], nrm[1], nrm[2], dist};
    if (dist < 0)
        for (int i = 0; i < 4; i++) pw[i] = -pw[i];
    double ps[4];
    for (int i = 0; i < 4; i++) ps[i] = ((T[0 * 4 + i] * pw[0] + T[1 * 4 + i] * pw[1]) + T[2 * 4 + i] * pw[2]) + T[3 * 4 + i] * pw[3];
    double top[3];
    g_plane_hit(T, invK, ps, c[1], top);
    scale[2] = top[2] / 2;
}

/* skew_ratio of the lifted cuboid, NaN when a scale is negative (the proposal is then dropped, box_proposal_detail.cpp:493) */
__device__ __forceinline__ double g_skew_of(const D2 *c, const CsPose &ps, const double *invK)
{
    double sc3[3];
    g_lift_scale(c, ps.ground, ps.T, invK, sc3);
    if (sc3[0] < 0 || sc3[1] < 0 || sc3[2] < 0) return nan("");
    const double r = g_max(sc3[0], sc3[1]) / g_min(sc3[0], sc3[1]);
    return isnan(r) ? __longlong_as_double(0x7ff0000000000000ll) : r; /* NaN skew (degenerate lift) ranks as +inf, still a cuboid */
}

/* VP_support_edge_infos for ONE vanishing point by ONE lane (object_3d_util.cpp:380-425): a plain loop over the line set, so
 * the first-occurrence semantics of maxCoeff / minCoeff and of smooth_jump_angles' base angle come for free. */
__device__ __forceinline__ void vp_support_lane(const double *ang, const double *midx, const double *midy, int n_lines, D2 vp, double thre,
                                                int vp_id, double *out2)
{
    bool have = false;
    double base = 0, vmax = 0, vmin = 0;
    int imax = 0, imin = 0;
    for (int e = 0; e < n_lines; e++) {
        const double raw = cs_pm_atan2(midy[e] - vp.y, midx[e] - vp.x);
        const double nrm = g_normalize_to_pi(raw);
        double d = fabs(ang[e] - nrm);
        d = g_min(d, CS_PI - d);
        if (d < thre) {
            if (!have) {
                have = true;
                base = raw;
                vmax = vmin = raw;
                imax = imin = e;
            } else {
                double v = raw;
                if ((raw - base) < -CS_PI)
                    v = raw + 2 * CS_PI;
                else if ((raw - base) > CS_PI)
                    v = raw - 2 * CS_PI;
                if (v > vmax) {
                    vmax = v;
                    imax = e;
                }
                if (v < vmin) {
                    vmin = v;
                    imin = e;
                }
            }
        }
    }
    if (!have) {
        out2[0] = nan("");
        out2[1] = nan("");
        return;
    }
    int low = imax, top = imin;
    if (vp_id > 0) {
        const int t = low;
        low = top;
        top = t;
    }
    out2[0] = ang[low];
    out2[1] = ang[top];
}

/* One warp per (ROI job, pose, group of SWW_YAWS yaws).  Per yaw: VP support by the warp, one lane per (top-x, config)
 * candidate for the FP64 corner chain; valid candidates are compacted into the warp's slot list and scored 32 at a time, so
 * the expensive part (99/77 dist-map gathers, 6 atan2, the 3D lift for the skew) runs with full lanes.  No block barrier
 * after the line set is staged. */
__global__ void __launch_bounds__(32 * SWW_WARPS) k_sweep_warp(const CsJob *__restrict__ jobs, const CsFrame *__restrict__ frames,
                                                               const CsPose *__restrict__ poses, const double *__restrict__ yaw_table,
                                                               const int4 *__restrict__ blocks /* (job, pose, yaw0, n) */,
                                                               const double *__restrict__ merged_lines, const int32_t *__restrict__ line_counts,
                                                               const float *__restrict__ dist_arena, uint8_t *__restrict__ c_valid,
                                                               double *__restrict__ c_dist, double *__restrict__ c_angle,
                                                               double *__restrict__ c_skew, cs_cuboid_params prm)
{
    __shared__ SweepWarpShared S;
    const int4 bk = blocks[blockIdx.x];
    const CsJob &jb = jobs[bk.x];
    const CsFrame &fr = frames[jb.frame];
    const CsPose &pose = poses[fr.pose_off + bk.y];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const unsigned FULL = 0xffffffffu;
    const int n_lines = line_counts[bk.x * 2 + 1];
    {
        const double *ml = merged_lines + (size_t)bk.x * CS_MAXL_OUT * 7;
        for (int i = tid; i < n_lines; i += 32 * SWW_WARPS) {
            S.ang[i] = ml[4 * CS_MAXL_OUT + i];
            S.midx[i] = ml[5 * CS_MAXL_OUT + i];
            S.midy[i] = ml[6 * CS_MAXL_OUT + i];
        }
    }
    __syncthreads();
    /* phase A: one lane per (yaw, VP) -- vanishing point + its two supporting line angles.  The vertical VP does not depend on
     * the yaw: it is evaluated once per block and copied. */
    {
        const int n_tasks = 2 * bk.w + 1;
        for (int t = tid; t < n_tasks; t += 32 * SWW_WARPS) {
            const int ys = (t < 2 * bk.w) ? (t >> 1) : 0, vp_id = (t < 2 * bk.w) ? (t & 1) : 2;
            D2 v3[3];
            g_vanishing_points(pose.KinvR, yaw_table + 3 * (size_t)(fr.yaw_off + bk.z + ys), v3);
            const double thre = ((vp_id != 2) ? prm.vp12_edge_angle_thre : prm.vp3_edge_angle_thre) / 180.0 * CS_PI;
            double o2[2];
            vp_support_lane(S.ang, S.midx, S.midy, n_lines, v3[vp_id], thre, vp_id, o2);
            if (vp_id < 2) {
                S.vps[ys][vp_id] = v3[vp_id];
                S.vp_angles[ys][vp_id * 2] = o2[0];
                S.vp_angles[ys][vp_id * 2 + 1] = o2[1];
            } else {
                for (int k = 0; k < bk.w; k++) {
                    S.vps[k][2] = v3[2];
                    S.vp_angles[k][4] = o2[0];
                    S.vp_angles[k][5] = o2[1];
                }
            }
        }
    }
    __syncthreads();
    const int y_first = bk.z + wid * SWW_YAWS, y_end = min(bk.z + bk.w, y_first + SWW_YAWS);
    if (y_first >= y_end) return;
    const int n_top = jb.n_top, n_yaw = fr.n_yaw;
    const float *dist = dist_arena + jb.px_off;
    const int64_t cbase = jb.cand_off + (int64_t)bk.y * n_yaw * n_top * 2;
    const bool cfg1 = prm.consider_config_1 != 0, cfg2 = prm.consider_config_2 != 0;
    int n_pending = 0;

    auto score_slots = [&](int count) { /* lanes < count score slot `lane` */
        if (lane < count) {
            const D2 *c = S.corners[wid][lane];
            const int cfg = S.slot_cfg[wid][lane];
            const int64_t ci = cbase + S.slot_cand[wid][lane];
            const double sum_dist = g_edge_sum_dists(dist, jb.dpitch, jb.roi_w, jb.roi_h, c, (double)jb.roi_l, (double)jb.roi_t, cfg,
                                                     prm.reweight_edge_distance != 0);
            c_dist[ci] = sum_dist / jb.diag;
            c_angle[ci] = g_angle_error(S.vp_angles[S.slot_yaw[wid][lane]], cfg, c);
            c_skew[ci] = g_skew_of(c, pose, fr.invK);
        }
        __syncwarp();
    };

    for (int yy = 0; y_first + yy < y_end; yy++) {
        const int yi = y_first + yy;
        const int ys = yi - bk.z; /* yaw slot inside the block */
        for (int c0 = 0; c0 < n_top * 2; c0 += 32) {
            const int ci = c0 + lane;
            bool valid = false;
            D2 c[8];
            int config_id = 1;
            if (ci < n_top * 2) {
                const int ti = ci >> 1;
                config_id = (ci & 1) + 1;
                int vp1pos;
                if ((config_id == 1) ? cfg1 : cfg2) valid = g_build_corners(jb, S.vps[ys], g_top_x(jb, ti), config_id, prm.shorted_edge_thre, c, vp1pos);
                c_valid[cbase + (int64_t)yi * n_top * 2 + ci] = valid ? 1 : 0;
            }
            const unsigned m = __ballot_sync(FULL, valid);
            if (valid) {
                const int slot = n_pending + __popc(m & ((1u << lane) - 1u));
#pragma unroll
                for (int k = 0; k < 8; k++) S.corners[wid][slot][k] = c[k];
                S.slot_cand[wid][slot] = yi * n_top * 2 + ci;
                S.slot_yaw[wid][slot] = (int8_t)ys;
                S.slot_cfg[wid][slot] = (int8_t)config_id;
            }
            n_pending += __popc(m);
            __syncwarp();
            if (n_pending >= 32) {
                score_slots(32);
                const int rest = n_pending - 32; /* < 32: move the tail to the front */
                D2 tc[8];
                int tcand = 0, ty = 0, tcf = 0;
                if (lane < rest) {
#pragma unroll
                    for (int k = 0; k < 8; k++) tc[k] = S.corners[wid][32 + lane][k];
                    tcand = S.slot_cand[wid][32 + lane];
                    ty = S.slot_yaw[wid][32 + lane];
                    tcf = S.slot_cfg[wid][32 + lane];
                }
                __syncwarp();
                if (lane < rest) {
#pragma unroll
                    for (int k = 0; k < 8; k++) S.corners[wid][lane][k] = tc[k];
                    S.slot_cand[wid][lane] = tcand;
                    S.slot_yaw[wid][lane] = (int8_t)ty;
                    S.slot_cfg[wid][lane] = (int8_t)tcf;
                }
                n_pending = rest;
                __syncwarp();
            }
        }
    }
    if (n_pending > 0) score_slots(n_pending);
}

/* ---- selection, one warp per 2D box (all valid counts <= FW_CAP) ---- */
#define FW_CAP 1024
#define FW_WARPS 2

struct FuseWarpShared {
    uint64_t key[FW_CAP];
    uint16_t idx[FW_CAP];
    uint16_t vlist[FW_CAP];
    uint16_t keep[FW_CAP];
    uint8_t flag[FW_CAP];
};

__device__ __forceinline__ void warp_bitonic(uint64_t *key, uint16_t *idx, int P)
{
    const int lane = threadIdx.x & 31;
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncwarp();
            for (int i = lane; i < P; i += 32) {
                const int l = i ^ j;
                if (l > i) {
                    const uint64_t ki = key[i], kl = key[l];
                    const uint16_t ii = idx[i], il = idx[l];
                    const bool gt = (ki > kl) || (ki == kl && ii > il);
                    const bool up = ((i & k) == 0);
                    if (gt == up) {
                        key[i] = kl;
                        key[l] = ki;
                        idx[i] = il;
                        idx[l] = ii;
                    }
                }
            }
        }
    __syncwarp();
}

__device__ __forceinline__ double warp_min_d(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = g_min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max_d(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = g_max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

extern __shared__ unsigned char fw_smem_raw[];

__global__ void __launch_bounds__(32 * FW_WARPS) k_fuse_warp(const CsObj *__restrict__ objs, int n_objs, const CsJob *__restrict__ jobs,
                                                             const CsFrame *__restrict__ frames, const CsPose *__restrict__ poses,
                                                             const double *__restrict__ yaw_table, const uint8_t *__restrict__ c_valid,
                                                             const double *__restrict__ c_dist, const double *__restrict__ c_angle,
                                                             const double *__restrict__ c_skew, int32_t *__restrict__ w_vlist,
                                                             int32_t *__restrict__ w_keep, double *__restrict__ w_norm,
                                                             double *__restrict__ w_score, int32_t *__restrict__ job_counts,
                                                             cs_cuboid_rec *__restrict__ out, int32_t *__restrict__ out_counts, int topk,
                                                             cs_cuboid_params prm)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int oi = blockIdx.x * FW_WARPS + wid;
    if (oi >= n_objs) return;
    FuseWarpShared &S = reinterpret_cast<FuseWarpShared *>(fw_smem_raw)[wid];
    const unsigned FULL = 0xffffffffu;
    const CsObj ob = objs[oi];
    const CsFrame &fr = frames[ob.frame];

    for (int jj = 0; jj < ob.n_jobs; jj++) {
        const int job = ob.job_off + jj;
        const CsJob &jb = jobs[job];
        const int64_t co = jb.cand_off;
        /* 1. valid proposals in enumeration order */
        int n = 0;
        for (int base = 0; base < jb.n_cand; base += 32) {
            const int i = base + lane;
            const bool v = (i < jb.n_cand) && c_valid[co + i];
            const unsigned m = __ballot_sync(FULL, v);
            if (v) S.vlist[n + __popc(m & ((1u << lane) - 1u))] = (uint16_t)i;
            n += __popc(m);
        }
        __syncwarp();
        int n_keep = 0;
        /* 2. fuse_normalize_scores_v2 */
        if (n > 4) {
            const int bn = (int)round((double)((float)n) / 3.0 * 2.0);
            int P = 1;
            while (P < n) P <<= 1;
            for (int i = lane; i < P; i += 32) {
                S.key[i] = (i < n) ? sort_key(c_dist[co + S.vlist[i]]) : ~0ull;
                S.idx[i] = (i < n) ? (uint16_t)i : (uint16_t)0xffff;
            }
            warp_bitonic(S.key, S.idx, P);
            for (int i = lane; i < n; i += 32) S.flag[i] = 0;
            __syncwarp();
            for (int i = lane; i < bn - 1; i += 32) {
                S.flag[S.idx[i]] = 1;
                S.keep[i] = S.idx[i];
            }
            __syncwarp();
            for (int i = lane; i < P; i += 32) {
                S.key[i] = (i < n) ? sort_key(c_angle[co + S.vlist[i]]) : ~0ull;
                S.idx[i] = (i < n) ? (uint16_t)i : (uint16_t)0xffff;
            }
            warp_bitonic(S.key, S.idx, P);
            const double a1 = c_angle[co + S.vlist[S.idx[bn - 1]]], a2 = c_angle[co + S.vlist[S.idx[bn - 2]]];
            if (a1 > a2) {
                for (int i = lane; i < bn - 1; i += 32) S.flag[S.idx[i]] |= 2;
                __syncwarp();
                int cnt = 0;
                for (int base = 0; base < n; base += 32) {
                    const int i = base + lane;
                    const bool v = (i < n) && (S.flag[i] == 3);
                    const unsigned m = __ballot_sync(FULL, v);
                    if (v) S.keep[cnt + __popc(m & ((1u << lane) - 1u))] = (uint16_t)i;
                    cnt += __popc(m);
                }
                n_keep = cnt;
            } else
                n_keep = bn - 1;
            __syncwarp();
        } else {
            for (int i = lane; i < n; i += 32) S.keep[i] = (uint16_t)i;
            n_keep = n;
            __syncwarp();
        }
        double mn_d = 1e6, mx_d = -1, mn_a = 1e6, mx_a = -1;
        for (int i = lane; i < n_keep; i += 32) {
            const int cand = S.vlist[S.keep[i]];
            const double td = c_dist[co + cand], ta = c_angle[co + cand];
            mn_d = g_min(mn_d, td);
            mx_d = g_max(mx_d, td);
            mn_a = g_min(mn_a, ta);
            mx_a = g_max(mx_a, ta);
        }
        mn_d = warp_min_d(mn_d);
        mx_d = warp_max_d(mx_d);
        mn_a = warp_min_d(mn_a);
        mx_a = warp_max_d(mx_a);
        /* 3. normalised score + skew penalty per kept proposal */
        for (int i = lane; i < n_keep; i += 32) {
            const int raw = S.keep[i];
            const int cand = S.vlist[raw];
            const double dk = c_dist[co + cand];
            double ak = c_angle[co + cand];
            double comb;
            if (prm.whether_normalize_two_errors && n_keep > 1) {
                comb = (dk - mn_d) / (mx_d - mn_d);
                if ((mx_a - mn_a) > 0) ak = (ak - mn_a) / (mx_a - mn_a);
                comb = (comb + prm.weight_vp_angle * ak) / (1 + prm.weight_vp_angle);
            } else
                comb = (dk + prm.weight_vp_angle * ak) / (1 + prm.weight_vp_angle);
            const double skew_ratio = c_skew[co + cand]; /* from the sweep; NaN == negative scale == dropped */
            double sc;
            if (isnan(skew_ratio))
                sc = nan("");
            else {
                double skew_error = prm.weight_skew_error * g_max(skew_ratio - prm.nominal_skew_ratio, 0.0);
                if (skew_ratio > prm.max_cut_skew) skew_error = 100;
                sc = comb + prm.weight_skew_error * skew_error;
                if (isnan(sc)) sc = __longlong_as_double(0x7ff0000000000000ll);
            }
            w_score[co + i] = sc;
            w_norm[co + i] = comb;
            w_keep[co + i] = raw;
            w_vlist[co + i] = cand; /* NOTE: indexed by kept position here (the CTA kernel indexes by valid row) */
        }
        if (lane == 0) {
            job_counts[job * 2 + 0] = n;
            job_counts[job * 2 + 1] = n_keep;
        }
        __syncwarp();
    }
    __threadfence_block();
    __syncwarp();
    /* 4. final ranking: K rounds of arg-min by (score, position) */
    const int K = min(topk, CS_MAX_TOPK);
    long long chosen[CS_MAX_TOPK];
    int n_out = 0;
    for (int round = 0; round < K; round++) {
        double bv = 0;
        long long bp = -1;
        for (int jj = 0; jj < ob.n_jobs; jj++) {
            const int job = ob.job_off + jj;
            const int64_t co = jobs[job].cand_off;
            const int nk = job_counts[job * 2 + 1];
            for (int i = lane; i < nk; i += 32) {
                const double sc = w_score[co + i];
                if (isnan(sc)) continue;
                const long long p = ((long long)jj << 32) | (long long)i;
                bool taken = false;
                for (int r = 0; r < round; r++) taken |= (chosen[r] == p);
                if (taken) continue;
                if (bp < 0 || sc < bv || (sc == bv && p < bp)) {
                    bv = sc;
                    bp = p;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(FULL, bv, o);
            const long long op = __shfl_xor_sync(FULL, bp, o);
            if (op >= 0 && (bp < 0 || ov < bv || (ov == bv && op < bp))) {
                bv = ov;
                bp = op;
            }
        }
        chosen[round] = bp;
        if (bp < 0) break;
        n_out++;
        if (lane == 0) {
            const int jj = (int)(bp >> 32), i = (int)(bp & 0xffffffffll);
            const int job = ob.job_off + jj;
            const CsJob &jb = jobs[job];
            const int64_t co = jb.cand_off;
            const int raw = w_keep[co + i];
            const int cand = w_vlist[co + i];
            D2 c[8];
            int vp1pos, config_id, pose_id, top_id;
            const double *yaw;
            rebuild_corners(jb, fr, poses, yaw_table, prm, cand, c, vp1pos, config_id, yaw, pose_id, top_id);
            cs_cuboid_rec &o = out[(size_t)oi * topk + round];
            const CsPose &ps = poses[fr.pose_off + pose_id];
            g_lift_to_3d(c, (double)config_id, (double)vp1pos, yaw, ps.ground, ps.T, fr.invK, o);
            o.rect_detect_2d[0] = ob.left;
            o.rect_detect_2d[1] = ob.top;
            o.rect_detect_2d[2] = ob.width_raw;
            o.rect_detect_2d[3] = ob.height_raw;
            o.edge_distance_error = c_dist[co + cand];
            o.edge_angle_error = c_angle[co + cand];
            o.normalized_error = w_norm[co + i];
            o.skew_ratio = g_max(o.scale[0], o.scale[1]) / g_min(o.scale[0], o.scale[1]);
            o.down_expand_height = (double)jb.down_expand;
            if (prm.whether_sample_cam_roll_pitch) {
                o.camera_roll_delta = ps.roll - fr.euler_raw[0];
                o.camera_pitch_delta = ps.pitch - fr.euler_raw[1];
            } else {
                o.camera_roll_delta = 0;
                o.camera_pitch_delta = 0;
            }
            o.combined_score = g_record_score(w_score[co + i], o, prm);
            o.proposal_index = raw;
            o.height_sample_id = jb.hs;
            o.valid = 1;
            o.pad_ = 0;
        }
    }
    if (lane == 0) out_counts[oi] = n_out;
}

/* ------------------------------------------------------------------------------------------ launchers */
void cs_launch_sweep(const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw, const int2 *d_blocks,
                     int n_blocks, const double *d_mlines, const int32_t *d_line_counts, const float *d_dist, uint8_t *c_valid, double *c_dist,
                     double *c_angle, const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches)
{
    if (n_blocks <= 0) return;
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(k_sweep_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SweepShared)));
    k_sweep_score<<<n_blocks, SW_THREADS, sizeof(SweepShared), st>>>(d_jobs, d_frames, d_poses, d_yaw, d_blocks, d_mlines, d_line_counts, d_dist,
                                                                     c_valid, c_dist, c_angle, *prm);
    (*launches)++;
}

void cs_launch_fuse(const CsObj *d_objs, int n_objs, const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw,
                    const uint8_t *c_valid, const double *c_dist, const double *c_angle, int32_t *w_vlist, uint64_t *w_key, uint32_t *w_idx,
                    uint8_t *w_flag, int32_t *w_keep, double *w_norm, double *w_score, int32_t *job_counts, cs_cuboid_rec *d_out,
                    int32_t *d_out_counts, int topk, const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches)
{
    if (n_objs <= 0) return;
    const size_t smem = (sizeof(uint64_t) + sizeof(uint32_t)) * FU_SMEM_SORT;
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(k_fuse_rank, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_fuse_rank<<<n_objs, FU_THREADS, smem, st>>>(d_objs, d_jobs, d_frames, d_poses, d_yaw, c_valid, c_dist, c_angle, w_vlist, w_key, w_idx, w_flag,
                                                  w_keep, w_norm, w_score, job_counts, d_out, d_out_counts, topk, *prm);
    (*launches)++;
}

void cs_launch_sweep_warp(const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw, const int4 *d_blocks,
                          int n_blocks, const double *d_mlines, const int32_t *d_line_counts, const float *d_dist, uint8_t *c_valid,
                          double *c_dist, double *c_angle, double *c_skew, const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches)
{
    if (n_blocks <= 0) return;
    CS_APPLY_CARVEOUT(k_sweep_warp);
    k_sweep_warp<<<n_blocks, 32 * SWW_WARPS, 0, st>>>(d_jobs, d_frames, d_poses, d_yaw, d_blocks, d_mlines, d_line_counts, d_dist, c_valid, c_dist,
                                                      c_angle, c_skew, *prm);
    (*launches)++;
}

int cs_fuse_warp_cap(void) { return FW_CAP; }
int cs_sweep_warp_yaws(void) { return SWW_WARPS * SWW_YAWS; }

void cs_launch_fuse_warp(const CsObj *d_objs, int n_objs, const CsJob *d_jobs, const CsFrame *d_frames, const CsPose *d_poses, const double *d_yaw,
                         const uint8_t *c_valid, const double *c_dist, const double *c_angle, const double *c_skew, int32_t *w_vlist, int32_t *w_keep,
                         double *w_norm, double *w_score, int32_t *job_counts, cs_cuboid_rec *d_out, int32_t *d_out_counts, int topk,
                         const cs_cuboid_params *prm, cudaStream_t st, int64_t *launches)
{
    if (n_objs <= 0) return;
    const size_t smem = sizeof(FuseWarpShared) * FW_WARPS;
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(k_fuse_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CS_APPLY_CARVEOUT(k_fuse_warp);
    k_fuse_warp<<<(n_objs + FW_WARPS - 1) / FW_WARPS, 32 * FW_WARPS, smem, st>>>(d_objs, n_objs, d_jobs, d_frames, d_poses, d_yaw, c_valid, c_dist,
                                                                                 c_angle, c_skew, w_vlist, w_keep, w_norm, w_score, job_counts, d_out,
                                                                                 d_out_counts, topk, *prm);
    (*launches)++;
}
